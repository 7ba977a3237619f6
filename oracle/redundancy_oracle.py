"""CPU oracle for the data-redundancy analysis -- TEST INFRASTRUCTURE ONLY.

A restatement, with Python sets as the reference uses them, of ``duplicates``, ``count_triplets`` and
``cartesian_product_relations`` of torchkge v0.17.7 (torchkge/utils/data_redundancy.py), with the two
deviations ``torchkge_b200.data_redundancy`` documents: every pair of ``range(kg_tr.n_rel)`` is compared
(not ``range(1345)``), and a relation without facts belongs to no pair and is never a Cartesian-product
relation (the reference divides by zero).  No progress bars; the printed lines are the reference's.
``tests/test_utils_data_redundancy_cpu.py`` pins it against outputs of the unmodified reference
(``tests/golden/redundancy.npz``).
"""
from itertools import combinations

import torch


def concat_kgs(kg_tr, kg_val, kg_te):
    h = torch.cat((kg_tr.head_idx, kg_val.head_idx, kg_te.head_idx))
    t = torch.cat((kg_tr.tail_idx, kg_val.tail_idx, kg_te.tail_idx))
    r = torch.cat((kg_tr.relations, kg_val.relations, kg_te.relations))
    return h, t, r


def _pair_sets(h, t, r):
    """relation -> set of (h, t), and the number of facts per relation (with multiplicity)"""
    sets, lengths = {}, {}
    for a, b, c in zip(h.tolist(), t.tolist(), r.tolist()):
        sets.setdefault(c, set()).add((a, b))
        lengths[c] = lengths.get(c, 0) + 1
    return sets, lengths


def count_triplets(kg1, kg2, duplicates, rev_duplicates):
    s1, _ = _pair_sets(kg1.head_idx, kg1.tail_idx, kg1.relations)
    s2, _ = _pair_sets(kg2.head_idx, kg2.tail_idx, kg2.relations)
    empty = set()

    def ht(s, r):
        return s.get(r, empty)

    def th(s, r):
        return {(b, a) for a, b in s.get(r, empty)}

    n_duplicates = 0
    for r1, r2 in duplicates:
        n_duplicates += len(ht(s2, r1) & ht(s1, r2)) + len(ht(s2, r2) & ht(s1, r1))
    n_rev_duplicates = 0
    for r1, r2 in rev_duplicates:
        n_rev_duplicates += len(ht(s2, r1) & th(s1, r2)) + len(ht(s2, r2) & th(s1, r1))
    return n_duplicates, n_rev_duplicates


def duplicates(kg_tr, kg_val, kg_te, theta1=0.8, theta2=0.8, verbose=False, counts=False, reverses=None):
    if verbose:
        print('Computing Ts')
    if reverses is None:
        reverses = []
    sets, lengths = _pair_sets(*concat_kgs(kg_tr, kg_val, kg_te))
    T = {r: sets.get(r, set()) for r in range(kg_tr.n_rel)}
    T_inv = {r: {(b, a) for a, b in T[r]} for r in range(kg_tr.n_rel)}
    if verbose:
        print('Finding duplicate relations')
    dupl, rev = [], []
    nonempty = [r for r in range(kg_tr.n_rel) if lengths.get(r, 0) > 0]
    for r1, r2 in combinations(nonempty, 2):
        n = len(T[r1] & T[r2])
        if n / lengths[r1] > theta1 and n / lengths[r2] > theta2:
            dupl.append((r1, r2))
        if (r1, r2) not in reverses:
            n = len(T[r1] & T_inv[r2])
            if n / lengths[r1] > theta1 and n / lengths[r2] > theta2:
                rev.append((r1, r2))
    if verbose:
        print('Duplicate relations: {}'.format(len(dupl)))
        print('Reverse duplicate relations: {}\n'.format(len(rev)))
    if counts:
        d, rv = count_triplets(kg_tr, kg_tr, dupl, rev)
        print('{} train triplets have duplicate in train set ({}%)'.format(d, int(d / len(kg_tr))))
        print('{} train triplets have reverse duplicate in train set ({}%)\n'.format(rv, int(rv / len(kg_tr) * 100)))
        d, rv = count_triplets(kg_tr, kg_te, dupl, rev)
        print('{} test triplets have duplicate in train set ({}%)'.format(d, int(d / len(kg_te))))
        print('{} test triplets have reverse duplicate in train set ({}%)\n'.format(rv, int(rv / len(kg_te) * 100)))
        d, rv = count_triplets(kg_te, kg_te, dupl, rev)
        print('{} test triplets have duplicate in test set ({}%)'.format(d, int(d / len(kg_te))))
        print('{} test triplets have reverse duplicate in test set ({}%)\n'.format(rv, int(rv / len(kg_te) * 100)))
    return dupl, rev


def cartesian_product_relations(kg_tr, kg_val, kg_te, theta=0.8):
    h, t, r = concat_kgs(kg_tr, kg_val, kg_te)
    S, O, lengths = {}, {}, {}
    for a, b, c in zip(h.tolist(), t.tolist(), r.tolist()):
        S.setdefault(c, set()).add(a)
        O.setdefault(c, set()).add(b)
        lengths[c] = lengths.get(c, 0) + 1
    return [r_ for r_ in range(kg_tr.n_rel)
            if lengths.get(r_, 0) > 0 and lengths[r_] / (len(S[r_]) * len(O[r_])) > theta]
