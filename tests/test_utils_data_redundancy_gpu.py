"""Data redundancy on the GPU (torchkge_b200.data_redundancy, csrc/redundancy.cu): equal to the outputs of
the unmodified reference stored in tests/golden/redundancy.npz -- lists, order, counts and printed text --
and to the CPU oracle (oracle/redundancy_oracle.py) on graphs the reference cannot take: other relation
counts, empty splits, relations without facts, one entity pair carrying 500 relations, self-loops only,
and a graph of a million facts."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import redundancy_oracle as oracle
from tests.test_utils_data_redundancy_cpu import CART_THETAS, REVERSES, THETAS, RefStyleKG, golden_graphs, pairs
from torchkge_b200 import data_redundancy as dr

pytestmark = pytest.mark.gpu


def as_package_kg(kg):
    return tk.KnowledgeGraph(kg.head_idx, kg.tail_idx, kg.relations, kg.n_ent, kg.n_rel)


def same_as_oracle(tr, va, te, capsys, theta1=0.8, theta2=0.8, reverses=None, counts=True):
    """duplicates (with its printed lines), cartesian_product_relations at two thresholds and count_triplets
    of the found lists equal the oracle's; returns the duplicate lists."""
    want = oracle.duplicates(tr, va, te, theta1, theta2, verbose=True, counts=counts, reverses=reverses)
    want_text = capsys.readouterr().out
    got = dr.duplicates(tr, va, te, theta1, theta2, verbose=True, counts=counts, reverses=reverses)
    assert capsys.readouterr().out == want_text
    assert got == want
    assert all(type(x) is int for p in got[0] + got[1] for x in p)
    for th in (0.8, 0.3):
        assert dr.cartesian_product_relations(tr, va, te, theta=th) == oracle.cartesian_product_relations(
            tr, va, te, theta=th)
    for kg1, kg2 in ((tr, te), (tr, tr), (te, tr)):
        assert dr.count_triplets(kg1, kg2, *got) == oracle.count_triplets(kg1, kg2, *got)
    return got


@pytest.mark.parametrize("kind", ["reference-style", "package"])
def test_equal_to_the_reference_golden(kind, capsys):
    z, kgs = golden_graphs()
    tr, va, te = kgs if kind == "reference-style" else [as_package_kg(kg) for kg in kgs]
    for i, (t1, t2) in enumerate(THETAS):
        for tag, rev in REVERSES.items():
            d, rd = dr.duplicates(tr, va, te, theta1=t1, theta2=t2, reverses=rev)
            assert d == pairs(z["dup_%d_%s" % (i, tag)]), (i, tag)
            assert rd == pairs(z["rev_%d_%s" % (i, tag)]), (i, tag)
    d_listed, rd_listed = pairs(z["count_dup_listed"]), pairs(z["count_rev_listed"])
    assert dr.count_triplets(tr, te, d_listed, rd_listed) == tuple(z["count_tr_te"].tolist())
    assert dr.count_triplets(te, te, d_listed, rd_listed) == tuple(z["count_te_te"].tolist())
    for i, th in enumerate(CART_THETAS):
        assert dr.cartesian_product_relations(tr, va, te, theta=th) == z["cart_%d" % i].tolist()
    capsys.readouterr()
    dr.duplicates(tr, va, te, verbose=True, counts=True)
    assert capsys.readouterr().out == str(z["stdout"])


def random_graph(n_rel, n_facts, n_ent, seed, split=(0.7, 0.15)):
    """Random facts plus planted structure: copies of a relation's pairs (some reversed, some with extra
    facts) under other relations, and repeated facts; split into three graphs."""
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, n_ent, (n_facts,), generator=g)
    t = torch.randint(0, n_ent, (n_facts,), generator=g)
    r = torch.randint(0, n_rel, (n_facts,), generator=g)
    if n_rel >= 2:
        k = max(1, n_rel // 4)
        src = torch.randint(0, n_rel, (k,), generator=g)
        dst = torch.randint(0, n_rel, (k,), generator=g)
        extra = []
        for i, (a, b) in enumerate(zip(src.tolist(), dst.tolist())):
            m = r == a
            keep = torch.rand(int(m.sum()), generator=g) < 0.9
            hh, tt = h[m][keep], t[m][keep]
            if i % 2:
                hh, tt = tt, hh
            extra.append(torch.stack([hh, tt, torch.full_like(hh, b)], 1))
        extra = torch.cat(extra)
        h, t, r = torch.cat([h, extra[:, 0]]), torch.cat([t, extra[:, 1]]), torch.cat([r, extra[:, 2]])
    rep = torch.randint(0, h.numel(), (h.numel() // 20,), generator=g)
    h, t, r = torch.cat([h, h[rep]]), torch.cat([t, t[rep]]), torch.cat([r, r[rep]])
    perm = torch.randperm(h.numel(), generator=g)
    h, t, r = h[perm], t[perm], r[perm]
    n_tr, n_va = int(split[0] * h.numel()), int(split[1] * h.numel())
    cuts = [(0, n_tr), (n_tr, n_tr + n_va), (n_tr + n_va, h.numel())]
    return [RefStyleKG(h[a:b], t[a:b], r[a:b], n_ent, n_rel) for a, b in cuts]


@pytest.mark.parametrize("n_rel,n_facts,n_ent", [(1, 300, 20), (2, 500, 25), (37, 4000, 60), (300, 20000, 150),
                                                 (2000, 30000, 400)])
def test_random_graphs_equal_the_oracle(n_rel, n_facts, n_ent, capsys):
    tr, va, te = random_graph(n_rel, n_facts, n_ent, seed=n_rel)
    same_as_oracle(tr, va, te, capsys)
    d, rd = same_as_oracle(tr, va, te, capsys, theta1=0.2, theta2=0.1, counts=False)
    if n_rel >= 37:
        assert d and rd     # the planted copies are found
        same_as_oracle(tr, va, te, capsys, theta1=0.2, theta2=0.1, reverses=rd[::2], counts=False)


def test_empty_validation_and_test_graphs(capsys):
    tr, _, _ = random_graph(37, 4000, 60, seed=5)
    empty = RefStyleKG([], [], [], 60, 37)
    assert dr.duplicates(tr, empty, empty, 0.2, 0.1) == oracle.duplicates(tr, empty, empty, 0.2, 0.1)
    assert dr.cartesian_product_relations(tr, empty, empty, 0.3) == oracle.cartesian_product_relations(
        tr, empty, empty, 0.3)
    d, rd = dr.duplicates(tr, empty, empty, 0.2, 0.1)
    assert dr.count_triplets(tr, empty, d, rd) == (0, 0) == dr.count_triplets(empty, tr, d, rd)
    assert dr.duplicates(empty, empty, empty) == ([], [])
    assert dr.cartesian_product_relations(empty, empty, empty) == []


def test_relations_without_facts(capsys):
    tr, va, te = random_graph(37, 4000, 60, seed=7)
    drop = lambda kg: RefStyleKG(kg.head_idx[kg.relations % 5 != 3], kg.tail_idx[kg.relations % 5 != 3],  # noqa: E731
                                 kg.relations[kg.relations % 5 != 3], kg.n_ent, kg.n_rel)
    tr, va, te = drop(tr), drop(va), drop(te)
    d, rd = same_as_oracle(tr, va, te, capsys, theta1=0.0, theta2=0.0)
    assert not any(a % 5 == 3 or b % 5 == 3 for a, b in d + rd)
    assert not any(x % 5 == 3 for x in dr.cartesian_product_relations(tr, va, te, theta=0.0))


def test_one_entity_pair_carrying_500_relations(capsys):
    """A segment of 500 keys on both sides of the join: the warp's strided loop over 500 x 500 products."""
    tr, va, te = random_graph(600, 6000, 300, seed=11)
    h = torch.cat([tr.head_idx, torch.full((500,), 3), torch.full((400,), 5), torch.full((50,), 7)])
    t = torch.cat([tr.tail_idx, torch.full((500,), 5), torch.full((400,), 3), torch.full((50,), 7)])
    r = torch.cat([tr.relations, torch.arange(500), torch.arange(100, 500), torch.arange(550, 600)])
    tr = RefStyleKG(h, t, r, 300, 600)
    same_as_oracle(tr, va, te, capsys)
    same_as_oracle(tr, va, te, capsys, theta1=0.0, theta2=0.0, counts=False)
    big = [(a, a + 1) for a in range(0, 499, 7)]
    assert dr.count_triplets(tr, tr, big, big) == oracle.count_triplets(tr, tr, big, big)


def test_self_loop_only_relations(capsys):
    g = torch.Generator().manual_seed(13)
    e = torch.randint(0, 30, (600,), generator=g)
    r = torch.randint(0, 12, (600,), generator=g)
    tr = RefStyleKG(e[:400], e[:400], r[:400], 30, 12)
    va = RefStyleKG(e[400:500], e[400:500], r[400:500], 30, 12)
    te = RefStyleKG(e[500:], e[500:], r[500:], 30, 12)
    d, rd = same_as_oracle(tr, va, te, capsys, theta1=0.3, theta2=0.3)
    assert d == rd and d     # a self-loop is its own reverse


def test_count_triplets_with_repeated_and_out_of_range_pairs():
    tr, va, te = random_graph(37, 4000, 60, seed=17)
    d, rd = dr.duplicates(tr, va, te, 0.2, 0.1)
    listed = d + d[:3] + [(5, 5), (36, 0), (37, 1), (-1, 4), (2, 10 ** 6), (1 << 70, 3), [4, 9]]
    rlisted = rd + rd[:1] * 3 + [(7, 7), (-3, -3), (0, 37)]
    for kg1, kg2 in ((tr, te), (te, tr), (va, va)):
        assert dr.count_triplets(kg1, kg2, listed, rlisted) == oracle.count_triplets(kg1, kg2, listed, rlisted)
    assert dr.count_triplets(tr, te, [], []) == (0, 0)


def test_million_facts_with_planted_duplicates(capsys):
    tr, va, te = random_graph(200, 1_000_000, 20_000, seed=19)
    assert len(tr) + len(va) + len(te) > 1_000_000
    d, rd = same_as_oracle(tr, va, te, capsys, theta1=0.4, theta2=0.4)
    assert d and rd
