"""``duplicates``, ``count_triplets`` and ``cartesian_product_relations`` with the reference's names,
signatures and results (torchkge/utils/data_redundancy.py): the analysis of Akrami et al. (SIGMOD 2020)
that finds duplicate, reverse-duplicate and Cartesian-product relations, to be run before trusting
link-prediction numbers on FB15k-like data.

Facts are the concatenation of the three graphs (``concat_kgs``).  ``T[r]`` is the set of distinct
``(h, t)`` with relation ``r``, ``T_inv[r]`` the set of ``(t, h)``, and ``lengths[r]`` counts the facts
of ``r`` WITH multiplicity, so repeated facts raise the length but not the intersections.  A pair
``r1 < r2`` is a duplicate when ``|T[r1] & T[r2]| / lengths[r1] > theta1`` and ``... / lengths[r2] >
theta2`` (float64 division of exact integers: the bits of Python's true division), a reverse duplicate
when the same holds for ``T[r1] & T_inv[r2]`` and ``(r1, r2) not in reverses``.  A relation is a
Cartesian-product relation when ``lengths[r] / (|S_r| * |O_r|) > theta`` (distinct heads and tails).
Only ``head_idx``, ``tail_idx``, ``relations``, ``n_ent``, ``n_rel`` and ``len()`` of a graph are read,
so the reference's ``KnowledgeGraph`` works as well as this package's.

How it runs (DESIGN.md, "Data redundancy"): each graph becomes one sorted, deduplicated int64 key array
``(h * n_ent + t) * n_rel + r`` cut into segments of equal ``(h, t)``; ``kge_cooccurrence``
(csrc/redundancy.cu) joins two such arrays on ``(h, t)`` -- or ``(t, h)`` -- and counts relation pairs
into a dense ``n_rel x n_rel`` matrix of 64-bit counters.  The threshold tests run on the device over
its upper triangle, whose row-major order is the reference's ``combinations`` order.  Work runs on the
current CUDA device; without one ``KgeLibraryError`` is raised (there is no CPU path).  Nothing prints
progress bars; ``verbose`` and ``counts`` print the reference's lines verbatim.

Deviations, on purpose:

1. All relations are compared: pairs run over ``range(kg_tr.n_rel)``, where the reference hard-codes
   ``combinations(range(1345), 2)`` (data_redundancy.py:147) -- KeyError with fewer relations, relations
   past 1,344 silently skipped with more.  On graphs of 1,345 relations the two agree.
2. A relation with no facts (``lengths[r] == 0``) belongs to no pair and is never a Cartesian-product
   relation; the reference raises ZeroDivisionError (data_redundancy.py:150, 234).
3. Input checks, each a ``ValueError`` raised on the host before any device work: relation ids outside
   ``[0, kg_tr.n_rel)`` in any of the three graphs (``count_triplets``: each graph's ids outside
   ``[0, kg.n_rel)``), which the reference ignores; entity ids outside ``[0, n_ent)``; ``theta1`` or
   ``theta2`` outside ``[0, 1]``; ``n_ent^2 * n_rel >= 2^63`` (the key packing, as in ``FilterIndex``);
   and a counter matrix of more than ``MAX_COUNTER_BYTES`` (512 MiB: up to 8,192 relations; the usual
   benchmarks have 11 to 1,345, Wikidata5M 822).
"""
import torch

from . import _lib
from .engine import _ptr, _stream

#: bytes of one n_rel x n_rel matrix of 64-bit counters, at most (n_rel <= 8192)
MAX_COUNTER_BYTES = 1 << 29


def _check_ids(what, x, hi):
    if x.numel() and (int(x.min()) < 0 or int(x.max()) >= hi):
        raise ValueError("%s outside [0, %d)" % (what, hi))


def _check_sizes(n_ent, n_rel, counters):
    if n_ent * n_ent * n_rel >= 2 ** 63:
        raise ValueError("the (head, tail, relation) key does not fit in int64: n_ent^2 * n_rel = %d^2 * %d"
                         % (n_ent, n_rel))
    if counters and 8 * n_rel * n_rel > MAX_COUNTER_BYTES:
        raise ValueError("%d relations need %d bytes per counter matrix; at most %d are allowed (%d relations)"
                         % (n_rel, 8 * n_rel * n_rel, MAX_COUNTER_BYTES, int((MAX_COUNTER_BYTES // 8) ** 0.5)))


def _check_graph(kg, n_ent, n_rel, name):
    _check_ids(name + " relation ids", kg.relations, n_rel)
    _check_ids(name + " head ids", kg.head_idx, n_ent)
    _check_ids(name + " tail ids", kg.tail_idx, n_ent)


def _device():
    if not torch.cuda.is_available():
        raise _lib.KgeLibraryError("the data-redundancy analysis runs on a CUDA device; there is no CPU fallback")
    _lib.load()
    return torch.device("cuda", torch.cuda.current_device())


def _facts(kgs, dev):
    """(h, t, r) of the concatenated graphs, int64 on ``dev``."""
    return tuple(torch.cat([getattr(kg, a).to(dev, torch.int64) for kg in kgs])
                 for a in ("head_idx", "tail_idx", "relations"))


class _Segments:
    """The distinct keys (h * n_ent + t) * n_rel + r of a set of facts, sorted, and their segments of equal
    (h, t): keys[offs[s]:offs[s+1]] share the pair pairs[s] = h * n_ent + t."""

    def __init__(self, h, t, r, n_ent, n_rel):
        self.keys = torch.unique((h * n_ent + t) * n_rel + r)
        self.pairs, size = torch.unique_consecutive(torch.div(self.keys, n_rel, rounding_mode="floor"),
                                                    return_counts=True)
        self.offs = torch.zeros(self.pairs.numel() + 1, dtype=torch.int64, device=h.device)
        torch.cumsum(size, 0, out=self.offs[1:])


def _cooccurrence(left, right, n_ent, n_rel, flip, upper):
    """counts[a][b] = |{(h, t) of a in left} & {(h, t) of b in right}| -- (t, h) on the right when flip --
    as an (n_rel, n_rel) int64 matrix; upper: only a < b, the rest zero."""
    dev = left.keys.device
    counts = torch.zeros((n_rel, n_rel), dtype=torch.int64, device=dev)
    _lib.check(_lib.load().kge_cooccurrence(
        _ptr(left.keys), _ptr(left.offs), _ptr(left.pairs), left.pairs.numel(),
        _ptr(right.keys), _ptr(right.offs), _ptr(right.pairs), right.pairs.numel(),
        n_ent, n_rel, int(flip), int(upper), _ptr(counts), _stream(dev)), "kge_cooccurrence")
    return counts


def _pairs_above(counts, lengths, theta1, theta2):
    """[(r1, r2)] with r1 < r2, both relations non-empty, counts / lengths[r1] > theta1 and counts /
    lengths[r2] > theta2, in row-major (``combinations``) order."""
    inter = counts.double()
    length = lengths.double()
    keep = (inter / length[:, None] > theta1) & (inter / length[None, :] > theta2)
    nonempty = lengths > 0
    keep &= torch.triu(nonempty[:, None] & nonempty[None, :], diagonal=1)
    return [(a, b) for a, b in keep.nonzero().tolist()]


def count_triplets(kg1, kg2, duplicates, rev_duplicates):
    """(n_duplicates, n_rev_duplicates): the number of triplets of ``kg2`` that have their duplicate
    (reverse duplicate) triplet in ``kg1`` (torchkge/utils/data_redundancy.py:35-79).

    For every listed pair ``(r1, r2)``, as often as it is listed, adds ``|pairs_kg2(r1) & pairs_kg1(r2)|
    + |pairs_kg2(r2) & pairs_kg1(r1)|``, with the (t, h) pairs of ``kg1`` for the reverse count.  Ids
    outside ``[0, max(kg1.n_rel, kg2.n_rel))`` contribute 0, as the empty sets do in the reference."""
    n_rel = max(int(kg1.n_rel), int(kg2.n_rel))
    n_ent = max(int(kg1.n_ent), int(kg2.n_ent))
    _check_sizes(n_ent, n_rel, counters=True)
    _check_graph(kg1, n_ent, int(kg1.n_rel), "kg1")
    _check_graph(kg2, n_ent, int(kg2.n_rel), "kg2")
    dev = _device()
    seg1 = _Segments(*_facts([kg1], dev), n_ent, n_rel)
    seg2 = _Segments(*_facts([kg2], dev), n_ent, n_rel)
    out = []
    for listed, flip in ((duplicates, False), (rev_duplicates, True)):
        valid = [(int(a), int(b)) for a, b in listed]
        valid = [(a, b) for a, b in valid if 0 <= a < n_rel and 0 <= b < n_rel]
        if not valid:
            out.append(0)
            continue
        counts = _cooccurrence(seg2, seg1, n_ent, n_rel, flip, upper=False)
        a, b = torch.tensor(valid, dtype=torch.int64, device=dev).unbind(1)
        out.append(int((counts[a, b] + counts[b, a]).sum()))
    return out[0], out[1]


def duplicates(kg_tr, kg_val, kg_te, theta1=0.8, theta2=0.8, verbose=False, counts=False, reverses=None):
    """(duplicates, rev_duplicates): lists of ``(r1, r2)`` with ``r1 < r2`` in lexicographic order, the
    duplicate and reverse duplicate relations of Akrami et al. (torchkge/utils/data_redundancy.py:82-187)
    over the facts of the three graphs.  ``reverses``: known reverse relations; a qualifying pair is
    dropped from the reverse list when ``(r1, r2) in reverses``.  ``counts``: print, as the reference
    does, how many train and test triplets have a (reverse) duplicate in the train and test sets."""
    theta1, theta2 = float(theta1), float(theta2)
    for name, th in (("theta1", theta1), ("theta2", theta2)):
        if not 0.0 <= th <= 1.0:
            raise ValueError("%s must be in [0, 1], got %r" % (name, th))
    n_rel = int(kg_tr.n_rel)
    n_ent = max(int(kg.n_ent) for kg in (kg_tr, kg_val, kg_te))
    _check_sizes(n_ent, n_rel, counters=True)
    for name, kg in (("kg_tr", kg_tr), ("kg_val", kg_val), ("kg_te", kg_te)):
        _check_graph(kg, n_ent, n_rel, name)
    dev = _device()

    if verbose:
        print('Computing Ts')
    if reverses is None:
        reverses = []
    h, t, r = _facts([kg_tr, kg_val, kg_te], dev)
    lengths = torch.bincount(r, minlength=n_rel)
    seg = _Segments(h, t, r, n_ent, n_rel)

    if verbose:
        print('Finding duplicate relations')
    dupl = _pairs_above(_cooccurrence(seg, seg, n_ent, n_rel, flip=False, upper=True), lengths, theta1, theta2)
    rev_dupl = [p for p in _pairs_above(_cooccurrence(seg, seg, n_ent, n_rel, flip=True, upper=True), lengths,
                                        theta1, theta2)
                if p not in reverses]

    if verbose:
        print('Duplicate relations: {}'.format(len(dupl)))
        print('Reverse duplicate relations: '
              '{}\n'.format(len(rev_dupl)))

    if counts:
        # the reference's lines, its percentages included (the duplicate ones are not multiplied by 100)
        d, rv = count_triplets(kg_tr, kg_tr, dupl, rev_dupl)
        print('{} train triplets have duplicate in train set '
              '({}%)'.format(d, int(d / len(kg_tr))))
        print('{} train triplets have reverse duplicate in train set '
              '({}%)\n'.format(rv, int(rv / len(kg_tr) * 100)))

        d, rv = count_triplets(kg_tr, kg_te, dupl, rev_dupl)
        print('{} test triplets have duplicate in train set '
              '({}%)'.format(d, int(d / len(kg_te))))
        print('{} test triplets have reverse duplicate in train set '
              '({}%)\n'.format(rv, int(rv / len(kg_te) * 100)))

        d, rv = count_triplets(kg_te, kg_te, dupl, rev_dupl)
        print('{} test triplets have duplicate in test set '
              '({}%)'.format(d, int(d / len(kg_te))))
        print('{} test triplets have reverse duplicate in test set '
              '({}%)\n'.format(rv, int(rv / len(kg_te) * 100)))

    return dupl, rev_dupl


def cartesian_product_relations(kg_tr, kg_val, kg_te, theta=0.8):
    """Ids, ascending, of the relations with ``lengths[r] / (|S_r| * |O_r|) > theta`` over the facts of the
    three graphs (torchkge/utils/data_redundancy.py:190-237); the ratio exceeds 1 when facts repeat."""
    n_rel = int(kg_tr.n_rel)
    n_ent = max(int(kg.n_ent) for kg in (kg_tr, kg_val, kg_te))
    _check_sizes(n_ent, n_rel, counters=False)
    for name, kg in (("kg_tr", kg_tr), ("kg_val", kg_val), ("kg_te", kg_te)):
        _check_graph(kg, n_ent, n_rel, name)
    dev = _device()
    h, t, r = _facts([kg_tr, kg_val, kg_te], dev)
    lengths = torch.bincount(r, minlength=n_rel)
    n_heads = torch.bincount(torch.div(torch.unique(r * n_ent + h), n_ent, rounding_mode="floor"), minlength=n_rel)
    n_tails = torch.bincount(torch.div(torch.unique(r * n_ent + t), n_ent, rounding_mode="floor"), minlength=n_rel)
    # n_rel integers per vector: the test runs in Python's exact integer-over-integer division
    return [i for i, (n, s, o) in enumerate(zip(lengths.tolist(), n_heads.tolist(), n_tails.tolist()))
            if n > 0 and n / (s * o) > theta]
