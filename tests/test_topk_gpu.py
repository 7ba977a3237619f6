"""Top-k inference (EntityInference / RelationInference, csrc/topk.cu) against an exact CPU
reference -- the predicted ids and the bits of their scores -- where the selection leaves its small
single-pass form: several collect passes (csrc/api.cu: kge_topk_side), the bitonic merge, k up to
TOPK_MAX_K, the query split of inference.py, NaN and signed-zero scores, and RESCAL's dense path
(kge_rescal_rel_scores + kge_topk_dense).  Each test that targets one of these branches asserts
that it ran, so that a change of a budget constant cannot quietly turn it into a one-pass test."""
import copy
from collections import defaultdict

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200 import _lib, inference
from torchkge_b200 import engine as engine_mod

pytestmark = pytest.mark.gpu

N_ENT, N_REL, DIM = 5000, 13, 16
#: the first call of EntityInference takes 16,384 queries (three collect passes: 2048 + 2048 + 904
#: rows), the second the remaining 1,000 (one pass)
N_QUERIES = 17384
NAN_ROWS = list(range(3000, 3012))     # rows of the second collect pass of the 16,384-query call
SORT_N = 2048                          # keys per bitonic sort in topk_merge_kernel (csrc/topk.cu)


# ------------------------------------------------------------------ reference
def topk_chunk_rows(n, n_rows):
    """Candidate rows per collect pass of kge_topk_side, as topk_chunk_rows in csrc/api.cu computes
    them: the (score, id) lists of one pass (8 bytes an entry) hold at most 256 MB over n queries;
    a multiple of the candidate tile, at least one tile, at most the (tile-rounded) table."""
    rows = (256 << 20) // (8 * max(n, 1))
    rows = max(rows // _lib.TILE_C * _lib.TILE_C, _lib.TILE_C)
    return min(rows, -(-n_rows // _lib.TILE_C) * _lib.TILE_C)


def collect_passes(n, n_rows):
    return -(-n_rows // topk_chunk_rows(n, n_rows))


def expected_topk(dense, k, block=1024):
    """(ids int64 (n, k), scores float32 (n, k)) of the k best columns of every row of ``dense``
    (masked entries already -inf): NaN first, then scores descending, exact ties by ascending id.
    +0.0 and -0.0 do not tie: +0.0 comes first, as the kernel orders them (csrc/topk.cu)."""
    ids, vals = [], []
    for lo in range(0, dense.shape[0], block):
        s = dense[lo:lo + block]
        key = s.double()
        key[(s == 0) & torch.signbit(s)] = -1e-300      # below +0.0, above every negative float32
        key[torch.isnan(s)] = float("nan")              # one NaN, whatever its sign bit
        # a stable descending sort keeps equal keys in ascending id order and puts NaN first
        order = torch.sort(key, dim=1, descending=True, stable=True).indices[:, :k]
        ids.append(order)
        vals.append(s.gather(1, order))
    return torch.cat(ids), torch.cat(vals)


def assert_topk(pred, vals, want_ids, want_vals):
    """ids exactly; scores bit for bit, NaN matched as NaN (the kernel returns one canonical NaN)."""
    pred, vals = pred.cpu(), vals.cpu()
    assert pred.shape == want_ids.shape and vals.shape == want_vals.shape
    bad = (pred != want_ids).any(1).nonzero().flatten()
    assert bad.numel() == 0, "%d / %d lists differ, first at query %d:\n got  %s\n want %s" % (
        bad.numel(), pred.shape[0], bad[0], pred[bad[0]].tolist()[:40], want_ids[bad[0]].tolist()[:40])
    nan_g, nan_w = torch.isnan(vals), torch.isnan(want_vals)
    assert torch.equal(nan_g, nan_w)
    same = vals.view(torch.int32) == want_vals.view(torch.int32)
    assert (same | nan_w).all(), "score bits differ at %s" % (~(same | nan_w)).nonzero()[:5].tolist()


def _masked(dense, key1, key2, dictionary):
    out = dense.clone()
    for i, (a, b) in enumerate(zip(key1.tolist(), key2.tolist())):
        s = dictionary.get((a, b))
        if s:
            out[i, sorted(s)] = -float("inf")
    return out


@pytest.fixture
def calls(monkeypatch):
    """A fresh default engine that records every top-k call: ('side', queries, mask entries) or
    ('dense', rows, columns, k, mask entries)."""
    eng = engine_mod.CudaEngine()
    seen = []
    topk_side, topk_dense = eng.topk_side, eng.topk_dense

    def side(spec, packed, s, hrows, trows, r_idx, k, mask=None):
        seen.append(("side", hrows.shape[0], 0 if mask is None else mask[1].numel()))
        return topk_side(spec, packed, s, hrows, trows, r_idx, k, mask)

    def dense(scores, k, mask=None):
        seen.append(("dense", scores.shape[0], scores.shape[1], k, 0 if mask is None else mask[1].numel()))
        return topk_dense(scores, k, mask)

    monkeypatch.setattr(eng, "topk_side", side)
    monkeypatch.setattr(eng, "topk_dense", dense)
    monkeypatch.setattr(engine_mod, "_default_engine", eng)
    return seen


# ------------------------------------------------------------------ 5,000 entities, 17,384 queries
def _entity_planes(model):
    return [getattr(model, n).weight for n in ("ent_emb", "re_ent_emb", "im_ent_emb") if hasattr(model, n)]


_CASES = {}


def _case(kind, missing, device):
    """Model, queries, dictionary and the oracle's (unmasked and masked) dense scores, built once
    per (kind, missing) for the whole module."""
    key = (kind, missing)
    if key in _CASES:
        return _CASES[key]
    model = helpers.make_model(kind, DIM, N_ENT, N_REL, seed=11)
    with torch.no_grad():
        for w in _entity_planes(model):
            if kind in ("distmult", "complex"):
                w[100:120] *= 3.0                  # larger rows: they lead many lists of the bilinear kinds
            w[2100:2120] = w[100:120]              # exact copies in the second and third passes:
            w[4100:4120] = w[100:120]              # ties across pass boundaries
    model = model.to(device)
    P = helpers.oracle_params(kind, model)
    g = torch.Generator().manual_seed(7)
    known = torch.randint(0, N_ENT, (N_QUERIES,), generator=g)
    rels = torch.randint(0, N_REL, (N_QUERIES,), generator=g)
    side = "tail" if missing == "tails" else "head"
    dense = torch.cat([oracle.scores_all(kind, P, known[lo:lo + 1024], known[lo:lo + 1024], rels[lo:lo + 1024], side)
                       for lo in range(0, N_QUERIES, 1024)])
    # every third query masks ids of passes 2 and 3: those of its unmasked top 12, four random ones
    # and, every ninth query, the first NaN rows of the NaN tests
    best = expected_topk(dense, 12)[0]
    dictionary = defaultdict(set)
    for i in range(0, N_QUERIES, 3):
        s = dictionary[(int(known[i]), int(rels[i]))]
        s.update(x for x in best[i].tolist() if x >= 2048)
        s.update(torch.randint(2048, N_ENT, (4,), generator=g).tolist())
        if i % 9 == 0:
            s.update(NAN_ROWS[:3])
    masked = _masked(dense, known, rels, dictionary)
    # masked ids that would be in the top k, on both sides of the 16,384 split
    hit = torch.isinf(masked.gather(1, best[:, :10])).any(1)
    assert hit[:16384].any() and hit[16384:].any()
    _CASES[key] = c = dict(model=model, known=known, rels=rels, dictionary=dictionary, dense=dense, masked=masked)
    return c


def _run_entity(c, k, missing, calls):
    inf = tk.EntityInference(c["model"], c["known"], c["rels"], top_k=k, missing=missing, dictionary=c["dictionary"])
    inf.evaluate(b_size=256, verbose=False)
    # the query split of inference.py, each call with a mask, three collect passes then one
    assert inference._MAX_QUERIES_PER_CALL == 16384
    assert [x[:2] for x in calls] == [("side", 16384), ("side", 1000)] and all(x[2] > 0 for x in calls)
    assert collect_passes(16384, N_ENT) == 3 and topk_chunk_rows(16384, N_ENT) == 2048
    assert collect_passes(1000, N_ENT) == 1
    return inf


@pytest.mark.parametrize("kind,missing,k", [
    ("distmult", "tails", 1), ("distmult", "tails", 10),
    ("distmult", "tails", 32), ("distmult", "tails", 33),      # warp insert / bitonic boundary
    ("distmult", "tails", 1024),                               # TOPK_MAX_K: the first pass sorts twice
    ("transe_l2", "heads", 10), ("complex", "tails", 10), ("rotate", "heads", 10)])
def test_entity_topk_over_several_passes(kind, missing, k, calls, cuda_device):
    c = _case(kind, missing, cuda_device)
    inf = _run_entity(c, k, missing, calls)
    want_ids, want_vals = expected_topk(c["masked"], k + 1)
    # exact ties at the k-th place between ids of different passes of the first call
    kth, nxt = want_ids[:16384, k - 1], want_ids[:16384, k]
    tied = (want_vals[:16384, k - 1] == want_vals[:16384, k]) & (kth // 2048 != nxt // 2048)
    assert tied.any()
    assert_topk(inf.predictions, inf.scores, want_ids[:, :k], want_vals[:, :k])


def test_top_k_above_the_limit_raises(cuda_device):
    model = helpers.make_model("distmult", 8, 2000, 3).to(cuda_device)
    e, r = torch.arange(5), torch.zeros(5, dtype=torch.long)
    with pytest.raises(_lib.KgeLibraryError):
        tk.EntityInference(model, e, r, top_k=1025).evaluate(b_size=4)


@pytest.mark.parametrize("n_nan", [1, 12])
def test_nan_rows_in_a_later_pass(n_nan, calls, cuda_device):
    """NaN rows in the second pass come first in every list that does not mask them.  With 12 of
    them and k = 10 the threshold becomes NaN, so the third pass collects all of its 904 rows
    (!(s < NaN)) and merges them on the bitonic path."""
    k = 10
    c = _case("distmult", "tails", cuda_device)
    rows = NAN_ROWS[:n_nan]
    model = copy.deepcopy(c["model"])
    with torch.no_grad():
        model.ent_emb.weight[rows] = float("nan")
    dense = c["dense"].clone()
    # a DistMult score is NaN when the candidate's row or the query's known entity holds a NaN
    dense[:, rows] = float("nan")
    dense[torch.isin(c["known"], torch.tensor(rows))] = float("nan")
    masked = _masked(dense, c["known"], c["rels"], c["dictionary"])
    inf = _run_entity(dict(c, model=model), k, "tails", calls)
    want_ids, want_vals = expected_topk(masked, k)
    # lists that do not mask the first NaN row, of queries that are not NaN themselves
    open_ = ~torch.isinf(masked[:, rows[0]]) & ~torch.isin(c["known"], torch.tensor(rows))
    assert open_.any() and torch.isinf(masked[:, rows[0]]).any()
    assert (inf.predictions[open_, 0] == rows[0]).all()
    if n_nan > k:
        nan_thr = torch.isnan(want_vals[:16384, k - 1])
        assert nan_thr.any() and N_ENT - 2 * 2048 > 128      # pass 3 lists exceed the warp path
    assert_topk(inf.predictions, inf.scores, want_ids, want_vals)


# ------------------------------------------------------------------ signed zeros
def test_zero_rows_tie_in_id_order(calls, cuda_device):
    """Candidate rows of +0.0 and of -0.0, interleaved by id, against positive queries: their scores
    are sums that start from +0.0 in ATen, so every one of them is +0.0; they tie, in id order."""
    n_ent, n_rel, d, k = 64, 2, 8, 40
    model = helpers.make_model("distmult", d, n_ent, n_rel, seed=1)
    with torch.no_grad():
        w = model.ent_emb.weight
        w[:4] = w[:4].abs() + 0.5
        w[4::2] = 0.0
        w[5::2] = -0.0
        model.rel_emb.weight.copy_(model.rel_emb.weight.abs() + 0.5)
    model = model.to(cuda_device)
    P = helpers.oracle_params("distmult", model)
    known = torch.tensor([0, 1, 2, 3, 0, 3])
    rels = torch.tensor([0, 0, 1, 1, 1, 0])
    dense = oracle.scores_all("distmult", P, known, known, rels, "tail")
    assert (dense[:, 4:].view(torch.int32) == 0).all()
    inf = tk.EntityInference(model, known, rels, top_k=k, missing="tails")
    inf.evaluate(b_size=8, verbose=False)
    assert calls == [("side", 6, 0)] and collect_passes(6, n_ent) == 1
    assert_topk(inf.predictions, inf.scores, *expected_topk(dense, k))


@pytest.mark.parametrize("k", [20, 64])
def test_signed_zero_order(k, cuda_device):
    """The merge kernel's order of +0.0 and -0.0, pinned on a dense matrix (kge_topk_dense): they do
    not tie -- +0.0 above -0.0, each group by ascending id -- and the sign bit of the score is kept.
    k = 20 takes the warp insert path (100 candidates), k = 64 the bitonic sort."""
    n, n_c = 8, 100
    g = torch.Generator().manual_seed(k)
    s = torch.where(torch.arange(n_c) % 8 == 0, torch.tensor(0.0), torch.tensor(-0.0)).repeat(n, 1)
    s[:, 90:] = torch.randn(n, 10, generator=g)          # a few non-zero scores around them
    s[1] = s[1].flip(0)
    s[2, ::3] = 0.0
    want_ids, want_vals = expected_topk(s, k)
    z = want_vals == 0
    assert torch.signbit(want_vals[z]).any() and (~torch.signbit(want_vals[z])).any()
    pred, vals = engine_mod.CudaEngine().topk_dense(s.to(cuda_device), k)
    assert_topk(pred, vals, want_ids, want_vals)


# ------------------------------------------------------------------ RESCAL relation inference
def _rescal_relation_case(d, n_ent, n_rel, n, seed):
    model = helpers.make_model("rescal", d, n_ent, n_rel, seed=seed)
    h, t, r = helpers.random_graph(n_ent, min(n_rel, 40), max(4 * n, 400), seed=seed)
    return model, h[:n], t[:n], r[:n]


@pytest.mark.parametrize("k", [5, 40])
def test_rescal_relation_topk_many_relations(k, calls, cuda_device):
    """2,100 relation matrices: kge_topk_dense merges more candidates than one bitonic sort takes
    (SORT_N - k new ones), so every list is sorted several times; copies of matrices 10..19 make
    exact ties, and the dictionary masks relations that would be in the top k."""
    d, n_ent, n_rel, n = 8, 300, 2100, 500
    model, h, t, r = _rescal_relation_case(d, n_ent, n_rel, n, seed=5)
    with torch.no_grad():
        m = model.rel_mat.weight
        m[1010:1020] = m[10:20]
        m[2010:2020] = m[10:20]
    model = model.to(cuda_device)
    P = helpers.oracle_params("rescal", model)
    dense = oracle.relation_scores_all("rescal", P, h, t)
    dr = oracle.build_rel_dict(h, t, r)
    best = expected_topk(dense, 3)[0]
    for i in range(0, n, 2):
        dr[(int(h[i]), int(t[i]))].update(best[i].tolist())
    masked = _masked(dense, h, t, dr)
    inf = tk.RelationInference(model, h, t, top_k=k, dictionary=dr)
    inf.evaluate(b_size=64, verbose=False)
    assert calls == [("dense", n, n_rel, k, calls[0][4])] and calls[0][4] > 0
    assert n_rel > SORT_N - k
    if not helpers.rescal_order_matches_here(d):
        pytest.skip("oneMKL on this CPU sums RESCAL's batched matmul in another order than the authoring machine")
    want_ids, want_vals = expected_topk(masked, k + 1)
    assert (want_vals[:, :k] == want_vals[:, 1:]).any()   # exact ties inside the lists
    assert_topk(inf.predictions, inf.scores, want_ids[:, :k], want_vals[:, :k])


def test_rescal_relation_topk_large_dim(calls, cuda_device):
    """dim = 800: kge_rescal_rel_scores needs more than 48 KB of dynamic shared memory (8 facts x
    2 x 800 floats per CTA); the scores of every relation equal the oracle's bits."""
    d, n_ent, n_rel, n = 800, 40, 5, 24
    assert 2 * 8 * d * 4 > 48 * 1024
    model, h, t, _ = _rescal_relation_case(d, n_ent, n_rel, n, seed=6)
    model = model.to(cuda_device)
    P = helpers.oracle_params("rescal", model)
    dense = oracle.relation_scores_all("rescal", P, h, t)
    inf = tk.RelationInference(model, h, t, top_k=n_rel)
    inf.evaluate(b_size=8, verbose=False)
    assert [x[:4] for x in calls] == [("dense", n, n_rel, n_rel)]
    want_ids, want_vals = expected_topk(dense, n_rel)
    if not helpers.rescal_order_matches_here(d):     # this CPU's MKL sums differently
        torch.testing.assert_close(inf.scores, want_vals, rtol=1e-5, atol=1e-5)
        return
    assert_topk(inf.predictions, inf.scores, want_ids, want_vals)
