"""Top-k inference over a range-partitioned entity table: per-shard kge_topk_side calls (global ids
through ``ent_lo``) merged by kge_topk_merge must give the unsharded result bit for bit -- ids,
score bits and the order among exact ties.  Shards are emulated on one device, then the public API
runs in two processes (gloo on one GPU; NCCL when two GPUs are present)."""

import numpy as np
import pytest
import torch

import torchkge_b200 as tk
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard, ModelSpec, QueryShard
from torchkge_b200.inference import _mask_csr

DEV = "cuda:0"
ALL_KINDS = ["transe_l1", "transe_l2", "toruse_l1", "toruse_l2", "distmult", "rescal", "complex",
             "analogy", "rotate"]


# ------------------------------------------------------------------ helpers
def _queries(n_ent, n_rel, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n_ent, (n,), generator=g), torch.randint(0, n_rel, (n,), generator=g)


def _dictionary(ents, rels, n_ent, seed, per_key=25):
    g = torch.Generator().manual_seed(seed)
    d = {}
    for i in range(0, ents.shape[0], 3):
        d[(int(ents[i]), int(rels[i]))] = set(torch.randint(0, n_ent, (per_key,), generator=g).tolist())
    return d


def unsharded(model, ents, rels, k, missing, dictionary):
    inf = tk.EntityInference(model, ents, rels, top_k=k, missing=missing, dictionary=dictionary)
    inf.evaluate(b_size=64)
    return inf.predictions, inf.scores


def emulated(model, ents, rels, k, missing, dictionary, world, eng):
    """One kge_topk_side per shard range [lo, hi) of the table (global ids through ent_lo), padded
    to k with empty slots, then kge_topk_merge -- what topk_entity_inference does per chunk."""
    spec = ModelSpec.from_model(model)
    side = _lib.SIDE_TAIL if missing == "tails" else _lib.SIDE_HEAD
    e, r = ents.to(DEV), rels.to(DEV)
    n = e.shape[0]
    mask = None
    if dictionary is not None:
        offs, ids = _mask_csr(dictionary, ents, rels)
        mask = (offs.to(DEV), ids.to(DEV))
    rows = eng.gather_rows(spec, e)
    pred_in = torch.full((world, n, k), -1, dtype=torch.int64, device=DEV)
    scores_in = torch.full((world, n, k), float("-inf"), dtype=torch.float32, device=DEV)
    for rank in range(world):
        sh = EntityShard(spec.n_ent, rank, world)
        k_loc = min(k, sh.hi - sh.lo)
        if k_loc == 0:
            continue
        sub = spec.narrowed(sh.lo, sh.hi)
        p, s = eng.topk_side(sub, eng.pack(sub), side, rows, rows, r, k_loc, mask)
        pred_in[rank, :, :k_loc], scores_in[rank, :, :k_loc] = p, s
    pred, vals = eng.topk_merge(pred_in, scores_in, k)
    return pred.cpu(), vals.cpu()


def assert_same(got, want):
    (gp, gs), (wp, ws) = got, want
    assert gp.shape == wp.shape
    bad = (gp != wp).any(1).nonzero().flatten()
    assert bad.numel() == 0, "%d lists differ, first at %d:\n got  %s\n want %s" % (
        bad.numel(), bad[0], gp[bad[0]].tolist()[:30], wp[bad[0]].tolist()[:30])
    assert torch.equal(gs.view(torch.int32), ws.view(torch.int32))


def _model(kind, dim, n_ent, n_rel, seed):
    return helpers.make_model(kind, dim, n_ent, n_rel, seed=seed).to(DEV)


# ------------------------------------------------------------------ 1. emulated shards, every model
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_emulated_shards_equal_unsharded(kind):
    n_ent, n_rel, dim = 3000, 7, 16
    model = _model(kind, dim, n_ent, n_rel, seed=5)
    eng = CudaEngine(tensor_core=False)
    ents, rels = _queries(n_ent, n_rel, 300, seed=6)
    dictionary = _dictionary(ents, rels, n_ent, seed=7)
    for missing in ("tails", "heads"):
        for dic in (None, dictionary):
            for k in (1, 10, 100, 1024):
                want = unsharded(model, ents, rels, k, missing, dic)
                for world in (2, 3, 8):
                    assert_same(emulated(model, ents, rels, k, missing, dic, world, eng), want)


# ------------------------------------------------------------------ 2. hard cases
def _entity_weights(model):
    return [getattr(model, n).weight for n in ("ent_emb", "sc_ent_emb", "re_ent_emb", "im_ent_emb")
            if hasattr(model, n)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["distmult", "transe_l2", "complex"])
def test_ties_across_shard_boundaries(kind):
    """Copies of one row and zero rows in every shard: exact ties whose order (ascending global id)
    spans shard boundaries."""
    n_ent, n_rel, dim = 600, 3, 16
    model = _model(kind, dim, n_ent, n_rel, seed=8)
    with torch.no_grad():
        for w in _entity_weights(model):
            for i in (7, 150, 299, 300, 451, 599):
                w[i] = w[3]
            for i in (11, 210, 333, 590):
                w[i] = 0.0
    ents = torch.tensor([3, 7, 11, 42, 150, 333, 590] * 9)
    rels = torch.arange(ents.shape[0]) % n_rel
    eng = CudaEngine(tensor_core=False)
    for missing in ("tails", "heads"):
        for k in (1, 5, 20, 600):
            want = unsharded(model, ents, rels, k, missing, None)
            for world in (2, 3, 8):
                assert_same(emulated(model, ents, rels, k, missing, None, world, eng), want)


@pytest.mark.gpu
def test_nan_rows_in_one_shard():
    n_ent, n_rel, dim = 500, 3, 16
    model = _model("distmult", dim, n_ent, n_rel, seed=9)
    with torch.no_grad():
        model.ent_emb.weight[[260, 263, 300]] = float("nan")     # shard 1 of 2 only
    ents, rels = _queries(n_ent, n_rel, 40, seed=10)
    eng = CudaEngine(tensor_core=False)
    for k in (1, 2, 3, 4, 10):
        want = unsharded(model, ents, rels, k, "tails", None)
        assert torch.isnan(want[1][:, 0]).all()
        assert_same(emulated(model, ents, rels, k, "tails", None, 2, eng), want)


@pytest.mark.gpu
@pytest.mark.parametrize("n_ent,world,k", [(50, 8, 30), (5, 8, 5), (3, 8, 1), (40, 3, 40)])
def test_small_and_empty_shards(n_ent, world, k):
    """Shards with fewer rows than k (padded with empty slots) and, for n_ent < world, shards with
    no rows at all."""
    model = _model("complex", 8, n_ent, 2, seed=11)
    ents, rels = _queries(n_ent, 2, 20, seed=12)
    eng = CudaEngine(tensor_core=False)
    for missing in ("tails", "heads"):
        want = unsharded(model, ents, rels, k, missing, None)
        assert_same(emulated(model, ents, rels, k, missing, None, world, eng), want)


@pytest.mark.gpu
def test_masks_straddling_shards():
    """Mask sets across every shard and k above the unmasked count: the masked -inf entries fill
    the tail of the lists in ascending id order, across the shards."""
    n_ent, n_rel = 40, 2
    model = _model("transe_l2", 8, n_ent, n_rel, seed=13)
    ents = torch.tensor([0, 1, 2, 3, 39])
    rels = torch.tensor([0, 1, 0, 1, 0])
    dictionary = {(0, 0): set(range(2, 38)), (1, 1): set(range(0, 40, 2)), (3, 1): set(range(40)),
                  (39, 0): {5, 12, 13, 14, 26, 27, 39}}
    eng = CudaEngine(tensor_core=False)
    for k in (10, 35, 40):
        want = unsharded(model, ents, rels, k, "tails", dictionary)
        assert torch.isinf(want[1][0, -1]) and torch.isinf(want[1][3]).all()
        for world in (2, 3, 8):
            assert_same(emulated(model, ents, rels, k, "tails", dictionary, world, eng), want)


# ------------------------------------------------------------------ 3. kge_topk_merge on its own
def _score_key(bits):
    """score_key of csrc/topk.cu on the bits of non-NaN floats"""
    u = bits.astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)


def _host_merge(pred_in, scores_in, k):
    """Host restatement: key = (score key << 32) | (0xffffffff - id), descending, empty (-1) last."""
    lists, n, k_in = pred_in.shape
    ids = pred_in.transpose(1, 0, 2).reshape(n, -1)
    s = scores_in.transpose(1, 0, 2).reshape(n, -1)
    skey = _score_key(s.view(np.uint32))
    skey = np.where(np.isnan(s), np.uint64(0xffffffff), skey)
    key = (skey << np.uint64(32)) | ((np.uint64(0xffffffff) - ids.astype(np.uint64)) & np.uint64(0xffffffff))
    key = np.where(ids < 0, np.uint64(0), key)
    order = np.argsort(key, axis=1)[:, ::-1][:, :k]     # keys are unique but for the empty ones
    top = np.take_along_axis(key, order, 1)
    pred = np.where(top == 0, -1, 0xffffffff - (top & np.uint64(0xffffffff)).astype(np.int64))
    sk = (top >> np.uint64(32)).astype(np.uint64)
    sbits = np.where(sk == 0xffffffff, np.uint64(0x7fc00000),
                     np.where(sk & 0x80000000, sk & 0x7fffffff, ~sk & 0xffffffff)).astype(np.uint32)
    vals = sbits.view(np.float32).copy()
    vals[top == 0] = -np.inf
    return pred.astype(np.int64), vals


def _random_lists(rng, n_lists, n, k_in, n_ids, adversarial):
    """Sorted (pred, scores) lists with ids unique per query across the lists and trailing empty
    slots.  Adversarial: scores drawn from a handful of values (±0.0, NaN, ±inf, ties)."""
    pred = np.full((n_lists, n, k_in), -1, np.int64)
    scores = np.full((n_lists, n, k_in), -np.inf, np.float32)
    pool = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.5, -1.5, 2.0], np.float32)
    for q in range(n):
        ids = rng.choice(n_ids, size=n_lists * k_in, replace=False)
        for li in range(n_lists):
            length = int(rng.integers(0, k_in + 1))
            mine = ids[li * k_in:li * k_in + length]
            s = rng.choice(pool, size=length) if adversarial else rng.standard_normal(length).astype(np.float32)
            if length:       # sorted best first by the host restatement of the key order
                p, v = _host_merge(mine.reshape(1, 1, -1), s.reshape(1, 1, -1), length)
                pred[li, q, :length], scores[li, q, :length] = p[0], v[0]
    return pred, scores


@pytest.mark.gpu
@pytest.mark.parametrize("n_lists,k_in,k,adversarial", [(2, 10, 10, False), (3, 7, 5, True), (8, 64, 100, True),
                                                        (64, 16, 1024, False), (64, 1024, 1024, True),
                                                        (5, 1, 1, True), (1, 30, 12, False)])
def test_merge_kernel_against_host(n_lists, k_in, k, adversarial):
    rng = np.random.default_rng(n_lists * 1000 + k)
    n = 4 if k_in == 1024 else 24
    pred_in, scores_in = _random_lists(rng, n_lists, n, k_in, 1 << 30, adversarial)
    eng = CudaEngine()
    got_p, got_s = eng.topk_merge(torch.from_numpy(pred_in).to(DEV), torch.from_numpy(scores_in).to(DEV), k)
    want_p, want_s = _host_merge(pred_in, scores_in, k)
    assert np.array_equal(got_p.cpu().numpy(), want_p)
    assert np.array_equal(got_s.cpu().numpy().view(np.uint32), want_s.view(np.uint32))


@pytest.mark.gpu
def test_merge_signed_zero_across_lists():
    """+0.0 ranks above -0.0 whatever the ids, and the sign bit survives the merge."""
    pred_in = torch.tensor([[[1, 4]], [[9, -1]], [[2, 3]]], dtype=torch.int64, device=DEV)
    scores_in = torch.tensor([[[-0.0, -0.0]], [[0.0, 0.0]], [[0.0, -1.0]]], device=DEV)
    pred, vals = CudaEngine().topk_merge(pred_in, scores_in, 6)
    assert pred.tolist() == [[2, 9, 1, 4, 3, -1]]
    assert torch.signbit(vals[0, :4]).tolist() == [False, False, True, True]
    assert vals[0, 5].item() == float("-inf")


def test_merge_rejects_arguments_out_of_range():
    """Checked before anything touches a device."""
    lib = _lib.load()
    for n_lists, k_in, k in ((0, 4, 4), (65, 4, 4), (2, 4, 0), (2, 4, 1025), (2, 0, 4), (2, 1025, 4)):
        assert lib.kge_topk_merge(None, None, n_lists, 3, k_in, k, None, None, None) == 1
        assert b"kge_topk_merge" in lib.kge_last_error()


# ------------------------------------------------------------------ 4./5. public API, two processes
def _api_worker(rank, world, backend):
    dev = torch.device("cuda:%d" % (rank if backend == "nccl" else 0))
    torch.cuda.set_device(dev)
    try:
        results = {}
        n_ent, n_rel, dim = 1100, 9, 16
        for kind in ("distmult", "complex"):
            model = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
            ents, rels = _queries(n_ent, n_rel, 45, seed=22)
            e2, _ = _queries(n_ent, n_rel, 45, seed=23)
            dictionary = _dictionary(ents, rels, n_ent, seed=24)
            rdict = {(int(a), int(b)): {1, 4} for a, b in zip(ents[::4].tolist(), e2[::4].tolist())}
            ref_e = tk.EntityInference(model, ents, rels, top_k=30, missing="heads", dictionary=dictionary)
            ref_e.evaluate(b_size=8)
            ref_r = tk.RelationInference(model, ents, e2, top_k=4, dictionary=rdict)
            ref_r.evaluate(b_size=8)
            full = EntityShard.from_group(n_ent)
            for name, shard, m in (
                    ("entity-full", full, model),
                    ("entity-local", EntityShard.from_group(n_ent, local_storage=True),
                     helpers.local_model(kind, model, full.lo, full.hi, n_rel, dim)),
                    ("query", QueryShard.from_group(ents.shape[0]), model)):
                got_e = tk.EntityInference(m, ents, rels, top_k=30, missing="heads", dictionary=dictionary,
                                           shard=shard)
                got_e.evaluate(b_size=8)
                got_r = tk.RelationInference(m, ents, e2, top_k=4, dictionary=rdict, shard=shard)
                got_r.evaluate(b_size=8)
                results["%s/%s/entity" % (kind, name)] = (
                    torch.equal(got_e.predictions, ref_e.predictions)
                    and torch.equal(got_e.scores.view(torch.int32), ref_e.scores.view(torch.int32)))
                results["%s/%s/relation" % (kind, name)] = (
                    torch.equal(got_r.predictions, ref_r.predictions)
                    and torch.equal(got_r.scores.view(torch.int32), ref_r.scores.view(torch.int32)))
        return results
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


def _run_two_ranks(backend):
    ret = gloo.spawn(2, _api_worker, backend, backend=backend)
    for rank in (0, 1):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        assert all(res.values()) and len(res) == 12, "rank %d: %s" % (rank, res)


@pytest.mark.gpu
def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
