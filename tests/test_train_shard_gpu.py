"""The entity-sharded fused margin step: per-rank kernel calls on row ranges of one table (the sharded
ring kernel and the generic sharded kernels), summed over the ranks and scattered as the host logic
does, must reproduce the unsharded fused step -- loss within 1e-5 relative, gradients under the
atomics-order rule of tests/test_train_gpu.py.  Shards are emulated on one device, then the public
API trains in two processes (gloo on one GPU; NCCL when two GPUs are present)."""
import ctypes

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import gloo, helpers
from tests import train_kit as kit
from tests.train_kit import DEV
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, _ptr

pytestmark = pytest.mark.gpu
ALL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "analogy", "toruse_l1",
             "toruse_l2"]


# ---------------------------------------------------------------- 1. emulated shards vs unsharded
RING = [(k, d) for k in ("transe_l1", "transe_l2", "distmult") for d in (36, 200, 256)]
GENERIC = [(k, 50 if k != "rescal" else 12) for k in ALL_KINDS] + [(k, 64 if k != "rescal" else 16) for k in ALL_KINDS]
CASES = [(k, d, (1, 33, 256)[i % 3]) for i, (k, d) in enumerate(RING + GENERIC)]


@pytest.mark.parametrize("kind,d,n_neg", CASES, ids=["%s-d%d-neg%d" % c for c in CASES])
def test_emulated_shards_equal_unsharded(kind, d, n_neg):
    # 40 relations: a relation row sums ~b n_neg / 40 hinge terms, which keeps the atomics-order noise of
    # the relation gradients inside the rtol of the rule
    n_ent, n_rel, b = 700, 40, 160
    model = kit.train_model(kind, d, n_ent, n_rel, seed=3)
    h, t, r, probs = kit.batch(n_ent, n_rel, b, d + n_neg)
    kw = dict(n_neg=n_neg, probs=probs, margin=1.0 if kind not in ("transe_l1", "transe_l2") else 0.3, seed=99,
              offset=5)
    want = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        kit.compare(kit.emulated(model, h, t, r, world, eng, **kw), want)


@pytest.mark.parametrize("kind,d", [("distmult", 200), ("transe_l2", 36), ("complex", 50), ("rotate", 64)])
def test_emulated_shards_equal_oracle_autograd(kind, d):
    """Against the oracle's CPU autograd on the negatives kge_corrupt_batch draws at the same seed / offset."""
    n_ent, n_rel, b, n_neg, seed, offset = 500, 5, 96, 33, 4242, 17
    model = kit.train_model(kind, d, n_ent, n_rel, seed=8)
    h, t, r, probs = kit.batch(n_ent, n_rel, b, 9)
    nh, nt = kit.corrupt_batch(h, t, r, probs, n_neg, n_ent, seed, offset)
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    pos, neg = oracle.forward_pos_neg(kind, P, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    ref = oracle.margin_loss(pos, neg, 1.0)
    ref.backward()
    keys = {"distmult": ("ent", None, "rel", None), "transe_l2": ("ent", None, "rel", None)}.get(
        kind, ("re_ent", "im_ent", "re_rel", "im_rel"))
    want = (ref.item(), [None if k is None else P[k].grad for k in keys])
    eng = CudaEngine()
    for world in (2, 3, 8):
        got = kit.emulated(model, h, t, r, world, eng, n_neg=n_neg, probs=probs, margin=1.0, seed=seed,
                           offset=offset)
        assert got[0] == pytest.approx(want[0], rel=2e-5)
        for a, c in zip(got[1], want[1]):
            if c is not None:
                kit.close_grad(a, c, rtol=2e-4)


# ---------------------------------------------------------------- 2. hard cases
HARD = [("distmult", 200), ("transe_l1", 36), ("complex", 50), ("analogy", 64), ("rescal", 12)]


@pytest.mark.parametrize("kind,d", HARD)
@pytest.mark.parametrize("case", ["empty_shards", "tiny", "self_loops", "one_owner"])
def test_hard_cases(kind, d, case):
    n_rel, b, n_neg = 4, 64, 33
    n_ent = {"empty_shards": 5, "tiny": 17}.get(case, 300)
    model = kit.train_model(kind, d, n_ent, n_rel, seed=13)
    h, t, r, _ = kit.batch(n_ent, n_rel, b, 14)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.25], device=DEV)    # Bernoulli 0 and 1: one side only
    if case == "self_loops":
        h[::2] = t[::2]
    if case == "one_owner":                 # every positive held by rank 0 of 8 (rows [0, 38))
        h, t = h % 38, t % 38
    # tiny n_ent: most draws hit a shard's first or last row and many negatives equal their positive
    kw = dict(n_neg=n_neg, probs=probs, margin=1.0, seed=7, offset=3)
    want = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (2, 3, 8):
        kit.compare(kit.emulated(model, h, t, r, world, eng, **kw), want)


# ---------------------------------------------------------------- 3. kge_scatter_rows_add
@pytest.mark.parametrize("kind,planes", [("distmult", 1), ("complex", 2), ("analogy", 3)])
def test_scatter_rows_add_equals_index_add(kind, planes):
    code = {"distmult": _lib.DISTMULT, "complex": _lib.COMPLEX, "analogy": _lib.ANALOGY}[kind]
    n_rows, lo, dim, n = 50, 20, 37, 400
    g = torch.Generator().manual_seed(planes)
    idx = torch.randint(0, 100, (n,), generator=g)          # ids repeat; ids outside [20, 70) are ignored
    idx[:5] = torch.tensor([-3, 19, 20, 69, 70])
    rows = torch.randn(n, planes, dim, generator=g)
    base = torch.randn(planes, n_rows, dim, generator=g)
    want = base.clone()
    own = (idx >= lo) & (idx < lo + n_rows)
    for p in range(planes):
        want[p].index_add_(0, idx[own] - lo, rows[own, p])
    grad = base.to(DEV).contiguous()
    g0, g1 = (grad, None) if planes == 3 else (grad[0], grad[1] if planes == 2 else None)
    CudaEngine().scatter_rows_add(code, dim, g0, g1, lo, idx.to(DEV), rows.to(DEV))
    torch.testing.assert_close(grad.cpu(), want, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------- 4. ABI
def test_margin_step_args_field_order_matches_the_header():
    assert kit.header_fields("kge_margin_step_args_t") == [n for n, _ in _lib.MarginStepArgs._fields_]


def _args(x, hrows=True):
    """Arguments of a sharded step over the float tensor x (pointers only; nothing is launched)."""
    a = _lib.MarginStepArgs()
    a.tb.model, a.tb.dim = _lib.DISTMULT, 4
    a.tb.ent0 = a.tb.rel0 = a.loss = a.bern_probs = _ptr(x)
    a.h = a.t = a.r = _ptr(x)
    a.n_neg, a.b, a.n_ent, a.ent_lo, a.n_rows = 2, 1, 10, 0, 5
    if hrows:
        a.hrows = a.trows = a.grad_hrows = a.grad_trows = _ptr(x)
    return a


def test_sharded_argument_errors():
    lib = _lib.load()
    x = torch.zeros(64, device=DEV)
    g = _lib.Grads()
    g.ent0 = g.rel0 = _ptr(x)
    for field in ("nh", "pos_out", "neg_out", "nh_out"):
        a = _args(x)
        setattr(a, field, _ptr(x))
        if field == "nh":
            a.nt = _ptr(x)
        if field == "nh_out":
            a.nt_out = _ptr(x)
        assert lib.kge_margin_step_fwd(ctypes.byref(a)) == 1      # KGE_ERR_ARG
        assert lib.kge_margin_step_bwd(ctypes.byref(a), ctypes.byref(g), _ptr(x)) == 1
    a = _args(x)
    a.trows = None
    assert lib.kge_margin_step_fwd(ctypes.byref(a)) == 1
    for field in ("grad_hrows", "grad_trows"):
        a = _args(x)
        setattr(a, field, None)
        assert lib.kge_margin_step_bwd(ctypes.byref(a), ctypes.byref(g), _ptr(x)) == 1
    a = _args(x)
    a.n_rows = 0                               # a shard holding no rows: valid, nothing to do
    a.tb.ent0 = None
    assert lib.kge_margin_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()


def test_legacy_calls_still_accept_their_arguments():
    """hrows == NULL: external negatives and every optional output, as before."""
    model = kit.train_model("distmult", 36, 100, 3, seed=1)
    h, t, r, probs = kit.batch(100, 3, 8, 1)
    nh, nt = h.repeat(2), (t.repeat(2) + 1) % 100
    out = kit.forward_outputs(model, h, t, r, margin=1.0, negatives=(nh, nt))
    assert torch.equal(out["nh"], nh) and torch.equal(out["nt"], nt)
    assert out["loss"].item() == pytest.approx(torch.relu(1.0 - out["pos"].repeat(2) + out["neg"]).sum().item(),
                                               rel=1e-5)


# ---------------------------------------------------------------- 5. public API, two processes
def _api_worker(rank, world, backend):
    dev = torch.device("cuda:%d" % (rank if backend == "nccl" else 0))
    torch.cuda.set_device(dev)
    try:
        res, kg, batches, local, shard = kit.whole_against_shard(
            (("distmult", 200, 1.0), ("complex", 50, 1.0)),
            lambda kg: tk.BernoulliNegativeSampler(kg, n_neg=16, seed=3), dev, 5, on_ranks=True)
        # a seed that differs between the ranks raises on every rank instead of hanging
        sampler = tk.BernoulliNegativeSampler(kg, n_neg=4, seed=100 + rank)
        try:
            sampler.fused_step(local, *batches[0], 1.0, shard=shard)
            res["seed_mismatch_raises"] = False
        except ValueError:
            res["seed_mismatch_raises"] = True
        return res
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


def _run_two_ranks(backend):
    kit.every_rank_ok(gloo.spawn(2, _api_worker, backend, backend=backend), 2, min_checks=12)


def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
