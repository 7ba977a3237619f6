"""The entity-sharded fused margin step: per-rank kernel calls on row ranges of one table (the sharded
ring kernel and the generic sharded kernels), summed over the ranks and scattered as the host logic
does, must reproduce the unsharded fused step -- loss within 1e-5 relative, gradients under the
atomics-order rule of tests/test_train_gpu.py.  Shards are emulated on one device, then the public
API trains in two processes (gloo on one GPU; NCCL when two GPUs are present)."""
import ctypes
import os
import re

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard, _ptr, _stream
from torchkge_b200.training import _MarginStep

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "analogy", "toruse_l1",
             "toruse_l2"]


def _batch(n_ent, n_rel, b, seed):
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, n_ent, (b,), generator=g)
    t = torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, n_rel, (b,), generator=g)
    probs = torch.rand(n_rel, generator=g)
    return h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)


def _compare(got, want, rtol=1e-4):
    (gl, gg), (wl, wg) = got, want
    assert gl == pytest.approx(wl, rel=1e-5, abs=1e-6)
    for a, b in zip(gg, wg):
        if b is not None:
            helpers.close_grad(a, b, rtol)


# ---------------------------------------------------------------- 1. emulated shards vs unsharded
RING = [(k, d) for k in ("transe_l1", "transe_l2", "distmult") for d in (36, 200, 256)]
GENERIC = [(k, 50 if k != "rescal" else 12) for k in ALL_KINDS] + [(k, 64 if k != "rescal" else 16) for k in ALL_KINDS]
CASES = [(k, d, (1, 33, 256)[i % 3]) for i, (k, d) in enumerate(RING + GENERIC)]


@pytest.mark.parametrize("kind,d,n_neg", CASES, ids=["%s-d%d-neg%d" % c for c in CASES])
def test_emulated_shards_equal_unsharded(kind, d, n_neg):
    # 40 relations: a relation row sums ~b n_neg / 40 hinge terms, which keeps the atomics-order noise of
    # the relation gradients inside the rtol of the rule
    n_ent, n_rel, b = 700, 40, 160
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=3)
    h, t, r, probs = _batch(n_ent, n_rel, b, seed=d + n_neg)
    margin = 1.0 if kind not in ("transe_l1", "transe_l2") else 0.3
    want = helpers.unsharded(model, h, t, r, probs, margin, n_neg, 99, 5)
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        _compare(helpers.emulated(model, h, t, r, probs, margin, n_neg, 99, 5, world, eng), want)


@pytest.mark.parametrize("kind,d", [("distmult", 200), ("transe_l2", 36), ("complex", 50), ("rotate", 64)])
def test_emulated_shards_equal_oracle_autograd(kind, d):
    """Against the oracle's CPU autograd on the negatives kge_corrupt_batch draws at the same seed / offset."""
    n_ent, n_rel, b, n_neg, seed, offset = 500, 5, 96, 33, 4242, 17
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=8)
    h, t, r, probs = _batch(n_ent, n_rel, b, seed=9)
    nh = torch.empty(b * n_neg, dtype=torch.int64, device=DEV)
    nt = torch.empty_like(nh)
    _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), b, n_neg, _ptr(probs), n_ent, seed, offset,
                                             _ptr(nh), _ptr(nt), _stream(h.device)), "kge_corrupt_batch")
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    pos, neg = oracle.forward_pos_neg(kind, P, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    ref = oracle.margin_loss(pos, neg, 1.0)
    ref.backward()
    keys = {"distmult": ("ent", None, "rel", None), "transe_l2": ("ent", None, "rel", None)}.get(
        kind, ("re_ent", "im_ent", "re_rel", "im_rel"))
    want = (ref.item(), [None if k is None else P[k].grad for k in keys])
    eng = CudaEngine()
    for world in (2, 3, 8):
        got = helpers.emulated(model, h, t, r, probs, 1.0, n_neg, seed, offset, world, eng)
        assert got[0] == pytest.approx(want[0], rel=2e-5)
        for a, c in zip(got[1], want[1]):
            if c is not None:
                helpers.close_grad(a, c, rtol=2e-4)


# ---------------------------------------------------------------- 2. hard cases
HARD = [("distmult", 200), ("transe_l1", 36), ("complex", 50), ("analogy", 64), ("rescal", 12)]


@pytest.mark.parametrize("kind,d", HARD)
@pytest.mark.parametrize("case", ["empty_shards", "tiny", "self_loops", "one_owner"])
def test_hard_cases(kind, d, case):
    n_rel, b, n_neg = 4, 64, 33
    n_ent = {"empty_shards": 5, "tiny": 17}.get(case, 300)
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=13)
    h, t, r, _ = _batch(n_ent, n_rel, b, seed=14)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.25], device=DEV)    # Bernoulli 0 and 1: one side only
    if case == "self_loops":
        h[::2] = t[::2]
    if case == "one_owner":                 # every positive held by rank 0 of 8 (rows [0, 38))
        h, t = h % 38, t % 38
    # tiny n_ent: most draws hit a shard's first or last row and many negatives equal their positive
    want = helpers.unsharded(model, h, t, r, probs, 1.0, n_neg, 7, 3)
    eng = CudaEngine()
    for world in (2, 3, 8):
        _compare(helpers.emulated(model, h, t, r, probs, 1.0, n_neg, 7, 3, world, eng), want)


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
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "kge_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^{}]*)\}\s*kge_margin_step_args_t\s*;", header, flags=re.S).group(1)
    names = [re.findall(r"[A-Za-z_][A-Za-z0-9_]*", part)[-1]
             for decl in body.split(";") if decl.strip() for part in decl.split(",")]
    assert names == [n for n, _ in _lib.MarginStepArgs._fields_]


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
    model = helpers.train_model("distmult", 36, 100, 3, seed=1)
    h, t, r, probs = _batch(100, 3, 8, seed=1)
    code, dim, ts = helpers.train_leaves(model)
    tabs = [None if x is None else x.detach() for x in ts]
    nh, nt = h.repeat(2), (t.repeat(2) + 1) % 100
    out = [torch.zeros(16, device=DEV), torch.zeros(8, device=DEV)]
    ids = [torch.zeros(16, dtype=torch.int64, device=DEV) for _ in range(2)]
    loss = torch.zeros((), device=DEV)
    a = _MarginStep._args(code, dim, 100, 1.0, 2, h, t, r, nh, nt, None, 0, 0, tabs, loss, h.device)
    a.pos_out, a.neg_out, a.nh_out, a.nt_out = _ptr(out[1]), _ptr(out[0]), _ptr(ids[0]), _ptr(ids[1])
    assert _lib.load().kge_margin_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()
    assert torch.equal(ids[0], nh) and torch.equal(ids[1], nt)
    assert loss.item() == pytest.approx(torch.relu(1.0 - out[1].repeat(2) + out[0]).sum().item(), rel=1e-5)


# ---------------------------------------------------------------- 5. public API, two processes
def _local_model(kind, model, lo, hi, n_rel, dim):
    part = helpers.make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part.to(next(model.parameters()).device)


def _train(model, kg, batches, shard, steps, seed):
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=16, seed=seed)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for h, t, r in batches[:steps]:
        opt.zero_grad()
        loss = sampler.fused_step(model, h, t, r, 1.0, shard=shard)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return losses


def _api_worker(rank, world, backend):
    dev = torch.device("cuda:%d" % (rank if backend == "nccl" else 0))
    torch.cuda.set_device(dev)
    try:
        res = {}
        n_ent, n_rel = 3001, 7
        hh, tt, rr = helpers.random_graph(n_ent, n_rel, 6000, seed=5)
        kg = tk.KnowledgeGraph(hh, tt, rr, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
        batches = [(hh[i:i + 512].to(dev), tt[i:i + 512].to(dev), rr[i:i + 512].to(dev)) for i in range(0, 2560, 512)]
        for kind, dim in (("distmult", 200), ("complex", 50)):
            full = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
            shard = EntityShard.from_group(n_ent, local_storage=True)
            local = _local_model(kind, full, shard.lo, shard.hi, n_rel, dim)
            want = _train(full, kg, batches, None, 5, seed=3)
            got = _train(local, kg, batches, shard, 5, seed=3)
            everyone = shard.stack_all(torch.tensor(got, dtype=torch.float64, device=dev))
            res[kind + "/losses_equal_on_ranks"] = bool((everyone == everyone[0]).all())
            res[kind + "/losses_close"] = all(abs(a - b) <= 1e-5 * abs(b) for a, b in zip(got, want))
            for name, p in local.named_parameters():
                ref = dict(full.named_parameters())[name]
                if "ent_emb" in name:
                    res[kind + "/" + name] = torch.allclose(p, ref[shard.lo:shard.hi], rtol=1e-4, atol=1e-5)
                else:
                    allp = shard.stack_all(p.detach())
                    res[kind + "/" + name + "/bitwise_on_ranks"] = bool((allp == allp[0]).all())
                    res[kind + "/" + name] = torch.allclose(p, ref, rtol=1e-4, atol=1e-5)
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
    ret = gloo.spawn(2, _api_worker, backend, backend=backend)
    for rank in (0, 1):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad and len(res) >= 12, "rank %d: %s" % (rank, res)


def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
