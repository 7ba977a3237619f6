"""The entity-sharded fused step with LogisticLoss and BinaryCrossEntropyLoss: per-rank kernel calls on
row ranges of one table, summed over the ranks and scattered as the host logic does, must reproduce the
unsharded fused step of the same loss -- loss within 1e-5 relative, gradients under the atomics-order
rule of tests/test_train_gpu.py.  Every rank counts the positive's term only for the negatives it owns.
Then the public API trains in two processes over gloo on one GPU; the NCCL form needs two GPUs and is
skipped on a machine with one."""

import pytest
import torch

import torchkge_b200 as tk
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ALL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "analogy", "toruse_l1",
             "toruse_l2"]
KINDS = {"logistic": _lib.LOSS_LOGISTIC, "bce": _lib.LOSS_BCE}


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
GENERIC = [(k, 50 if k != "rescal" else 12) for k in ALL_KINDS]
CASES = [(k, d, (1, 33, 256)[i % 3]) for i, (k, d) in enumerate(RING + GENERIC)]


@pytest.mark.parametrize("loss", sorted(KINDS))
@pytest.mark.parametrize("kind,d,n_neg", CASES, ids=["%s-d%d-neg%d" % c for c in CASES])
def test_emulated_shards_equal_unsharded(kind, d, n_neg, loss):
    n_ent, n_rel, b = 700, 40, 160
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=3)
    h, t, r, probs = _batch(n_ent, n_rel, b, seed=d + n_neg)
    want = helpers.unsharded(model, h, t, r, probs, 0.0, n_neg, 99, 5, loss_kind=KINDS[loss])
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        _compare(helpers.emulated(model, h, t, r, probs, 0.0, n_neg, 99, 5, world, eng, loss_kind=KINDS[loss]), want)


@pytest.mark.parametrize("loss", sorted(KINDS))
@pytest.mark.parametrize("kind,d", [("distmult", 200), ("transe_l1", 36), ("complex", 50), ("analogy", 64),
                                    ("toruse_l2", 40)])
def test_empty_shards_and_one_sided_draws(kind, d, loss):
    """17 entities over 8 ranks (one row per rank or none), Bernoulli probabilities 0 and 1."""
    n_ent, n_rel, b, n_neg = 17, 4, 64, 33
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=13)
    h, t, r, _ = _batch(n_ent, n_rel, b, seed=14)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.25], device=DEV)
    want = helpers.unsharded(model, h, t, r, probs, 0.0, n_neg, 7, 3, loss_kind=KINDS[loss])
    eng = CudaEngine()
    for world in (2, 3, 8):
        _compare(helpers.emulated(model, h, t, r, probs, 0.0, n_neg, 7, 3, world, eng, loss_kind=KINDS[loss]), want)


# ---------------------------------------------------------------- 2. public API, two processes
def _local_model(kind, model, lo, hi, n_rel, dim):
    part = helpers.make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part.to(next(model.parameters()).device)


def _train(model, kg, batches, shard, steps, seed, crit):
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=16, seed=seed)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for h, t, r in batches[:steps]:
        opt.zero_grad()
        loss = sampler.fused_step(model, h, t, r, criterion=crit, shard=shard)
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
        for kind, dim, crit in (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.BinaryCrossEntropyLoss())):
            full = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
            shard = EntityShard.from_group(n_ent, local_storage=True)
            local = _local_model(kind, full, shard.lo, shard.hi, n_rel, dim)
            want = _train(full, kg, batches, None, 5, 3, crit)
            got = _train(local, kg, batches, shard, 5, 3, crit)
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
        # a loss kind that differs between the ranks raises on every rank instead of hanging
        sampler = tk.BernoulliNegativeSampler(kg, n_neg=4, seed=100)
        crit = tk.LogisticLoss() if rank == 0 else tk.BinaryCrossEntropyLoss()
        try:
            sampler.fused_step(local, *batches[0], criterion=crit, shard=shard)
            res["loss_mismatch_raises"] = False
        except ValueError:
            res["loss_mismatch_raises"] = True
        return res
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


def _run_two_ranks(backend):
    ret = gloo.spawn(2, _api_worker, backend, backend=backend)
    for rank in (0, 1):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad and len(res) >= 14, "rank %d: %s" % (rank, res)


def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                    reason="needs two GPUs (one NCCL rank per device)")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
