"""The entity-sharded fused step with LogisticLoss and BinaryCrossEntropyLoss: per-rank kernel calls on
row ranges of one table, summed over the ranks and scattered as the host logic does, must reproduce the
unsharded fused step of the same loss -- loss within 1e-5 relative, gradients under the atomics-order
rule of tests/test_train_gpu.py.  Every rank counts the positive's term only for the negatives it owns.
Then the public API trains in two processes over gloo on one GPU; the NCCL form needs two GPUs and is
skipped on a machine with one."""

import pytest
import torch

import torchkge_b200 as tk
from tests import gloo
from tests import train_kit as kit
from torchkge_b200.engine import CudaEngine

pytestmark = pytest.mark.gpu
ALL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "analogy", "toruse_l1",
             "toruse_l2"]
KINDS = ("bce", "logistic")


# ---------------------------------------------------------------- 1. emulated shards vs unsharded
RING = [(k, d) for k in ("transe_l1", "transe_l2", "distmult") for d in (36, 200, 256)]
GENERIC = [(k, 50 if k != "rescal" else 12) for k in ALL_KINDS]
CASES = [(k, d, (1, 33, 256)[i % 3]) for i, (k, d) in enumerate(RING + GENERIC)]


@pytest.mark.parametrize("loss", KINDS)
@pytest.mark.parametrize("kind,d,n_neg", CASES, ids=["%s-d%d-neg%d" % c for c in CASES])
def test_emulated_shards_equal_unsharded(kind, d, n_neg, loss):
    n_ent, n_rel, b = 700, 40, 160
    model = kit.train_model(kind, d, n_ent, n_rel, seed=3)
    h, t, r, probs = kit.batch(n_ent, n_rel, b, d + n_neg)
    kw = dict(n_neg=n_neg, probs=probs, loss=loss, seed=99, offset=5)
    want = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        kit.compare(kit.emulated(model, h, t, r, world, eng, **kw), want)


@pytest.mark.parametrize("loss", KINDS)
@pytest.mark.parametrize("kind,d", [("distmult", 200), ("transe_l1", 36), ("complex", 50), ("analogy", 64),
                                    ("toruse_l2", 40)])
def test_empty_shards_and_one_sided_draws(kind, d, loss):
    """17 entities over 8 ranks (one row per rank or none), Bernoulli probabilities 0 and 1."""
    n_ent, n_rel, b, n_neg = 17, 4, 64, 33
    model = kit.train_model(kind, d, n_ent, n_rel, seed=13)
    h, t, r, _ = kit.batch(n_ent, n_rel, b, 14)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.25], device=kit.DEV)
    kw = dict(n_neg=n_neg, probs=probs, loss=loss, seed=7, offset=3)
    want = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (2, 3, 8):
        kit.compare(kit.emulated(model, h, t, r, world, eng, **kw), want)


# ---------------------------------------------------------------- 2. public API, two processes
def _api_worker(rank, world, backend):
    dev = torch.device("cuda:%d" % (rank if backend == "nccl" else 0))
    torch.cuda.set_device(dev)
    try:
        res, kg, batches, local, shard = kit.whole_against_shard(
            (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.BinaryCrossEntropyLoss())),
            lambda kg: tk.BernoulliNegativeSampler(kg, n_neg=16, seed=3), dev, 5, on_ranks=True)
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
    kit.every_rank_ok(gloo.spawn(2, _api_worker, backend, backend=backend), 2, min_checks=14)


def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                    reason="needs two GPUs (one NCCL rank per device)")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
