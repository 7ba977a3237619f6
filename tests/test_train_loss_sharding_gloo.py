"""Multi-process (gloo, CPU) tests of the sharded fused step's host logic with LogisticLoss and
BinaryCrossEntropyLoss: the loss kind travels to every rank's kernels, the ranks' sums give the
unsharded loss and gradients, the collectives are the margin step's (stack_all and three all-reduces),
ranks that disagree on the loss kind raise on every rank, and an unsupported criterion raises before
any collective.  The CUDA engine is an oracle-backed stand-in; tests/test_train_loss_shard_gpu.py runs
the kernels."""
import pytest
import torch

import torchkge_b200 as tk
from tests import gloo, helpers
from tests.train_kit import (CountingShard, NoCollectiveShard, OracleStepEngine, every_rank_ok, grads_match,
                             oracle_loss, stand_in_draws)
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard
from torchkge_b200.training import fused_loss_step, sharded_margin_step


def _reference(kind, loss_kind, model, h, t, r, probs, seed, offset, n_neg, n_ent):
    head, e = stand_in_draws(seed, offset, r, n_neg, probs, n_ent)
    nh = torch.where(head, e, h.repeat(n_neg))
    nt = torch.where(head, t.repeat(n_neg), e)
    return oracle_loss(kind, loss_kind, model, h, t, r, nh, nt)


def _run(rank, world, kind, loss_kind, n_ent, b, n_neg, steps):
    n_rel, dim = 4, 8
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.3])
    eng = OracleStepEngine()
    ok = {}
    for s in range(steps):
        g = torch.Generator().manual_seed(100 + s)
        h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
        r = torch.randint(0, n_rel, (b,), generator=g)
        h[:3] = t[:3]
        local.zero_grad()
        shard.collectives.clear()
        loss = sharded_margin_step(local, h, t, r, 0.0, n_neg, probs, 7, s + 1, shard, engine=eng,
                                   loss_kind=loss_kind)
        loss.backward()
        step_collectives = list(shard.collectives)
        want_loss, want = _reference(kind, loss_kind, model, h, t, r, probs, 7, s + 1, n_neg, n_ent)
        ok["loss%d" % s] = abs(loss.item() - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
        ok.update(grads_match(kind, local, want, shard, str(s)))
        ok["collectives%d" % s] = [c[0] for c in step_collectives] == ["stack_all", "all_reduce", "all_reduce",
                                                                       "all_reduce"]
        ok["agreement_fields%d" % s] = step_collectives[0][1] == 6     # the loss kind joins the check
    ok["empty_rank_skips_kernels"] = (shard.hi > shard.lo) or eng.calls == []
    return ok


def _worker(rank, world, case):
    try:
        if case[0] == "mismatch":
            shard = EntityShard.from_group(30, local_storage=True)
            whole = helpers.make_model("distmult", 8, 30, 4, seed=1)
            model = helpers.local_model("distmult", whole, shard.lo, shard.hi, 4, 8)
            h = torch.arange(5)
            crit = tk.LogisticLoss() if rank == 0 else tk.BinaryCrossEntropyLoss()
            try:
                fused_loss_step(model, h, h, h % 4, crit, n_neg=3, bern_probs=torch.full((4,), 0.5), seed=11,
                                offset=1, shard=shard)
                return {"raised": False}
            except ValueError as e:
                return {"raised": "loss kind" in str(e)}
        return _run(rank, world, *case)
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


# (world, kind, loss kind, n_ent, b, n_neg, steps)
CASES = [
    (2, "distmult", _lib.LOSS_LOGISTIC, 40, 12, 5, 2),
    (2, "complex", _lib.LOSS_BCE, 31, 9, 4, 1),
    (3, "complex", _lib.LOSS_LOGISTIC, 31, 9, 4, 1),
    (3, "transe_l2", _lib.LOSS_BCE, 2, 6, 3, 1),       # n_ent < world: rank 2 holds nothing
]


@pytest.mark.parametrize("case", CASES, ids=["%s-loss%d-w%d-n%d" % (c[1], c[2], c[0], c[3]) for c in CASES])
def test_sharded_loss_step_equals_oracle(case):
    every_rank_ok(gloo.spawn(case[0], _worker, case[1:]), case[0])


def test_loss_kind_mismatch_raises_on_every_rank():
    ret = gloo.spawn(2, _worker, ("mismatch",))
    assert ret == {0: {"raised": True}, 1: {"raised": True}}


def test_unsupported_criterion_raises_before_any_collective():
    model = helpers.make_model("distmult", 8, 10, 4, seed=2)
    h = torch.arange(4)
    with pytest.raises(TypeError, match="MSELoss"):
        fused_loss_step(model, h, h, h, torch.nn.MSELoss(), n_neg=2, bern_probs=torch.full((4,), 0.5), seed=1,
                        offset=1, shard=NoCollectiveShard(20, 0, 2, local_storage=True))
