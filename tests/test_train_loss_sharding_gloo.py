"""Multi-process (gloo, CPU) tests of the sharded fused step's host logic with LogisticLoss and
BinaryCrossEntropyLoss: the loss kind travels to every rank's kernels, the ranks' sums give the
unsharded loss and gradients, the collectives are the margin step's (stack_all and three all-reduces),
ranks that disagree on the loss kind raise on every rank, and an unsupported criterion raises before
any collective.  The CUDA engine is an oracle-backed stand-in; tests/test_train_loss_shard_gpu.py runs
the kernels."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import gloo, helpers
from tests.test_train_sharding_gloo import (_ENT_KEYS, _KIND_OF_CODE, _REL_KEYS, CountingShard, OracleStepEngine,
                                            Shard, _local_model, draws)
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard
from torchkge_b200.training import fused_loss_step, sharded_margin_step


def pair_loss(kind, pos, neg):
    """utils/losses.py:47-112 with torch's modules, summed over the pairs."""
    if kind == _lib.LOSS_LOGISTIC:
        crit = torch.nn.SoftMarginLoss(reduction="sum")
        return crit(pos, torch.ones_like(pos)) + crit(neg, -torch.ones_like(neg))
    crit = torch.nn.BCELoss(reduction="sum")
    return crit(torch.sigmoid(pos), torch.ones_like(pos)) + crit(torch.sigmoid(neg), torch.zeros_like(neg))


class LossStepEngine(OracleStepEngine):
    """The stand-in engine with the step's loss kind: pair terms of the negatives this shard owns, the
    positive's term once per owned negative."""

    def _partial(self, step, tables, h, t, r, probs, hrows, trows, grad):
        kind = _KIND_OF_CODE[step.code]
        b, n = h.shape[0], step.n_rows
        ent = [x for x in tables[:2] if x is not None]
        P = {}
        for p, key in enumerate(_ENT_KEYS[kind]):
            P[key] = torch.cat([ent[p], hrows[:, p], trows[:, p]]).clone().requires_grad_(grad)
        for p, key in enumerate(_REL_KEYS[kind]):
            P[key] = tables[2 + p].clone().requires_grad_(grad)
        head, e = draws(step.seed, step.offset, r, step.n_neg, probs, step.n_ent)
        own = (e >= step.ent_lo) & (e < step.ent_lo + n)
        i = torch.arange(b).repeat(step.n_neg)[own]
        loc, head = e[own] - step.ent_lo, head[own]
        nh = torch.where(head, loc, n + i)
        nt = torch.where(head, loc.new_full(loc.shape, n) + b + i, loc)
        pos = oracle.score_triples(kind, P, n + i, n + b + i, r[i])
        neg = oracle.score_triples(kind, P, nh, nt, r[i])
        return pair_loss(step.loss_kind, pos, neg), P


def _reference(kind, loss_kind, model, h, t, r, probs, seed, offset, n_neg, n_ent):
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    head, e = draws(seed, offset, r, n_neg, probs, n_ent)
    nh = torch.where(head, e, h.repeat(n_neg))
    nt = torch.where(head, t.repeat(n_neg), e)
    pos, neg = oracle.forward_pos_neg(kind, P, h, t, r, nh, nt)
    loss = pair_loss(loss_kind, pos, neg)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in P.items()}


def _run(rank, world, kind, loss_kind, n_ent, b, n_neg, steps):
    n_rel, dim = 4, 8
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = _local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.3])
    eng = LossStepEngine()
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
        names = dict(zip(_ENT_KEYS[kind], ("ent_emb.weight",) if kind != "complex" else
                         ("re_ent_emb.weight", "im_ent_emb.weight")))
        names.update(zip(_REL_KEYS[kind], ("rel_emb.weight",) if kind != "complex" else
                         ("re_rel_emb.weight", "im_rel_emb.weight")))
        params = dict(local.named_parameters())
        for key, name in names.items():
            ref = want[key][shard.lo:shard.hi] if "ent" in key else want[key]
            ok["%s%d" % (key, s)] = torch.allclose(params[name].grad, ref, rtol=1e-4, atol=1e-6)
        ok["collectives%d" % s] = [c[0] for c in step_collectives] == ["stack_all", "all_reduce", "all_reduce",
                                                                       "all_reduce"]
        ok["agreement_fields%d" % s] = step_collectives[0][1] == 6     # the loss kind joins the check
    ok["empty_rank_skips_kernels"] = (shard.hi > shard.lo) or eng.calls == []
    return ok


def _worker(rank, world, case):
    try:
        if case[0] == "mismatch":
            shard = EntityShard.from_group(30, local_storage=True)
            model = _local_model("distmult", helpers.make_model("distmult", 8, 30, 4, seed=1), shard.lo, shard.hi, 4, 8)
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


def _spawn(world, case):
    return gloo.spawn(world, _worker, case)


# (world, kind, loss kind, n_ent, b, n_neg, steps)
CASES = [
    (2, "distmult", _lib.LOSS_LOGISTIC, 40, 12, 5, 2),
    (2, "complex", _lib.LOSS_BCE, 31, 9, 4, 1),
    (3, "complex", _lib.LOSS_LOGISTIC, 31, 9, 4, 1),
    (3, "transe_l2", _lib.LOSS_BCE, 2, 6, 3, 1),       # n_ent < world: rank 2 holds nothing
]


@pytest.mark.parametrize("case", CASES, ids=["%s-loss%d-w%d-n%d" % (c[1], c[2], c[0], c[3]) for c in CASES])
def test_sharded_loss_step_equals_oracle(case):
    world = case[0]
    ret = _spawn(world, case[1:])
    for rank in range(world):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad, "rank %d: %s" % (rank, bad)


def test_loss_kind_mismatch_raises_on_every_rank():
    ret = _spawn(2, ("mismatch",))
    assert ret == {0: {"raised": True}, 1: {"raised": True}}


def test_unsupported_criterion_raises_before_any_collective():
    model = helpers.make_model("distmult", 8, 10, 4, seed=2)
    h = torch.arange(4)
    with pytest.raises(TypeError, match="MSELoss"):
        fused_loss_step(model, h, h, h, torch.nn.MSELoss(), n_neg=2, bern_probs=torch.full((4,), 0.5), seed=1,
                        offset=1, shard=Shard(20, 0, 2, local_storage=True))
