"""Multi-process (gloo, CPU) tests of the entity-sharded fused training step's host logic
(torchkge_b200.training.sharded_margin_step): the positive-row exchange, the loss all-reduce, the single
backward all-reduce of grad_hrows / grad_trows / relation gradients, the scatter into the local entity
gradient, and the argument errors raised before any collective.  The CUDA engine is replaced by an
oracle-backed stand-in with the same methods -- this tests the plumbing, not the kernels;
tests/test_train_shard_gpu.py runs the kernels."""
import pytest
import torch

from tests import gloo, helpers
from tests.train_kit import (_ENT_KEYS, _REL_KEYS, CountingShard, NoCollectiveShard, OracleStepEngine, every_rank_ok,
                             grads_match, oracle_loss, param_names, stand_in_draws)
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard, QueryShard
from torchkge_b200.training import fused_margin_step, sharded_margin_step


def _reference(kind, model, h, t, r, probs, seed, offset, n_neg, margin, n_ent):
    head, e = stand_in_draws(seed, offset, r, n_neg, probs, n_ent)
    nh = torch.where(head, e, h.repeat(n_neg))
    nt = torch.where(head, t.repeat(n_neg), e)
    return oracle_loss(kind, _lib.LOSS_MARGIN, model, h, t, r, nh, nt, margin=margin)


def _run(rank, world, kind, n_ent, b, n_neg, steps):
    n_rel, dim, margin = 4, 8, 0.7
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.3])             # Bernoulli probabilities 0 and 1 included
    eng = OracleStepEngine()
    ok = {}
    for s in range(steps):
        g = torch.Generator().manual_seed(100 + s)
        h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
        r = torch.randint(0, n_rel, (b,), generator=g)
        h[:3] = t[:3]                                       # self loops
        local.zero_grad()
        shard.collectives.clear()
        loss = sharded_margin_step(local, h, t, r, margin, n_neg, probs, 7, s + 1, shard, engine=eng)
        loss.backward()
        step_collectives = list(shard.collectives)
        want_loss, want = _reference(kind, model, h, t, r, probs, 7, s + 1, n_neg, margin, n_ent)
        ok["loss%d" % s] = abs(loss.item() - want_loss) <= 1e-5 * max(1.0, abs(want_loss))
        ok.update(grads_match(kind, local, want, shard, str(s)))
        for key in _REL_KEYS[kind]:    # relation gradients are the output of one all-reduce: equal everywhere
            g = dict(local.named_parameters())[param_names(kind)[key]].grad
            ok["same_%s%d" % (key, s)] = bool((shard.stack_all(g) == g).all())
        # exactly: the agreement check, the row exchange, the loss, ONE backward all-reduce
        kinds = [c[0] for c in step_collectives]
        ok["collectives%d" % s] = kinds == ["stack_all", "all_reduce", "all_reduce", "all_reduce"]
        planes = len(_ENT_KEYS[kind])
        ok["row_floats%d" % s] = step_collectives[1][1] == 2 * b * planes * dim
        ok["bwd_floats%d" % s] = step_collectives[3][1] == 2 * b * planes * dim + planes * n_rel * dim
    ok["empty_rank_skips_kernels"] = (shard.hi > shard.lo) or eng.calls == []
    return ok


def _worker(rank, world, case):
    try:
        if case[0] == "mismatch":
            shard = EntityShard.from_group(30, local_storage=True)
            whole = helpers.make_model("distmult", 8, 30, 4, seed=1)
            model = helpers.local_model("distmult", whole, shard.lo, shard.hi, 4, 8)
            h = torch.arange(5)
            try:
                sharded_margin_step(model, h, h, h % 4, 1.0, 3, torch.full((4,), 0.5), 11 + rank, 1, shard,
                                    engine=OracleStepEngine())
                return {"raised": False}
            except ValueError:
                return {"raised": True}
        return _run(rank, world, *case)
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


# (world, kind, n_ent, b, n_neg, steps)
CASES = [
    (2, "distmult", 40, 12, 5, 2),
    (3, "complex", 31, 9, 4, 2),
    (3, "transe_l2", 2, 6, 3, 1),       # n_ent < world: rank 2 holds nothing
]


@pytest.mark.parametrize("case", CASES, ids=["%s-w%d-n%d" % (c[1], c[0], c[2]) for c in CASES])
def test_sharded_step_equals_oracle(case):
    every_rank_ok(gloo.spawn(case[0], _worker, case[1:]), case[0])


def test_seed_mismatch_raises_on_every_rank():
    ret = gloo.spawn(2, _worker, ("mismatch",))
    assert ret == {0: {"raised": True}, 1: {"raised": True}}


def test_argument_errors_come_before_any_collective():
    model = helpers.make_model("distmult", 8, 10, 4, seed=2)
    h = torch.arange(4)
    probs = torch.full((4,), 0.5)

    def run(shard, m=model, **kw):
        kw.setdefault("bern_probs", probs)
        return fused_margin_step(m, h, h, h, 1.0, n_neg=2, seed=1, offset=1, shard=shard, **kw)

    with pytest.raises(ValueError, match="QueryShard"):
        run(QueryShard(4, 0, 2))
    with pytest.raises(ValueError, match="local_storage"):
        run(NoCollectiveShard(20, 0, 2, local_storage=False))
    with pytest.raises(ValueError, match="external negatives"):
        run(NoCollectiveShard(20, 0, 2, local_storage=True), negatives=(h, h))
    with pytest.raises(ValueError, match="holds 10 entity rows"):
        run(NoCollectiveShard(30, 0, 2, local_storage=True))          # rows [0, 15) expected
    with pytest.raises(ValueError, match="bern_probs"):
        run(NoCollectiveShard(20, 0, 2, local_storage=True), bern_probs=None)


def test_sampler_entity_count_must_match_the_shard():
    import torchkge_b200 as tk
    hh, tt, rr = helpers.random_graph(50, 4, 200, seed=3)
    kg = tk.KnowledgeGraph(hh, tt, rr, 50, 4, dict_of_heads={}, dict_of_tails={})
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=2, seed=1)
    model = helpers.make_model("distmult", 8, 25, 4, seed=2)
    with pytest.raises(ValueError, match="sampler draws on 50"):
        sampler.fused_step(model, hh[:4], tt[:4], rr[:4], 1.0,
                           shard=NoCollectiveShard(60, 0, 2, local_storage=True))
