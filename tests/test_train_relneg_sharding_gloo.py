"""CPU tests of the relation-corrupting step (BernoulliRelationNegativeSampler): the host logic of the
entity-sharded step over gloo with an oracle-backed stand-in engine (a relation negative is scored by
the rank that holds the positive's head; the ranks' sums give the unsharded loss and gradients; the
collectives are those of the entity step), the rel_share agreement, the sampler's argument checks, and
the argument errors of the three new entry points in a child process that sees no GPU."""
import pytest
import torch

import torchkge_b200 as tk
from tests import gloo, helpers
from tests.train_kit import (CountingShard, OracleStepEngine, every_rank_ok, grads_match, header_fields,
                             malformed_calls, oracle_loss, stand_in_rel_draws)
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard
from torchkge_b200.training import fused_loss_step, sharded_margin_step


def _reference(kind, loss_kind, model, h, t, r, probs, seed, offset, n_neg, n_ent, n_rel, share):
    k, e = stand_in_rel_draws(seed, offset, h, r, n_neg, probs, n_ent, n_rel, share)
    nh = torch.where(k == 1, e, h.repeat(n_neg))
    nt = torch.where(k == 0, e, t.repeat(n_neg))
    nr = torch.where(k == 2, e, r.repeat(n_neg))
    return oracle_loss(kind, loss_kind, model, h, t, r, nh, nt, nr)


def _run(rank, world, kind, loss_kind, n_ent, b, n_neg, share):
    n_rel, dim = 5, 8
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.3, 0.8])
    eng = OracleStepEngine()
    g = torch.Generator().manual_seed(100)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, n_rel, (b,), generator=g)
    loss = sharded_margin_step(local, h, t, r, 0.0, n_neg, probs, 7, 1, shard, engine=eng, loss_kind=loss_kind,
                               rel_share=share)
    loss.backward()
    want_loss, want = _reference(kind, loss_kind, model, h, t, r, probs, 7, 1, n_neg, n_ent, n_rel, share)
    ok = {"loss": abs(loss.item() - want_loss) <= 1e-5 * max(1.0, abs(want_loss))}
    ok.update(grads_match(kind, local, want, shard))
    ok["collectives"] = [c[0] for c in shard.collectives] == ["stack_all", "all_reduce", "all_reduce", "all_reduce"]
    ok["agreement_fields"] = shard.collectives[0][1] == 6
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
                fused_loss_step(model, h, h, h % 4, tk.LogisticLoss(), n_neg=3, bern_probs=torch.full((4,), 0.5),
                                seed=11, offset=1, shard=shard, rel_share=0.33 if rank == 0 else case[1])
                return {"raised": False}
            except ValueError as e:
                return {"raised": "rel_share" in str(e)}
        return _run(rank, world, *case)
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


# (world, kind, loss kind, n_ent, b, n_neg, rel_share)
CASES = [
    (2, "distmult", _lib.LOSS_LOGISTIC, 40, 12, 5, 0.33),
    (2, "complex", _lib.LOSS_BCE, 31, 9, 4, 0.0),
    (3, "transe_l2", _lib.LOSS_MARGIN, 2, 6, 3, 0.5),       # n_ent < world: rank 2 holds nothing
]


@pytest.mark.parametrize("case", CASES, ids=["%s-loss%d-w%d-share%g" % (c[1], c[2], c[0], c[6]) for c in CASES])
def test_sharded_rel_step_equals_oracle(case):
    every_rank_ok(gloo.spawn(case[0], _worker, case[1:]), case[0])


@pytest.mark.parametrize("other", [0.5, None])
def test_rel_share_mismatch_raises_on_every_rank(other):
    """Ranks that disagree on rel_share -- or where one runs the entity step -- raise on every rank."""
    assert gloo.spawn(2, _worker, ("mismatch", other)) == {0: {"raised": True}, 1: {"raised": True}}


def test_sampler_arguments():
    kg, _, _ = helpers.make_kg(50, 1, n_facts=100, n_test=5, seed=1)
    with pytest.raises(ValueError, match="n_rel >= 2"):
        tk.BernoulliRelationNegativeSampler(kg)
    s = tk.BernoulliRelationNegativeSampler(kg, rel_share=1.0, seed=3)
    assert s.rel_share == 1.0 and s.bern_probs.tolist() == pytest.approx([float(tk.sampling.get_bernoulli_probs(kg)
                                                                                [0])])
    kg2, _, _ = helpers.make_kg(50, 6, n_facts=100, n_test=5, seed=1)
    with pytest.raises(ValueError, match="rel_share"):
        tk.BernoulliRelationNegativeSampler(kg2, rel_share=1.5)
    s2 = tk.BernoulliRelationNegativeSampler(kg2, n_neg=3)
    assert s2.n_neg == 3 and s2.rel_share == pytest.approx(0.33) and s2.bern_probs.dtype == torch.float32
    model = helpers.make_model("distmult", 8, 50, 6, seed=2)
    h = torch.arange(4)
    # argument errors before any collective or kernel, and before the call count moves
    with pytest.raises(ValueError, match="exactly one"):
        s2.fused_step(model, h, h, h)
    with pytest.raises(TypeError, match="MSELoss"):
        s2.fused_step(model, h, h, h, criterion=torch.nn.MSELoss())
    assert s2._calls == 0


_ABI_CHILD = r"""
step_cases(_lib.RelStepArgs, dict(n_rel=5, rel_share=0.5), lib.kge_rel_step_fwd, lib.kge_rel_step_bwd, {
    "null": lambda a: None,
    "n_rel_0": lambda a: setattr(a, "n_rel", 0),
    "one_relation": lambda a: setattr(a, "n_rel", 1),
    "share_above_1": lambda a: setattr(a, "rel_share", 1.5),
    "share_nan": lambda a: setattr(a, "rel_share", float("nan")),
    "share_negative": lambda a: setattr(a, "rel_share", -0.1),
    "nr_without_nh": lambda a: setattr(a, "nr", F),
    "nh_without_nr": lambda a: (setattr(a.base, "nh", F), setattr(a.base, "nt", F)),
    "bad_loss_kind": lambda a: setattr(a.base, "loss_kind", 7),
    "no_loss": lambda a: setattr(a.base, "loss", None),
    "sharded_nr_out": lambda a: (setattr(a.base, "hrows", F), setattr(a.base, "trows", F),
                                 setattr(a.base, "n_rows", 10), setattr(a, "nr_out", F)),
    "sharded_external": lambda a: (setattr(a.base, "hrows", F), setattr(a.base, "trows", F),
                                   setattr(a.base, "n_rows", 10), setattr(a.base, "nh", F),
                                   setattr(a.base, "nt", F), setattr(a, "nr", F)),
})
cb = lib.kge_corrupt_batch_rel
res["corrupt_null"] = cb(F, F, F, 4, 1, F, 10, 5, 0.5, 1, 1, F, F, None, None)
res["corrupt_n_neg_0"] = cb(F, F, F, 4, 0, F, 10, 5, 0.5, 1, 1, F, F, F, None)
res["corrupt_one_relation"] = cb(F, F, F, 4, 1, F, 10, 1, 0.5, 1, 1, F, F, F, None)
res["corrupt_share"] = cb(F, F, F, 4, 1, F, 10, 5, 2.0, 1, 1, F, F, F, None)
res["corrupt_b_negative"] = cb(F, F, F, -1, 1, F, 10, 5, 0.5, 1, 1, F, F, F, None)
res["corrupt_empty_ok"] = cb(None, None, None, 0, 1, None, 10, 5, 0.5, 1, 1, None, None, None, None)
"""


def test_new_entry_points_reject_malformed_calls_without_a_gpu():
    res = malformed_calls(_ABI_CHILD)
    assert res == {k: (0 if k == "corrupt_empty_ok" else 1) for k in res}    # KGE_OK / KGE_ERR_ARG


def test_rel_step_struct_matches_the_header_in_order():
    """kge_rel_step_args_t in include/kge_b200.h, field by field, is _lib.RelStepArgs."""
    assert header_fields("kge_rel_step_args_t") == [n for n, _ in _lib.RelStepArgs._fields_]
    assert _lib.RelStepArgs._fields_[0] == ("base", _lib.MarginStepArgs)


def test_negatives_and_rel_share_are_checked_on_the_host():
    model = helpers.make_model("distmult", 8, 20, 4, seed=2)
    h = torch.arange(4)
    with pytest.raises(ValueError, match="rel_share"):        # two-part negatives with a relation draw
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), negatives=(h, h), rel_share=0.5)
    with pytest.raises(ValueError, match="rel_share"):        # three-part negatives: nothing is drawn
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), negatives=(h, h, h), rel_share=0.5)
    with pytest.raises(ValueError, match="common length"):
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), negatives=(h, h, h[:3]))
    with pytest.raises(ValueError, match="multiple of the batch"):
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), negatives=(h[:3], h[:3], h[:3]))
    with pytest.raises(ValueError, match="rel_share must lie"):
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), bern_probs=torch.full((4,), 0.5), rel_share=-0.5)
