"""CPU tests of the positional fused step (PositionalNegativeSampler.fused_step, fused_*_step(positional=...)):
the host logic of the entity-sharded step over gloo with an oracle-backed stand-in engine (a negative is
scored by the rank holding the entity it draws; the ranks' sums give the unsharded loss and gradients; the
agreement tells the positional step from the entity step and compares the candidate CSRs' sizes), the
argument errors raised before any collective or kernel, the argument rules of kge_pos_step_* in a child
process that sees no GPU, and kge_pos_step_args_t against its binding."""
import pytest
import torch

import torchkge_b200 as tk
from tests import gloo, helpers
from tests.train_kit import (CountingShard, OracleStepEngine, csr, every_rank_ok, grads_match, header_fields,
                             malformed_calls, oracle_loss, stand_in_pos_draws)
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard, QueryShard
from torchkge_b200.training import fused_loss_step, fused_margin_step, sharded_margin_step


def positional_of(n_ent, n_rel, seed, n=40):
    g = torch.Generator().manual_seed(seed)
    rel = torch.randint(1, n_rel, (n,), generator=g)            # relation 0 has no candidates
    hd, tl = torch.randint(0, n_ent, (n,), generator=g), torch.randint(0, n_ent, (n,), generator=g)
    return csr(rel, hd, n_rel, n_ent) + csr(rel, tl, n_rel, n_ent)


def _reference(kind, loss_kind, model, h, t, r, probs, seed, offset, n_neg, n_ent, pos):
    head, e = stand_in_pos_draws(seed, offset, r, n_neg, probs, n_ent, pos)
    nh = torch.where(head, e, h.repeat(n_neg))
    nt = torch.where(head, t.repeat(n_neg), e)
    return oracle_loss(kind, loss_kind, model, h, t, r, nh, nt)


def _run(rank, world, kind, loss_kind, n_ent, b, n_neg):
    n_rel, dim = 5, 8
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.5, 1.0, 0.0, 0.3, 0.8])
    pos = positional_of(n_ent, n_rel, seed=2)
    eng = OracleStepEngine()
    g = torch.Generator().manual_seed(100)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, n_rel, (b,), generator=g)
    loss = sharded_margin_step(local, h, t, r, 0.0, n_neg, probs, 7, 1, shard, engine=eng, loss_kind=loss_kind,
                               positional=pos)
    loss.backward()
    want_loss, want = _reference(kind, loss_kind, model, h, t, r, probs, 7, 1, n_neg, n_ent, pos)
    ok = {"loss": abs(loss.item() - want_loss) <= 1e-5 * max(1.0, abs(want_loss))}
    ok.update(grads_match(kind, local, want, shard))
    # the entity step's collectives, plus one for the CSR sizes
    ok["collectives"] = [c[0] for c in shard.collectives] == ["stack_all", "stack_all", "all_reduce", "all_reduce",
                                                               "all_reduce"]
    ok["agreement_fields"] = [c[1] for c in shard.collectives[:2]] == [6, 4]
    ok["empty_rank_skips_kernels"] = (shard.hi > shard.lo) or eng.calls == []
    return ok


def _worker(rank, world, case):
    try:
        if case[0] in ("csr", "kind"):
            shard = EntityShard.from_group(30, local_storage=True)
            whole = helpers.make_model("distmult", 8, 30, 4, seed=1)
            model = helpers.local_model("distmult", whole, shard.lo, shard.hi, 4, 8)
            h = torch.arange(5)
            pos = positional_of(30, 4, seed=3, n=40 if rank == 0 else 41)
            if case[0] == "kind" and rank == 1:
                pos = None
            try:
                fused_loss_step(model, h, h, h % 4, tk.LogisticLoss(), n_neg=3, bern_probs=torch.full((4,), 0.5),
                                seed=11, offset=1, shard=shard, positional=pos)
                return {"raised": False}
            except ValueError as e:
                return {"raised": ("CSR" if case[0] == "csr" else "positional") in str(e)}
        return _run(rank, world, *case)
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


# (world, kind, loss kind, n_ent, b, n_neg)
CASES = [
    (2, "distmult", _lib.LOSS_LOGISTIC, 40, 12, 5),
    (2, "complex", _lib.LOSS_MARGIN, 31, 9, 4),
    (3, "transe_l2", _lib.LOSS_BCE, 2, 6, 3),       # n_ent < world: rank 2 holds nothing
    (3, "distmult", _lib.LOSS_MARGIN, 50, 10, 3),
]


@pytest.mark.parametrize("case", CASES, ids=["%s-loss%d-w%d" % (c[1], c[2], c[0]) for c in CASES])
def test_sharded_pos_step_equals_oracle(case):
    every_rank_ok(gloo.spawn(case[0], _worker, case[1:]), case[0])


@pytest.mark.parametrize("what", ["csr", "kind"])
def test_mismatch_raises_on_every_rank(what):
    """Ranks whose CSRs differ in size, or where one runs the entity step, raise on every rank."""
    assert gloo.spawn(2, _worker, (what,)) == {0: {"raised": True}, 1: {"raised": True}}


def test_argument_errors():
    kg, _, _ = helpers.make_kg(60, 5, n_facts=200, n_test=5, seed=1)
    s = tk.PositionalNegativeSampler(kg, seed=4)
    u = tk.UniformNegativeSampler(kg, seed=4)
    model = helpers.make_model("distmult", 8, 60, 5, seed=2)
    h = torch.arange(4)
    for sampler in (s, u):
        with pytest.raises(ValueError, match="exactly one"):
            sampler.fused_step(model, h, h, h)
        with pytest.raises(TypeError, match="MSELoss"):
            sampler.fused_step(model, h, h, h, criterion=torch.nn.MSELoss())
        with pytest.raises(ValueError, match="QueryShard"):
            sampler.fused_step(model, h, h, h, margin=1.0, shard=QueryShard(10, 0, 1))
        with pytest.raises(_lib.KgeLibraryError, match="CUDA"):    # CPU tensors: no CPU path
            sampler.fused_step(model, h, h, h, margin=1.0)
    calls = s._calls
    with pytest.raises(ValueError, match="entities"):     # before the call count moves
        s.fused_step(helpers.make_model("distmult", 8, 61, 5, seed=2), h, h, h, margin=1.0)
    with pytest.raises(ValueError, match="entities"):
        s.fused_step(model, h, h, h, margin=1.0, shard=EntityShard(99, 0, 2, local_storage=True))
    assert s._calls == calls
    with pytest.raises(ValueError, match="relations"):
        s.fused_step(helpers.make_model("distmult", 8, 60, 6, seed=2), h, h, h, margin=1.0)
    pos = positional_of(60, 5, seed=1)
    probs = torch.full((5,), 0.5)
    with pytest.raises(ValueError, match="caller negatives"):
        fused_loss_step(model, h, h, h, tk.LogisticLoss(), negatives=(h, h), positional=pos)
    with pytest.raises(ValueError, match="rel_share"):
        fused_margin_step(model, h, h, h, 1.0, bern_probs=probs, positional=pos, rel_share=0.5)
    with pytest.raises(ValueError, match="rel_share"):
        fused_margin_step(model, h, h, h, 1.0, bern_probs=probs, positional=pos, rel_share=0.5,
                          shard=EntityShard(60, 0, 1, local_storage=True))
    with pytest.raises(ValueError, match="covers 4 relations"):
        fused_margin_step(model, h, h, h, 1.0, bern_probs=probs, positional=positional_of(60, 4, seed=1))
    with pytest.raises(ValueError, match="covers 4 relations"):
        fused_margin_step(model, h, h, h, 1.0, bern_probs=probs, positional=positional_of(60, 4, seed=1),
                          shard=EntityShard(60, 0, 1, local_storage=True))
    with pytest.raises(ValueError, match="head_offs, head_ents"):
        fused_margin_step(model, h, h, h, 1.0, bern_probs=probs, positional=pos[:2])


_ABI_CHILD = r"""
fields = dict(n_rel=5, head_offs=F, head_ents=F, tail_offs=F, tail_ents=F)
step_cases(_lib.PosStepArgs, fields, lib.kge_pos_step_fwd, lib.kge_pos_step_bwd, {
    "null": lambda a: None,
    "n_rel_0": lambda a: setattr(a, "n_rel", 0),
    "no_head_offs": lambda a: setattr(a, "head_offs", None),
    "no_tail_offs": lambda a: setattr(a, "tail_offs", None),
    "caller_negatives": lambda a: (setattr(a.base, "nh", F), setattr(a.base, "nt", F)),
    "no_probs": lambda a: setattr(a.base, "bern_probs", None),
    "bad_loss_kind": lambda a: setattr(a.base, "loss_kind", 7),
    "no_loss": lambda a: setattr(a.base, "loss", None),
    "sharded_nh_out": lambda a: (setattr(a.base, "hrows", F), setattr(a.base, "trows", F),
                                 setattr(a.base, "n_rows", 10), setattr(a.base, "nh_out", F),
                                 setattr(a.base, "nt_out", F)),
    "sharded_rows_past_n_ent": lambda a: (setattr(a.base, "hrows", F), setattr(a.base, "trows", F),
                                          setattr(a.base, "n_rows", 11)),
})
"""


def test_entry_points_reject_malformed_calls_without_a_gpu():
    res = malformed_calls(_ABI_CHILD)
    assert res == {k: 1 for k in res}    # KGE_ERR_ARG


def test_pos_step_struct_matches_the_header_in_order():
    """kge_pos_step_args_t in include/kge_b200.h, field by field, is _lib.PosStepArgs."""
    assert header_fields("kge_pos_step_args_t") == [n for n, _ in _lib.PosStepArgs._fields_]
    assert _lib.PosStepArgs._fields_[0] == ("base", _lib.MarginStepArgs)
