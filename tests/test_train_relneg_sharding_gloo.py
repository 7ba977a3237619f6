"""CPU tests of the relation-corrupting step (BernoulliRelationNegativeSampler): the host logic of the
entity-sharded step over gloo with an oracle-backed stand-in engine (a relation negative is scored by
the rank that holds the positive's head; the ranks' sums give the unsharded loss and gradients; the
collectives are those of the entity step), the rel_share agreement, the sampler's argument checks, and
the argument errors of the three new entry points in a child process that sees no GPU."""
import os
import subprocess
import sys

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import gloo, helpers
from tests.test_train_loss_sharding_gloo import pair_loss
from tests.test_train_sharding_gloo import _ENT_KEYS, _KIND_OF_CODE, _REL_KEYS, CountingShard, OracleStepEngine, \
    _local_model
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard
from torchkge_b200.training import fused_loss_step, sharded_margin_step

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_draws(seed, offset, h, r, n_neg, probs, n_ent, n_rel, rel_share):
    """The stand-in's negatives (kind 0 tail, 1 head, 2 relation; replacement), a function of (seed,
    offset) and the global sizes only (the kernels use Philox; any fixed law serves the plumbing)."""
    g = torch.Generator().manual_seed((seed * 1000003 + offset) % (1 << 62))
    n = n_neg * h.shape[0]
    u, z = torch.rand(n, generator=g), torch.rand(n, generator=g)
    e = torch.randint(1, max(n_ent, 2), (n,), generator=g)
    q = torch.randint(1, max(n_rel, 2), (n,), generator=g)
    kind = torch.where(z < rel_share, (u < probs[r.repeat(n_neg)]).long(), torch.full_like(e, 2))
    return kind, torch.where(kind == 2, q, e)


class RelStepEngine(OracleStepEngine):
    """The stand-in engine for a relation-corrupting step: entity negatives on the rank holding their
    replaced entity, relation negatives on the rank holding the positive's head."""

    def _partial(self, step, tables, h, t, r, probs, hrows, trows, grad):
        assert step.n_rel > 0
        kind = _KIND_OF_CODE[step.code]
        b, n = h.shape[0], step.n_rows
        ent = [x for x in tables[:2] if x is not None]
        P = {}
        for p, key in enumerate(_ENT_KEYS[kind]):
            P[key] = torch.cat([ent[p], hrows[:, p], trows[:, p]]).clone().requires_grad_(grad)
        for p, key in enumerate(_REL_KEYS[kind]):
            P[key] = tables[2 + p].clone().requires_grad_(grad)
        k, e = rel_draws(step.seed, step.offset, h, r, step.n_neg, probs, step.n_ent, step.n_rel, step.rel_share)
        H = h.repeat(step.n_neg)
        holder = torch.where(k == 2, H, e)
        own = (holder >= step.ent_lo) & (holder < step.ent_lo + n)
        i = torch.arange(b).repeat(step.n_neg)[own]
        k, e = k[own], e[own]
        loc = e - step.ent_lo
        nh = torch.where(k == 1, loc, n + i)
        nt = torch.where(k == 0, loc, n + b + i)
        nr = torch.where(k == 2, e, r[i])
        pos = oracle.score_triples(kind, P, n + i, n + b + i, r[i])
        neg = oracle.score_triples(kind, P, nh, nt, nr)
        return pair_loss(step.loss_kind, pos, neg), P


def _reference(kind, loss_kind, model, h, t, r, probs, seed, offset, n_neg, n_ent, n_rel, share):
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    k, e = rel_draws(seed, offset, h, r, n_neg, probs, n_ent, n_rel, share)
    nh = torch.where(k == 1, e, h.repeat(n_neg))
    nt = torch.where(k == 0, e, t.repeat(n_neg))
    nr = torch.where(k == 2, e, r.repeat(n_neg))
    pos = oracle.score_triples(kind, P, h, t, r).repeat(n_neg)
    neg = oracle.score_triples(kind, P, nh, nt, nr)
    loss = pair_loss(loss_kind, pos, neg)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in P.items()}


def _run(rank, world, kind, loss_kind, n_ent, b, n_neg, share):
    n_rel, dim = 5, 8
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = _local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
    probs = torch.tensor([0.0, 1.0, 0.5, 0.3, 0.8])
    eng = RelStepEngine()
    g = torch.Generator().manual_seed(100)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, n_rel, (b,), generator=g)
    loss = sharded_margin_step(local, h, t, r, 0.0, n_neg, probs, 7, 1, shard, engine=eng, loss_kind=loss_kind,
                               rel_share=share)
    loss.backward()
    want_loss, want = _reference(kind, loss_kind, model, h, t, r, probs, 7, 1, n_neg, n_ent, n_rel, share)
    ok = {"loss": abs(loss.item() - want_loss) <= 1e-5 * max(1.0, abs(want_loss))}
    names = dict(zip(_ENT_KEYS[kind], ("ent_emb.weight",) if kind != "complex" else
                     ("re_ent_emb.weight", "im_ent_emb.weight")))
    names.update(zip(_REL_KEYS[kind], ("rel_emb.weight",) if kind != "complex" else
                     ("re_rel_emb.weight", "im_rel_emb.weight")))
    params = dict(local.named_parameters())
    for key, name in names.items():
        ref = want[key][shard.lo:shard.hi] if "ent" in key else want[key]
        ok[key] = torch.allclose(params[name].grad, ref, rtol=1e-4, atol=1e-6)
    ok["collectives"] = [c[0] for c in shard.collectives] == ["stack_all", "all_reduce", "all_reduce", "all_reduce"]
    ok["agreement_fields"] = shard.collectives[0][1] == 6
    ok["empty_rank_skips_kernels"] = (shard.hi > shard.lo) or eng.calls == []
    return ok


def _worker(rank, world, case):
    try:
        if case[0] == "mismatch":
            shard = EntityShard.from_group(30, local_storage=True)
            model = _local_model("distmult", helpers.make_model("distmult", 8, 30, 4, seed=1), shard.lo, shard.hi, 4, 8)
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
    world = case[0]
    ret = gloo.spawn(world, _worker, case[1:])
    for rank in range(world):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad, "rank %d: %s" % (rank, bad)


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
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from torchkge_b200 import _lib
lib = _lib.load()
F = 8   # a non-NULL stand-in pointer: every call below fails its checks before touching memory
res = {}
def ok_args():
    a = _lib.RelStepArgs()
    b = a.base
    b.tb.model, b.tb.dim, b.tb.ent0, b.tb.rel0 = _lib.DISTMULT, 8, F, F
    b.n_neg, b.b, b.n_ent, b.h, b.t, b.r, b.bern_probs, b.loss = 2, 4, 10, F, F, F, F, F
    a.n_rel, a.rel_share = 5, 0.5
    return a
g = _lib.Grads(F, None, F, None)
cases = {
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
}
for name, edit in cases.items():
    a = ok_args()
    edit(a)
    p = None if name == "null" else ctypes.byref(a)
    res["fwd_" + name] = lib.kge_rel_step_fwd(p)
    res["bwd_" + name] = lib.kge_rel_step_bwd(p, ctypes.byref(g), F)
a = ok_args()
res["bwd_no_grad_loss"] = lib.kge_rel_step_bwd(ctypes.byref(a), ctypes.byref(g), None)
res["bwd_no_grads"] = lib.kge_rel_step_bwd(ctypes.byref(a), None, F)
a.base.hrows, a.base.trows, a.base.n_rows = F, F, 10
res["bwd_sharded_no_grad_rows"] = lib.kge_rel_step_bwd(ctypes.byref(a), ctypes.byref(g), F)
cb = lib.kge_corrupt_batch_rel
res["corrupt_null"] = cb(F, F, F, 4, 1, F, 10, 5, 0.5, 1, 1, F, F, None, None)
res["corrupt_n_neg_0"] = cb(F, F, F, 4, 0, F, 10, 5, 0.5, 1, 1, F, F, F, None)
res["corrupt_one_relation"] = cb(F, F, F, 4, 1, F, 10, 1, 0.5, 1, 1, F, F, F, None)
res["corrupt_share"] = cb(F, F, F, 4, 1, F, 10, 5, 2.0, 1, 1, F, F, F, None)
res["corrupt_b_negative"] = cb(F, F, F, -1, 1, F, 10, 5, 0.5, 1, 1, F, F, F, None)
res["corrupt_empty_ok"] = cb(None, None, None, 0, 1, None, 10, 5, 0.5, 1, 1, None, None, None, None)
print(json.dumps(res))
"""


def test_new_entry_points_reject_malformed_calls_without_a_gpu():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _ABI_CHILD, ROOT], env=env, capture_output=True, text=True,
                          timeout=300)
    assert proc.returncode == 0, proc.stderr[-3000:]
    import json
    res = json.loads(proc.stdout.strip().splitlines()[-1])
    assert res == {k: (0 if k == "corrupt_empty_ok" else 1) for k in res}    # KGE_OK / KGE_ERR_ARG


def test_rel_step_struct_matches_the_header_in_order():
    """kge_rel_step_args_t in include/kge_b200.h, field by field, is _lib.RelStepArgs."""
    import re
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "kge_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^{}]*)\}\s*kge_rel_step_args_t\s*;", header, flags=re.S).group(1)
    names = [re.findall(r"[A-Za-z_][A-Za-z0-9_]*", part)[-1]
             for decl in body.split(";") if decl.strip() for part in decl.split(",")]
    assert names == [n for n, _ in _lib.RelStepArgs._fields_]
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
