"""Multi-process (gloo, CPU) tests of the entity-sharded fused training step's host logic
(torchkge_b200.training.sharded_margin_step): the positive-row exchange, the loss all-reduce, the single
backward all-reduce of grad_hrows / grad_trows / relation gradients, the scatter into the local entity
gradient, and the argument errors raised before any collective.  The CUDA engine is replaced by an
oracle-backed stand-in with the same methods -- this tests the plumbing, not the kernels;
tests/test_train_shard_gpu.py runs the kernels."""
import pytest
import torch

from oracle import kge_oracle as oracle
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard, QueryShard
from torchkge_b200.training import fused_margin_step, sharded_margin_step

_KIND_OF_CODE = {_lib.TRANSE_L2: "transe_l2", _lib.DISTMULT: "distmult", _lib.COMPLEX: "complex"}
_ENT_KEYS = {"transe_l2": ("ent",), "distmult": ("ent",), "complex": ("re_ent", "im_ent")}
_REL_KEYS = {"transe_l2": ("rel",), "distmult": ("rel",), "complex": ("re_rel", "im_rel")}


def draws(seed, offset, r, n_neg, probs, n_ent):
    """The stand-in's negatives: (head?, replacement) of negative j of fact i at index j * b + i, a
    function of (seed, offset) and the global n_ent only (the kernels use Philox; any fixed law
    serves the plumbing)."""
    g = torch.Generator().manual_seed((seed * 1000003 + offset) % (1 << 62))
    b = r.shape[0]
    u = torch.rand(n_neg * b, generator=g)
    e = torch.randint(1, max(n_ent, 2), (n_neg * b,), generator=g)
    return u < probs[r.repeat(n_neg)], e


class OracleStepEngine:
    """CPU stand-in for CudaEngine's sharded-step methods (tests only)."""

    def __init__(self):
        self.calls = []

    def gather_rows(self, spec, idx):
        planes = [spec.ent0] + ([spec.ent1] if spec.ent1 is not None else [])
        out = torch.zeros(idx.shape[0], len(planes), spec.dim)
        own = (idx >= spec.ent_lo) & (idx < spec.ent_lo + spec.n_rows)
        for p, tab in enumerate(planes):
            out[own, p] = tab[idx[own] - spec.ent_lo]
        return out

    def _partial(self, step, tables, h, t, r, probs, hrows, trows, grad):
        """Loss of the negatives this shard owns, from a table [local rows | hrows | trows]."""
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
        return torch.relu(step.margin - pos + neg).sum(), P

    def margin_step_fwd(self, step, tables, h, t, r, probs, hrows, trows):
        self.calls.append("fwd")
        with torch.no_grad():
            return self._partial(step, tables, h, t, r, probs, hrows, trows, False)[0].float()

    def margin_step_bwd(self, step, tables, grads, h, t, r, probs, gloss, hrows, trows, grad_hrows, grad_trows):
        self.calls.append("bwd")
        kind = _KIND_OF_CODE[step.code]
        with torch.enable_grad():          # autograd's backward runs with grad mode off
            loss, P = self._partial(step, tables, h, t, r, probs, hrows, trows, True)
            (loss * gloss).backward()
        n, b = step.n_rows, h.shape[0]
        for p, key in enumerate(_ENT_KEYS[kind]):
            gx = P[key].grad
            grads[p] += gx[:n]
            grad_hrows[:, p] += gx[n:n + b]
            grad_trows[:, p] += gx[n + b:]
        for p, key in enumerate(_REL_KEYS[kind]):
            grads[2 + p] += P[key].grad

    def scatter_rows_add(self, code, dim, grad0, grad1, ent_lo, idx, rows):
        self.calls.append("scatter")
        own = (idx >= ent_lo) & (idx < ent_lo + grad0.shape[0])
        for p, g in enumerate(x for x in (grad0, grad1) if x is not None):
            g.index_add_(0, idx[own] - ent_lo, rows[own, p])


def _local_model(kind, model, lo, hi, n_rel, dim):
    """The same model holding only entity rows [lo, hi)."""
    part = helpers.make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part


def _reference(kind, model, h, t, r, probs, seed, offset, n_neg, margin, n_ent):
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    head, e = draws(seed, offset, r, n_neg, probs, n_ent)
    nh = torch.where(head, e, h.repeat(n_neg))
    nt = torch.where(head, t.repeat(n_neg), e)
    pos, neg = oracle.forward_pos_neg(kind, P, h, t, r, nh, nt)
    loss = oracle.margin_loss(pos, neg, margin)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in P.items()}


class CountingShard(EntityShard):
    """EntityShard that counts its collectives."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.collectives = []

    def all_reduce_sum(self, t):
        self.collectives.append(("all_reduce", t.numel()))
        return super().all_reduce_sum(t)

    def stack_all(self, t):
        self.collectives.append(("stack_all", t.numel()))
        return super().stack_all(t)


def _run(rank, world, kind, n_ent, b, n_neg, steps):
    n_rel, dim, margin = 4, 8, 0.7
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=31)
    shard = CountingShard(n_ent, rank, world, None, local_storage=True)
    local = _local_model(kind, model, shard.lo, shard.hi, n_rel, dim)
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
        names = dict(zip(_ENT_KEYS[kind], ("ent_emb.weight",) if kind != "complex" else
                         ("re_ent_emb.weight", "im_ent_emb.weight")))
        names.update(zip(_REL_KEYS[kind], ("rel_emb.weight",) if kind != "complex" else
                         ("re_rel_emb.weight", "im_rel_emb.weight")))
        params = dict(local.named_parameters())
        for key, name in names.items():
            ref = want[key][shard.lo:shard.hi] if "ent" in key else want[key]
            ok["%s%d" % (key, s)] = torch.allclose(params[name].grad, ref, rtol=1e-4, atol=1e-6)
            if "rel" in key:    # relation gradients are the output of one all-reduce: equal everywhere
                ok["same_%s%d" % (key, s)] = bool((shard.stack_all(params[name].grad) == params[name].grad).all())
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
            model = _local_model("distmult", helpers.make_model("distmult", 8, 30, 4, seed=1), shard.lo, shard.hi, 4, 8)
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


def _spawn(world, case):
    return gloo.spawn(world, _worker, case)


# (world, kind, n_ent, b, n_neg, steps)
CASES = [
    (2, "distmult", 40, 12, 5, 2),
    (3, "complex", 31, 9, 4, 2),
    (3, "transe_l2", 2, 6, 3, 1),       # n_ent < world: rank 2 holds nothing
]


@pytest.mark.parametrize("case", CASES, ids=["%s-w%d-n%d" % (c[1], c[0], c[2]) for c in CASES])
def test_sharded_step_equals_oracle(case):
    world = case[0]
    ret = _spawn(world, case[1:])
    for rank in range(world):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad, "rank %d: %s" % (rank, bad)


def test_seed_mismatch_raises_on_every_rank():
    ret = _spawn(2, ("mismatch",))
    assert ret == {0: {"raised": True}, 1: {"raised": True}}


class Shard(EntityShard):
    """An EntityShard whose collectives fail: argument errors must come before any of them."""

    def all_reduce_sum(self, t):
        raise AssertionError("collective reached")

    stack_all = all_reduce_sum


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
        run(Shard(20, 0, 2, local_storage=False))
    with pytest.raises(ValueError, match="external negatives"):
        run(Shard(20, 0, 2, local_storage=True), negatives=(h, h))
    with pytest.raises(ValueError, match="holds 10 entity rows"):
        run(Shard(30, 0, 2, local_storage=True))          # rows [0, 15) expected
    with pytest.raises(ValueError, match="bern_probs"):
        run(Shard(20, 0, 2, local_storage=True), bern_probs=None)


def test_sampler_entity_count_must_match_the_shard():
    import torchkge_b200 as tk
    hh, tt, rr = helpers.random_graph(50, 4, 200, seed=3)
    kg = tk.KnowledgeGraph(hh, tt, rr, 50, 4, dict_of_heads={}, dict_of_tails={})
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=2, seed=1)
    model = helpers.make_model("distmult", 8, 25, 4, seed=2)
    with pytest.raises(ValueError, match="sampler draws on 50"):
        sampler.fused_step(model, hh[:4], tt[:4], rr[:4], 1.0, shard=Shard(60, 0, 2, local_storage=True))
