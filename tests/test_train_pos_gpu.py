"""Positional and uniform negatives in the fused training step on the GPU: the positional draw (draw_pos)
against a numpy statement of it, bit for bit, on the ring and the generic kernels; its law on a large draw;
the loss and gradients against float64 autograd on the CPU for every training code and the three losses,
with the kernel that ran checked (and again under KGE_TRAIN_RING=0); UniformNegativeSampler.fused_step
against corrupt_batch; the entity-sharded step emulated over three ranks and over gloo in two processes.

Tolerances as in tests/test_train_relneg_gpu.py."""
import ctypes
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats

import torchkge_b200 as tk
from tests import gloo, helpers
from tests.test_train_paths_gpu import RING_MAX_NEG, SMEM_MAX, _cuda_kernel_names, last_n_neg_within, \
    margin_between, ring_smem_bytes
from tests.test_train_relneg_gpu import philox_words
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard, _exchanged_rows
from torchkge_b200.training import ShardedStep, _MarginStep, _row_spec

DEV = helpers.DEV
pytestmark = pytest.mark.gpu

CODES = ("transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "toruse_l1", "toruse_l2", "analogy")
RING_KINDS = ("transe_l1", "transe_l2", "distmult")
SEED, OFFSET = 777, 3


# ---------------------------------------------------------------- the candidate graph
def csr(rel, ent, n_rel, n_ent):
    """Sorted CSR of the distinct (relation, entity) pairs, as PositionalNegativeSampler builds it."""
    key = torch.unique(rel * n_ent + ent)
    offs = torch.zeros(n_rel + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.bincount(key // n_ent, minlength=n_rel), 0)
    return offs, key % n_ent


def graph(n_ent, n_rel, seed):
    """Candidate CSRs where relation 0 has no candidates on either side, relation 1 exactly one per side, and
    relation 2 more than 2^16 heads; the others a few hundred random ones."""
    g = torch.Generator().manual_seed(seed)
    rels, heads, tails = [], [], []
    rels.append(torch.tensor([1])); heads.append(torch.tensor([5])); tails.append(torch.tensor([n_ent - 1]))
    big = torch.randperm(n_ent, generator=g)[:70_001]
    rels.append(torch.full((big.shape[0],), 2)); heads.append(big)
    tails.append(torch.randint(0, n_ent, (big.shape[0],), generator=g) % 37)
    for r in range(3, n_rel):
        k = int(torch.randint(20, 400, (1,), generator=g))
        rels.append(torch.full((k,), r)); heads.append(torch.randint(0, n_ent, (k,), generator=g))
        tails.append(torch.randint(0, n_ent, (k,), generator=g))
    rel, hd, tl = torch.cat(rels), torch.cat(heads), torch.cat(tails)
    ho, he = csr(rel, hd, n_rel, n_ent)
    to, te = csr(rel, tl, n_rel, n_ent)
    return ho, he, to, te


def pos_draws(seed, offset, r, n_neg, probs, n_ent, pos):
    """The numpy statement of draw_pos: (head?, replacement) of negative j of fact i at index j b + i."""
    ho, he, to, te = (x.numpy().astype(np.int64) for x in pos)
    R = np.tile(r.numpy(), n_neg)
    x, y, _, _ = philox_words(seed, offset, np.arange(R.shape[0]))
    u = (x >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    head = u < probs.numpy().astype(np.float32)[R]
    lo = np.where(head, ho[R], to[R])
    n = np.where(head, ho[R + 1] - ho[R], to[R + 1] - to[R])
    k = ((y * n.astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
    e_any = ((y * np.uint64(n_ent)) >> np.uint64(32)).astype(np.int64)
    pick = np.where(n > 0, lo + k, 0)
    e = np.where(n > 0, np.where(head, he[np.minimum(pick, max(he.size - 1, 0))] if he.size else 0,
                                 te[np.minimum(pick, max(te.size - 1, 0))] if te.size else 0), e_any)
    return torch.from_numpy(head), torch.from_numpy(e)


def expected_draws(h, t, r, n_neg, probs, n_ent, pos):
    head, e = pos_draws(SEED, OFFSET, r.cpu(), n_neg, probs.cpu(), n_ent, pos)
    H, T = h.cpu().repeat(n_neg), t.cpu().repeat(n_neg)
    return torch.where(head, e, H), torch.where(head, T, e)


def drawn_step(model, h, t, r, probs, n_neg, loss, margin, pos, n_ent):
    """The fused positional step on its own draws: (loss, leaves with grads, nh, nt, neg scores), the negatives
    and scores read back through nh_out / nt_out / neg_out of kge_pos_step_fwd."""
    code, dim, ts = helpers.train_leaves(model)
    lk = helpers.LOSS_KINDS[loss]
    pos_dev = tuple(x.to(DEV) for x in pos)
    got = _MarginStep.apply(code, dim, n_ent, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *ts, lk, None,
                            None, pos_dev)
    got.backward()
    b = h.shape[0]
    ids = [torch.full((b * n_neg,), -1, dtype=torch.int64, device=DEV) for _ in range(2)]
    neg_out = torch.full((b * n_neg,), float("nan"), device=DEV)
    out = torch.zeros((), device=DEV)
    tabs = [None if x is None else x.detach() for x in ts]
    a = _MarginStep._args(code, dim, n_ent, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, tabs, out,
                          h.device, lk, None, None, pos_dev)
    assert isinstance(a, _lib.PosStepArgs)
    a.base.nh_out, a.base.nt_out, a.base.neg_out = _ptr(ids[0]), _ptr(ids[1]), _ptr(neg_out)
    assert _lib.load().kge_pos_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()
    assert out.item() == pytest.approx(got.item(), rel=1e-5, abs=1e-7)   # fp32 atomics in another order
    return got.item(), ts, ids[0], ids[1], neg_out


def _ptr(x):
    return x.data_ptr()


_STEP_KERNEL = re.compile(r"(margin_step_(?:ring_pos|ring_rel|ring|fast|shard_fwd|shard_bwd|fwd|bwd)_kernel)")


def expected_kernels(kind, d, n_neg, shard):
    """The kernels a positional step launches: the ring kernel's positional kind for TransE-L1 / L2 and
    DistMult where the ring applies (not under KGE_TRAIN_RING=0), else the generic kernels -- never the
    register-resident form."""
    ring_on = os.environ.get("KGE_TRAIN_RING", "")[:1] != "0"
    if (kind in RING_KINDS and d % 4 == 0 and d <= 256 and ring_on and n_neg <= RING_MAX_NEG and
            ring_smem_bytes(d, n_neg) <= SMEM_MAX):
        return {"margin_step_ring_pos_kernel"}
    return {"margin_step_shard_fwd_kernel", "margin_step_shard_bwd_kernel"} if shard else \
        {"margin_step_fwd_kernel", "margin_step_bwd_kernel"}


def launched(fn, expected, tries=4):
    ran = set()
    for _ in range(tries):
        ran |= {m.group(1) for m in map(_STEP_KERNEL.search, _cuda_kernel_names(fn)) if m}
        if ran >= expected:
            break
    return ran


# ---------------------------------------------------------------- 1. the draws, bit for bit
@pytest.mark.parametrize("kind,d,n_neg", [("distmult", 8, 7), ("transe_l2", 36, 1), ("complex", 8, 5),
                                          ("distmult", 8, last_n_neg_within(8, SMEM_MAX) + 1)])
def test_draws_equal_the_numpy_statement(kind, d, n_neg):
    """Relation 0 (empty: entity 0 can be drawn), 1 (one candidate), 2 (> 2^16 candidates) and others, on the
    ring kernel (DistMult, TransE) and on the generic kernels (ComplEx, and DistMult past the ring)."""
    n_ent, n_rel = 100_003, 9
    pos = graph(n_ent, n_rel, seed=1)
    model = helpers.train_model(kind, d, n_ent, n_rel, seed=2)
    g = torch.Generator().manual_seed(3)
    b = 600 if n_neg < 100 else 8
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.arange(b) % n_rel
    probs = torch.rand(n_rel, generator=g)
    probs[:3] = torch.tensor([0.5, 0.5, 0.9])
    h, t, r, probs = h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)
    _, _, nh, nt, _ = drawn_step(model, h, t, r, probs, n_neg, "logistic", 0.0, pos, n_ent)
    want_nh, want_nt = expected_draws(h, t, r, n_neg, probs, n_ent, pos)
    assert torch.equal(nh.cpu(), want_nh) and torch.equal(nt.cpu(), want_nt)
    R = r.cpu().repeat(n_neg)
    e = torch.where(nh.cpu() != h.cpu().repeat(n_neg), nh.cpu(), nt.cpu())
    if n_neg * b > 2000:      # relation 0 draws from [0, n_ent); somewhere a low id shows it is not [1, n_ent)
        assert int(e[R == 0].min()) < n_ent // 100
    assert set(nh.cpu()[(R == 1) & (nh.cpu() != h.cpu().repeat(n_neg))].tolist()) <= {5}
    assert set(nt.cpu()[(R == 1) & (nt.cpu() != t.cpu().repeat(n_neg))].tolist()) <= {n_ent - 1}
    code, dim, _ = helpers.train_leaves(model)
    pos_dev = tuple(x.to(DEV) for x in pos)

    def step():
        leaves = helpers.train_leaves(model)[2]
        _MarginStep.apply(code, dim, n_ent, 0.0, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *leaves,
                          _lib.LOSS_LOGISTIC, None, None, pos_dev).backward()
    want = expected_kernels(kind, d, n_neg, shard=False)
    assert launched(step, want) == want


def test_the_law_of_a_large_draw():
    """Support inside the candidate lists, head share per relation near bern_probs[r], uniform inside a slice."""
    n_ent, n_rel = 100_003, 9
    pos = graph(n_ent, n_rel, seed=4)
    ho, he, to, te = pos
    b, n_neg = 100_000, 4
    g = torch.Generator().manual_seed(5)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, n_rel, (b,), generator=g)
    probs = torch.rand(n_rel, generator=g)
    model = helpers.train_model("distmult", 4, n_ent, n_rel, seed=6)
    _, _, nh, nt, _ = drawn_step(model, h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV), n_neg, "logistic", 0.0,
                                 pos, n_ent)
    nh, nt = nh.cpu(), nt.cpu()
    head, e = pos_draws(SEED, OFFSET, r, n_neg, probs, n_ent, pos)
    R = r.repeat(n_neg)
    assert torch.equal(nh, torch.where(head, e, h.repeat(n_neg))) and torch.equal(nt, torch.where(head, t.repeat(n_neg), e))
    for rel in range(n_rel):
        m = R == rel
        p = float(probs[rel])
        f = float(head[m].double().mean())
        assert abs(f - p) <= 5 * math.sqrt(max(p * (1 - p), 1e-12) / int(m.sum())) + 1e-12, rel
        for side, offs, ents in ((head, ho, he), (~head, to, te)):
            drawn = e[m & side]
            cand = ents[offs[rel]:offs[rel + 1]]
            if cand.numel():
                assert bool(torch.isin(drawn, cand).all()), rel
            else:
                assert int(drawn.min()) >= 0 and int(drawn.max()) < n_ent
    # uniform inside relation 3's head slice (a few hundred distinct candidates, each a bin)
    m = (R == 3) & head
    cand = he[ho[3]:ho[4]]
    counts = torch.bincount(torch.searchsorted(cand, e[m]), minlength=cand.numel()).numpy()
    assert stats.chisquare(counts).pvalue > 1e-4


# ---------------------------------------------------------------- 2. against float64 autograd
N_ENT, N_REL = 700, 13


def small_graph(seed=8):
    g = torch.Generator().manual_seed(seed)
    n = 3000
    rel = torch.randint(1, N_REL, (n,), generator=g)            # relation 0: no candidates
    hd, tl = torch.randint(0, N_ENT, (n,), generator=g), torch.randint(0, N_ENT, (n,), generator=g)
    hd[rel == 1], tl[rel == 1] = 9, 11                          # relation 1: one candidate per side
    return csr(rel, hd, N_REL, N_ENT) + csr(rel, tl, N_REL, N_ENT)


def problem(kind, d, n_neg, seed, b=23, n_ent=N_ENT):
    model = helpers.train_model(kind, d, n_ent, N_REL, seed=seed)
    gen = torch.Generator().manual_seed(seed + n_neg)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, N_REL, (b,), generator=gen)
    probs = torch.rand(N_REL, generator=gen)
    return model, h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)


def reference(kind, ts, h, t, r, nh, nt, loss, margin):
    cpu = helpers.cpu_leaves(ts, torch.float64)
    pos, neg = helpers.cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    want = helpers.torch_loss(loss, pos, neg, margin)
    want.backward()
    return want.item(), [None if x is None else x.grad for x in cpu], neg.detach()


def _cases():
    out = [(k, 16, n, loss) for k in CODES for n in (1, 7) for loss in ("margin", "logistic", "bce")]
    out += [(k, 36, last_n_neg_within(36, SMEM_MAX) + 1, loss) for k in RING_KINDS for loss in ("margin", "bce")]
    out += [(k, 200, 256, "logistic") for k in RING_KINDS]
    return out


CASES = _cases()


@pytest.mark.parametrize("kind,d,n_neg,loss", CASES, ids=["%s-d%d-neg%d-%s" % c for c in CASES])
def test_drawn_step_matches_float64_autograd(kind, d, n_neg, loss):
    model, h, t, r, probs = problem(kind, d, n_neg, seed=d + n_neg)
    pos = small_graph()
    want_nh, want_nt = expected_draws(h, t, r, n_neg, probs, N_ENT, pos)
    margin = 0.0
    if loss == "margin":    # no hinge so near its kink that float32 and float64 could disagree on it
        cpu = helpers.cpu_leaves(helpers.train_leaves(model)[2], torch.float64)
        p_, n_ = helpers.cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), want_nh, want_nt)
        margin = margin_between((p_ - n_).detach())
    got, ts, nh, nt, neg_out = drawn_step(model, h, t, r, probs, n_neg, loss, margin, pos, N_ENT)
    assert torch.equal(nh.cpu(), want_nh) and torch.equal(nt.cpu(), want_nt)
    want_loss, want_grads, neg = reference(kind, ts, h, t, r, nh, nt, loss, margin)
    torch.testing.assert_close(neg_out.cpu().double(), neg.double(), rtol=1e-5, atol=1e-5)
    assert got == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    for a, c in zip(ts, want_grads):
        if c is None:
            continue
        if n_neg <= 1000:
            helpers.close_grad(a.grad, c, rtol=2e-4)
        else:
            # past the ring the generic kernels add every pair's gradient by its own fp32 atomics: ~10^4 of them
            # per row of the 700-entity table, whose rounding error scales with the table's largest entry
            torch.testing.assert_close(a.grad.cpu().float(), c.float(), rtol=2e-4, atol=2e-4 * float(c.abs().max()))
    code, dim, _ = helpers.train_leaves(model)
    pos_dev = tuple(x.to(DEV) for x in pos)

    def step():
        leaves = helpers.train_leaves(model)[2]
        _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *leaves,
                          helpers.LOSS_KINDS[loss], None, None, pos_dev).backward()
    want = expected_kernels(kind, d, n_neg, shard=False)
    assert launched(step, want) == want


# ---------------------------------------------------------------- 3. the samplers
def test_positional_sampler_fused_step_equals_loop_on_its_draws():
    kg, _, _ = helpers.make_kg(400, 9, n_facts=3000, n_test=100, seed=5)
    h, t, r = kg.head_idx[:512].to(DEV), kg.tail_idx[:512].to(DEV), kg.relations[:512].to(DEV)
    s = tk.PositionalNegativeSampler(kg, seed=21)
    m = helpers.train_model("distmult", 32, 400, 9, seed=6)
    loss = s.fused_step(m, h, t, r, criterion=tk.LogisticLoss(), n_neg=3)
    assert s._calls == 1
    offs_h, ents_h, _ = s._csr["heads"]
    offs_t, ents_t, _ = s._csr["tails"]
    pos = (offs_h, ents_h, offs_t, ents_t)
    head, e = pos_draws(s.seed, 1, r.cpu(), 3, s.bern_probs.cpu(), 400, pos)
    nh = torch.where(head, e, h.cpu().repeat(3))
    nt = torch.where(head, t.cpu().repeat(3), e)
    m2 = helpers.train_model("distmult", 32, 400, 9, seed=6)
    want = tk.training.fused_loss_step(m2, h, t, r, tk.LogisticLoss(), negatives=(nh.to(DEV), nt.to(DEV)))
    assert loss.item() == pytest.approx(want.item(), rel=1e-5)
    loss.backward()
    want.backward()
    for a, c in zip(m.parameters(), m2.parameters()):
        helpers.close_grad(a.grad, c.grad, rtol=1e-4)
    with pytest.raises(ValueError, match="entities"):     # before the call count moves
        s.fused_step(helpers.train_model("distmult", 8, 401, 9, seed=1), h, t, r, margin=1.0)
    assert s._calls == 1
    with pytest.raises(ValueError, match="relations"):
        s.fused_step(helpers.train_model("distmult", 8, 400, 10, seed=1), h, t, r, margin=1.0)


@pytest.mark.parametrize("loss", ["margin", "bce"])
def test_uniform_fused_step_draws_what_corrupt_batch_draws(loss):
    kg, _, _ = helpers.make_kg(500, 7, n_facts=3000, n_test=100, seed=9)
    h, t, r = kg.head_idx[:700].to(DEV), kg.tail_idx[:700].to(DEV), kg.relations[:700].to(DEV)
    crit = tk.MarginLoss(0.8) if loss == "margin" else tk.BinaryCrossEntropyLoss()
    s1, s2 = tk.UniformNegativeSampler(kg, seed=31), tk.UniformNegativeSampler(kg, seed=31)
    s1.corrupt_batch(h, t, r, n_neg=2)          # both samplers at call 2 next
    s2.corrupt_batch(h, t, r, n_neg=2)
    m1, m2 = helpers.train_model("transe_l2", 24, 500, 7, seed=3), helpers.train_model("transe_l2", 24, 500, 7, seed=3)
    got = s1.fused_step(m1, h, t, r, criterion=crit, n_neg=5)
    nh, nt = s2.corrupt_batch(h, t, r, n_neg=5)
    want = tk.training.fused_loss_step(m2, h, t, r, crit, negatives=(nh, nt))
    assert got.item() == pytest.approx(want.item(), rel=1e-6, abs=1e-7)
    got.backward()
    want.backward()
    for a, c in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a.grad, c.grad, rtol=1e-5, atol=1e-6 * float(c.grad.abs().max()) + 1e-9)
    # the draws themselves, through nh_out / nt_out of the entity step at the sampler's (seed, call count)
    code, dim, ts = helpers.train_leaves(m1)
    out = torch.zeros((), device=DEV)
    ids = [torch.full((h.shape[0] * 5,), -1, dtype=torch.int64, device=DEV) for _ in range(2)]
    a = _MarginStep._args(code, dim, 500, 1.0, 5, h, t, r, None, None, s1._halves, s1.seed, 2,
                          [None if x is None else x.detach() for x in ts], out, h.device)
    a.nh_out, a.nt_out = _ptr(ids[0]), _ptr(ids[1])
    assert _lib.load().kge_margin_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()
    assert torch.equal(ids[0], nh) and torch.equal(ids[1], nt)


# ---------------------------------------------------------------- 4. entity-sharded, emulated
def emulated(model, h, t, r, probs, margin, n_neg, world, eng, lk, pos, n_ent):
    """Every rank's kernels on its row range, the all-reduces as sums, then every rank's scatter."""
    code, dim, ts = helpers.train_leaves(model)
    tabs = [None if x is None else x.detach() for x in ts]
    b = h.shape[0]
    full = ShardedStep(code, dim, n_ent, 0, n_ent, n_neg, float(margin), SEED, OFFSET, lk, 0, 1.0, pos)
    rows = _exchanged_rows(_row_spec(full, tabs), torch.cat([h, t]), EntityShard(n_ent), eng)
    hrows, trows = rows[:b], rows[b:]
    loss = torch.zeros((), dtype=torch.float32, device=DEV)
    grad_rows = torch.zeros_like(rows)
    grel = [None if x is None else torch.zeros_like(x) for x in tabs[2:]]
    gent = [None if x is None else torch.zeros_like(x) for x in tabs[:2]]
    parts = []
    for rank in range(world):
        sh = EntityShard(n_ent, rank, world, local_storage=True)
        n = sh.hi - sh.lo
        local = [None if x is None else x.narrow(-2, sh.lo, n) for x in tabs[:2]] + tabs[2:]
        lg = [None if x is None else x.narrow(-2, sh.lo, n) for x in gent]
        parts.append((sh, lg))
        if n == 0:
            continue
        step = ShardedStep(code, dim, n_ent, sh.lo, n, n_neg, float(margin), SEED, OFFSET, lk, 0, 1.0, pos)
        loss += eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
        g_rows = torch.zeros_like(rows)
        g_rel = [None if x is None else torch.zeros_like(x) for x in tabs[2:]]
        gl = torch.ones((), dtype=torch.float32, device=DEV)
        eng.margin_step_bwd(step, local, lg + g_rel, h, t, r, probs, gl, hrows, trows, g_rows[:b], g_rows[b:])
        grad_rows += g_rows
        for a, c in zip(grel, g_rel):
            if a is not None:
                a += c
    for sh, lg in parts:
        if sh.hi > sh.lo:
            eng.scatter_rows_add(code, dim, lg[0], lg[1], sh.lo, torch.cat([h, t]), grad_rows)
    return loss.item(), gent + grel


SHARD_CASES = ([(k, 16, 6, loss) for k in ("transe_l2", "distmult", "complex", "rescal", "analogy")
                for loss in ("margin", "logistic")] + [(k, 200, 256, "bce") for k in RING_KINDS])


@pytest.mark.parametrize("kind,d,n_neg,loss", SHARD_CASES, ids=["%s-d%d-neg%d-%s" % c for c in SHARD_CASES])
def test_sharded_step_sums_to_unsharded(kind, d, n_neg, loss):
    margin = 0.5
    model, h, t, r, probs = problem(kind, d, n_neg, seed=13)
    lk = helpers.LOSS_KINDS[loss]
    pos = tuple(x.to(DEV) for x in small_graph())
    code, dim, ts = helpers.train_leaves(model)
    one = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *ts, lk, None,
                            None, pos)
    one.backward()
    eng = CudaEngine()
    for world in (1, 3):
        got_loss, got_grads = emulated(model, h, t, r, probs, margin, n_neg, world, eng, lk, pos, N_ENT)
        assert got_loss == pytest.approx(one.item(), rel=1e-5, abs=1e-6), world
        for a, c in zip(got_grads, ts):
            if c is not None:
                helpers.close_grad(a, c.grad, rtol=1e-4)
    want = expected_kernels(kind, d, n_neg, shard=True)
    ran = launched(lambda: emulated(model, h, t, r, probs, margin, n_neg, 3, eng, lk, pos, N_ENT), want)
    assert ran == want


def test_sharded_step_with_a_rank_that_holds_no_rows():
    """2 entities over 3 ranks: rank 2 holds nothing and scores nothing."""
    model, h, t, r, probs = problem("distmult", 8, 4, seed=19, b=9, n_ent=2)
    g = torch.Generator().manual_seed(1)
    rel = torch.randint(1, N_REL, (30,), generator=g)
    hd, tl = torch.randint(0, 2, (30,), generator=g), torch.randint(0, 2, (30,), generator=g)
    pos = tuple(x.to(DEV) for x in csr(rel, hd, N_REL, 2) + csr(rel, tl, N_REL, 2))
    code, dim, ts = helpers.train_leaves(model)
    one = _MarginStep.apply(code, dim, 2, 0.0, 4, h, t, r, None, None, probs, SEED, OFFSET, *ts,
                            _lib.LOSS_LOGISTIC, None, None, pos)
    one.backward()
    got_loss, got_grads = emulated(model, h, t, r, probs, 0.0, 4, 3, CudaEngine(), _lib.LOSS_LOGISTIC, pos, 2)
    assert got_loss == pytest.approx(one.item(), rel=1e-5, abs=1e-6)
    for a, c in zip(got_grads, ts):
        if c is not None:
            helpers.close_grad(a, c.grad, rtol=1e-4)


# ---------------------------------------------------------------- 5. public API, two processes on one GPU
def _local_model(kind, model, lo, hi, n_rel, dim):
    part = helpers.make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part.to(next(model.parameters()).device)


def _train(model, kg, batches, shard, crit):
    sampler = tk.PositionalNegativeSampler(kg, seed=3)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for h, t, r in batches:
        opt.zero_grad()
        loss = sampler.fused_step(model, h, t, r, criterion=crit, n_neg=16, shard=shard)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return losses


def _api_worker(rank, world, _):
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    try:
        from torchkge_b200.engine import EntityShard as Shard
        res = {}
        n_ent, n_rel = 3001, 7
        hh, tt, rr = helpers.random_graph(n_ent, n_rel, 6000, seed=5)
        kg = tk.KnowledgeGraph(hh, tt, rr, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
        batches = [(hh[i:i + 512].to(dev), tt[i:i + 512].to(dev), rr[i:i + 512].to(dev)) for i in range(0, 2048, 512)]
        # DistMult d=200 takes the ring kernel's positional kind, ComplEx the generic kernels
        for kind, dim, crit in (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.MarginLoss(1.0))):
            full = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
            shard = Shard.from_group(n_ent, local_storage=True)
            local = _local_model(kind, full, shard.lo, shard.hi, n_rel, dim)
            want = _train(full, kg, batches, None, crit)
            got = _train(local, kg, batches, shard, crit)
            res[kind + "/losses_close"] = all(abs(a - b) <= 1e-5 * abs(b) + 1e-6 for a, b in zip(got, want))
            for name, p in local.named_parameters():
                ref = dict(full.named_parameters())[name]
                res[kind + "/" + name] = torch.allclose(p, ref[shard.lo:shard.hi] if "ent_emb" in name else ref,
                                                        rtol=1e-4, atol=1e-5)
        other = kg if rank == 0 else tk.KnowledgeGraph(hh[:5000], tt[:5000], rr[:5000], n_ent, n_rel,
                                                       dict_of_heads={}, dict_of_tails={})
        try:
            tk.PositionalNegativeSampler(other, seed=100).fused_step(local, *batches[0], criterion=tk.LogisticLoss(),
                                                                     shard=shard)
            res["csr_mismatch_raises"] = False
        except ValueError as e:
            res["csr_mismatch_raises"] = "CSR" in str(e)
        return res
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


def test_public_api_two_processes_gloo_one_gpu():
    ret = gloo.spawn(2, _api_worker, None)
    for rank in (0, 1):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad and len(res) >= 6, "rank %d: %s" % (rank, res)


# ---------------------------------------------------------------- 6. KGE_TRAIN_RING=0
def test_without_the_ring():
    """The draw, float64 and sharded cases of the ring kinds once more in a child process under
    KGE_TRAIN_RING=0: every positional step then takes the generic kernels (expected_kernels reads the
    switch)."""
    if "KGE_TRAIN_RING" in os.environ:
        pytest.skip("runs in the parent process only")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
         "(draws_equal or drawn_step or sharded_step_sums) and (transe or distmult)"]
    proc = subprocess.run(cmd, cwd=root, env=dict(os.environ, KGE_TRAIN_RING="0"), capture_output=True, text=True,
                          timeout=1200)
    assert proc.returncode == 0, proc.stdout[-6000:] + proc.stderr[-3000:]
    assert " passed" in proc.stdout, proc.stdout[-2000:]
