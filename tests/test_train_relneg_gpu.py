"""Relation-corrupting negatives (BernoulliRelationNegativeSampler) on the GPU: the law of
kge_corrupt_batch_rel, the fused step against the unfused loop and against float64 autograd on the
CPU for every training code, and the entity-sharded step emulated over 1, 2, 3 and 8 ranks.

Tolerances as in tests/test_train_paths_gpu.py: losses within 2e-5 of float64 (1e-5 against the
float32 loop), gradients under helpers.close_grad."""
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
from tests.test_train_paths_gpu import RING_MAX_NEG, SMEM_MAX, _cuda_kernel_names, ring_smem_bytes
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard, _exchanged_rows, _ptr, _stream
from torchkge_b200.training import ShardedStep, _MarginStep, _row_spec

DEV = helpers.DEV
pytestmark = pytest.mark.gpu

CODES = ("transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "toruse_l1", "toruse_l2", "analogy")
N_ENT, N_REL = 700, 13
SEED, OFFSET = 2024, 5


def corrupt_rel(h, t, r, probs, n_neg, n_ent, n_rel, rel_share, seed=SEED, offset=OFFSET):
    nh, nt, nr = (torch.empty(h.shape[0] * n_neg, dtype=torch.int64, device=DEV) for _ in range(3))
    _lib.check(_lib.load().kge_corrupt_batch_rel(_ptr(h), _ptr(t), _ptr(r), h.shape[0], n_neg, _ptr(probs), n_ent,
                                                 n_rel, rel_share, seed, offset, _ptr(nh), _ptr(nt), _ptr(nr),
                                                 _stream(h.device)), "kge_corrupt_batch_rel")
    return nh, nt, nr


def corrupt_ent(h, t, r, probs, n_neg, n_ent, seed=SEED, offset=OFFSET):
    nh, nt = (torch.empty(h.shape[0] * n_neg, dtype=torch.int64, device=DEV) for _ in range(2))
    _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), h.shape[0], n_neg, _ptr(probs), n_ent, seed,
                                             offset, _ptr(nh), _ptr(nt), _stream(h.device)), "kge_corrupt_batch")
    return nh, nt


# ---------------------------------------------------------------- 1. the law of the draws
def philox_words(seed, offset, idx):
    """Philox4x32-10 with counter (idx, offset) and key seed, in numpy (csrc/train.cu: philox4x32)."""
    M = np.uint64(0xFFFFFFFF)
    idx = idx.astype(np.uint64)
    c0, c1 = idx & M, idx >> np.uint64(32)
    c2 = np.full_like(c0, offset & 0xFFFFFFFF)
    c3 = np.full_like(c0, offset >> 32)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & M
        hi1, lo1 = p1 >> np.uint64(32), p1 & M
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def test_bernoulli_draws_are_those_of_the_philox_statement():
    """kge_corrupt_batch (BernoulliNegativeSampler) still draws what draw_one states: head iff
    (x >> 8) / 2^24 < p_r, entity 1 + (y (n_ent - 1)) >> 32."""
    b, n_neg, n_ent = 4099, 3, 100003
    g = torch.Generator().manual_seed(1)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, N_REL, (b,), generator=g)
    probs = torch.rand(N_REL, generator=g)
    nh, nt = corrupt_ent(h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV), n_neg, n_ent)
    x, y, _, _ = philox_words(SEED, OFFSET, np.arange(b * n_neg))
    u = (x >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    e = torch.from_numpy((1 + ((y * np.uint64(n_ent - 1)) >> np.uint64(32))).astype(np.int64))
    head = torch.from_numpy(u) < probs[r.repeat(n_neg)]
    assert torch.equal(nh.cpu(), torch.where(head, e, h.repeat(n_neg)))
    assert torch.equal(nt.cpu(), torch.where(head, t.repeat(n_neg), e))


def test_relation_draws_follow_the_law():
    b, n_neg, n_ent, n_rel, share = 250_000, 4, 5003, 97, 0.33
    g = torch.Generator().manual_seed(2)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, 6, (b,), generator=g)
    probs = torch.zeros(n_rel)
    probs[:6] = torch.tensor([0.0, 1.0, 0.5, 0.2, 0.9, 0.35])
    hd, td, rd, pd = h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)
    nh, nt, nr = (x.cpu() for x in corrupt_rel(hd, td, rd, pd, n_neg, n_ent, n_rel, share))
    H, T, R = h.repeat(n_neg), t.repeat(n_neg), r.repeat(n_neg)
    ch, ct, cr = nh != H, nt != T, nr != R
    # a replaced position may redraw its old value: then nothing changes; never more than one changes
    assert int((ch.int() + ct.int() + cr.int()).max()) <= 1
    n = b * n_neg
    # which kind: the same words through the numpy statement
    x, y, z, w = philox_words(SEED, OFFSET, np.arange(n))
    u_ent = (z >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    is_rel = torch.from_numpy(~(u_ent < np.float32(share)))
    frac = float(is_rel.double().mean())
    assert abs(frac - (1 - share)) <= 5 * math.sqrt(share * (1 - share) / n)
    new_r = torch.from_numpy((1 + ((w * np.uint64(n_rel - 1)) >> np.uint64(32))).astype(np.int64))
    assert torch.equal(nr, torch.where(is_rel, new_r, R))
    assert torch.equal(nh[is_rel], H[is_rel]) and torch.equal(nt[is_rel], T[is_rel])
    head = torch.from_numpy((x >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)) < probs[R]
    e = torch.from_numpy((1 + ((y * np.uint64(n_ent - 1)) >> np.uint64(32))).astype(np.int64))
    ent = ~is_rel
    assert torch.equal(nh[ent], torch.where(head, e, H)[ent]) and torch.equal(nt[ent], torch.where(head, T, e)[ent])
    # head fraction among the entity negatives, per relation
    for rel in range(6):
        m = ent & (R == rel)
        p = float(probs[rel])
        f = float(head[m].double().mean())
        assert abs(f - p) <= 5 * math.sqrt(max(p * (1 - p), 1e-12) / int(m.sum())) + 1e-12, rel
    # replacements: never 0, uniform on [1, n)
    rep_r = new_r[is_rel]
    rep_e = e[ent]
    assert int(rep_r.min()) >= 1 and int(rep_r.max()) < n_rel
    assert int(rep_e.min()) >= 1 and int(rep_e.max()) < n_ent
    for vals, k in ((rep_r, n_rel), (rep_e, n_ent)):
        counts = torch.bincount(vals, minlength=k)[1:].numpy()
        assert stats.chisquare(counts).pvalue > 1e-4
    # the same (seed, offset) gives the same draws; another offset others
    again = [x.cpu() for x in corrupt_rel(hd, td, rd, pd, n_neg, n_ent, n_rel, share)]
    assert all(torch.equal(a, c) for a, c in zip(again, (nh, nt, nr)))
    other = corrupt_rel(hd, td, rd, pd, n_neg, n_ent, n_rel, share, offset=OFFSET + 1)[2].cpu()
    assert not torch.equal(other, nr)


@pytest.mark.parametrize("share", [0.0, 1.0])
def test_rel_share_extremes(share):
    b, n_neg, n_ent, n_rel = 5000, 3, 800, 9
    g = torch.Generator().manual_seed(3)
    h, t = torch.randint(0, n_ent, (b,), generator=g).to(DEV), torch.randint(0, n_ent, (b,), generator=g).to(DEV)
    r = torch.randint(0, n_rel, (b,), generator=g).to(DEV)
    probs = torch.rand(n_rel, generator=g).to(DEV)
    nh, nt, nr = corrupt_rel(h, t, r, probs, n_neg, n_ent, n_rel, share)
    if share == 1.0:      # exactly BernoulliNegativeSampler's draws
        eh, et = corrupt_ent(h, t, r, probs, n_neg, n_ent)
        assert torch.equal(nh, eh) and torch.equal(nt, et) and torch.equal(nr, r.repeat(n_neg))
    else:
        assert torch.equal(nh, h.repeat(n_neg)) and torch.equal(nt, t.repeat(n_neg))
        assert int(nr.min()) >= 1


def test_sampler_api():
    kg, _, _ = helpers.make_kg(300, 7, n_facts=2000, n_test=10, seed=4)
    s = tk.BernoulliRelationNegativeSampler(kg, n_neg=5, seed=9)
    assert s.rel_share == pytest.approx(0.33) and s.bern_probs.shape == (7,)
    h, t, r = kg.head_idx.to(DEV), kg.tail_idx.to(DEV), kg.relations.to(DEV)
    nh, nt, nr = s.corrupt_batch(h, t, r, n_neg=4)
    assert nh.shape == h.shape and nh.dtype == torch.int64 and nh.device == h.device   # one per fact
    twin = tk.BernoulliNegativeSampler(kg, seed=9)
    s1 = tk.BernoulliRelationNegativeSampler(kg, rel_share=1.0, seed=9)
    a = s1.corrupt_batch(h, t, r)
    c = twin.corrupt_batch(h, t, r, n_neg=1)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]) and torch.equal(a[2], r)
    out = tk.BernoulliRelationNegativeSampler(kg, seed=9).corrupt_kg(512, True)
    assert len(out) == 3 and all(x.shape == (kg.n_facts,) and x.device.type == "cpu" for x in out)


# ---------------------------------------------------------------- 2. fused step == the unfused loop
def _loss_of(name, margin=1.0):
    return {"margin": tk.MarginLoss(margin), "logistic": tk.LogisticLoss(), "bce": tk.BinaryCrossEntropyLoss()}[name]


@pytest.mark.parametrize("loss", ["margin", "logistic", "bce"])
@pytest.mark.parametrize("kind", ["transe_l2", "distmult", "complex"])
def test_fused_step_equals_unfused_loop(kind, loss):
    kg, _, _ = helpers.make_kg(400, 9, n_facts=3000, n_test=257, seed=5)
    crit = _loss_of(loss, margin=0.7)
    h, t, r = kg.head_idx.to(DEV), kg.tail_idx.to(DEV), kg.relations.to(DEV)
    m1 = helpers.train_model(kind, 32, 400, 9, seed=6)
    m2 = helpers.train_model(kind, 32, 400, 9, seed=6)
    s1 = tk.BernoulliRelationNegativeSampler(kg, rel_share=0.5, seed=77)
    s2 = tk.BernoulliRelationNegativeSampler(kg, rel_share=0.5, seed=77)
    got = s1.fused_step(m1, h, t, r, criterion=crit)
    got.backward()
    pos, neg = m2(h, t, r, *s2.corrupt_batch(h, t, r))
    want = crit(pos, neg)
    want.backward()
    assert got.item() == pytest.approx(want.item(), rel=1e-5)
    for (name, a), (_, c) in zip(m1.named_parameters(), m2.named_parameters()):
        if c.grad is not None:
            helpers.close_grad(a.grad, c.grad, rtol=1e-4)


def test_fused_step_argument_errors():
    kg, _, _ = helpers.make_kg(100, 5, n_facts=300, n_test=20, seed=7)
    s = tk.BernoulliRelationNegativeSampler(kg, seed=1)
    m = helpers.train_model("distmult", 8, 100, 5, seed=1)
    h = kg.head_idx[:10].to(DEV)
    with pytest.raises(ValueError, match="exactly one"):
        s.fused_step(m, h, h, h % 5)
    with pytest.raises(TypeError):
        s.fused_step(m, h, h, h % 5, criterion=torch.nn.MSELoss())
    with pytest.raises(ValueError, match="entities"):
        s.fused_step(m, h, h, h % 5, margin=1.0, shard=EntityShard(99, 0, 2, local_storage=True))
    assert s._calls == 0


# ---------------------------------------------------------------- 3. against float64 autograd
def reference(kind, ts, h, t, r, nh, nt, nr, loss, margin):
    cpu = helpers.cpu_leaves(ts, torch.float64)
    n_neg = nh.shape[0] // h.shape[0]
    pos = helpers.cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), h.cpu(), t.cpu())[0].repeat(n_neg)
    neg = helpers.cpu_pos_neg(kind, cpu, nh.cpu(), nt.cpu(), nr.cpu(), nh.cpu(), nt.cpu())[1]
    want = helpers.torch_loss(loss, pos, neg, margin)
    want.backward()
    return want.item(), [None if x is None else x.grad for x in cpu], pos.detach(), neg.detach()


def problem(kind, d, n_neg, seed, b=23, n_ent=N_ENT):
    model = helpers.train_model(kind, d, n_ent, N_REL, seed=seed)
    gen = torch.Generator().manual_seed(seed + n_neg)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, N_REL, (b,), generator=gen)
    probs = torch.rand(N_REL, generator=gen)
    return model, h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)


def drawn_step(model, h, t, r, probs, n_neg, share, loss, margin):
    """The fused step on its own draws; returns (loss, grads, nh, nt, nr, neg scores) with the negatives and
    scores the kernel wrote out through nh_out / nt_out / nr_out / neg_out."""
    code, dim, ts = helpers.train_leaves(model)
    lk = helpers.LOSS_KINDS[loss]
    got = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *ts, lk, None,
                            (N_REL, share))
    got.backward()
    b = h.shape[0]
    ids = [torch.full((b * n_neg,), -1, dtype=torch.int64, device=DEV) for _ in range(3)]
    neg_out = torch.full((b * n_neg,), float("nan"), device=DEV)
    out = torch.zeros((), device=DEV)
    tabs = [None if x is None else x.detach() for x in ts]
    a = _MarginStep._args(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, tabs, out,
                          h.device, lk, None, (N_REL, share))
    a.base.nh_out, a.base.nt_out, a.nr_out, a.base.neg_out = _ptr(ids[0]), _ptr(ids[1]), _ptr(ids[2]), _ptr(neg_out)
    assert _lib.load().kge_rel_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()
    assert out.item() == pytest.approx(got.item(), rel=1e-6)
    return got.item(), ts, ids, neg_out


RING_KINDS = ("transe_l1", "transe_l2", "distmult")
_STEP_KERNEL = re.compile(r"(margin_step_(?:ring_rel|ring|fast|shard_fwd|shard_bwd|fwd|bwd)_kernel)")


def expected_kernels(kind, d, n_neg, shard):
    """The kernels a relation-corrupting step with rel_share < 1 launches: the ring kernel's relation kind
    for TransE-L1 / L2 and DistMult where the ring applies (not under KGE_TRAIN_RING=0), else the generic
    kernels."""
    ring_on = os.environ.get("KGE_TRAIN_RING", "")[:1] != "0"
    if (kind in RING_KINDS and d % 4 == 0 and d <= 256 and ring_on and n_neg <= RING_MAX_NEG and
            ring_smem_bytes(d, n_neg) <= SMEM_MAX):
        return {"margin_step_ring_rel_kernel"}
    return {"margin_step_shard_fwd_kernel", "margin_step_shard_bwd_kernel"} if shard else \
        {"margin_step_fwd_kernel", "margin_step_bwd_kernel"}


def launched(fn, expected, tries=4):
    """Fused-step kernels that ran while fn() ran (retried: torch.profiler now and then drops a kernel)."""
    ran = set()
    for _ in range(tries):
        ran |= {m.group(1) for m in map(_STEP_KERNEL.search, _cuda_kernel_names(fn)) if m}
        if ran >= expected:
            break
    return ran


def check(kind, got_loss, ts, want_loss, want_grads, rtol=2e-4):
    assert got_loss == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    for a, c in zip(ts, want_grads):
        if c is not None:
            helpers.close_grad(a.grad, c, rtol=rtol)


RING_SHAPES = [(k, d, n) for k in ("transe_l1", "transe_l2", "distmult") for d, n in
               ((4, 1), (36, 7), (200, 256), (256, 1000))]
CODE_CASES = [(k, 16, 9) for k in CODES] + RING_SHAPES


@pytest.mark.parametrize("share", [0.0, 0.33, 1.0])
@pytest.mark.parametrize("kind,d,n_neg", CODE_CASES, ids=["%s-d%d-neg%d" % c for c in CODE_CASES])
def test_drawn_step_matches_float64_autograd(kind, d, n_neg, share):
    model, h, t, r, probs = problem(kind, d, n_neg, seed=d + n_neg)
    loss = "margin" if n_neg % 2 else "logistic"
    margin = 0.5
    got, ts, (nh, nt, nr), neg_out = drawn_step(model, h, t, r, probs, n_neg, share, loss, margin)
    want_nh, want_nt, want_nr = corrupt_rel(h, t, r, probs, n_neg, N_ENT, N_REL, share)
    assert torch.equal(nh, want_nh) and torch.equal(nt, want_nt) and torch.equal(nr, want_nr)
    want_loss, want_grads, _, neg = reference(kind, ts, h, t, r, nh, nt, nr, loss, margin)
    torch.testing.assert_close(neg_out.cpu().double(), neg.double(), rtol=1e-5, atol=1e-5)
    check(kind, got, ts, want_loss, want_grads)
    if share < 1.0:
        code, dim, _ = helpers.train_leaves(model)

        def step():
            leaves = helpers.train_leaves(model)[2]
            _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *leaves,
                              helpers.LOSS_KINDS[loss], None, (N_REL, share)).backward()
        want = expected_kernels(kind, d, n_neg, shard=False)
        assert launched(step, want) == want
    if share == 1.0:      # the entity step's negatives, loss and gradients
        code, dim, ts2 = helpers.train_leaves(model)
        ent = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *ts2,
                                helpers.LOSS_KINDS[loss])
        ent.backward()
        assert got == pytest.approx(ent.item(), rel=1e-6, abs=1e-7)
        for a, c in zip(ts, ts2):
            if a is not None:
                torch.testing.assert_close(a.grad, c.grad, rtol=1e-6, atol=1e-6 * float(c.grad.abs().max()) + 1e-9)


@pytest.mark.parametrize("kind", CODES)
def test_external_negatives_changing_several_positions(kind):
    n_neg = 5
    model, h, t, r, probs = problem(kind, 16, n_neg, seed=41)
    g = torch.Generator().manual_seed(5)
    b = h.shape[0]
    nh, nt, nr = h.repeat(n_neg).cpu(), t.repeat(n_neg).cpu(), r.repeat(n_neg).cpu()
    which = torch.randint(0, 7, (b * n_neg,), generator=g)     # bit 0: head, 1: tail, 2: relation
    nh = torch.where(which & 1 > 0, torch.randint(1, N_ENT, nh.shape, generator=g), nh)
    nt = torch.where(which & 2 > 0, torch.randint(1, N_ENT, nt.shape, generator=g), nt)
    nr = torch.where(which & 4 > 0, torch.randint(1, N_REL, nr.shape, generator=g), nr)
    code, dim, ts = helpers.train_leaves(model)
    want_loss, want_grads, _, _ = reference(kind, ts, h, t, r, nh, nt, nr, "logistic", 0.0)
    public = tk.training.fused_loss_step(model, h, t, r, tk.LogisticLoss(),
                                         negatives=(nh.to(DEV), nt.to(DEV), nr.to(DEV)))
    assert public.item() == pytest.approx(want_loss, rel=2e-5)
    got2 = _MarginStep.apply(code, dim, N_ENT, 0.0, n_neg, h, t, r, nh.to(DEV), nt.to(DEV), None, 0, 0, *ts,
                             _lib.LOSS_LOGISTIC, nr.to(DEV), (N_REL, 1.0))
    got2.backward()
    check(kind, got2.item(), ts, want_loss, want_grads)


# ---------------------------------------------------------------- 5. entity-sharded, emulated
def emulated(model, h, t, r, probs, margin, n_neg, world, eng, lk, share):
    """As helpers.emulated, for the relation-corrupting step: every rank's kernels on its row range, the
    all-reduces as sums, then every rank's scatter into its own rows."""
    code, dim, ts = helpers.train_leaves(model)
    tabs = [None if x is None else x.detach() for x in ts]
    n_ent, b = model.n_ent, h.shape[0]
    full = ShardedStep(code, dim, n_ent, 0, n_ent, n_neg, float(margin), SEED, OFFSET, lk, N_REL, share)
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
        step = ShardedStep(code, dim, n_ent, sh.lo, n, n_neg, float(margin), SEED, OFFSET, lk, N_REL, share)
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


SHARD_CASES = ([(k, 16, 6, loss) for k in CODES for loss in ("margin", "logistic", "bce")] +
               [(k, 200, 256, "logistic") for k in RING_KINDS])


@pytest.mark.parametrize("kind,d,n_neg,loss", SHARD_CASES, ids=["%s-d%d-neg%d-%s" % c for c in SHARD_CASES])
def test_sharded_step_sums_to_unsharded(kind, d, n_neg, loss):
    share, margin = 0.4, 0.5
    model, h, t, r, probs = problem(kind, d, n_neg, seed=13)
    lk = helpers.LOSS_KINDS[loss]
    code, dim, ts = helpers.train_leaves(model)
    one = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET, *ts, lk, None,
                            (N_REL, share))
    one.backward()
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        got_loss, got_grads = emulated(model, h, t, r, probs, margin, n_neg, world, eng, lk, share)
        assert got_loss == pytest.approx(one.item(), rel=1e-5, abs=1e-6), world
        for a, c in zip(got_grads, ts):
            if c is not None:
                helpers.close_grad(a, c.grad, rtol=1e-4)
    want = expected_kernels(kind, d, n_neg, shard=True)
    ran = launched(lambda: emulated(model, h, t, r, probs, margin, n_neg, 3, eng, lk, share), want)
    assert ran == want


def test_sharded_step_with_ranks_that_hold_no_rows():
    """3 entities over 8 ranks: five ranks hold nothing and score nothing."""
    model, h, t, r, probs = problem("distmult", 8, 4, seed=19, b=9, n_ent=3)
    code, dim, ts = helpers.train_leaves(model)
    one = _MarginStep.apply(code, dim, 3, 0.0, 4, h, t, r, None, None, probs, SEED, OFFSET, *ts,
                            _lib.LOSS_LOGISTIC, None, (N_REL, 0.5))
    one.backward()
    got_loss, got_grads = emulated(model, h, t, r, probs, 0.0, 4, 8, CudaEngine(), _lib.LOSS_LOGISTIC, 0.5)
    assert got_loss == pytest.approx(one.item(), rel=1e-5, abs=1e-6)
    for a, c in zip(got_grads, ts):
        if c is not None:
            helpers.close_grad(a, c.grad, rtol=1e-4)


# ---------------------------------------------------------------- 6. public API, two processes on one GPU
def _local_model(kind, model, lo, hi, n_rel, dim):
    part = helpers.make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part.to(next(model.parameters()).device)


def _train(model, kg, batches, shard, crit, share):
    sampler = tk.BernoulliRelationNegativeSampler(kg, n_neg=16, rel_share=share, seed=3)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for h, t, r in batches:
        opt.zero_grad()
        loss = sampler.fused_step(model, h, t, r, criterion=crit, shard=shard)
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
        # DistMult d=200 takes the ring kernel's relation kind, ComplEx the generic kernels
        for kind, dim, crit in (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.MarginLoss(1.0))):
            full = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
            shard = Shard.from_group(n_ent, local_storage=True)
            local = _local_model(kind, full, shard.lo, shard.hi, n_rel, dim)
            want = _train(full, kg, batches, None, crit, 0.33)
            got = _train(local, kg, batches, shard, crit, 0.33)
            res[kind + "/losses_close"] = all(abs(a - b) <= 1e-5 * abs(b) + 1e-6 for a, b in zip(got, want))
            for name, p in local.named_parameters():
                ref = dict(full.named_parameters())[name]
                res[kind + "/" + name] = torch.allclose(p, ref[shard.lo:shard.hi] if "ent_emb" in name else ref,
                                                        rtol=1e-4, atol=1e-5)
        sampler = tk.BernoulliRelationNegativeSampler(kg, n_neg=4, rel_share=0.33 if rank == 0 else 0.5, seed=100)
        try:
            sampler.fused_step(local, *batches[0], criterion=tk.LogisticLoss(), shard=shard)
            res["rel_share_mismatch_raises"] = False
        except ValueError as e:
            res["rel_share_mismatch_raises"] = "rel_share" in str(e)
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


# ---------------------------------------------------------------- 7. KGE_TRAIN_RING=0
def test_without_the_ring():
    """The float64 and sharded cases of the ring kinds once more in a child process under KGE_TRAIN_RING=0:
    every relation-corrupting step then takes the generic kernels (expected_kernels reads the switch)."""
    if "KGE_TRAIN_RING" in os.environ:
        pytest.skip("runs in the parent process only")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
         "(drawn_step or sharded_step_sums) and (transe or distmult)"]
    proc = subprocess.run(cmd, cwd=root, env=dict(os.environ, KGE_TRAIN_RING="0"), capture_output=True, text=True,
                          timeout=1200)
    assert proc.returncode == 0, proc.stdout[-6000:] + proc.stderr[-3000:]
    assert " passed" in proc.stdout, proc.stdout[-2000:]
