"""Relation-corrupting negatives (BernoulliRelationNegativeSampler) on the GPU: the law of
kge_corrupt_batch_rel, the fused step against the unfused loop and against float64 autograd on the
CPU for every training code, and the entity-sharded step emulated over 1, 2, 3 and 8 ranks.

Tolerances as in tests/test_train_paths_gpu.py: losses within 2e-5 of float64 (1e-5 against the
float32 loop), gradients under train_kit.close_grad."""
import math
import os

import pytest
import torch
from scipy import stats

import torchkge_b200 as tk
from tests import gloo, helpers
from tests import train_kit as kit
from tests.train_kit import DEV, expected_kernels, launched
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, EntityShard, _ptr, _stream

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


# ---------------------------------------------------------------- 1. the law of the draws
def test_bernoulli_draws_are_those_of_the_philox_statement():
    """kge_corrupt_batch (BernoulliNegativeSampler) still draws what draw_one states: head iff
    (x >> 8) / 2^24 < p_r, entity 1 + (y (n_ent - 1)) >> 32."""
    b, n_neg, n_ent = 4099, 3, 100003
    g = torch.Generator().manual_seed(1)
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.randint(0, N_REL, (b,), generator=g)
    probs = torch.rand(N_REL, generator=g)
    nh, nt = kit.corrupt_batch(h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV), n_neg, n_ent, SEED, OFFSET)
    head, e = kit.philox_draws(SEED, OFFSET, r, n_neg, probs, n_ent)
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
    is_rel, new_r, head, e = kit.philox_rel_draws(SEED, OFFSET, r, n_neg, probs, n_ent, n_rel, share)
    frac = float(is_rel.double().mean())
    assert abs(frac - (1 - share)) <= 5 * math.sqrt(share * (1 - share) / n)
    assert torch.equal(nr, torch.where(is_rel, new_r, R))
    assert torch.equal(nh[is_rel], H[is_rel]) and torch.equal(nt[is_rel], T[is_rel])
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
        eh, et = kit.corrupt_batch(h, t, r, probs, n_neg, n_ent, SEED, OFFSET)
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
    m1 = kit.train_model(kind, 32, 400, 9, seed=6)
    m2 = kit.train_model(kind, 32, 400, 9, seed=6)
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
            kit.close_grad(a.grad, c.grad, rtol=1e-4)


def test_fused_step_argument_errors():
    kg, _, _ = helpers.make_kg(100, 5, n_facts=300, n_test=20, seed=7)
    s = tk.BernoulliRelationNegativeSampler(kg, seed=1)
    m = kit.train_model("distmult", 8, 100, 5, seed=1)
    h = kg.head_idx[:10].to(DEV)
    with pytest.raises(ValueError, match="exactly one"):
        s.fused_step(m, h, h, h % 5)
    with pytest.raises(TypeError):
        s.fused_step(m, h, h, h % 5, criterion=torch.nn.MSELoss())
    with pytest.raises(ValueError, match="entities"):
        s.fused_step(m, h, h, h % 5, margin=1.0, shard=EntityShard(99, 0, 2, local_storage=True))
    assert s._calls == 0


# ---------------------------------------------------------------- 3. against float64 autograd
RING_KINDS = ("transe_l1", "transe_l2", "distmult")


def check(got_loss, grads, want_loss, want_grads, rtol=2e-4):
    assert got_loss == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    for a, c in zip(grads, want_grads):
        if c is not None:
            kit.close_grad(a, c, rtol=rtol)


RING_SHAPES = [(k, d, n) for k in ("transe_l1", "transe_l2", "distmult") for d, n in
               ((4, 1), (36, 7), (200, 256), (256, 1000))]
CODE_CASES = [(k, 16, 9) for k in CODES] + RING_SHAPES


@pytest.mark.parametrize("share", [0.0, 0.33, 1.0])
@pytest.mark.parametrize("kind,d,n_neg", CODE_CASES, ids=["%s-d%d-neg%d" % c for c in CODE_CASES])
def test_drawn_step_matches_float64_autograd(kind, d, n_neg, share):
    model, h, t, r, probs = kit.problem(kind, d, n_neg, d + n_neg, N_ENT, N_REL)
    loss = "margin" if n_neg % 2 else "logistic"
    kw = dict(n_neg=n_neg, loss=loss, margin=0.5, probs=probs, seed=SEED, offset=OFFSET)
    # the negatives and scores the kernel writes out through nh_out / nt_out / nr_out / neg_out
    got, grads, out = kit.whole_table_step(model, h, t, r, rel_share=share, outputs=True, **kw)
    assert out["loss"].item() == pytest.approx(got, rel=1e-6)
    nh, nt, nr = out["nh"], out["nt"], out["nr"]
    want_nh, want_nt, want_nr = corrupt_rel(h, t, r, probs, n_neg, N_ENT, N_REL, share)
    assert torch.equal(nh, want_nh) and torch.equal(nt, want_nt) and torch.equal(nr, want_nr)
    want_loss, want_grads, _, neg = kit.reference(kind, kit.train_leaves(model)[2], h, t, r, nh, nt, loss, 0.5, nr)
    torch.testing.assert_close(out["neg"].cpu().double(), neg.double(), rtol=1e-5, atol=1e-5)
    check(got, grads, want_loss, want_grads)
    if share < 1.0:
        want = expected_kernels(kind, d, n_neg, loss, shard=False, negatives="relation")
        assert launched(lambda: kit.whole_table_step(model, h, t, r, rel_share=share, **kw), want) == want
    if share == 1.0:      # the entity step's negatives, loss and gradients
        ent, ent_grads = kit.whole_table_step(model, h, t, r, **kw)
        assert got == pytest.approx(ent, rel=1e-6, abs=1e-7)
        for a, c in zip(grads, ent_grads):
            if a is not None:
                torch.testing.assert_close(a, c, rtol=1e-6, atol=1e-6 * float(c.abs().max()) + 1e-9)


@pytest.mark.parametrize("kind", CODES)
def test_external_negatives_changing_several_positions(kind):
    n_neg = 5
    model, h, t, r, probs = kit.problem(kind, 16, n_neg, 41, N_ENT, N_REL)
    g = torch.Generator().manual_seed(5)
    b = h.shape[0]
    nh, nt, nr = h.repeat(n_neg).cpu(), t.repeat(n_neg).cpu(), r.repeat(n_neg).cpu()
    which = torch.randint(0, 7, (b * n_neg,), generator=g)     # bit 0: head, 1: tail, 2: relation
    nh = torch.where(which & 1 > 0, torch.randint(1, N_ENT, nh.shape, generator=g), nh)
    nt = torch.where(which & 2 > 0, torch.randint(1, N_ENT, nt.shape, generator=g), nt)
    nr = torch.where(which & 4 > 0, torch.randint(1, N_REL, nr.shape, generator=g), nr)
    want_loss, want_grads, _, _ = kit.reference(kind, kit.train_leaves(model)[2], h, t, r, nh, nt, "logistic", 0.0,
                                                nr)
    public = tk.training.fused_loss_step(model, h, t, r, tk.LogisticLoss(),
                                         negatives=(nh.to(DEV), nt.to(DEV), nr.to(DEV)))
    assert public.item() == pytest.approx(want_loss, rel=2e-5)
    got2, grads = kit.whole_table_step(model, h, t, r, loss="logistic", rel_share=1.0,
                                       negatives=(nh.to(DEV), nt.to(DEV), nr.to(DEV)))
    check(got2, grads, want_loss, want_grads)


# ---------------------------------------------------------------- 5. entity-sharded, emulated
SHARD_CASES = ([(k, 16, 6, loss) for k in CODES for loss in ("margin", "logistic", "bce")] +
               [(k, 200, 256, "logistic") for k in RING_KINDS])


@pytest.mark.parametrize("kind,d,n_neg,loss", SHARD_CASES, ids=["%s-d%d-neg%d-%s" % c for c in SHARD_CASES])
def test_sharded_step_sums_to_unsharded(kind, d, n_neg, loss):
    model, h, t, r, probs = kit.problem(kind, d, n_neg, 13, N_ENT, N_REL)
    kw = dict(n_neg=n_neg, loss=loss, margin=0.5, probs=probs, seed=SEED, offset=OFFSET, rel_share=0.4)
    one, one_grads = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (1, 2, 3, 8):
        got_loss, got_grads = kit.emulated(model, h, t, r, world, eng, **kw)
        assert got_loss == pytest.approx(one, rel=1e-5, abs=1e-6), world
        for a, c in zip(got_grads, one_grads):
            if c is not None:
                kit.close_grad(a, c, rtol=1e-4)
    want = expected_kernels(kind, d, n_neg, loss, shard=True, negatives="relation")
    ran = launched(lambda: kit.emulated(model, h, t, r, 3, eng, **kw), want)
    assert ran == want


def test_sharded_step_with_ranks_that_hold_no_rows():
    """3 entities over 8 ranks: five ranks hold nothing and score nothing."""
    model, h, t, r, probs = kit.problem("distmult", 8, 4, 19, 3, N_REL, b=9)
    kw = dict(n_neg=4, loss="logistic", probs=probs, seed=SEED, offset=OFFSET, rel_share=0.5)
    one, one_grads = kit.whole_table_step(model, h, t, r, **kw)
    got_loss, got_grads = kit.emulated(model, h, t, r, 8, CudaEngine(), **kw)
    assert got_loss == pytest.approx(one, rel=1e-5, abs=1e-6)
    for a, c in zip(got_grads, one_grads):
        if c is not None:
            kit.close_grad(a, c, rtol=1e-4)


# ---------------------------------------------------------------- 6. public API, two processes on one GPU
def _api_worker(rank, world, _):
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    try:
        # DistMult d=200 takes the ring kernel's relation kind, ComplEx the generic kernels
        res, kg, batches, local, shard = kit.whole_against_shard(
            (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.MarginLoss(1.0))),
            lambda kg: tk.BernoulliRelationNegativeSampler(kg, n_neg=16, rel_share=0.33, seed=3), dev, 4,
            loss_atol=1e-6)
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
    kit.every_rank_ok(gloo.spawn(2, _api_worker, None), 2, min_checks=6)


# ---------------------------------------------------------------- 7. KGE_TRAIN_RING=0
def test_without_the_ring():
    """The float64 and sharded cases of the ring kinds once more in a child process under KGE_TRAIN_RING=0:
    every relation-corrupting step then takes the generic kernels (expected_kernels reads the switch)."""
    if "KGE_TRAIN_RING" in os.environ:
        pytest.skip("runs in the parent process only")
    kit.rerun(__file__, "KGE_TRAIN_RING=0", "(drawn_step or sharded_step_sums) and (transe or distmult)")
