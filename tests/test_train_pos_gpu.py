"""Positional and uniform negatives in the fused training step on the GPU: the positional draw (draw_pos)
against a numpy statement of it, bit for bit, on the ring and the generic kernels; its law on a large draw;
the loss and gradients against float64 autograd on the CPU for every training code and the three losses,
with the kernel that ran checked (and again under KGE_TRAIN_RING=0); UniformNegativeSampler.fused_step
against corrupt_batch; the entity-sharded step emulated over three ranks and over gloo in two processes.

Tolerances as in tests/test_train_relneg_gpu.py."""
import math
import os

import pytest
import torch
from scipy import stats

import torchkge_b200 as tk
from tests import gloo, helpers
from tests import train_kit as kit
from tests.train_kit import DEV, SMEM_MAX, csr, expected_kernels, last_n_neg_within, launched
from torchkge_b200.engine import CudaEngine

pytestmark = pytest.mark.gpu

CODES = ("transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "toruse_l1", "toruse_l2", "analogy")
RING_KINDS = ("transe_l1", "transe_l2", "distmult")
SEED, OFFSET = 777, 3


# ---------------------------------------------------------------- the candidate graph
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


def expected_draws(h, t, r, n_neg, probs, n_ent, pos):
    head, e = kit.philox_pos_draws(SEED, OFFSET, r, n_neg, probs, n_ent, pos)
    H, T = h.cpu().repeat(n_neg), t.cpu().repeat(n_neg)
    return torch.where(head, e, H), torch.where(head, T, e)


def drawn_step(model, h, t, r, probs, n_neg, loss, margin, pos):
    """The fused positional step on its own draws: (loss, [grads], the outputs of kge_pos_step_fwd)."""
    got, grads, out = kit.whole_table_step(model, h, t, r, n_neg=n_neg, loss=loss, margin=margin, probs=probs,
                                           seed=SEED, offset=OFFSET, positional=pos, outputs=True)
    assert out["loss"].item() == pytest.approx(got, rel=1e-5, abs=1e-7)   # fp32 atomics in another order
    return got, grads, out


# ---------------------------------------------------------------- 1. the draws, bit for bit
@pytest.mark.parametrize("kind,d,n_neg", [("distmult", 8, 7), ("transe_l2", 36, 1), ("complex", 8, 5),
                                          ("distmult", 8, last_n_neg_within(8, SMEM_MAX) + 1)])
def test_draws_equal_the_numpy_statement(kind, d, n_neg):
    """Relation 0 (empty: entity 0 can be drawn), 1 (one candidate), 2 (> 2^16 candidates) and others, on the
    ring kernel (DistMult, TransE) and on the generic kernels (ComplEx, and DistMult past the ring)."""
    n_ent, n_rel = 100_003, 9
    pos = graph(n_ent, n_rel, seed=1)
    model = kit.train_model(kind, d, n_ent, n_rel, seed=2)
    g = torch.Generator().manual_seed(3)
    b = 600 if n_neg < 100 else 8
    h, t = torch.randint(0, n_ent, (b,), generator=g), torch.randint(0, n_ent, (b,), generator=g)
    r = torch.arange(b) % n_rel
    probs = torch.rand(n_rel, generator=g)
    probs[:3] = torch.tensor([0.5, 0.5, 0.9])
    h, t, r, probs = h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)
    out = drawn_step(model, h, t, r, probs, n_neg, "logistic", 0.0, pos)[2]
    nh, nt = out["nh"], out["nt"]
    want_nh, want_nt = expected_draws(h, t, r, n_neg, probs, n_ent, pos)
    assert torch.equal(nh.cpu(), want_nh) and torch.equal(nt.cpu(), want_nt)
    R = r.cpu().repeat(n_neg)
    e = torch.where(nh.cpu() != h.cpu().repeat(n_neg), nh.cpu(), nt.cpu())
    if n_neg * b > 2000:      # relation 0 draws from [0, n_ent); somewhere a low id shows it is not [1, n_ent)
        assert int(e[R == 0].min()) < n_ent // 100
    assert set(nh.cpu()[(R == 1) & (nh.cpu() != h.cpu().repeat(n_neg))].tolist()) <= {5}
    assert set(nt.cpu()[(R == 1) & (nt.cpu() != t.cpu().repeat(n_neg))].tolist()) <= {n_ent - 1}
    want = expected_kernels(kind, d, n_neg, "logistic", shard=False, negatives="positional")
    assert launched(lambda: kit.whole_table_step(model, h, t, r, n_neg=n_neg, loss="logistic", probs=probs, seed=SEED,
                                                 offset=OFFSET, positional=pos), want) == want


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
    model = kit.train_model("distmult", 4, n_ent, n_rel, seed=6)
    out = drawn_step(model, h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV), n_neg, "logistic", 0.0, pos)[2]
    nh, nt = out["nh"].cpu(), out["nt"].cpu()
    head, e = kit.philox_pos_draws(SEED, OFFSET, r, n_neg, probs, n_ent, pos)
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


def _cases():
    out = [(k, 16, n, loss) for k in CODES for n in (1, 7) for loss in ("margin", "logistic", "bce")]
    out += [(k, 36, last_n_neg_within(36, SMEM_MAX) + 1, loss) for k in RING_KINDS for loss in ("margin", "bce")]
    out += [(k, 200, 256, "logistic") for k in RING_KINDS]
    return out


CASES = _cases()


@pytest.mark.parametrize("kind,d,n_neg,loss", CASES, ids=["%s-d%d-neg%d-%s" % c for c in CASES])
def test_drawn_step_matches_float64_autograd(kind, d, n_neg, loss):
    model, h, t, r, probs = kit.problem(kind, d, n_neg, d + n_neg, N_ENT, N_REL)
    pos = small_graph()
    want_nh, want_nt = expected_draws(h, t, r, n_neg, probs, N_ENT, pos)
    margin = 0.0
    if loss == "margin":    # no hinge so near its kink that float32 and float64 could disagree on it
        cpu = kit.cpu_leaves(kit.train_leaves(model)[2], torch.float64)
        p_, n_ = kit.cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), want_nh, want_nt)
        margin = kit.margin_between((p_ - n_).detach())
    got, grads, out = drawn_step(model, h, t, r, probs, n_neg, loss, margin, pos)
    assert torch.equal(out["nh"].cpu(), want_nh) and torch.equal(out["nt"].cpu(), want_nt)
    want_loss, want_grads, _, neg = kit.reference(kind, kit.train_leaves(model)[2], h, t, r, out["nh"], out["nt"],
                                                  loss, margin)
    torch.testing.assert_close(out["neg"].cpu().double(), neg.double(), rtol=1e-5, atol=1e-5)
    assert got == pytest.approx(want_loss, rel=2e-5, abs=1e-6)
    for a, c in zip(grads, want_grads):
        if c is None:
            continue
        if n_neg <= 1000:
            kit.close_grad(a, c, rtol=2e-4)
        else:
            # past the ring the generic kernels add every pair's gradient by its own fp32 atomics: ~10^4 of them
            # per row of the 700-entity table, whose rounding error scales with the table's largest entry
            torch.testing.assert_close(a.cpu().float(), c.float(), rtol=2e-4, atol=2e-4 * float(c.abs().max()))
    want = expected_kernels(kind, d, n_neg, loss, shard=False, negatives="positional")
    assert launched(lambda: kit.whole_table_step(model, h, t, r, n_neg=n_neg, loss=loss, margin=margin, probs=probs,
                                                 seed=SEED, offset=OFFSET, positional=pos), want) == want


# ---------------------------------------------------------------- 3. the samplers
def test_positional_sampler_fused_step_equals_loop_on_its_draws():
    kg, _, _ = helpers.make_kg(400, 9, n_facts=3000, n_test=100, seed=5)
    h, t, r = kg.head_idx[:512].to(DEV), kg.tail_idx[:512].to(DEV), kg.relations[:512].to(DEV)
    s = tk.PositionalNegativeSampler(kg, seed=21)
    m = kit.train_model("distmult", 32, 400, 9, seed=6)
    loss = s.fused_step(m, h, t, r, criterion=tk.LogisticLoss(), n_neg=3)
    assert s._calls == 1
    offs_h, ents_h, _ = s._csr["heads"]
    offs_t, ents_t, _ = s._csr["tails"]
    pos = (offs_h, ents_h, offs_t, ents_t)
    head, e = kit.philox_pos_draws(s.seed, 1, r.cpu(), 3, s.bern_probs.cpu(), 400, pos)
    nh = torch.where(head, e, h.cpu().repeat(3))
    nt = torch.where(head, t.cpu().repeat(3), e)
    m2 = kit.train_model("distmult", 32, 400, 9, seed=6)
    want = tk.training.fused_loss_step(m2, h, t, r, tk.LogisticLoss(), negatives=(nh.to(DEV), nt.to(DEV)))
    assert loss.item() == pytest.approx(want.item(), rel=1e-5)
    loss.backward()
    want.backward()
    for a, c in zip(m.parameters(), m2.parameters()):
        kit.close_grad(a.grad, c.grad, rtol=1e-4)
    with pytest.raises(ValueError, match="entities"):     # before the call count moves
        s.fused_step(kit.train_model("distmult", 8, 401, 9, seed=1), h, t, r, margin=1.0)
    assert s._calls == 1
    with pytest.raises(ValueError, match="relations"):
        s.fused_step(kit.train_model("distmult", 8, 400, 10, seed=1), h, t, r, margin=1.0)


@pytest.mark.parametrize("loss", ["margin", "bce"])
def test_uniform_fused_step_draws_what_corrupt_batch_draws(loss):
    kg, _, _ = helpers.make_kg(500, 7, n_facts=3000, n_test=100, seed=9)
    h, t, r = kg.head_idx[:700].to(DEV), kg.tail_idx[:700].to(DEV), kg.relations[:700].to(DEV)
    crit = tk.MarginLoss(0.8) if loss == "margin" else tk.BinaryCrossEntropyLoss()
    s1, s2 = tk.UniformNegativeSampler(kg, seed=31), tk.UniformNegativeSampler(kg, seed=31)
    s1.corrupt_batch(h, t, r, n_neg=2)          # both samplers at call 2 next
    s2.corrupt_batch(h, t, r, n_neg=2)
    m1, m2 = kit.train_model("transe_l2", 24, 500, 7, seed=3), kit.train_model("transe_l2", 24, 500, 7, seed=3)
    got = s1.fused_step(m1, h, t, r, criterion=crit, n_neg=5)
    nh, nt = s2.corrupt_batch(h, t, r, n_neg=5)
    want = tk.training.fused_loss_step(m2, h, t, r, crit, negatives=(nh, nt))
    assert got.item() == pytest.approx(want.item(), rel=1e-6, abs=1e-7)
    got.backward()
    want.backward()
    for a, c in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a.grad, c.grad, rtol=1e-5, atol=1e-6 * float(c.grad.abs().max()) + 1e-9)
    # the draws themselves, through nh_out / nt_out of the entity step at the sampler's (seed, call count)
    out = kit.forward_outputs(m1, h, t, r, n_neg=5, margin=1.0, probs=s1._halves, seed=s1.seed, offset=2)
    assert torch.equal(out["nh"], nh) and torch.equal(out["nt"], nt)


# ---------------------------------------------------------------- 4. entity-sharded, emulated
SHARD_CASES = ([(k, 16, 6, loss) for k in ("transe_l2", "distmult", "complex", "rescal", "analogy")
                for loss in ("margin", "logistic")] + [(k, 200, 256, "bce") for k in RING_KINDS])


@pytest.mark.parametrize("kind,d,n_neg,loss", SHARD_CASES, ids=["%s-d%d-neg%d-%s" % c for c in SHARD_CASES])
def test_sharded_step_sums_to_unsharded(kind, d, n_neg, loss):
    model, h, t, r, probs = kit.problem(kind, d, n_neg, 13, N_ENT, N_REL)
    kw = dict(n_neg=n_neg, loss=loss, margin=0.5, probs=probs, seed=SEED, offset=OFFSET, positional=small_graph())
    one, one_grads = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    for world in (1, 3):
        got_loss, got_grads = kit.emulated(model, h, t, r, world, eng, **kw)
        assert got_loss == pytest.approx(one, rel=1e-5, abs=1e-6), world
        for a, c in zip(got_grads, one_grads):
            if c is not None:
                kit.close_grad(a, c, rtol=1e-4)
    want = expected_kernels(kind, d, n_neg, loss, shard=True, negatives="positional")
    ran = launched(lambda: kit.emulated(model, h, t, r, 3, eng, **kw), want)
    assert ran == want


def test_sharded_step_with_a_rank_that_holds_no_rows():
    """2 entities over 3 ranks: rank 2 holds nothing and scores nothing."""
    model, h, t, r, probs = kit.problem("distmult", 8, 4, 19, 2, N_REL, b=9)
    g = torch.Generator().manual_seed(1)
    rel = torch.randint(1, N_REL, (30,), generator=g)
    hd, tl = torch.randint(0, 2, (30,), generator=g), torch.randint(0, 2, (30,), generator=g)
    kw = dict(n_neg=4, loss="logistic", probs=probs, seed=SEED, offset=OFFSET,
              positional=csr(rel, hd, N_REL, 2) + csr(rel, tl, N_REL, 2))
    one, one_grads = kit.whole_table_step(model, h, t, r, **kw)
    got_loss, got_grads = kit.emulated(model, h, t, r, 3, CudaEngine(), **kw)
    assert got_loss == pytest.approx(one, rel=1e-5, abs=1e-6)
    for a, c in zip(got_grads, one_grads):
        if c is not None:
            kit.close_grad(a, c, rtol=1e-4)


# ---------------------------------------------------------------- 5. public API, two processes on one GPU
def _api_worker(rank, world, _):
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    try:
        # DistMult d=200 takes the ring kernel's positional kind, ComplEx the generic kernels
        res, kg, batches, local, shard = kit.whole_against_shard(
            (("distmult", 200, tk.LogisticLoss()), ("complex", 50, tk.MarginLoss(1.0))),
            lambda kg: tk.PositionalNegativeSampler(kg, seed=3), dev, 4, n_neg=16, loss_atol=1e-6)
        hh, tt, rr = helpers.random_graph(3001, 7, 6000, seed=5)
        other = kg if rank == 0 else tk.KnowledgeGraph(hh[:5000], tt[:5000], rr[:5000], 3001, 7,
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
    kit.every_rank_ok(gloo.spawn(2, _api_worker, None), 2, min_checks=6)


# ---------------------------------------------------------------- 6. KGE_TRAIN_RING=0
def test_without_the_ring():
    """The draw, float64 and sharded cases of the ring kinds once more in a child process under
    KGE_TRAIN_RING=0: every positional step then takes the generic kernels (expected_kernels reads the
    switch)."""
    if "KGE_TRAIN_RING" in os.environ:
        pytest.skip("runs in the parent process only")
    kit.rerun(__file__, "KGE_TRAIN_RING=0", "(draws_equal or drawn_step or sharded_step_sums) and (transe or distmult)")
