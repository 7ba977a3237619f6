"""GPU parity tests of the training-side kernels against the reference's golden outputs and
the CPU oracle.  Tolerances are the ones north_star / SURVEY.md section 8d state: scores and
loss within 1e-5 relative, gradients allclose(rtol=1e-4) (atomics order)."""
import numpy as np
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200.training import fused_margin_step

pytestmark = pytest.mark.gpu
RTOL_SCORE = 1e-5


def _close(a, b, rtol, atol):
    torch.testing.assert_close(a.detach().cpu().float(), b.detach().cpu().float(), rtol=rtol, atol=atol)


def _close_grad(a, b, rtol=1e-4):
    """Gradient tables are sums of hundreds of signed terms accumulated by atomics in arbitrary
    order: rtol on the element plus an absolute floor of 1e-5 of the table's largest entry
    (elements that are small only by cancellation cannot be held to a relative bound)."""
    b = b.detach().cpu().float()
    _close(a, b, rtol, 1e-5 * float(b.abs().max()) + 1e-9)


@pytest.mark.parametrize("case", helpers.GOLDEN_CASES)
def test_scoring_function_matches_reference(case, cuda_device):
    g = helpers.load_golden(case)
    model = helpers.model_from_golden(g).to(cuda_device)
    got = model.scoring_function(g["heads"].to(cuda_device), g["tails"].to(cuda_device),
                                 g["rels"].to(cuda_device))
    want = torch.from_numpy(g["raw"]["triple_scores"])
    _close(got, want, RTOL_SCORE, 1e-6)


@pytest.mark.parametrize("case", helpers.GOLDEN_CASES)
def test_forward_loss_and_gradients_match_reference(case, cuda_device):
    """model(h, t, r, nh, nt) + MarginLoss(0.5) + backward, negatives fixed by the fixture."""
    g = helpers.load_golden(case)
    model = helpers.model_from_golden(g).to(cuda_device)
    dev = cuda_device
    pos, neg = model(g["heads"].to(dev), g["tails"].to(dev), g["rels"].to(dev),
                     g["neg_heads"].to(dev), g["neg_tails"].to(dev))
    _close(pos, torch.from_numpy(g["raw"]["fwd_pos"]), RTOL_SCORE, 1e-6)
    _close(neg, torch.from_numpy(g["raw"]["fwd_neg"]), RTOL_SCORE, 1e-6)
    loss = tk.MarginLoss(0.5)(pos, neg)
    assert loss.item() == pytest.approx(float(g["raw"]["loss_margin_0p5"]), rel=1e-5)
    loss.backward()
    for name, p in model.named_parameters():
        _close_grad(p.grad, g["grads"][name])


@pytest.mark.parametrize("case", helpers.GOLDEN_CASES)
def test_fused_step_with_given_negatives_matches_reference(case, cuda_device):
    g = helpers.load_golden(case)
    model = helpers.model_from_golden(g).to(cuda_device)
    dev = cuda_device
    loss = fused_margin_step(model, g["heads"].to(dev), g["tails"].to(dev), g["rels"].to(dev), 0.5,
                             negatives=(g["neg_heads"].to(dev), g["neg_tails"].to(dev)))
    assert loss.item() == pytest.approx(float(g["raw"]["loss_margin_0p5"]), rel=1e-5)
    loss.backward()
    for name, p in model.named_parameters():
        _close_grad(p.grad, g["grads"][name])


@pytest.mark.parametrize("kind", ["transe_l2", "distmult", "complex", "rotate", "transe_l1", "rescal"])
def test_scoring_function_matches_oracle_unnormalised_weights(kind, cuda_device):
    n_ent, n_rel, d = 500, 9, 33 if kind != "rescal" else 12
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=4)
    with torch.no_grad():
        for p in model.parameters():
            p.mul_(1.7)
    model = model.to(cuda_device)
    P = helpers.oracle_params(kind, model)
    gen = torch.Generator().manual_seed(1)
    h = torch.randint(0, n_ent, (700,), generator=gen)
    t = torch.randint(0, n_ent, (700,), generator=gen)
    r = torch.randint(0, n_rel, (700,), generator=gen)
    got = model.scoring_function(h.to(cuda_device), t.to(cuda_device), r.to(cuda_device))
    _close(got, oracle.score_triples(kind, P, h, t, r), 2e-5, 2e-6)


@pytest.mark.parametrize("kind", ["transe_l2", "distmult", "complex", "rotate"])
def test_gradients_match_torch_autograd_of_the_oracle(kind, cuda_device):
    n_ent, n_rel, d, b, n_neg = 200, 5, 24, 64, 4
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=8).to(cuda_device)
    gen = torch.Generator().manual_seed(2)
    h = torch.randint(0, n_ent, (b,), generator=gen)
    t = torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    nh = torch.randint(1, n_ent, (b * n_neg,), generator=gen)
    nt = t.repeat(n_neg)
    # oracle side, CPU autograd
    if kind == "rotate":
        P = {"re_ent": model.re_ent_emb.weight.detach().cpu().clone().requires_grad_(True),
             "im_ent": model.im_ent_emb.weight.detach().cpu().clone().requires_grad_(True)}
        phase = model.rel_emb.weight.detach().cpu().clone().requires_grad_(True)
        P["re_rel"], P["im_rel"] = torch.cos(phase), torch.sin(phase)
        leaves = {"re_ent_emb.weight": P["re_ent"], "im_ent_emb.weight": P["im_ent"], "rel_emb.weight": phase}
    else:
        P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
        names = {"ent": "ent_emb.weight", "rel": "rel_emb.weight", "re_ent": "re_ent_emb.weight",
                 "im_ent": "im_ent_emb.weight", "re_rel": "re_rel_emb.weight", "im_rel": "im_rel_emb.weight"}
        leaves = {names[k]: v for k, v in P.items()}
    pos, neg = oracle.forward_pos_neg(kind, P, h, t, r, nh, nt)
    ref_loss = oracle.margin_loss(pos, neg, 1.0)
    ref_loss.backward()
    dev = cuda_device
    loss = fused_margin_step(model, h.to(dev), t.to(dev), r.to(dev), 1.0, negatives=(nh.to(dev), nt.to(dev)))
    assert loss.item() == pytest.approx(ref_loss.item(), rel=2e-5)
    loss.backward()
    for name, p in model.named_parameters():
        _close_grad(p.grad, leaves[name].grad, rtol=2e-4)


@pytest.mark.parametrize("kind", ["transe_l1", "transe_l2", "distmult"])
@pytest.mark.parametrize("d", [200, 256, 36])
def test_fast_fused_step_matches_oracle_autograd(kind, d, cuda_device):
    """The fused step of the single-plane models at dim % 4 == 0, dim <= 256 -- at n_neg = 40 the ring
    kernel (csrc/train.cu: margin_step_ring_kernel; the register-resident margin_step_fast_kernel and the
    ring past 48 KB are tests/test_train_paths_gpu.py's): head- and tail-corrupted negatives mixed, a
    negative equal to the positive, a few pairs with BOTH ends replaced (the generic path inside the
    kernel), un-normalised weights."""
    n_ent, n_rel, b, n_neg = 900, 7, 96, 40
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=11)
    with torch.no_grad():
        model.ent_emb.weight.mul_(1.0 + torch.rand(n_ent, 1))
    model = model.to(cuda_device)
    gen = torch.Generator().manual_seed(5)
    h = torch.randint(0, n_ent, (b,), generator=gen)
    t = torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    nh, nt = h.repeat(n_neg), t.repeat(n_neg)
    which = torch.rand(b * n_neg, generator=gen) < 0.45
    rnd = torch.randint(1, n_ent, (b * n_neg,), generator=gen)
    nh = torch.where(which, rnd, nh)
    nt = torch.where(~which, rnd, nt)
    nt[5], nh[5] = t[5], h[5]                       # a "negative" identical to the positive
    both = torch.arange(17, b * n_neg, 301)
    nh[both] = (h.repeat(n_neg)[both] + 3) % n_ent  # both ends differ
    nt[both] = (t.repeat(n_neg)[both] + 5) % n_ent
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    pos, neg = oracle.forward_pos_neg(kind, P, h, t, r, nh, nt)
    margin = 1.0 if kind == "distmult" else 0.3
    ref_loss = oracle.margin_loss(pos, neg, margin)
    ref_loss.backward()
    frac_active = ((margin - pos + neg) > 0).float().mean().item()
    assert 0.05 < frac_active <= 1.0
    dev = cuda_device
    loss = fused_margin_step(model, h.to(dev), t.to(dev), r.to(dev), margin, negatives=(nh.to(dev), nt.to(dev)))
    assert loss.item() == pytest.approx(ref_loss.item(), rel=2e-5)
    loss.backward()
    _close_grad(model.ent_emb.weight.grad, P["ent"].grad, rtol=2e-4)
    _close_grad(model.rel_emb.weight.grad, P["rel"].grad, rtol=2e-4)


def test_sampler_probabilities_match_reference():
    pass  # CPU-side; see tests/test_host_logic.py::test_bernoulli_probs_match_golden


def test_corrupt_batch_layout_support_and_frequencies(cuda_device):
    n_ent, n_rel = 5000, 6
    h, t, r = helpers.random_graph(n_ent, n_rel, 40000, seed=3)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=16, seed=123)
    b = 4096
    hb, tb_, rb = h[:b].to(cuda_device), t[:b].to(cuda_device), r[:b].to(cuda_device)
    nh, nt = sampler.corrupt_batch(hb, tb_, rb)
    assert nh.dtype == torch.int64 and nh.shape == (b * 16,) and nh.device == hb.device
    H, T = hb.repeat(16), tb_.repeat(16)
    head_changed, tail_changed = nh != H, nt != T
    assert not (head_changed & tail_changed).any()          # never both
    corrupted = torch.where(head_changed, nh, nt)[head_changed | tail_changed]
    assert corrupted.min().item() >= 1 and corrupted.max().item() < n_ent   # entity 0 never drawn
    # head-corruption frequency per relation ~ bern_probs (binomial, 5 sigma)
    R = rb.repeat(16)
    probs = sampler.bern_probs.cpu()
    for rel in range(n_rel):
        m = (R == rel)
        n = int(m.sum())
        if n < 500:
            continue
        # a replaced head may coincide with the original with probability ~1/n_ent: negligible
        f = head_changed[m].float().mean().item()
        p = probs[rel].item()
        assert abs(f - p) < 5 * (p * (1 - p) / n) ** 0.5 + 2.0 / n_ent, (rel, f, p)
    # uniformity of the replacements over [1, n_ent): chi-square on 50 bins
    hist = torch.histc(corrupted.float().cpu(), bins=50, min=1, max=n_ent)
    exp = corrupted.numel() / 50
    chi2 = ((hist - exp) ** 2 / exp).sum().item()
    assert chi2 < 120, chi2   # 49 dof: mean 49, 120 is far in the tail
    # same seed + same call count => same draws; next call differs
    s2 = tk.BernoulliNegativeSampler(kg, n_neg=16, seed=123)
    nh2, nt2 = s2.corrupt_batch(hb, tb_, rb)
    assert torch.equal(nh, nh2) and torch.equal(nt, nt2)
    nh3, _ = s2.corrupt_batch(hb, tb_, rb)
    assert not torch.equal(nh, nh3)


def test_fused_step_draws_the_negatives_corrupt_batch_draws(cuda_device):
    n_ent, n_rel, d, b, n_neg = 800, 7, 40, 256, 8
    h, t, r = helpers.random_graph(n_ent, n_rel, 5000, seed=5)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    model = helpers.make_model("distmult", d, n_ent, n_rel, seed=5).to(cuda_device)
    hb, tb_, rb = h[:b].to(cuda_device), t[:b].to(cuda_device), r[:b].to(cuda_device)
    s1 = tk.BernoulliNegativeSampler(kg, n_neg=n_neg, seed=77)
    s2 = tk.BernoulliNegativeSampler(kg, n_neg=n_neg, seed=77)
    nh, nt = s1.corrupt_batch(hb, tb_, rb)
    pos, neg = model(hb, tb_, rb, nh, nt)
    unfused = tk.MarginLoss(1.0)(pos, neg)
    fused = s2.fused_step(model, hb, tb_, rb, 1.0)
    assert fused.item() == pytest.approx(unfused.item(), rel=1e-5)
    unfused.backward()
    g1 = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    fused.backward()
    for n, p in model.named_parameters():
        _close_grad(p.grad, g1[n])


def test_training_loop_reduces_loss(cuda_device):
    """The tutorial loop (docs/tutorials/transe.rst:41-64) runs unchanged and learns."""
    n_ent, n_rel, d = 300, 5, 32
    h, t, r = helpers.random_graph(n_ent, n_rel, 3000, seed=6)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel)
    model = helpers.make_model("transe_l2", d, n_ent, n_rel, seed=6).to(cuda_device)
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=4, seed=1)
    crit = tk.MarginLoss(0.5)
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    hb, tb_, rb = (x.to(cuda_device) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    losses = []
    for _ in range(15):
        opt.zero_grad()
        nh, nt = sampler.corrupt_batch(hb, tb_, rb)
        pos, neg = model(hb, tb_, rb, nh, nt)
        loss = crit(pos, neg)
        loss.backward()
        opt.step()
        model.normalize_parameters()
        losses.append(loss.item())
    assert losses[-1] < 0.7 * losses[0], losses


@pytest.mark.parametrize("name", ["LogisticLoss", "BinaryCrossEntropyLoss"])
def test_logistic_and_bce_losses_match_torch(name, cuda_device):
    """utils/losses.py:47-112 restated with the same torch modules on the CPU."""
    gen = torch.Generator().manual_seed(3)
    pos = (torch.randn(5000, generator=gen) * 4).requires_grad_(True)
    neg = (torch.randn(5000, generator=gen) * 4).requires_grad_(True)
    with torch.no_grad():
        pos[:3] = torch.tensor([40.0, -40.0, 0.0])      # saturated sigmoids
        neg[:3] = torch.tensor([-40.0, 40.0, 0.0])
    if name == "LogisticLoss":
        crit = torch.nn.SoftMarginLoss(reduction="sum")
        ref = crit(pos, torch.ones_like(pos)) + crit(neg, -torch.ones_like(neg))
    else:
        crit = torch.nn.BCELoss(reduction="sum")
        ref = crit(torch.sigmoid(pos), torch.ones_like(pos)) + crit(torch.sigmoid(neg), torch.zeros_like(neg))
    ref.backward()
    p = pos.detach().to(cuda_device).requires_grad_(True)
    n = neg.detach().to(cuda_device).requires_grad_(True)
    loss = getattr(tk, name)()(p, n)
    assert loss.item() == pytest.approx(ref.item(), rel=1e-5)
    (2.0 * loss).backward()
    _close(p.grad, 2.0 * pos.grad, 1e-4, 1e-6)
    _close(n.grad, 2.0 * neg.grad, 1e-4, 1e-6)


def test_uniform_sampler_support_and_frequencies(cuda_device):
    n_ent, n_rel = 3000, 4
    h, t, r = helpers.random_graph(n_ent, n_rel, 20000, seed=8)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    sampler = tk.UniformNegativeSampler(kg, n_neg=8, seed=5)
    b = 4096
    hb, tb_ = h[:b].to(cuda_device), t[:b].to(cuda_device)
    nh, nt = sampler.corrupt_batch(hb, tb_)          # relations are optional, as in the reference
    assert nh.shape == (b * 8,) and nh.dtype == torch.int64 and nh.device == hb.device
    H, T = hb.repeat(8), tb_.repeat(8)
    head_changed, tail_changed = nh != H, nt != T
    assert not (head_changed & tail_changed).any()
    f = head_changed.float().mean().item()
    assert abs(f - 0.5) < 5 * (0.25 / (b * 8)) ** 0.5 + 2.0 / n_ent
    corrupted = torch.where(head_changed, nh, nt)[head_changed | tail_changed]
    assert corrupted.min().item() >= 1 and corrupted.max().item() < n_ent
    nh2, nt2 = tk.UniformNegativeSampler(kg, n_neg=8, seed=5).corrupt_batch(hb, tb_)
    assert torch.equal(nh, nh2) and torch.equal(nt, nt2)
    ch, ct = sampler.corrupt_kg(1000, True)          # whole graph, n_neg = 1, CPU tensors out
    assert ch.shape == (kg.n_facts,) and not ch.is_cuda and ct.dtype == torch.int64
