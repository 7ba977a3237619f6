"""The fused training step with LogisticLoss and BinaryCrossEntropyLoss (training.fused_loss_step):
against the reference's golden loss and gradients, against CPU autograd of the oracle's scores with
torch's SoftMarginLoss / BCELoss for every training kind, on the ring kernel's shapes, on saturated
sigmoids, and through the sampler.  Tolerances as in tests/test_train_gpu.py: the loss within 1e-5
relative, gradients under its atomics-order rule."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import torchkge_b200 as tk
from tests import helpers
from tests import train_kit as kit
from tests.train_kit import DEV
from torchkge_b200 import _lib
from torchkge_b200.engine import _ptr
from torchkge_b200.training import fused_loss_step, fused_margin_step, loss_kind_of

pytestmark = pytest.mark.gpu
ALL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "rotate", "analogy", "toruse_l1",
             "toruse_l2"]
LOSSES = {"logistic": (tk.LogisticLoss, _lib.LOSS_LOGISTIC), "bce": (tk.BinaryCrossEntropyLoss, _lib.LOSS_BCE)}


# ---------------------------------------------------------------- 1. reference golden values
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("case", helpers.GOLDEN_CASES)
def test_fused_step_matches_reference_golden(case, loss):
    """The fixture's weights and negatives; loss and gradients of torchkge's own criterion."""
    g = helpers.load_golden(case)
    z = np.load(os.path.join(helpers.GOLDEN_DIR, "loss_" + case + ".npz"), allow_pickle=False)
    model = helpers.model_from_golden(g).to(DEV)
    got = fused_loss_step(model, g["heads"].to(DEV), g["tails"].to(DEV), g["rels"].to(DEV), LOSSES[loss][0](),
                          negatives=(g["neg_heads"].to(DEV), g["neg_tails"].to(DEV)))
    assert got.item() == pytest.approx(float(z["loss_" + loss]), rel=1e-5)
    got.backward()
    for name, p in model.named_parameters():
        kit.close_grad(p.grad, torch.from_numpy(z["g_%s:%s" % (loss, name)]))


# ---------------------------------------------------------------- 2. every training kind vs CPU autograd
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_every_kind_matches_cpu_autograd(kind, loss):
    n_ent, n_rel, b, n_neg = 300, 6, 64, 5
    d = 12 if kind == "rescal" else 40
    model = kit.train_model(kind, d, n_ent, n_rel, seed=4)
    gen = torch.Generator().manual_seed(6)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    nh, nt = kit.negatives(h, t, n_ent, n_neg, gen)
    kit.check_against_cpu(model, kind, loss, h, t, r, nh, nt)


# ---------------------------------------------------------------- 3. the ring kernel's shapes
RING = [(k, d, (1, 33, 256)[i % 3]) for i, (k, d) in
        enumerate((k, d) for k in ("transe_l1", "transe_l2", "distmult") for d in (36, 200, 256))]


@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("source", ["external", "drawn"])
@pytest.mark.parametrize("kind,d,n_neg", RING, ids=["%s-d%d-neg%d" % c for c in RING])
def test_ring_shapes_match_cpu_autograd(kind, d, n_neg, source, loss):
    """External negatives (mixed sides, one equal to its positive, some with both ends replaced) and
    Philox draws (the ring's own draw loop; the CPU side gets kge_corrupt_batch's negatives)."""
    n_ent, n_rel, b = 900, 7, 96
    model = kit.train_model(kind, d, n_ent, n_rel, seed=11)
    gen = torch.Generator().manual_seed(d + n_neg)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    if source == "external":
        nh, nt = kit.negatives(h, t, n_ent, n_neg, gen)
        kit.check_against_cpu(model, kind, loss, h, t, r, nh, nt)
        return
    probs = torch.rand(n_rel, generator=gen).to(DEV)
    hd, td, rd = h.to(DEV), t.to(DEV), r.to(DEV)
    nh, nt = kit.corrupt_batch(hd, td, rd, probs, n_neg, n_ent, 31, 2)
    got, grads = kit.whole_table_step(model, hd, td, rd, n_neg=n_neg, loss=loss, probs=probs, seed=31, offset=2)
    cpu = kit.cpu_leaves(kit.train_leaves(model)[2])
    pos, neg = kit.cpu_pos_neg(kind, cpu, h, t, r, nh.cpu(), nt.cpu())
    want = kit.torch_loss(loss, pos, neg)
    want.backward()
    assert got == pytest.approx(want.item(), rel=2e-5)
    for a, c in zip(grads, cpu):
        if a is not None:
            kit.close_grad(a, c.grad, rtol=2e-4)


# ---------------------------------------------------------------- 4. saturated sigmoids
@pytest.mark.parametrize("loss", sorted(LOSSES))
@pytest.mark.parametrize("kind,d", [("distmult", 200), ("distmult", 40), ("transe_l2", 36), ("complex", 24)])
def test_saturated_scores(kind, d, loss):
    """Relations 1 and 2 scaled so that every score of their pairs lies far beyond +-20 (DistMult /
    ComplEx: +-thousands on positive entity rows; TransE: -1e8): BCE's gradients are exactly 0 where
    torch's are, and its -100 clamps give the same loss.  The logistic loss is held to its softplus form
    there (torch_loss: SoftMarginLoss itself overflows to inf)."""
    n_ent, n_rel, b, n_neg = 200, 3, 96, 8
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=21)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "ent" in name:
                p.abs_()
            elif kind == "transe_l2":
                p[1:] *= 1e4
            elif name.startswith("im_"):
                p[1:] = 0.0
            else:
                p[1], p[2] = 1e4, -1e4
    model = model.to(DEV)
    gen = torch.Generator().manual_seed(22)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    nh, nt = kit.negatives(h, t, n_ent, n_neg, gen)
    with torch.no_grad():
        pos, neg = kit.cpu_pos_neg(kind, [None if x is None else x.cpu() for x in kit.train_leaves(model)[2]], h,
                                   t, r, nh, nt)
    sat = r.repeat(n_neg) > 0
    assert (pos[sat].abs() > 100).all() and (neg[sat].abs() > 100).all()
    assert (pos[~sat].abs() < 20).all()
    grads, cpu = kit.check_against_cpu(model, kind, loss, h, t, r, nh, nt,
                                       ref="logistic_stable" if loss == "logistic" else None)
    for a, c in zip(grads, cpu):
        if a is not None:
            assert torch.equal(a.cpu() == 0, c.grad == 0)
    if loss == "bce":      # every pair of relations 1 and 2 is saturated: their rows get exactly 0
        assert (grads[2][1:] == 0).all() and (cpu[2].grad[1:] == 0).all()


# ---------------------------------------------------------------- 5. through the sampler
@pytest.mark.parametrize("loss", sorted(LOSSES))
def test_sampler_fused_step_equals_three_calls(loss):
    n_ent, n_rel, d, b, n_neg = 800, 7, 40, 256, 8
    h, t, r = helpers.random_graph(n_ent, n_rel, 5000, seed=5)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    model = helpers.make_model("distmult", d, n_ent, n_rel, seed=5).to(DEV)
    hb, tb_, rb = h[:b].to(DEV), t[:b].to(DEV), r[:b].to(DEV)
    s1 = tk.BernoulliNegativeSampler(kg, n_neg=n_neg, seed=77)
    s2 = tk.BernoulliNegativeSampler(kg, n_neg=n_neg, seed=77)
    crit = LOSSES[loss][0]()
    for _ in range(2):             # the second call: the same call count on both samplers
        nh, nt = s1.corrupt_batch(hb, tb_, rb)
        unfused = crit(*model(hb, tb_, rb, nh, nt))
        fused = s2.fused_step(model, hb, tb_, rb, criterion=crit)
    assert fused.item() == pytest.approx(unfused.item(), rel=1e-5)
    model.zero_grad()
    unfused.backward()
    g1 = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    fused.backward()
    for n, p in model.named_parameters():
        kit.close_grad(p.grad, g1[n])


class MarginLoss(torch.nn.Module):
    """torchkge's MarginLoss as it stores its margin (utils/losses.py:12-44)."""

    def __init__(self, margin):
        super().__init__()
        self.loss = torch.nn.MarginRankingLoss(margin=margin, reduction="sum")


@pytest.mark.parametrize("crit", ["package", "torchkge"])
def test_margin_criterion_equals_fused_margin_step(crit):
    n_ent, n_rel, d, b = 500, 5, 200, 128
    model = kit.train_model("distmult", d, n_ent, n_rel, seed=2)
    gen = torch.Generator().manual_seed(3)
    h, t = torch.randint(0, n_ent, (b,), generator=gen).to(DEV), torch.randint(0, n_ent, (b,), generator=gen).to(DEV)
    r = torch.randint(0, n_rel, (b,), generator=gen).to(DEV)
    probs = torch.rand(n_rel, generator=gen).to(DEV)
    criterion = tk.MarginLoss(0.7) if crit == "package" else MarginLoss(0.7)
    assert loss_kind_of(criterion) == (_lib.LOSS_MARGIN, pytest.approx(0.7))
    want = fused_margin_step(model, h, t, r, 0.7, n_neg=33, bern_probs=probs, seed=5, offset=1)
    want.backward()
    g1 = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    got = fused_loss_step(model, h, t, r, criterion, n_neg=33, bern_probs=probs, seed=5, offset=1)
    got.backward()
    assert got.item() == pytest.approx(want.item(), rel=1e-6)
    for n, p in model.named_parameters():
        kit.close_grad(p.grad, g1[n])


# ---------------------------------------------------------------- 6. ABI and argument errors
def test_margin_step_args_field_order_and_abi_version():
    names = kit.header_fields("kge_margin_step_args_t")
    assert names == [n for n, _ in _lib.MarginStepArgs._fields_]
    assert names[-1] == "loss_kind"
    assert _lib.load().kge_abi_version() == 11 == _lib.ABI_VERSION
    assert re.search(r"#define KGE_LOSS_MARGIN 0\b", kit.header())


def test_unknown_loss_kind_is_an_argument_error():
    lib = _lib.load()
    x = torch.zeros(64, device=DEV)
    a = _lib.MarginStepArgs()
    a.tb.model, a.tb.dim = _lib.DISTMULT, 4
    a.tb.ent0 = a.tb.rel0 = a.loss = a.bern_probs = _ptr(x)
    a.h = a.t = a.r = _ptr(x)
    a.n_neg, a.b, a.n_ent = 2, 1, 10
    g = _lib.Grads()
    g.ent0 = g.rel0 = _ptr(x)
    for kind in (3, -1, 100):
        a.loss_kind = kind
        assert lib.kge_margin_step_fwd(ctypes.byref(a)) == 1          # KGE_ERR_ARG
        assert lib.kge_margin_step_bwd(ctypes.byref(a), ctypes.byref(g), _ptr(x)) == 1
    torch.cuda.synchronize()


def test_argument_errors():
    n_ent, n_rel = 50, 4
    h, t, r = helpers.random_graph(n_ent, n_rel, 200, seed=3)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=2, seed=1)
    model = helpers.make_model("distmult", 8, n_ent, n_rel, seed=2).to(DEV)
    hb, tb_, rb = h[:4].to(DEV), t[:4].to(DEV), r[:4].to(DEV)
    with pytest.raises(TypeError, match="MSELoss"):
        fused_loss_step(model, hb, tb_, rb, torch.nn.MSELoss(), n_neg=2, bern_probs=sampler.bern_probs)
    with pytest.raises(TypeError):
        sampler.fused_step(model, hb, tb_, rb, criterion=torch.nn.SoftMarginLoss())
    with pytest.raises(ValueError, match="exactly one"):
        sampler.fused_step(model, hb, tb_, rb, 1.0, criterion=tk.LogisticLoss())
    with pytest.raises(ValueError, match="exactly one"):
        sampler.fused_step(model, hb, tb_, rb)
    assert sampler.fused_step(model, hb, tb_, rb, 1.0).item() >= 0.0     # positional margin as before


# ---------------------------------------------------------------- 7. training learns
def test_logistic_training_loop_reduces_loss():
    n_ent, n_rel, d = 300, 5, 32
    h, t, r = helpers.random_graph(n_ent, n_rel, 3000, seed=6)
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel)
    model = helpers.make_model("distmult", d, n_ent, n_rel, seed=6).to(DEV)
    sampler = tk.BernoulliNegativeSampler(kg, n_neg=4, seed=1)
    crit = tk.LogisticLoss()
    opt = torch.optim.Adam(model.parameters(), lr=0.1)
    hb, tb_, rb = (x.to(DEV) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    losses = []
    for _ in range(20):
        opt.zero_grad()
        loss = sampler.fused_step(model, hb, tb_, rb, criterion=crit)
        loss.backward()
        opt.step()
        model.normalize_parameters()
        losses.append(loss.item())
    # DistMult on unit entity rows: the scores are bounded by the relation rows, which grow ~lr per step
    assert losses[-1] < 0.9 * losses[0], losses
