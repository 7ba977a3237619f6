"""The fused training step on every kernel its launcher can pick for TransE-L1, TransE-L2 and DistMult
(csrc/train.cu: launch_margin_step), against torch autograd in float64 on the CPU.

The launcher picks by the ring kernel's shared memory, 4 * pad128(8 * 4 dim + 4 pad4(n_neg) + 64) bytes
per block: up to 48 KB the ring kernel runs as is, up to 96 KB after raising its dynamic shared memory
limit, beyond that the register-resident margin_step_fast_kernel (margin loss, unsharded) or the generic
kernels (the other losses; every sharded step).  KGE_TRAIN_RING=0 takes the ring out of the choice and
KGE_TRAIN_BWD_BLOCKS=5 holds the unsharded margin backward to 96 registers; both are read once per
process, so test_environment_variants runs this module again in a child process under each.

Every step is profiled and the kernels that ran are checked against a Python statement of the launch
rule (expected_kernels), which test_launch_rule_mirrors_train_cu pins to the constants of train.cu.
Tolerances: the loss within 2e-5 relative of the float64 loss, gradients within rtol 2e-4 plus a floor
of 1e-5 of the table's largest entry (tests/test_train_gpu.py), scores written out within 1e-5."""
import os
import re

import pytest
import torch

from tests import train_kit as kit
from tests.train_kit import (DEV, FAST_MAX_DIM, RING_MAX_NEG, RING_SLOTS, SMEM_DEFAULT, SMEM_MAX, WARPS_PER_BLOCK,
                             expected_kernels, kernel_signature, last_n_neg_within, launched)
from torchkge_b200.engine import CudaEngine

SWITCHES = ("KGE_TRAIN_RING", "KGE_TRAIN_BWD_BLOCKS")


def forward_of(kernels):
    return {k for k in kernels if k[0] in ("fwd", "shard_fwd") or (k[0] in ("ring", "fast") and not k[2])}


def test_launch_rule_mirrors_train_cu():
    """The constants and branches of expected_kernels are the ones train.cu launches by."""
    src = re.sub(r"//[^\n]*", "", open(kit.TRAIN_CU).read())
    flat = re.sub(r"\s+", " ", src)

    def const(name):
        return int(re.search(r"constexpr int %s = (\d+);" % name, src).group(1))

    def body(head):
        return re.sub(r"\s+", " ", re.search(re.escape(head) + r".*?\n}", src, flags=re.S).group(0))

    def in_order(text, *parts):
        at = [text.find(p) for p in parts]
        assert -1 not in at and at == sorted(at), [p for p, i in zip(parts, at) if i < 0] or at

    assert const("RING") == RING_SLOTS
    assert const("WARPS_PER_BLOCK") == WARPS_PER_BLOCK
    assert "constexpr int FAST_MAX_DIM = 4 * 32 * FAST_NCH;" in src
    assert 4 * 32 * const("FAST_NCH") == FAST_MAX_DIM
    # ring_smem_bytes: RING rows of 4 dim bytes, n_neg codes padded to 4, RING 8-byte barriers, per warp
    # rounded up to 128 bytes
    assert ("const size_t per_warp = (size_t)RING * a.dim * 4 + (size_t)((a.n_neg + 3) & ~3) * 4 + "
            "RING * sizeof(uint64_t); return WARPS_PER_BLOCK * ((per_warp + 127) & ~(size_t)127);") in flat
    ok = body("bool ring_step_ok(")
    assert "a.n_neg <= %d" % RING_MAX_NEG in ok and "ring_smem_bytes(a) <= 96 * 1024" in ok
    assert "getenv(\"KGE_TRAIN_RING\"); return !(v && v[0] == '0');" in ok
    launch = body("cudaError_t launch_ring_variant(")
    assert "smem > 48 * 1024" in launch and "cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024" in launch
    assert ("return (a.model == KGE_TRANSE_L1 || a.model == KGE_TRANSE_L2 || a.model == KGE_DISTMULT) && "
            "a.dim % 4 == 0 && a.dim <= FAST_MAX_DIM;") in flat
    # the choice itself: a relation step at rel_share >= 1 without caller negatives or nr_out is the entity
    # step; then the ring; else the register form for the unsharded entity step with the margin loss only
    # (never for a relation or positional step); else the generic kernels
    step = body("cudaError_t launch_margin_step(")
    in_order(step, "if (a.n_rel > 0 && a.rel_share >= 1.f && !a.nh && !a.nr_out) a.n_rel = 0;",
             "if (fast_step_ok(a) && ring_step_ok(a)) return with_fast_model(a.model, [&](auto m) { return "
             "launch_ring<decltype(m)::value, BWD>(a, gr, gloss, st, pc); });",
             "if (a.n_rel <= 0 && !pc.head_offs) { if (!shard && fast_step_ok(a) && a.loss_kind == KGE_LOSS_MARGIN) "
             "{ return with_fast_model(a.model, [&](auto m) { margin_step_fast_kernel<decltype(m)::value, BWD><<<",
             "if (shard) margin_step_shard_bwd_kernel<<<", "else margin_step_bwd_kernel<<<",
             "if (shard) margin_step_shard_fwd_kernel<<<", "else margin_step_fwd_kernel<<<")
    assert step.count("margin_step_fast_kernel") == 1 and step.count("launch_ring<") == 1
    # the ring's kinds: positional, relation, then the entity step, where MINB = 5 (KGE_TRAIN_BWD_BLOCKS=5)
    # only for the unsharded margin backward; the kernels' template arguments in kernel_signature's order
    ring = body("cudaError_t launch_ring(")
    in_order(ring, "if (pc.head_offs) return a.hrows ? launch_ring_variant<MODEL, BWD, 0, true, LOSS, false, true>"
                   "(a, gr, gloss, st, pc) : launch_ring_variant<MODEL, BWD, 0, false, LOSS, false, true>(a, gr, "
                   "gloss, st, pc);",
             "if (a.n_rel > 0) return a.hrows ? launch_ring_variant<MODEL, BWD, 0, true, LOSS, true>(a, gr, gloss, "
             "st) : launch_ring_variant<MODEL, BWD, 0, false, LOSS, true>(a, gr, gloss, st);",
             "if (a.hrows) return launch_ring_variant<MODEL, BWD, 0, true, LOSS>(a, gr, gloss, st); "
             "if constexpr (BWD && LOSS == KGE_LOSS_MARGIN) { static const bool tight = [] { const char* v = "
             "getenv(\"KGE_TRAIN_BWD_BLOCKS\"); return v && v[0] == '5'; }(); if (tight) return "
             "launch_ring_variant<MODEL, true, 5, false, LOSS>(a, gr, gloss, st); } "
             "return launch_ring_variant<MODEL, BWD, 0, false, LOSS>(a, gr, gloss, st);",
             "case KGE_LOSS_LOGISTIC: return by_shard(std::integral_constant<int, KGE_LOSS_LOGISTIC>{}); "
             "case KGE_LOSS_BCE: return by_shard(std::integral_constant<int, KGE_LOSS_BCE>{}); "
             "default: return by_shard(std::integral_constant<int, KGE_LOSS_MARGIN>{});")
    assert ring.count("launch_ring_variant<") == 7
    assert ("if constexpr (POS) return margin_step_ring_pos_kernel<MODEL, BWD, SHARD, LOSS>; else if constexpr "
            "(REL) return margin_step_ring_rel_kernel<MODEL, BWD, SHARD, LOSS>; else return "
            "margin_step_ring_kernel<MODEL, BWD, MINB, SHARD, LOSS>;") in flat
    assert (SMEM_DEFAULT, SMEM_MAX) == (48 * 1024, 96 * 1024)
    # n_neg <= 8192 never decides: the codes alone pass 96 KB first, at every dim the ring takes
    assert all(last_n_neg_within(d, SMEM_MAX) < RING_MAX_NEG for d in range(4, FAST_MAX_DIM + 1, 4))


def test_kernel_signature_parses_both_name_forms():
    ns = "void kge::(anonymous namespace)::"
    assert kernel_signature(ns + "margin_step_ring_kernel<2, true, 5, false, 0>(kge::MarginStepParams, "
                            "kge::TrainGrads, float const*)") == ("ring", 2, True, 5, False, 0)
    assert kernel_signature(ns + "margin_step_fast_kernel<0, false>(kge::MarginStepParams)") == ("fast", 0, False)
    assert kernel_signature(ns + "margin_step_fwd_kernel(kge::MarginStepParams)") == ("fwd",)
    assert kernel_signature(ns + "margin_step_shard_fwd_kernel(kge::MarginStepParams)") == ("shard_fwd",)
    assert kernel_signature("_ZN3kge12_GLOBAL__N_123margin_step_ring_kernelILi1ELb0ELi0ELb1ELi2EEEvNS_16Margin"
                            "StepParamsENS_10TrainGradsEPKf") == ("ring", 1, False, 0, True, 2)
    assert kernel_signature("_ZN3kge12_GLOBAL__N_128margin_step_shard_bwd_kernelENS_16MarginStepParamsE") == \
        ("shard_bwd",)
    assert kernel_signature(ns + "margin_step_ring_rel_kernel<1, true, false, 2>(kge::MarginStepParams, "
                            "kge::TrainGrads, float const*)") == ("ring_rel", 1, True, False, 2)
    assert kernel_signature("_ZN3kge12_GLOBAL__N_127margin_step_ring_pos_kernelILi0ELb0ELb1ELi1EEEvNS_16Margin"
                            "StepParamsENS_10TrainGradsEPKfNS_6PosCSRE") == ("ring_pos", 0, False, True, 1)
    assert kernel_signature("void at::native::vectorized_elementwise_kernel<4>(int)") is None


# ---------------------------------------------------------------- data and the float64 reference
KINDS = tuple(kit.FAST_KINDS)
DIMS = (36, 200, 256)
N_ENT, N_REL = 1500, 11
SEED, OFFSET = 4099, 7


def boundaries(dim):
    """n_neg at the two limits: the last within 48 KB, the first past it, the last within 96 KB, the first
    past it."""
    a, b = last_n_neg_within(dim, SMEM_DEFAULT), last_n_neg_within(dim, SMEM_MAX)
    return (a, a + 1, b, b + 1)


def problem(kind, dim, n_neg, source, seed):
    """A model, a batch of 23 positives (the last block holds three warps) on the GPU, Bernoulli
    probabilities and the negatives: external ones (train_kit.negatives) or the kernel's own draws."""
    model = kit.train_model(kind, dim, N_ENT, N_REL, seed=seed)
    gen = torch.Generator().manual_seed(seed + n_neg)
    h, t, r, probs = kit.batch(N_ENT, N_REL, 23, gen)
    if source == "external":
        nh, nt = (x.to(DEV) for x in kit.negatives(h.cpu(), t.cpu(), N_ENT, n_neg, gen))
    else:
        nh, nt = kit.corrupt_batch(h, t, r, probs, n_neg, N_ENT, SEED, OFFSET)
    return model, h, t, r, probs, nh, nt


def reference_with_margin(kind, model, h, t, r, nh, nt, loss):
    """train_kit.reference on the model's leaves, (loss, [grads], pos, neg, margin), with the margin chosen
    here (margin_between) so that between 5 and 95 % of the hinges are active."""
    ts = kit.train_leaves(model)[2]
    margin = 0.0
    if loss == "margin":
        pos, neg = kit.cpu_pos_neg(kind, kit.cpu_leaves(ts, torch.float64), h.cpu(), t.cpu(), r.cpu(), nh.cpu(),
                                   nt.cpu())
        margin = kit.margin_between(pos - neg)
        active = float(((margin - pos + neg) > 0).double().mean())
        assert 0.05 <= active <= 0.95, active
    return kit.reference(kind, ts, h, t, r, nh, nt, loss, margin) + (margin,)


def assert_matches_reference(got_loss, got_grads, want_loss, want_grads, h, t):
    """The loss within 2e-5, every table under close_grad(rtol=2e-4) -- and the entity rows that only
    negatives touch once more on their own, so that the positives' large rows do not set their floor."""
    assert got_loss == pytest.approx(want_loss, rel=2e-5)
    for a, c in zip(got_grads, want_grads):
        if c is not None:
            kit.close_grad(a, c, rtol=2e-4)
    only_neg = torch.ones(N_ENT, dtype=torch.bool)
    only_neg[torch.cat([h, t]).cpu()] = False
    kit.close_grad(got_grads[0].cpu()[only_neg], want_grads[0][only_neg], rtol=2e-4)


def _unsharded_cases():
    margin = [(k, d, n, "margin") for k in KINDS for d in DIMS for n in boundaries(d)]
    small = [(k, d, n, "margin") for k in KINDS for d, n in ((36, 1), (200, 33), (256, 256))]
    # the other losses on the ring past 48 KB and at its largest n_neg, and on the generic kernels past 96 KB
    losses = [(k, d, boundaries(d)[i], loss) for k in KINDS for loss in ("logistic", "bce")
              for d, i in ((256, 1), (200, 2), (200, 3))]
    return margin + small + losses


UNSHARDED = _unsharded_cases()


# ---------------------------------------------------------------- 2. unsharded, at the boundaries
@pytest.mark.gpu
@pytest.mark.parametrize("source", ["external", "drawn"])
@pytest.mark.parametrize("kind,d,n_neg,loss", UNSHARDED, ids=["%s-d%d-neg%d-%s" % c for c in UNSHARDED])
def test_step_matches_float64_autograd(kind, d, n_neg, loss, source):
    model, h, t, r, probs, nh, nt = problem(kind, d, n_neg, source, seed=d + 3)
    want_loss, want_grads, _, _, margin = reference_with_margin(kind, model, h, t, r, nh, nt, loss)
    negs = dict(negatives=(nh, nt)) if source == "external" else dict(n_neg=n_neg, probs=probs, seed=SEED,
                                                                      offset=OFFSET)

    def step():
        return kit.whole_table_step(model, h, t, r, loss=loss, margin=margin, **negs)

    got, grads = step()
    assert_matches_reference(got, grads, want_loss, want_grads, h, t)
    expected = expected_kernels(kind, d, n_neg, loss, shard=False)
    assert launched(step, expected) == expected


# ---------------------------------------------------------------- 3. optional outputs
ROUTES = {"fast": ("margin", 3), "ring_past_48k": ("margin", 1), "generic": ("logistic", 3)}


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["external", "drawn"])
@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("kind", KINDS)
def test_optional_outputs(kind, route, source):
    """pos_out / neg_out / nh_out / nt_out through the C ABI (kge_margin_step_fwd)."""
    loss, which = ROUTES[route]
    d = 200
    n_neg = boundaries(d)[which]
    model, h, t, r, probs, nh, nt = problem(kind, d, n_neg, source, seed=17)
    want_loss, _, pos, neg, margin = reference_with_margin(kind, model, h, t, r, nh, nt, loss)
    b = h.shape[0]
    kw = dict(n_neg=n_neg, loss=loss, margin=margin, probs=probs, seed=SEED, offset=OFFSET,
              negatives=(nh, nt) if source == "external" else None)
    out = kit.forward_outputs(model, h, t, r, **kw)
    assert torch.equal(out["nh"], nh) and torch.equal(out["nt"], nt)
    torch.testing.assert_close(out["pos"].cpu().double(), pos[:b], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(out["neg"].cpu().double(), neg, rtol=1e-5, atol=1e-6)
    assert out["loss"].item() == pytest.approx(want_loss, rel=2e-5)
    expected = forward_of(expected_kernels(kind, d, n_neg, loss, shard=False))
    assert launched(lambda: kit.forward_outputs(model, h, t, r, **kw), expected) == expected


# ---------------------------------------------------------------- 4. sharded, at the boundaries
SHARDED = ([(k, d, boundaries(d)[i], "margin") for k in KINDS for d in DIMS for i in (1, 3)] +
           [(k, 200, boundaries(200)[3], loss) for k in KINDS for loss in ("logistic", "bce")])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d,n_neg,loss", SHARDED, ids=["%s-d%d-neg%d-%s" % c for c in SHARDED])
def test_sharded_step_matches_unsharded_and_float64_autograd(kind, d, n_neg, loss):
    """Emulated shards (train_kit.emulated: every rank's kernels on its row range, the all-reduces as sums)."""
    model, h, t, r, probs, nh, nt = problem(kind, d, n_neg, "drawn", seed=d + 5)
    want_loss, want_grads, _, _, margin = reference_with_margin(kind, model, h, t, r, nh, nt, loss)
    kw = dict(n_neg=n_neg, probs=probs, loss=loss, margin=margin, seed=SEED, offset=OFFSET)
    one_loss, one_grads = kit.whole_table_step(model, h, t, r, **kw)
    eng = CudaEngine()
    expected = expected_kernels(kind, d, n_neg, loss, shard=True)
    for world in (1, 3, 8):
        got_loss, got_grads = kit.emulated(model, h, t, r, world, eng, **kw)
        assert got_loss == pytest.approx(one_loss, rel=1e-5, abs=1e-6)
        for a, c in zip(got_grads, one_grads):
            if c is not None:
                kit.close_grad(a, c, rtol=1e-4)
        assert_matches_reference(got_loss, got_grads, want_loss, want_grads, h, t)
        ran = launched(lambda: kit.emulated(model, h, t, r, world, eng, **kw), expected)
        assert ran == expected, world


# ---------------------------------------------------------------- 5. the environment switches
@pytest.mark.gpu
@pytest.mark.parametrize("switch", ["KGE_TRAIN_RING=0", "KGE_TRAIN_BWD_BLOCKS=5"])
def test_environment_variants(switch):
    """This module once more in a fresh process with the switch set: every case then asserts the kernels
    expected_kernels names under it (KGE_TRAIN_RING=0: the register form for every unsharded margin step,
    the generic kernels for the other losses and every sharded step; KGE_TRAIN_BWD_BLOCKS=5: the
    96-register backward of the unsharded margin ring)."""
    if any(v in os.environ for v in SWITCHES):
        pytest.skip("runs in the parent process only (%s is set here)" % ", ".join(v for v in SWITCHES
                                                                                if v in os.environ))
    out = kit.rerun(__file__, switch)
    assert " skipped" in out, out[-2000:]
