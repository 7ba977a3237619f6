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
import ctypes
import os
import re
import subprocess
import sys
import time

import pytest
import torch

from tests import helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import CudaEngine, _ptr, _stream
from torchkge_b200.training import _MarginStep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN_CU = os.path.join(ROOT, "torchkge_b200", "csrc", "train.cu")
DEV = helpers.DEV
SWITCHES = ("KGE_TRAIN_RING", "KGE_TRAIN_BWD_BLOCKS")

# ---------------------------------------------------------------- the launch rule, restated
RING_SLOTS = 8                 # RING: rows in flight per warp
WARPS_PER_BLOCK = 4
FAST_MAX_DIM = 256             # 4 floats x 32 lanes x FAST_NCH chunks
SMEM_DEFAULT = 48 * 1024       # dynamic shared memory without cudaFuncSetAttribute
SMEM_MAX = 96 * 1024           # what launch_ring_variant raises the limit to
RING_MAX_NEG = 8192
FAST_KINDS = {"transe_l1": _lib.TRANSE_L1, "transe_l2": _lib.TRANSE_L2, "distmult": _lib.DISTMULT}


def _pad(x, m):
    return (x + m - 1) // m * m


def ring_smem_bytes(dim, n_neg):
    """Dynamic shared memory of one ring block: per warp RING rows, the codes of every negative and
    one mbarrier per slot, each warp's part rounded up to 128 bytes."""
    per_warp = RING_SLOTS * dim * 4 + _pad(n_neg, 4) * 4 + RING_SLOTS * 8
    return WARPS_PER_BLOCK * _pad(per_warp, 128)


def last_n_neg_within(dim, limit):
    """The largest n_neg whose ring block fits in `limit` bytes."""
    n = 1
    while ring_smem_bytes(dim, n + 1) <= limit:
        n += 1
    return n


def expected_kernels(kind, dim, n_neg, loss, shard, env=None):
    """Signatures (see kernel_signature) of the forward and backward kernels one step launches."""
    env = os.environ if env is None else env
    ring_on = env.get("KGE_TRAIN_RING", "")[:1] != "0"
    tight = env.get("KGE_TRAIN_BWD_BLOCKS", "")[:1] == "5"
    fast = kind in FAST_KINDS and dim % 4 == 0 and dim <= FAST_MAX_DIM
    if fast and ring_on and n_neg <= RING_MAX_NEG and ring_smem_bytes(dim, n_neg) <= SMEM_MAX:
        minb = 5 if tight and not shard and loss == "margin" else 0
        lk = helpers.LOSS_KINDS[loss]
        return {("ring", FAST_KINDS[kind], False, 0, shard, lk), ("ring", FAST_KINDS[kind], True, minb, shard, lk)}
    if fast and not shard and loss == "margin":
        return {("fast", FAST_KINDS[kind], False), ("fast", FAST_KINDS[kind], True)}
    return {("shard_fwd",), ("shard_bwd",)} if shard else {("fwd",), ("bwd",)}


def forward_of(kernels):
    return {k for k in kernels if k[0] in ("fwd", "shard_fwd") or (k[0] in ("ring", "fast") and not k[2])}


def test_launch_rule_mirrors_train_cu():
    """The constants and conditions above are the ones train.cu launches by."""
    src = open(TRAIN_CU).read()
    flat = re.sub(r"\s+", " ", src)

    def const(name):
        return int(re.search(r"constexpr int %s = (\d+);" % name, src).group(1))

    assert const("RING") == RING_SLOTS
    assert const("WARPS_PER_BLOCK") == WARPS_PER_BLOCK
    assert "constexpr int FAST_MAX_DIM = 4 * 32 * FAST_NCH;" in src
    assert 4 * 32 * const("FAST_NCH") == FAST_MAX_DIM
    # ring_smem_bytes: RING rows of 4 dim bytes, n_neg codes padded to 4, RING 8-byte barriers, per warp
    # rounded up to 128 bytes
    assert ("const size_t per_warp = (size_t)RING * a.dim * 4 + (size_t)((a.n_neg + 3) & ~3) * 4 + "
            "RING * sizeof(uint64_t); return WARPS_PER_BLOCK * ((per_warp + 127) & ~(size_t)127);") in flat
    body = re.search(r"bool ring_step_ok\(.*?\n}", src, flags=re.S).group(0)
    assert "a.n_neg <= %d" % RING_MAX_NEG in body and "ring_smem_bytes(a) <= 96 * 1024" in body
    assert "getenv(\"KGE_TRAIN_RING\"); return !(v && v[0] == '0');" in re.sub(r"\s+", " ", body)
    launch = re.search(r"cudaError_t launch_ring_variant\(.*?\n}", src, flags=re.S).group(0)
    assert "smem > 48 * 1024" in launch and "cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024" in launch
    assert "getenv(\"KGE_TRAIN_BWD_BLOCKS\"); return v && v[0] == '5';" in flat
    assert ("return (a.model == KGE_TRANSE_L1 || a.model == KGE_TRANSE_L2 || a.model == KGE_DISTMULT) && "
            "a.dim % 4 == 0 && a.dim <= FAST_MAX_DIM;") in flat
    # the choice itself: ring, else (unsharded margin) the register form, else the generic kernels
    assert ("if (fast_step_ok(a) && ring_step_ok(a)) return with_fast_model(" in flat and
            "if (!shard && fast_step_ok(a) && a.loss_kind == KGE_LOSS_MARGIN) {" in flat)
    assert (SMEM_DEFAULT, SMEM_MAX) == (48 * 1024, 96 * 1024)
    # n_neg <= 8192 never decides: the codes alone pass 96 KB first, at every dim the ring takes
    assert all(last_n_neg_within(d, SMEM_MAX) < RING_MAX_NEG for d in range(4, FAST_MAX_DIM + 1, 4))


# ---------------------------------------------------------------- which kernels ran
_KERNEL = r"margin_step_(ring|fast|shard_fwd|shard_bwd|fwd|bwd)_kernel"
_DEMANGLED = re.compile(r"(?<![\w])" + _KERNEL + r"(?:<([^<>]*)>)?\(")
_MANGLED = re.compile(r"\d" + _KERNEL + r"(?:I((?:L[ib]\d+E)+)E)?")


def kernel_signature(name):
    """("ring", model, bwd, minb, shard, loss), ("fast", model, bwd), ("fwd",), ("bwd",), ("shard_fwd",) or
    ("shard_bwd",) for a fused-step kernel's (demangled or mangled) name; None for any other kernel."""
    m = _DEMANGLED.search(name)
    if m:
        args = [] if m.group(2) is None else [a.strip() for a in m.group(2).split(",")]
        args = [a == "true" if a in ("true", "false") else int(re.sub(r"^\(\w+\)", "", a)) for a in args]
    else:
        m = _MANGLED.search(name)
        if not m:
            return None
        args = [bool(int(v)) if k == "b" else int(v) for k, v in re.findall(r"L([ib])(\d+)E", m.group(2) or "")]
    return (m.group(1),) + tuple(args)


def _cuda_kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def launched(fn, expected, tries=4):
    """The set of fused-step kernel signatures that ran on the GPU while fn() ran.  torch.profiler now and
    then leaves a kernel out of its record, so fn (which must be repeatable) runs up to `tries` times
    under it until every expected kernel has been seen; the union is returned, so a kernel that should
    not run still shows."""
    ran, names = set(), []
    for _ in range(tries):
        names = _cuda_kernel_names(fn)
        ran |= {s for s in map(kernel_signature, names) if s is not None}
        if ran >= expected:
            break
    if not ran:
        control = _cuda_kernel_names(lambda: torch.ones(4, device=DEV).add_(1))
        if not control:
            pytest.fail("torch.profiler records no CUDA kernels here, not even torch's own: the kernel each "
                        "step runs cannot be checked")
        if not names:
            pytest.fail("torch.profiler recorded a torch kernel but none while the fused step ran")
    return ran


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
    assert kernel_signature("void at::native::vectorized_elementwise_kernel<4>(int)") is None


# ---------------------------------------------------------------- data and the float64 reference
KINDS = tuple(FAST_KINDS)
DIMS = (36, 200, 256)
N_ENT, N_REL = 1500, 11
SEED, OFFSET = 4099, 7


def boundaries(dim):
    """n_neg at the two limits: the last within 48 KB, the first past it, the last within 96 KB, the first
    past it."""
    a, b = last_n_neg_within(dim, SMEM_DEFAULT), last_n_neg_within(dim, SMEM_MAX)
    return (a, a + 1, b, b + 1)


def draw(h, t, r, probs, n_neg):
    """kge_corrupt_batch's negatives: the ones every fused kernel draws at (SEED, OFFSET)."""
    nh = torch.empty(h.shape[0] * n_neg, dtype=torch.int64, device=DEV)
    nt = torch.empty_like(nh)
    _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), h.shape[0], n_neg, _ptr(probs), N_ENT, SEED,
                                             OFFSET, _ptr(nh), _ptr(nt), _stream(h.device)), "kge_corrupt_batch")
    return nh, nt


def problem(kind, dim, n_neg, source, seed):
    """A model, a batch of 23 positives (the last block holds three warps) on the GPU, Bernoulli
    probabilities and the negatives: external ones (helpers.negatives) or the kernel's own draws."""
    model = helpers.train_model(kind, dim, N_ENT, N_REL, seed=seed)
    gen = torch.Generator().manual_seed(seed + n_neg)
    b = 23
    h, t = torch.randint(0, N_ENT, (b,), generator=gen), torch.randint(0, N_ENT, (b,), generator=gen)
    r = torch.randint(0, N_REL, (b,), generator=gen)
    probs = torch.rand(N_REL, generator=gen)
    h, t, r, probs = h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)
    if source == "external":
        nh, nt = helpers.negatives(h.cpu(), t.cpu(), N_ENT, n_neg, gen)
        nh, nt = nh.to(DEV), nt.to(DEV)
    else:
        nh, nt = draw(h, t, r, probs, n_neg)
    return model, h, t, r, probs, nh, nt


def margin_between(diff, q=0.5):
    """A float32 margin m in the widest gap between neighbouring values of pos - neg near its q-quantile:
    about half the hinges are active, and none lies so close to its kink that float32 and float64 could
    disagree on whether it is."""
    s = torch.sort(diff.detach().flatten()).values
    k = int(q * (s.shape[0] - 1))
    w = min(200, s.shape[0] // 4)
    if w == 0:
        return float(torch.tensor(float(s[0]) + 0.5, dtype=torch.float32))
    lo, hi = k - w, k + w
    i = lo + int(torch.argmax(s[lo + 1:hi + 1] - s[lo:hi]))
    return float(torch.tensor(float(s[i] + s[i + 1]) / 2, dtype=torch.float32))


def reference(kind, ts, h, t, r, nh, nt, loss):
    """float64 CPU autograd of the oracle's scores on copies of the kernel's leaves:
    (loss, [grads], pos, neg, margin); the margin is chosen here (margin_between)."""
    cpu = helpers.cpu_leaves(ts, torch.float64)
    pos, neg = helpers.cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    margin = margin_between(pos - neg) if loss == "margin" else 0.0
    if loss == "margin":
        active = float(((margin - pos + neg) > 0).double().mean())
        assert 0.05 <= active <= 0.95, active
    want = helpers.torch_loss(loss, pos, neg, margin)
    want.backward()
    return want.item(), [None if x is None else x.grad for x in cpu], pos.detach(), neg.detach(), margin


def assert_matches_reference(got_loss, got_grads, want_loss, want_grads, h, t):
    """The loss within 2e-5, every table under close_grad(rtol=2e-4) -- and the entity rows that only
    negatives touch once more on their own, so that the positives' large rows do not set their floor."""
    assert got_loss == pytest.approx(want_loss, rel=2e-5)
    for a, c in zip(got_grads, want_grads):
        if c is not None:
            helpers.close_grad(a, c, rtol=2e-4)
    only_neg = torch.ones(N_ENT, dtype=torch.bool)
    only_neg[torch.cat([h, t]).cpu()] = False
    helpers.close_grad(got_grads[0].cpu()[only_neg], want_grads[0][only_neg], rtol=2e-4)


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
    code, dim, ts = helpers.train_leaves(model)
    want_loss, want_grads, _, _, margin = reference(kind, ts, h, t, r, nh, nt, loss)
    lk = helpers.LOSS_KINDS[loss]

    def step(leaves):
        if source == "external":
            got = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, nh, nt, None, 0, 0, *leaves, lk)
        else:
            got = _MarginStep.apply(code, dim, N_ENT, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET,
                                    *leaves, lk)
        got.backward()
        return got.item()

    got = step(ts)
    assert_matches_reference(got, [None if x is None else x.grad for x in ts], want_loss, want_grads, h, t)
    expected = expected_kernels(kind, d, n_neg, loss, shard=False)
    assert launched(lambda: step(helpers.train_leaves(model)[2]), expected) == expected


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
    code, dim, ts = helpers.train_leaves(model)
    want_loss, _, pos, neg, margin = reference(kind, ts, h, t, r, nh, nt, loss)
    b = h.shape[0]
    tabs = [None if x is None else x.detach() for x in ts]
    pos_out, neg_out = torch.full((b,), float("nan"), device=DEV), torch.full((b * n_neg,), float("nan"), device=DEV)
    ids = [torch.full((b * n_neg,), -1, dtype=torch.int64, device=DEV) for _ in range(2)]
    out = torch.zeros((), device=DEV)
    ext = source == "external"
    a = _MarginStep._args(code, dim, N_ENT, margin, n_neg, h, t, r, nh if ext else None, nt if ext else None,
                          probs, SEED, OFFSET, tabs, out, h.device, helpers.LOSS_KINDS[loss])
    a.pos_out, a.neg_out, a.nh_out, a.nt_out = _ptr(pos_out), _ptr(neg_out), _ptr(ids[0]), _ptr(ids[1])
    assert _lib.load().kge_margin_step_fwd(ctypes.byref(a)) == 0
    torch.cuda.synchronize()
    assert torch.equal(ids[0], nh) and torch.equal(ids[1], nt)
    torch.testing.assert_close(pos_out.cpu().double(), pos[:b], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(neg_out.cpu().double(), neg, rtol=1e-5, atol=1e-6)
    assert out.item() == pytest.approx(want_loss, rel=2e-5)
    expected = forward_of(expected_kernels(kind, d, n_neg, loss, shard=False))
    assert launched(lambda: _lib.load().kge_margin_step_fwd(ctypes.byref(a)), expected) == expected


# ---------------------------------------------------------------- 4. sharded, at the boundaries
SHARDED = ([(k, d, boundaries(d)[i], "margin") for k in KINDS for d in DIMS for i in (1, 3)] +
           [(k, 200, boundaries(200)[3], loss) for k in KINDS for loss in ("logistic", "bce")])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,d,n_neg,loss", SHARDED, ids=["%s-d%d-neg%d-%s" % c for c in SHARDED])
def test_sharded_step_matches_unsharded_and_float64_autograd(kind, d, n_neg, loss):
    """Emulated shards (helpers.emulated: every rank's kernels on its row range, the all-reduces as sums)."""
    model, h, t, r, probs, nh, nt = problem(kind, d, n_neg, "drawn", seed=d + 5)
    _, _, ts = helpers.train_leaves(model)
    want_loss, want_grads, _, _, margin = reference(kind, ts, h, t, r, nh, nt, loss)
    lk = helpers.LOSS_KINDS[loss]
    one_loss, one_grads = helpers.unsharded(model, h, t, r, probs, margin, n_neg, SEED, OFFSET, lk)
    eng = CudaEngine()
    expected = expected_kernels(kind, d, n_neg, loss, shard=True)
    for world in (1, 3, 8):
        got_loss, got_grads = helpers.emulated(model, h, t, r, probs, margin, n_neg, SEED, OFFSET, world, eng, lk)
        assert got_loss == pytest.approx(one_loss, rel=1e-5, abs=1e-6)
        for a, c in zip(got_grads, one_grads):
            if c is not None:
                helpers.close_grad(a, c, rtol=1e-4)
        assert_matches_reference(got_loss, got_grads, want_loss, want_grads, h, t)
        ran = launched(lambda: helpers.emulated(model, h, t, r, probs, margin, n_neg, SEED, OFFSET, world, eng, lk),
                       expected)
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
    name, value = switch.split("=")
    env = dict(os.environ, **{name: value})
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__)]
    start = time.time()
    proc = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    print("%s: %.0f s\n%s" % (switch, time.time() - start, proc.stdout[-600:]))
    assert proc.returncode == 0, "%s\n%s\n%s" % (switch, proc.stdout[-6000:], proc.stderr[-3000:])
    assert " passed" in proc.stdout and " skipped" in proc.stdout, proc.stdout[-2000:]
