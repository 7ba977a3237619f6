"""The DEVICE score arithmetic (torchkge_b200/csrc/reduce.cuh), compiled for the host with g++
(tests/host_arith.cpp + tests/host_shim/cuda_runtime.h: every rounded intrinsic mapped to the IEEE
operation it names, -ffp-contract=off), against ATen on the CPU, bit for bit:

  * replay : acc_step over the reduction schedule + acc_finish -- what true_scores_kernel,
             filter_kernel and the dense scan execute per (query, candidate) pair
  * natural: pair_score_natural -- the natural-order form used for small dims and as the
             definition the chain-parallel scorers are tested against on the GPU

for every element kind, including the TorusE kinds that have not run on a GPU yet.  This checks
the arithmetic the kernels are made of, not their tiling or pipelines (that is what -m gpu does).
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from torchkge_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# element kinds of csrc/reduce.cuh: (id, model code whose schedule it uses, QW, CW)
KINDS = {
    "dot1": (0, _lib.DISTMULT, 1, 1), "dot2": (1, _lib.COMPLEX, 2, 2),
    "l1_tail": (2, _lib.TRANSE_L1, 1, 1), "l1_head": (3, _lib.TRANSE_L1, 2, 1),
    "l2_tail": (4, _lib.TRANSE_L2, 1, 1), "l2_head": (5, _lib.TRANSE_L2, 2, 1),
    "rot": (6, _lib.ROTATE, 2, 2), "dot_mid": (7, _lib.DISTMULT, 2, 1),
    "tl1_tail": (8, _lib.TORUSE_L1, 1, 1), "tl1_head": (9, _lib.TORUSE_L1, 2, 1),
    "tl2_tail": (10, _lib.TORUSE_L2, 1, 1), "tl2_head": (11, _lib.TORUSE_L2, 2, 1),
    "dot3": (12, _lib.ANALOGY, 3, 3),
}


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    out = str(tmp_path_factory.mktemp("host_arith") / "host_arith.so")
    cmd = [gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
           "-I", os.path.join(ROOT, "tests", "host_shim"), os.path.join(ROOT, "tests", "host_arith.cpp"), "-o", out]
    subprocess.check_call(cmd)
    lib = ctypes.CDLL(out)
    lib.host_scores.restype = ctypes.c_int
    return lib


def _aten(kind, q, c):
    """(nq, nc) scores with the reference's tensor ops; q: (nq, QW, d), c: (nc, CW, d)."""
    nq, nc, d = q.shape[0], c.shape[0], q.shape[2]
    q0, q1 = q[:, 0].view(nq, 1, d), q[:, -1].view(nq, 1, d)
    c0, c1 = c[:, 0].view(1, nc, d).expand(nq, nc, d), c[:, -1].view(1, nc, d).expand(nq, nc, d)
    if kind == "dot1":
        return (q0 * c0).sum(dim=2)
    if kind == "dot2":
        return (q0 * c0 + q1 * c1).sum(dim=2)
    if kind == "dot3":       # Analogy, bilinear.py:695-698: scalar, real, imaginary planes
        qm, cm = q[:, 1].view(nq, 1, d), c[:, 1].view(1, nc, d).expand(nq, nc, d)
        return (q0 * c0 + qm * cm + q1 * c1).sum(dim=2)
    if kind == "dot_mid":
        return ((q0 * c0) * q1).sum(dim=2)
    if kind == "rot":
        return -torch.stack([q0 - c0, q1 - c1], dim=0).norm(dim=0).sum(dim=2)
    x = (q0 - c0) if kind.endswith("tail") else ((c0 + q0) - q1)
    if kind.startswith("l1"):
        return -x.norm(p=1, dim=-1)
    if kind.startswith("l2"):
        return -(x.norm(p=2, dim=-1) ** 2)
    if kind.startswith("tl1"):
        return -(2 * torch.min(torch.abs(x), 1 - torch.abs(x)).sum(dim=-1))
    return -(4 * torch.min(x ** 2, 1 - x ** 2).sum(dim=-1))


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("d", [1, 7, 8, 13, 50, 64, 200, 203, 520, 1001, 1024, 2049, 4095, 4096, 8191])
def test_device_arithmetic_equals_aten(kind, d, host_lib):
    el, model, qw, cw = KINDS[kind]
    g = torch.Generator().manual_seed(1000 * el + d)
    nq, nc = 3, 6
    scale = 1.0 if not kind.startswith("tl") else 3.0      # torus kinds: values beyond one period
    q = (torch.rand(nq, qw, d, generator=g) * 2 - 1) * scale
    c = (torch.rand(nc, cw, d, generator=g) * 2 - 1) * scale
    c[1] = c[0]                                            # exact ties
    c[2] = 0.0
    want = _aten(kind, q, c)
    perm, code = _lib.build_schedule(model, d)
    casc = int(bool((code & 0x04).any()))                  # SC_CASC1 present
    qn, cn = q.numpy().copy(), c.numpy().copy()
    P = ctypes.c_void_p
    for mode in (0, 1):
        if mode == 1 and kind.startswith("l1"):
            continue                                       # sequential norm: replay only
        out = np.full((nq, nc), np.nan, dtype=np.float32)
        rc = host_lib.host_scores(el, mode, casc, d, nq, nc, P(qn.ctypes.data), P(cn.ctypes.data),
                                  P(perm.ctypes.data), P(code.ctypes.data), P(out.ctypes.data))
        assert rc == 0
        got = torch.from_numpy(out)
        same = (got.view(torch.int32) == want.contiguous().view(torch.int32)) | (got == want)
        assert same.all(), "%s d=%d mode=%d: %d of %d scores differ" % (kind, d, mode, int((~same).sum()), same.numel())


#: the head side sums K-blocks of 384 while more than 768 terms remain, then two chains: dims at
#: and around every block boundary up to the library's limit
RESCAL_PREP_DIMS = [1, 2, 7, 13, 16, 19, 20, 21, 31, 32, 33, 50, 64, 100, 129, 200, 203, 256, 300, 384, 385,
                    400, 512, 767, 768, 769, 770, 1000, 1151, 1152, 1153, 1535, 1536, 1537, 1919, 2048, 2049,
                    3000, 4096, 8191]


@pytest.mark.parametrize("d", RESCAL_PREP_DIMS)
def test_rescal_query_preparation_equals_the_reference_matmul(d, host_lib):
    """`matmul(h.view(b, 1, d), M)` and `matmul(M, t.view(b, d, 1))` (bilinear.py:108, 113) against
    the device function the prep kernel is made of -- bit for bit.  This pins the oneMKL / ATen
    summation order the kernel replays (batches of >= 2 facts: a batch of one takes MKL's gemv path,
    whose order depends on memory alignment)."""
    g = torch.Generator().manual_seed(d)
    b = 3 if d <= 4096 else 2            # d = 8191: 2 x 268 MB of matrices
    v = torch.randn(b, d, generator=g)
    M = torch.randn(b, d, d, generator=g)
    v[1, : d // 2] = 0.0
    want_tail = torch.matmul(v.view(b, 1, d), M).view(b, d)
    want_head = torch.matmul(M, v.view(b, d, 1)).view(b, d)
    vn, Mn = v.numpy(), M.numpy()        # contiguous views: no second copy of the matrices
    P = ctypes.c_void_p
    for tail, want in ((1, want_tail), (0, want_head)):
        out = np.full((b, d), np.nan, dtype=np.float32)
        assert host_lib.host_rescal_prep(tail, d, b, P(vn.ctypes.data), P(Mn.ctypes.data), P(out.ctypes.data)) == 0
        got = torch.from_numpy(out)
        same = (got.view(torch.int32) == want.contiguous().view(torch.int32)) | (got == want)
        assert same.all(), "rescal %s d=%d: %d of %d components differ" % (
            "tail" if tail else "head", d, int((~same).sum()), same.numel())
