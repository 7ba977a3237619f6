"""Large embedding dims, up to the library's limit (dim <= 8191, csrc/kernels.h: SCAN_MAX_DIM): ranks,
dense scores and top-k lists against the CPU oracle on every scan path.

At these dims the scan runs up to 256 schedule stages, the tensor-core path streams K up to 3 x 8191
(Analogy) in k-blocks of 32 or 64, and RESCAL's head-side query preparation `M_r t` leaves its
two-chain form for oneMKL's K-blocking (csrc/reduce.cuh: rescal_query_component).  Tables are small
(300 entities, not a multiple of the 128-row candidate tile) so that the oracle stays cheap; 100 test
facts split the second 64-query tile; duplicate and zero rows send exact ties through the recheck and
filter kernels, near-copies of frequent test entities make ranks depend on the last bits of scores.  The oracle runs in batches of 24 facts: never a batch of one, whose RESCAL matmul
takes another MKL path in the reference (DESIGN.md 2.4)."""
import ctypes

import pytest
import torch

from oracle import kge_oracle as oracle
from tests import helpers
from tests.test_tc_gpu import _kernel_bound, _operands, _prefix_factor
from tests.test_topk_gpu import assert_topk, expected_topk
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import CudaEngine, ModelSpec, rank_link_prediction

pytestmark = pytest.mark.gpu

N_ENT, N_REL, N_FACTS, N_TEST, B_SIZE = 300, 3, 1200, 100, 24
WIDTHS = [2049, 4096, 8191]                     # plane widths (Analogy: three planes of this width)
RESCAL_DIMS = [769, 1000, 1537]                 # three, four and five K-blocks of M_r t
TC_KINDS = ["transe_l2", "distmult", "complex", "analogy"]
OTHER_KINDS = ["transe_l1", "rotate", "toruse_l2"]
TOPK = 40


def _emb_dim(kind, w):
    return 2 * w if kind == "analogy" else w    # Analogy: scalar and complex halves of emb_dim


_CASES = {}


def _case(kind, w, device):
    """Model on the device, its tables for the oracle, the test graph and the oracle's dense scores
    and ranks; built once per (kind, width) for the whole module."""
    key = (kind, w)
    if key in _CASES:
        return _CASES[key]
    kg, dh, dt = helpers.make_kg(N_ENT, N_REL, n_facts=N_FACTS, n_test=N_TEST, seed=w)
    assert kg.head_idx.shape[0] == N_TEST and N_TEST % B_SIZE != 1
    model = helpers.make_model(kind, _emb_dim(kind, w), N_ENT, N_REL, seed=w)
    g = torch.Generator().manual_seed(w)
    with torch.no_grad():
        for emb in [m for n, m in model.named_children() if "ent" in n]:
            x = emb.weight
            x[150:170] = x[10:30]                        # duplicate rows: exact ties
            # near-copies of the most frequent test entities (random half of the elements one ulp
            # off): scores within rounding noise of the true one, so a rank moves whenever a query
            # vector is off in its last bits
            src = x[0:40].clone()
            away = torch.where(torch.rand(src.shape, generator=g) < 0.5, -1.0, 1.0) * float("inf")
            x[170:210] = torch.where(torch.rand(src.shape, generator=g) < 0.5, torch.nextafter(src, away), src)
            x[285:] = 0.0                                # zero rows: many equal scores
    model = model.to(device)
    P = helpers.oracle_params(kind, model)
    h, t, r = kg.head_idx, kg.tail_idx, kg.relations
    dense = {}
    for side in ("tail", "head"):
        dense[side] = torch.cat([oracle.scores_all(kind, P, h[lo:lo + B_SIZE], t[lo:lo + B_SIZE],
                                                   r[lo:lo + B_SIZE], side)
                                 for lo in range(0, N_TEST, B_SIZE)])
    # oracle.link_prediction on the same scores (filtered_scores + rank_of_true are row-wise)
    ref = (oracle.rank_of_true(dense["head"], h),
           oracle.rank_of_true(dense["tail"], t),
           oracle.rank_of_true(oracle.filtered_scores(dense["head"], dh, t, r, h), h),
           oracle.rank_of_true(oracle.filtered_scores(dense["tail"], dt, h, r, t), t))
    _CASES[key] = c = dict(model=model, kg=kg, dh=dh, dt=dt, dense=dense, ref=ref)
    return c


def _gpu_ranks(c, eng, exact=False):
    dev = next(c["model"].parameters()).device
    kg = c["kg"]
    csr_t = tuple(x.to(dev) for x in filter_csr(c["dt"], kg.head_idx, kg.relations, kg.tail_idx))
    csr_h = tuple(x.to(dev) for x in filter_csr(c["dh"], kg.tail_idx, kg.relations, kg.head_idx))
    got = rank_link_prediction(ModelSpec.from_model(c["model"]), kg.head_idx.to(dev), kg.tail_idx.to(dev),
                               kg.relations.to(dev), csr_t, csr_h, engine=eng, exact=exact)
    torch.cuda.synchronize()
    return got


def _assert_ranks(got, ref, what):
    names = ["rank_true_heads", "rank_true_tails", "filt_rank_true_heads", "filt_rank_true_tails"]
    for name, a, b in zip(names, got, ref):
        a = a.cpu()
        bad = (a != b).nonzero().flatten()
        assert bad.numel() == 0, "%s %s: %d / %d ranks differ, first at %d: got %d want %d" % (
            what, name, bad.numel(), b.numel(), bad[0], a[bad[0]], b[bad[0]])


def _assert_refined(eng):
    """Both sides went through bound-and-refine, and neither near-tie list overflowed (an overflow
    would silently redo the ranks on the exact scan)."""
    assert len(eng.tc_stats) == 2
    for s in eng.tc_stats:
        found, cap = (int(x) for x in s.cpu())
        assert found <= cap


@pytest.fixture
def tc_layout():
    """Sets (bk, fp16) of the tensor-core scan; the layout in force before is restored afterwards."""
    lid = _lib.load().kge_tc_layout_id()
    yield lambda bk, fp16: _lib.tc_configure(bk=bk, fp16=fp16)
    _lib.tc_configure(bk=lid // 2, fp16=lid % 2)


def _needs_reference_mkl_order(d):
    if not helpers.rescal_order_matches_here(d):
        pytest.skip("oneMKL on this CPU sums RESCAL's batched matmul in another order than the machine "
                    "the golden fixtures come from: the reference's own bits differ here")


# ------------------------------------------------------------------ ranks
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("kind", TC_KINDS + OTHER_KINDS)
def test_exact_scan_ranks_equal_oracle(kind, w, cuda_device):
    c = _case(kind, w, cuda_device)
    _assert_ranks(_gpu_ranks(c, CudaEngine(tensor_core=False), exact=True), c["ref"], "%s w=%d exact" % (kind, w))


@pytest.mark.parametrize("bk", [32, 64])
@pytest.mark.parametrize("fp16", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("kind", TC_KINDS)
def test_tensor_core_ranks_equal_oracle(kind, w, fp16, bk, cuda_device, tc_layout):
    c = _case(kind, w, cuda_device)
    tc_layout(bk, fp16)
    eng = CudaEngine(tensor_core=True)
    got = _gpu_ranks(c, eng)
    _assert_refined(eng)
    _assert_ranks(got, c["ref"], "%s w=%d tensor cores bk=%d fp16=%d" % (kind, w, bk, fp16))


@pytest.mark.parametrize("w", WIDTHS)
def test_rotate_approximate_scan_ranks_equal_oracle(w, cuda_device):
    c = _case("rotate", w, cuda_device)
    eng = CudaEngine(tensor_core=True)            # RotatE: bound-and-refine on the fp32 pipes
    got = _gpu_ranks(c, eng)
    _assert_refined(eng)
    _assert_ranks(got, c["ref"], "rotate w=%d approximate scan" % w)


# ------------------------------------------------------------------ dense scores and top-k
def _rows(c):
    model = c["model"]
    dev = next(model.parameters()).device
    kg = c["kg"]
    eng = CudaEngine(tensor_core=False)
    spec = ModelSpec.from_model(model)
    h, t, r = kg.head_idx.to(dev), kg.tail_idx.to(dev), kg.relations.to(dev)
    return eng, spec, eng.pack(spec), eng.gather_rows(spec, h), eng.gather_rows(spec, t), r


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("kind", TC_KINDS + OTHER_KINDS)
def test_dense_scores_bit_equal_oracle(kind, w, cuda_device):
    c = _case(kind, w, cuda_device)
    eng, spec, packed, hrows, trows, r = _rows(c)
    for side, name in ((_lib.SIDE_TAIL, "tail"), (_lib.SIDE_HEAD, "head")):
        got = eng.score_all(spec, packed, side, hrows, trows, r).cpu()
        want = c["dense"][name]
        same = helpers.bits_equal(got, want)
        assert same.all(), "%s w=%d %s: %d of %d scores differ in bits (max abs diff %g)" % (
            kind, w, name, (~same).sum(), same.size, (got - want).abs().max())


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("kind", TC_KINDS + OTHER_KINDS)
def test_topk_equals_stable_sort_of_oracle_scores(kind, w, cuda_device):
    """The collect epilogue: the TOPK best ids (ties by ascending id, so the duplicate and zero rows
    are ordered) and the bits of their scores."""
    c = _case(kind, w, cuda_device)
    eng, spec, packed, hrows, trows, r = _rows(c)
    for side, name in ((_lib.SIDE_TAIL, "tail"), (_lib.SIDE_HEAD, "head")):
        pred, vals = eng.topk_side(spec, packed, side, hrows, trows, r, TOPK)
        want_ids, want_vals = expected_topk(c["dense"][name], TOPK)
        assert_topk(pred, vals, want_ids, want_vals)


# ------------------------------------------------------------------ RESCAL beyond d = 768
@pytest.mark.parametrize("d", RESCAL_DIMS)
def test_rescal_ranks_equal_oracle_on_both_scans(d, cuda_device, tc_layout):
    """M_r t sums K-blocks of 384 and then two chains (csrc/reduce.cuh: rescal_query_component): the
    exact scan and the tensor-core scan, whose near-ties are re-scored from the same query vectors."""
    _needs_reference_mkl_order(d)
    c = _case("rescal", d, cuda_device)
    _assert_ranks(_gpu_ranks(c, CudaEngine(tensor_core=False), exact=True), c["ref"], "rescal d=%d exact" % d)
    for fp16 in (0, 1):
        tc_layout(32, fp16)
        eng = CudaEngine(tensor_core=True)
        got = _gpu_ranks(c, eng)
        _assert_refined(eng)
        _assert_ranks(got, c["ref"], "rescal d=%d tensor cores fp16=%d" % (d, fp16))


@pytest.mark.parametrize("d", RESCAL_DIMS)
def test_rescal_dense_scores_bit_equal_oracle(d, cuda_device):
    _needs_reference_mkl_order(d)
    c = _case("rescal", d, cuda_device)
    eng, spec, packed, hrows, trows, r = _rows(c)
    for side, name in ((_lib.SIDE_TAIL, "tail"), (_lib.SIDE_HEAD, "head")):
        got = eng.score_all(spec, packed, side, hrows, trows, r).cpu()
        same = helpers.bits_equal(got, c["dense"][name])
        assert same.all(), "rescal d=%d %s: %d of %d scores differ in bits" % (d, name, (~same).sum(), same.size)


# ------------------------------------------------------------------ the error bound at large K
@pytest.mark.parametrize("fp16", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("shape", ["normalised", "same_sign"])
@pytest.mark.parametrize("kind,d", [("distmult", 8191), ("complex", 4096)])
def test_error_bound_holds_at_large_k(kind, d, shape, fp16, cuda_device, tc_layout):
    """|tensor-core score - reference fp32 score| <= the kernel's bound, pair by pair, at K = 8191
    and 8192: kappa grows with sqrt(K) and the running-magnitude factor with K (the same check as
    tests/test_tc_gpu.py at K <= 1024)."""
    tc_layout(32, fp16)
    g = torch.Generator().manual_seed(2000 + d)
    n_q, n_c = 70, 520
    dev = cuda_device
    if kind == "complex":
        a0, b0 = _operands(shape, n_q, n_c, d, g)
        a1, b1 = _operands(shape, n_q, n_c, d, g)
        ent0, ent1 = torch.cat([b0, a0]), torch.cat([b1, a1])
        P = {"re_ent": ent0, "im_ent": ent1, "re_rel": torch.ones(1, d), "im_rel": torch.zeros(1, d)}
        spec = ModelSpec(_lib.COMPLEX, d, n_c, 1, ent0[:n_c].contiguous().to(dev), ent1[:n_c].contiguous().to(dev),
                         P["re_rel"].to(dev), P["im_rel"].to(dev))
        hrows = torch.stack([a0, a1], 1).contiguous().to(dev)        # q = h o (1 + 0i) = h
        qv, cv = torch.cat([a0, a1], 1).double(), torch.cat([b0, b1], 1).double()
        k_total = 2 * d
    else:
        a, b = _operands(shape, n_q, n_c, d, g)
        ent = torch.cat([b, a])
        P = {"ent": ent, "rel": torch.ones(1, d)}                     # q = h * 1 = h
        spec = ModelSpec(_lib.DISTMULT, d, n_c, 1, ent[:n_c].contiguous().to(dev), None, P["rel"].to(dev), None)
        hrows = a.view(n_q, 1, d).contiguous().to(dev)
        qv, cv = a.double(), b.double()
        k_total = d
    h_idx = torch.arange(n_c, n_c + n_q)
    r_idx = torch.zeros(n_q, dtype=torch.int64)
    want = torch.cat([oracle.scores_all(kind, P, h_idx[lo:lo + 10], h_idx[lo:lo + 10], r_idx[lo:lo + 10],
                                        "tail")[:, :n_c] for lo in range(0, n_q, 10)]).double()
    eng = CudaEngine(tensor_core=True)
    tcp = eng.pack_tc(spec)
    dump = torch.full((n_q, n_c), float("nan"), device=dev)
    raw = torch.zeros(n_q, dtype=torch.int32, device=dev)
    eng.rank_side(spec, None, _lib.SIDE_TAIL, hrows, hrows, r_idx.to(dev), r_idx.to(dev), None, raw,
                  torch.zeros_like(raw), tc_packed=tcp, tc_dump=dump)
    torch.cuda.synchronize()
    got = dump.cpu().double()
    assert torch.isfinite(got).all()
    na, nb = qv.norm(dim=1).view(-1, 1), cv.norm(dim=1).view(1, -1)
    bound = _kernel_bound(spec.code, d, k_total, na, nb, qv.abs().max().item(), cv.abs().max().item(),
                          (cv ** 2).sum(1).max().item(), False, _prefix_factor(qv, k_total).view(-1, 1),
                          _prefix_factor(cv, k_total).view(1, -1))
    ratio = ((got - want).abs() / bound).max().item()
    assert ratio <= 1.0, "%s %s d=%d fp16=%d: error / bound = %.3f" % (kind, shape, d, fp16, ratio)
    print("tc bound %s %s d=%d fp16=%d: max error / bound = %.3f" % (kind, shape, d, fp16, ratio))


# ------------------------------------------------------------------ the limit
def test_dim_8191_is_the_limit_of_every_scan_entry_point(cuda_device):
    """dim = 8191 is accepted and dim = 8192 answered with KGE_ERR_UNSUPPORTED by kge_rank_side,
    kge_score_all, kge_topk_side, kge_pack_table and kge_tc_pack_table.  Every buffer is sized for
    the call at 8192, so that a call that wrongly got past its checks would still stay in bounds."""
    lib = _lib.load()
    dev = cuda_device
    n_rows, k = 130, 8
    P = ctypes.c_void_p
    for dim, want in ((8191, 0), (8192, 3)):
        ent = torch.randn(n_rows, dim, device=dev)
        rel = torch.randn(1, dim, device=dev)
        rows = ent[:1].reshape(1, 1, dim).contiguous()
        r_idx = torch.zeros(1, dtype=torch.int64, device=dev)
        packed = torch.zeros(max(lib.kge_packed_table_floats(_lib.DISTMULT, n_rows, 8192), 1), device=dev)
        tcp = torch.zeros(max(lib.kge_tc_packed_bytes(_lib.DISTMULT, n_rows, 8192), 1), dtype=torch.uint8, device=dev)
        got = {"kge_pack_table": lib.kge_pack_table(_lib.DISTMULT, P(ent.data_ptr()), None, n_rows, dim,
                                                    P(packed.data_ptr()), None)}
        torch.cuda.synchronize()
        got["kge_tc_pack_table"] = lib.kge_tc_pack_table(_lib.DISTMULT, P(ent.data_ptr()), None, n_rows, dim,
                                                         P(tcp.data_ptr()), None)
        torch.cuda.synchronize()
        ws = torch.zeros(max(lib.kge_rank_workspace_bytes(_lib.DISTMULT, _lib.SIDE_TAIL, 8192, 1, n_rows, 0),
                             lib.kge_topk_workspace_bytes(_lib.DISTMULT, _lib.SIDE_TAIL, 8192, 1, n_rows, k)),
                         dtype=torch.uint8, device=dev)
        raw, sub = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        a = _lib.RankArgs()
        a.model, a.side, a.dim, a.n, a.n_ent, a.n_rows = _lib.DISTMULT, _lib.SIDE_TAIL, dim, 1, n_rows, n_rows
        a.packed, a.ent0, a.rel0 = packed.data_ptr(), ent.data_ptr(), rel.data_ptr()
        a.hrows, a.trows, a.r_idx, a.true_idx = rows.data_ptr(), rows.data_ptr(), r_idx.data_ptr(), r_idx.data_ptr()
        a.raw_count, a.filt_sub = raw.data_ptr(), sub.data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        got["kge_rank_side"] = lib.kge_rank_side(ctypes.byref(a))
        torch.cuda.synchronize()
        scores = torch.zeros(1, n_rows, device=dev)
        s = _lib.ScoreAllArgs()
        s.model, s.side, s.dim, s.n, s.n_rows = _lib.DISTMULT, _lib.SIDE_TAIL, dim, 1, n_rows
        s.packed, s.rel0, s.hrows, s.trows, s.r_idx = (packed.data_ptr(), rel.data_ptr(), rows.data_ptr(),
                                                       rows.data_ptr(), r_idx.data_ptr())
        s.scores, s.workspace, s.workspace_bytes = scores.data_ptr(), ws.data_ptr(), ws.numel()
        got["kge_score_all"] = lib.kge_score_all(ctypes.byref(s))
        torch.cuda.synchronize()
        pred, vals = torch.zeros(1, k, dtype=torch.int64, device=dev), torch.zeros(1, k, device=dev)
        t = _lib.TopkArgs()
        t.model, t.side, t.dim, t.k, t.n, t.n_rows = _lib.DISTMULT, _lib.SIDE_TAIL, dim, k, 1, n_rows
        t.packed, t.rel0, t.hrows, t.trows, t.r_idx = (packed.data_ptr(), rel.data_ptr(), rows.data_ptr(),
                                                       rows.data_ptr(), r_idx.data_ptr())
        t.pred, t.scores, t.workspace, t.workspace_bytes = pred.data_ptr(), vals.data_ptr(), ws.data_ptr(), ws.numel()
        got["kge_topk_side"] = lib.kge_topk_side(ctypes.byref(t))
        torch.cuda.synchronize()
        assert got == {name: want for name in got}, "dim %d: %s (%s)" % (dim, got, lib.kge_last_error())
