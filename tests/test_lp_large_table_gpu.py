"""Link prediction on a table with more than twice as many candidate tiles as the GPU has SMs:
ranks, dense scores and top-k lists against the CPU oracle.

The scalar scan (csrc/scan.cu: scan_kernel) is persistent.  launch_one starts min(n_qt * n_ct, SMs)
CTAs, and each CTA walks the (query tile, candidate tile) pairs tile = blockIdx.x + i * gridDim.x,
qt = tile / n_ct.  Three pieces of per-thread state change only when qt changes: the counters cnt[]
(flushed into the rank counters then), the true scores st[] (the collect epilogue's k-th best
thresholds) and RotatE's approximate-scan thresholds.  Between two tiles of one query tile they are
carried, and so is the ring's stage / phase.  A CTA meets two tiles of one query tile in a row only
when n_ct > SMs, that is past 132 x 128 = 16,896 entities on a 132-SM H100: every real dataset past
FB15k, but none of the other rank tests, whose tables stay below 10,000 entities.

Here n_ent = 50,001 gives n_ct = 391 = 2 x 132 + 127: each CTA walks two or three candidate tiles of
one query tile and then crosses into the next query tile mid-walk; the last candidate tile holds 81
rows.  Every test asserts n_ct >= 2 x SMs + 1, so that on a GPU with more SMs it fails instead of
silently losing that path.  260 test facts make five 64-query tiles, the last one partial.  The
entity planes hold exact copies of the first candidate tile SMs tiles further on (the same CTA scans
both for one query tile), one-ulp near-copies of the most frequent test entities 2 x SMs tiles on
(a CTA's third tile), and zero rows in the partial last tile; filter sets reach past row 16,896.
The oracle runs in batches of 24 facts, never one (DESIGN.md 2.4)."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from tests.test_topk_gpu import assert_topk, collect_passes, expected_topk, topk_chunk_rows
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import CudaEngine, ModelSpec, rank_link_prediction

pytestmark = pytest.mark.gpu

N_ENT, N_REL, N_FACTS, N_TEST, B_SIZE = 50_001, 5, 40_000, 260, 24
N_CT = -(-N_ENT // _lib.TILE_C)
#: 40: two 32-position stages of the scan's ring, the second partial, so that the ring wraps inside a
#: tile and across tiles.  Analogy: emb_dim, three planes of 6
DIMS = {"transe_l1": 40, "transe_l2": 40, "distmult": 40, "toruse_l1": 40, "toruse_l2": 40,
        "complex": 16, "rotate": 16, "rescal": 12, "analogy": 12}
KINDS = list(DIMS)
TC_KINDS = ["transe_l2", "distmult", "rescal", "complex", "analogy"]
TOPK = 50
#: the top-k queries are the test facts repeated: 1,300 queries split the table into two collect
#: passes, so that the second pass scans against real k-th best thresholds (st[] of the collect epilogue)
TOPK_REPEAT = 5
RANGES = ((0, 20_011), (20_011, N_ENT))     # row ranges of more than 16,896 rows, ent_lo not a multiple of 128


def _sms(device):
    return torch.cuda.get_device_properties(device).multi_processor_count


_CASES = {}


def _case(kind, device):
    """Model on the device, the test graph, its filter CSRs and the oracle's dense scores and ranks;
    built once per kind for the whole module."""
    if kind in _CASES:
        return _CASES[kind]
    sms = _sms(device)
    assert N_CT >= 2 * sms + 1, (
        "%d candidate tiles against %d SMs: no CTA would scan three candidate tiles of one query tile"
        % (N_CT, sms))
    d = DIMS[kind]
    if kind == "rescal" and not helpers.rescal_order_matches_here(d):
        pytest.skip("oneMKL on this CPU sums RESCAL's batched matmul in another order than the machine "
                    "the golden fixtures come from: the reference's own bits differ here")
    kg, dh, dt = helpers.make_kg(N_ENT, N_REL, n_facts=N_FACTS, n_test=N_TEST, seed=17)
    assert kg.n_facts == N_TEST and N_TEST % B_SIZE != 1 and -(-N_TEST // _lib.TILE_Q) == 5
    model = helpers.make_model(kind, d, N_ENT, N_REL, seed=17)
    tie = sms * _lib.TILE_C         # tiles ct and ct + sms of one query tile go to the same CTA
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for emb in [m for n, m in model.named_children() if "ent" in n]:
            x = emb.weight
            x[tie:tie + 128] = x[0:128]                  # exact ties, a whole tile
            src = x[0:64].clone()                        # near-copies: a random half of the elements one ulp off
            away = torch.where(torch.rand(src.shape, generator=g) < 0.5, -1.0, 1.0) * float("inf")
            x[2 * tie:2 * tie + 64] = torch.where(torch.rand(src.shape, generator=g) < 0.5,
                                                  torch.nextafter(src, away), src)
            x[N_ENT - 41:] = 0.0                         # zero rows in the last, 81-row tile
    model = model.to(device)
    P = helpers.oracle_params(kind, model)
    h, t, r = kg.head_idx, kg.tail_idx, kg.relations
    dense = {}
    for side in ("tail", "head"):
        dense[side] = torch.cat([oracle.scores_all(kind, P, h[lo:lo + B_SIZE], t[lo:lo + B_SIZE],
                                                   r[lo:lo + B_SIZE], side)
                                 for lo in range(0, N_TEST, B_SIZE)])
    ref = (oracle.rank_of_true(dense["head"], h),
           oracle.rank_of_true(dense["tail"], t),
           oracle.rank_of_true(oracle.filtered_scores(dense["head"], dh, t, r, h), h),
           oracle.rank_of_true(oracle.filtered_scores(dense["tail"], dt, h, r, t), t))
    csr = {"tail": filter_csr(dt, h, r, t), "head": filter_csr(dh, t, r, h)}
    for side, true in (("tail", t), ("head", h)):
        # filter entries past a CTA's first tile that score at least the true score: the filter pass
        # discounts counts the scan made on such tiles
        offs, ids = csr[side]
        row = torch.repeat_interleave(torch.arange(N_TEST), offs[1:] - offs[:-1])
        s = dense[side]
        far = ids >= tie
        assert (s[row[far], ids[far]] >= s[row[far], true[row[far]]]).any(), side
    _CASES[kind] = c = dict(model=model, kg=kg, dh=dh, dt=dt, csr=csr, dense=dense, ref=ref, sms=sms)
    return c


def _device_csrs(c):
    dev = next(c["model"].parameters()).device
    return tuple(tuple(x.to(dev) for x in c["csr"][side]) for side in ("tail", "head"))


def _gpu_ranks(c, eng, exact=False):
    dev = next(c["model"].parameters()).device
    kg = c["kg"]
    ft, fh = _device_csrs(c)
    got = rank_link_prediction(ModelSpec.from_model(c["model"]), kg.head_idx.to(dev), kg.tail_idx.to(dev),
                               kg.relations.to(dev), ft, fh, engine=eng, exact=exact)
    torch.cuda.synchronize()
    return got


def _assert_ranks(got, ref, what):
    names = ["rank_true_heads", "rank_true_tails", "filt_rank_true_heads", "filt_rank_true_tails"]
    for name, a, b in zip(names, got, ref):
        a = a.cpu()
        bad = (a != b).nonzero().flatten()
        assert bad.numel() == 0, "%s %s: %d / %d ranks differ, first at %d: got %d want %d" % (
            what, name, bad.numel(), b.numel(), bad[0], a[bad[0]], b[bad[0]])


def _assert_refined(eng, calls):
    """One stats row per bound-and-refine call, and no near-tie list overflowed (an overflow would
    silently redo the ranks on the exact scan)."""
    assert len(eng.tc_stats) == calls
    for s in eng.tc_stats:
        found, cap = (int(x) for x in s.cpu())
        assert found <= cap


@pytest.fixture
def tc_layout():
    """Sets (bk, fp16) of the tensor-core scan; the layout in force before is restored afterwards."""
    lid = _lib.load().kge_tc_layout_id()
    yield lambda bk, fp16: _lib.tc_configure(bk=bk, fp16=fp16)
    _lib.tc_configure(bk=lid // 2, fp16=lid % 2)


# ------------------------------------------------------------------ ranks
@pytest.mark.parametrize("kind", KINDS)
def test_exact_scan_ranks_equal_oracle(kind, cuda_device):
    c = _case(kind, cuda_device)
    _assert_ranks(_gpu_ranks(c, CudaEngine(tensor_core=False), exact=True), c["ref"], "%s exact" % kind)


@pytest.mark.parametrize("fp16", [0, 1], ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", TC_KINDS)
def test_tensor_core_ranks_equal_oracle(kind, fp16, cuda_device, tc_layout):
    c = _case(kind, cuda_device)
    tc_layout(32, fp16)
    eng = CudaEngine(tensor_core=True)
    got = _gpu_ranks(c, eng)
    _assert_refined(eng, 2)
    _assert_ranks(got, c["ref"], "%s tensor cores fp16=%d" % (kind, fp16))


def test_rotate_approximate_scan_ranks_equal_oracle(cuda_device):
    """RotatE's default path: the approximate fp32 scan (KGE_FLAG_APPROX_SCAN), whose thresholds are
    set per query tile like st[], and the exact recheck of its near-ties."""
    c = _case("rotate", cuda_device)
    eng = CudaEngine(tensor_core=True)
    got = _gpu_ranks(c, eng)
    _assert_refined(eng, 2)
    _assert_ranks(got, c["ref"], "rotate approximate scan")


# ------------------------------------------------------------------ dense scores and top-k
def _rows(c, repeat=1):
    model = c["model"]
    dev = next(model.parameters()).device
    kg = c["kg"]
    eng = CudaEngine(tensor_core=False)
    spec = ModelSpec.from_model(model)
    h, t, r = (x.repeat(repeat).to(dev) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    return eng, spec, eng.pack(spec), eng.gather_rows(spec, h), eng.gather_rows(spec, t), r


@pytest.mark.parametrize("kind", KINDS)
def test_dense_scores_bit_equal_oracle(kind, cuda_device):
    """The scan with the store epilogue: tells a score error from a counting error in the rank tests."""
    c = _case(kind, cuda_device)
    eng, spec, packed, hrows, trows, r = _rows(c)
    for side, name in ((_lib.SIDE_TAIL, "tail"), (_lib.SIDE_HEAD, "head")):
        got = eng.score_all(spec, packed, side, hrows, trows, r).cpu()
        want = c["dense"][name]
        same = helpers.bits_equal(got, want)
        assert same.all(), "%s %s: %d of %d scores differ in bits (max abs diff %g)" % (
            kind, name, (~same).sum(), same.size, (got - want).abs().max())


@pytest.mark.parametrize("kind", KINDS)
def test_topk_equals_stable_sort_of_oracle_scores(kind, cuda_device):
    """The collect epilogue over two passes, each of more candidate tiles than SMs: the second pass
    keeps what is not below each query's k-th best so far, loaded into st[] per query tile."""
    c = _case(kind, cuda_device)
    n = TOPK_REPEAT * N_TEST
    rows = topk_chunk_rows(n, N_ENT)
    assert collect_passes(n, N_ENT) == 2 and min(rows, N_ENT - rows) > c["sms"] * _lib.TILE_C
    eng, spec, packed, hrows, trows, r = _rows(c, TOPK_REPEAT)
    for side, name in ((_lib.SIDE_TAIL, "tail"), (_lib.SIDE_HEAD, "head")):
        pred, vals = eng.topk_side(spec, packed, side, hrows, trows, r, TOPK)
        want_ids, want_vals = expected_topk(c["dense"][name], TOPK)
        assert_topk(pred, vals, want_ids.repeat(TOPK_REPEAT, 1), want_vals.repeat(TOPK_REPEAT, 1))


# ------------------------------------------------------------------ entity row ranges
@pytest.mark.parametrize("kind,tensor_core", [("transe_l1", False), ("toruse_l2", False), ("distmult", True)])
def test_entity_row_ranges_add_up(kind, tensor_core, cuda_device):
    """Two row ranges scanned separately, each with its filter pass, as the ranks of an EntityShard
    group do: the summed counters give the ranks of the whole table, which equal the oracle's."""
    c = _case(kind, cuda_device)
    dev = cuda_device
    kg = c["kg"]
    spec = ModelSpec.from_model(c["model"])
    h, t, r = (x.to(dev) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    ft, fh = _device_csrs(c)
    eng = CudaEngine(tensor_core=tensor_core)
    whole = rank_link_prediction(spec, h, t, r, ft, fh, engine=eng)
    eng.tc_stats.clear()
    counters = torch.zeros((4, N_TEST), dtype=torch.int32, device=dev)
    hrows, trows = eng.gather_rows(spec, h), eng.gather_rows(spec, t)
    keep = []
    assert RANGES[1][0] % _lib.TILE_C != 0
    for lo, hi in RANGES:
        part = spec.narrowed(lo, hi)
        assert part.ent_lo == lo and part.n_rows == hi - lo
        assert -(-part.n_rows // _lib.TILE_C) > c["sms"]
        # filter entries inside this range: the filter pass has work with this ent_lo
        assert all(((f[1] >= lo) & (f[1] < hi)).any() for f in (ft, fh))
        if tensor_core:
            args = dict(tc_packed=eng.pack_tc(part))
            assert args["tc_packed"] is not None
            packed = None
        else:
            packed = eng.pack(part)
            args = {}
        keep.append(eng.rank_side(part, packed, 0, hrows, trows, r, t, ft, counters[0], counters[1], **args))
        keep.append(eng.rank_side(part, packed, 1, hrows, trows, r, h, fh, counters[2], counters[3], **args))
    _assert_refined(eng, 4 if tensor_core else 0)
    rank_t, filt_t = eng.finalize(counters[0], counters[1])
    rank_h, filt_h = eng.finalize(counters[2], counters[3])
    torch.cuda.synchronize()
    _assert_ranks((rank_h, rank_t, filt_h, filt_t), [x.cpu() for x in whole], "%s row ranges" % kind)
    _assert_ranks(whole, c["ref"], "%s whole table" % kind)


# ------------------------------------------------------------------ public API
def test_evaluator_ranks_equal_oracle(cuda_device):
    """LinkPredictionEvaluator.evaluate: the filter CSRs built from the graph's dictionaries, the
    host chunking and the one device -> host copy on top of the exact scan (TransE-L1 has no other)."""
    c = _case("transe_l1", cuda_device)
    ev = tk.LinkPredictionEvaluator(c["model"], c["kg"])
    ev.evaluate(b_size=64, verbose=False)
    _assert_ranks((ev.rank_true_heads, ev.rank_true_tails, ev.filt_rank_true_heads, ev.filt_rank_true_tails),
                  c["ref"], "transe_l1 LinkPredictionEvaluator")
