"""rank_link_prediction on the CUDA engine where it leaves its usual single call over the whole
table: a near-tie list that overflows and the exact recomputation behind it (LazyRanks), facts split
over several calls (CSR cuts, the rebased row ids of a three-array CSR, one stats row per call), and
entity row ranges scanned separately (what the ranks of an EntityShard group do), filter pass
included.  Ranks are compared with the CPU oracle, and each test asserts that its path ran."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200 import engine as engine_mod
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import CudaEngine, ModelSpec, rank_link_prediction

pytestmark = pytest.mark.gpu


def _entity_planes(model):
    return [getattr(model, n).weight for n in ("ent_emb", "sc_ent_emb", "re_ent_emb", "im_ent_emb")
            if hasattr(model, n)]


def _assert_ranks(got, want):
    """got, want: (rank_heads, rank_tails, filt_rank_heads, filt_rank_tails)"""
    names = ("rank_heads", "rank_tails", "filt_rank_heads", "filt_rank_tails")
    for name, a, b in zip(names, got, want):
        a, b = a.cpu(), b.cpu()
        bad = (a != b).nonzero().flatten()
        assert bad.numel() == 0, "%s: %d / %d ranks differ, first at %d: got %d want %d" % (
            name, bad.numel(), b.numel(), bad[0], a[bad[0]], b[bad[0]])


def _device_csrs(dh, dt, h, t, r, dev):
    ft = tuple(x.to(dev) for x in filter_csr(dt, h, r, t))
    fh = tuple(x.to(dev) for x in filter_csr(dh, t, r, h))
    return ft, fh


# ------------------------------------------------------------------ near-tie list overflow
@pytest.mark.parametrize("kind", ["distmult", "transe_l2", "complex", "rotate"])
def test_near_tie_overflow_falls_back_to_exact_ranks(kind, cuda_device, monkeypatch):
    """Every entity row is the same row, so every (query, entity) pair is a near tie of the
    bound-and-refine scan (tensor cores; RotatE: its approximate fp32 scan): 128 x 2,000 pairs per
    query tile against room for 8,192.  The call reports found = capacity + 1, the ranks are
    recomputed on the exact scan with a RuntimeWarning, and equal the oracle's."""
    n_ent, n_rel, d = 2000, 5, 24
    kg, dh, dt = helpers.make_kg(n_ent, n_rel, n_facts=3000, n_test=300, seed=4)
    assert kg.n_facts == 300
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=4)
    with torch.no_grad():
        for w in _entity_planes(model):
            w[:] = w[7].clone()
        assert all(w[7].abs().min() > 0 for w in _entity_planes(model))
    model = model.to(cuda_device)
    P = helpers.oracle_params(kind, model)
    ref = oracle.link_prediction(kind, P, kg.head_idx, kg.tail_idx, kg.relations, dh, dt, b_size=100)
    eng = CudaEngine(tensor_core=True)
    monkeypatch.setattr(engine_mod, "_default_engine", eng)

    ev = tk.LinkPredictionEvaluator(model, kg)
    with pytest.warns(RuntimeWarning, match="overflowed"):
        ev.evaluate(b_size=64, verbose=False)
    _assert_ranks((ev.rank_true_heads, ev.rank_true_tails, ev.filt_rank_true_heads, ev.filt_rank_true_tails), ref)

    eng.tc_stats.clear()
    h, t, r = (x.to(cuda_device) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    ft, fh = _device_csrs(dh, dt, kg.head_idx, kg.tail_idx, kg.relations, cuda_device)
    lazy = rank_link_prediction(ModelSpec.from_model(model), h, t, r, ft, fh, engine=eng, sync=False)
    assert int(lazy.overflow) > 0
    stats = [s.tolist() for s in eng.tc_stats]
    assert len(stats) == 2 and all(found == cap + 1 for found, cap in stats), stats
    with pytest.warns(RuntimeWarning, match="overflowed"):
        ranks = lazy.get()
    _assert_ranks(ranks, ref)


# ------------------------------------------------------------------ several calls
@pytest.mark.parametrize("filters", ["filter_csr", "filter_index"])
@pytest.mark.parametrize("tensor_core", [True, False], ids=["bound_and_refine", "exact_scan"])
@pytest.mark.parametrize("kind", ["transe_l2", "distmult", "complex", "rotate"])
def test_several_calls_equal_one(kind, tensor_core, filters, cuda_device):
    """530 facts in calls of 200, 200 and 130 (not multiples of the 64- or 128-query tiles): the
    filter CSRs are cut per call -- with the row-id array rebased when the CSR has one
    (FilterIndex.csr) -- and the ranks equal those of a single call and the oracle's."""
    n_ent, n_rel, d, n = 1500, 9, 32, 530
    h, t, r = helpers.random_graph(n_ent, n_rel, 6000, seed=8)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    th, tt, tr = h[:n], t[:n], r[:n]
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=8)
    with torch.no_grad():
        for w in _entity_planes(model):
            w[700:760] = w[0:60]                    # exact ties
    model = model.to(cuda_device)
    P = helpers.oracle_params(kind, model)
    ref = oracle.link_prediction(kind, P, th, tt, tr, dh, dt, b_size=128)
    h_d, t_d, r_d = (x.to(cuda_device) for x in (th, tt, tr))
    if filters == "filter_csr":
        ft, fh = _device_csrs(dh, dt, th, tt, tr, cuda_device)
        assert len(ft) == len(fh) == 2
    else:
        kg = tk.KnowledgeGraph(th, tt, tr, n_ent, n_rel, filter_facts=(h, t, r))
        ft = kg.filter_index.csr("tail", h_d, r_d, t_d)
        fh = kg.filter_index.csr("head", t_d, r_d, h_d)
        assert len(ft) == len(fh) == 3
    for f in (ft, fh):   # every call has entries to discount
        assert all(int(f[0][hi]) > int(f[0][lo]) for lo, hi in ((0, 200), (200, 400), (400, n)))
    spec = ModelSpec.from_model(model)
    eng = CudaEngine(tensor_core=tensor_core)
    several = rank_link_prediction(spec, h_d, t_d, r_d, ft, fh, engine=eng, chunk=200)
    stats = [s.tolist() for s in eng.tc_stats]
    # bound-and-refine (tensor cores; RotatE: approximate scan): one stats row per call and side,
    # none overflowed (no exact recomputation behind the result)
    assert len(stats) == (6 if tensor_core else 0)
    assert all(found <= cap for found, cap in stats), stats
    one = rank_link_prediction(spec, h_d, t_d, r_d, ft, fh, engine=eng)
    _assert_ranks(several, one)
    _assert_ranks(several, ref)


# ------------------------------------------------------------------ entity row ranges
@pytest.mark.parametrize("tensor_core", [True, False], ids=["tensor_core", "exact_scan"])
@pytest.mark.parametrize("kind", ["transe_l2", "distmult", "complex", "analogy"])
def test_entity_row_ranges_add_up(kind, tensor_core, cuda_device):
    """Three row ranges of the table ([0, 389), [389, 1201), [1201, 2000): no bound a multiple of 32,
    128 or 256) scanned separately, each with its filter pass (ent_lo != 0 for two of them), as the
    ranks of an EntityShard group do: the summed counters give the ranks of the whole table, which
    equal the oracle's.  Extends test_analogy_gpu.py::test_entity_sharded_counts_add_up (two ranges,
    exact scan) to the tensor-core scan and to the other kinds that have one."""
    n_ent, n_rel, d = 2000, 5, 48
    kg, dh, dt = helpers.make_kg(n_ent, n_rel, n_facts=8000, n_test=300, seed=3)
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=3)
    with torch.no_grad():
        for w in _entity_planes(model):
            w[1300:1340] = w[300:340]               # exact ties across the ranges
    model = model.to(cuda_device)
    spec = ModelSpec.from_model(model)
    h, t, r = (x.to(cuda_device) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    ft, fh = _device_csrs(dh, dt, kg.head_idx, kg.tail_idx, kg.relations, cuda_device)
    eng = CudaEngine(tensor_core=tensor_core)
    whole = rank_link_prediction(spec, h, t, r, ft, fh, engine=eng)
    eng.tc_stats.clear()
    n = h.shape[0]
    counters = torch.zeros((4, n), dtype=torch.int32, device=cuda_device)
    hrows, trows = eng.gather_rows(spec, h), eng.gather_rows(spec, t)
    keep = []
    for lo, hi in ((0, 389), (389, 1201), (1201, n_ent)):
        part = spec.narrowed(lo, hi)
        assert part.ent_lo == lo and part.n_rows == hi - lo
        # filter entries inside this range: the filter pass has work with this ent_lo
        assert any(((f[1] >= lo) & (f[1] < hi)).any() for f in (ft, fh))
        if tensor_core:
            img = eng.pack_tc(part)
            assert img is not None
            args = dict(tc_packed=img)
            packed = None
        else:
            packed = eng.pack(part)
            args = {}
        keep.append(eng.rank_side(part, packed, 0, hrows, trows, r, t, ft, counters[0], counters[1], **args))
        keep.append(eng.rank_side(part, packed, 1, hrows, trows, r, h, fh, counters[2], counters[3], **args))
    stats = [s.tolist() for s in eng.tc_stats]
    assert len(stats) == (6 if tensor_core else 0)
    assert all(found <= cap for found, cap in stats), stats
    rank_t, filt_t = eng.finalize(counters[0], counters[1])
    rank_h, filt_h = eng.finalize(counters[2], counters[3])
    _assert_ranks((rank_h, rank_t, filt_h, filt_t), whole)
    P = helpers.oracle_params(kind, model)
    ref = oracle.link_prediction(kind, P, kg.head_idx, kg.tail_idx, kg.relations, dh, dt, b_size=100)
    _assert_ranks(whole, ref)
