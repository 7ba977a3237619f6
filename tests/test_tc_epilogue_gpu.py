"""Threshold epilogue of the tensor-core rank scan (csrc/tc.cu, tc_scan_kernel): ranks must equal
those of the exact scalar scan, and the oracle's, on the inputs that leave the epilogue's hot path --
a last candidate tile of 1 to 255 columns, padding rows of the last query tile, blocks whose pairs
are all exact ties (more near-ties than a warp buffers), NaN and inf operands -- in both operand
formats and in both the resident (k_total <= 224) and the streamed scan geometry."""
import pytest
import torch

from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import CudaEngine, ModelSpec, rank_link_prediction

pytestmark = pytest.mark.gpu

# (kind, d): k_total = d + 3 (TransE-L2), d (DistMult), 2 d (ComplEx); <= 224 keeps the query
# tile's operand image resident in shared memory, > 224 streams it
CASES = [("transe_l2", 200), ("transe_l2", 240), ("distmult", 64), ("distmult", 256), ("complex", 48)]
CASE_IDS = ["%s_d%d" % c for c in CASES]


@pytest.fixture(params=[0, 1], ids=["bf16", "fp16"])
def operand_format(request):
    default = _lib.tc_bound_constants(_lib.DISTMULT, 16)[3]
    _lib.tc_configure(fp16=request.param)
    yield request.param
    _lib.tc_configure(fp16=int(default))


def _entity_planes(model):
    return [getattr(model, n).weight for n in ("ent_emb", "re_ent_emb", "im_ent_emb") if hasattr(model, n)]


def _relation_planes(model):
    return [getattr(model, n).weight for n in ("rel_emb", "re_rel_emb", "im_rel_emb") if hasattr(model, n)]


def _triples(n_ent, n_rel, n_q, seed, heads=None, tails=None):
    g = torch.Generator().manual_seed(seed)
    pick = lambda pool: pool[torch.randint(0, pool.numel(), (n_q,), generator=g)]   # noqa: E731
    h = pick(torch.arange(n_ent) if heads is None else heads)
    t = pick(torch.arange(n_ent) if tails is None else tails)
    r = torch.randint(0, n_rel, (n_q,), generator=g)
    return h, t, r


def _ranks(model, h, t, r, dh, dt, dev, tensor_core):
    eng = CudaEngine(tensor_core=tensor_core)
    spec = ModelSpec.from_model(model)
    csr_t = tuple(x.to(dev) for x in filter_csr(dt, h, r, t))
    csr_h = tuple(x.to(dev) for x in filter_csr(dh, t, r, h))
    got = rank_link_prediction(spec, h.to(dev), t.to(dev), r.to(dev), csr_t, csr_h, engine=eng)
    stats = [s.tolist() for s in eng.tc_stats]
    return [x.cpu() for x in got], stats


def _check(kind, model, h, t, r, dev, with_oracle=True):
    """tensor-core ranks == exact-scan ranks (== oracle ranks); returns the near-ties found."""
    dh, dt = oracle.build_filter_dicts(h, t, r)
    got, stats = _ranks(model, h, t, r, dh, dt, dev, True)
    # both sides ran on the tensor cores and their near-tie lists did not overflow, so the ranks
    # are the epilogue's own and not those of the exact recomputation behind an overflow
    assert len(stats) == 2 and all(found <= cap for found, cap in stats), stats
    want, _ = _ranks(model, h, t, r, dh, dt, dev, False)
    names = ("rank_heads", "rank_tails", "filt_rank_heads", "filt_rank_tails")
    for name, a, b in zip(names, got, want):
        bad = (a != b).nonzero().flatten()
        assert bad.numel() == 0, "%s: %d ranks differ from the exact scan, first at %d: %d vs %d" % (
            name, bad.numel(), bad[0], a[bad[0]], b[bad[0]])
    if with_oracle:
        ref = oracle.link_prediction(kind, helpers.oracle_params(kind, model), h, t, r, dh, dt, 128)
        for name, a, b in zip(names, got, ref):
            assert torch.equal(a, b), name
    return sum(found for found, _ in stats)


@pytest.mark.parametrize("last_cols", [1, 31, 32, 33, 255])
@pytest.mark.parametrize("kind,d", CASES, ids=CASE_IDS)
def test_last_candidate_tile_widths(kind, d, last_cols, cuda_device, operand_format):
    """Tables of 2 x 256 + last_cols entities: the last candidate tile ends inside a 32-column block
    (1, 33, 255), on a block boundary (32) or one short of it (31); 137 queries (9 in the last tile)."""
    n_ent, n_rel = 512 + last_cols, 7
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=last_cols).to(cuda_device)
    # test facts whose true entity sits in the partial last tile too
    h, t, r = _triples(n_ent, n_rel, 137, seed=last_cols, tails=torch.arange(n_ent - last_cols, n_ent))
    _check(kind, model, h, t, r, cuda_device)


@pytest.mark.parametrize("q_rem", [1, 8, 9, 64, 65, 127])
@pytest.mark.parametrize("kind,d", CASES, ids=CASE_IDS)
def test_last_query_tile_fill(kind, d, q_rem, cuda_device, operand_format):
    """256 + q_rem queries: the last 128-query tile holds q_rem of them, the rest are padding rows
    (one or both rows of a thread, whole warps, a whole warpgroup)."""
    n_ent, n_rel = 512 + 33, 7
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=q_rem).to(cuda_device)
    h, t, r = _triples(n_ent, n_rel, 256 + q_rem, seed=q_rem)
    _check(kind, model, h, t, r, cuda_device)


@pytest.mark.parametrize("kind,d", CASES, ids=CASE_IDS)
def test_blocks_of_exact_ties(kind, d, cuda_device, operand_format):
    """Entities 256..287 are one row repeated, and so are 769..800 (the last of which is the only
    column of the last candidate tile); every test tail lies in the first group and every test
    head in the second.  Each query then ties with all 32 columns of a block: 512 near-ties per warp
    and block, more than the warp's buffer holds, some of them in the partial last tile."""
    n_ent, n_rel, n_q = 801, 5, 200
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=d)
    with torch.no_grad():
        for w in _entity_planes(model):
            w[256:288] = w[256].clone()
            w[769:801] = w[769].clone()
    model = model.to(cuda_device)
    h, t, r = _triples(n_ent, n_rel, n_q, seed=d, heads=torch.arange(769, 801), tails=torch.arange(256, 288))
    found = _check(kind, model, h, t, r, cuda_device)
    assert found >= 2 * 32 * n_q


@pytest.mark.parametrize("where", ["entity", "relation"])
@pytest.mark.parametrize("kind,d", CASES, ids=CASE_IDS)
def test_nan_and_inf_operands(kind, d, where, cuda_device, operand_format):
    """A NaN row and an inf row among the entities (candidate table and the queries built from them)
    or among the relations (queries only).  Such an operand invalidates its whole operand image, so
    every pair becomes a near-tie and is decided by the exact arithmetic: 40 entities and one query
    tile keep all of them inside the near-tie list."""
    n_ent, n_rel, n_q = 40, 4, 100
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=d)
    with torch.no_grad():
        for w in (_entity_planes(model) if where == "entity" else _relation_planes(model))[:1]:
            w[1] = float("nan")
            w[2] = float("inf")
    model = model.to(cuda_device)
    h, t, r = _triples(n_ent, n_rel, n_q, seed=d)
    if where == "entity":
        h[:10], t[10:20] = 1, 1
        h[20:30], t[30:40] = 2, 2
    else:
        r[:20], r[20:40] = 1, 2
    found = _check(kind, model, h, t, r, cuda_device, with_oracle=False)
    assert found == 2 * n_q * n_ent
