"""world_size-2 (gloo, CPU) test of the multi-GPU host logic in
torchkge_b200.engine.rank_link_prediction: range partition, query-row exchange, the single
all-reduce of the counters.  The CUDA engine is replaced by an oracle-backed stand-in with the
same interface -- this is a test of the sharding plumbing, not of the kernels."""
import pytest
import torch

from oracle import kge_oracle as oracle
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import EntityShard, ModelSpec, rank_link_prediction

_KIND_OF_CODE = {_lib.TRANSE_L1: "transe_l1", _lib.TRANSE_L2: "transe_l2",
                 _lib.DISTMULT: "distmult", _lib.COMPLEX: "complex", _lib.ANALOGY: "analogy"}


class OracleEngine:
    """CPU stand-in for CudaEngine (tests only)."""

    def pack(self, spec):
        return torch.zeros(1)

    def gather_rows(self, spec, idx):
        planes = [spec.ent0] + ([spec.ent1] if spec.ent1 is not None else [])
        planes += [spec.ent2] if getattr(spec, "ent2", None) is not None else []
        out = torch.zeros(idx.shape[0], len(planes), spec.dim)
        own = (idx >= spec.ent_lo) & (idx < spec.ent_lo + spec.n_rows)
        for p, tab in enumerate(planes):
            out[own, p] = tab[idx[own] - spec.ent_lo]
        return out

    def rank_side(self, spec, packed, side, hrows, trows, r_idx, true_idx, filt, raw, sub,
                  true_score=None):
        kind = _KIND_OF_CODE[spec.code]
        n, rows = r_idx.shape[0], spec.n_rows
        # candidates = shard rows, then the n head rows, then the n tail rows
        if spec.ent1 is None:
            P = {"ent": torch.cat([spec.ent0, hrows[:, 0], trows[:, 0]]), "rel": spec.rel0}
        elif kind == "analogy":     # three planes: scalar, real, imaginary
            P = {"sc_ent": torch.cat([spec.ent0, hrows[:, 0], trows[:, 0]]),
                 "re_ent": torch.cat([spec.ent1, hrows[:, 1], trows[:, 1]]),
                 "im_ent": torch.cat([spec.ent2, hrows[:, 2], trows[:, 2]]),
                 "sc_rel": spec.rel0, "re_rel": spec.rel1, "im_rel": spec.rel2}
        else:
            P = {"re_ent": torch.cat([spec.ent0, hrows[:, 0], trows[:, 0]]),
                 "im_ent": torch.cat([spec.ent1, hrows[:, 1], trows[:, 1]]),
                 "re_rel": spec.rel0, "im_rel": spec.rel1}
        ar = torch.arange(n)
        s = oracle.scores_all(kind, P, rows + ar, rows + n + ar, r_idx,
                              "tail" if side == _lib.SIDE_TAIL else "head")
        s_true = s[ar, rows + n + ar] if side == _lib.SIDE_TAIL else s[ar, rows + ar]
        shard_scores = s[:, :rows]
        raw += (shard_scores >= s_true.view(-1, 1)).sum(1).int()
        if filt is not None:
            offs, ids = filt
            for i in range(n):
                for c in ids[offs[i]:offs[i + 1]].tolist():
                    if spec.ent_lo <= c < spec.ent_lo + rows:
                        sc = shard_scores[i, c - spec.ent_lo]
                        sub[i] += int(sc >= s_true[i]) - int(s_true[i] == float("-inf"))
        return (side, s_true, shard_scores, spec)

    def filter_side(self, handle, filt, sub):
        side, s_true, shard_scores, spec = handle
        offs, ids = filt
        for i in range(s_true.shape[0]):
            for c in ids[offs[i]:offs[i + 1]].tolist():
                if spec.ent_lo <= c < spec.ent_lo + spec.n_rows:
                    sc = shard_scores[i, c - spec.ent_lo]
                    sub[i] += int(sc >= s_true[i]) - int(s_true[i] == float("-inf"))

    def finalize(self, raw, sub):
        return raw.long(), raw.long() - sub.long()


def _worker(rank, world, kind, storage):
    n_ent, n_rel, d = 203, 5, 24
    kg, dh, dt = helpers.make_kg(n_ent, n_rel, n_facts=1500, n_test=90, seed=21)
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=21)
    spec = ModelSpec.from_model(model)
    shard = EntityShard.from_group(n_ent, local_storage=storage == "local_storage")
    if storage == "local_storage":  # each rank only HOLDS its rows
        spec = spec.narrowed(shard.lo, shard.hi)
    csr_t = filter_csr(dt, kg.head_idx, kg.relations, kg.tail_idx)
    csr_h = filter_csr(dh, kg.tail_idx, kg.relations, kg.head_idx)
    out = rank_link_prediction(spec, kg.head_idx, kg.tail_idx, kg.relations, csr_t, csr_h,
                               shard=shard, engine=OracleEngine(), chunk=32)
    P = helpers.oracle_params(kind, model)
    ref = oracle.link_prediction(kind, P, kg.head_idx, kg.tail_idx, kg.relations, dh, dt, 30)
    return all(torch.equal(a, b) for a, b in zip(out, ref))


@pytest.mark.parametrize("kind,storage", [("distmult", "full"), ("transe_l2", "local_storage"),
                                          ("complex", "local_storage"), ("analogy", "local_storage")])
def test_two_rank_sharded_ranking_equals_single_process(kind, storage):
    assert gloo.spawn(2, _worker, kind, storage) == {0: True, 1: True}


def test_single_process_stand_in_agrees_with_oracle():
    """Sanity of the stand-in itself (world 1, chunked CSR slicing path)."""
    n_ent, n_rel, d = 120, 4, 16
    kg, dh, dt = helpers.make_kg(n_ent, n_rel, n_facts=800, n_test=70, seed=5)
    model = helpers.make_model("transe_l1", d, n_ent, n_rel, seed=5)
    spec = ModelSpec.from_model(model)
    csr_t = filter_csr(dt, kg.head_idx, kg.relations, kg.tail_idx)
    csr_h = filter_csr(dh, kg.tail_idx, kg.relations, kg.head_idx)
    out = rank_link_prediction(spec, kg.head_idx, kg.tail_idx, kg.relations, csr_t, csr_h,
                               engine=OracleEngine(), chunk=16)
    ref = oracle.link_prediction("transe_l1", helpers.oracle_params("transe_l1", model),
                                 kg.head_idx, kg.tail_idx, kg.relations, dh, dt, 64)
    for a, b in zip(out, ref):
        assert torch.equal(a, b)


def _worker_queries(rank, world, kind, n_test):
    """The second decomposition (bench.py at N > 1 for tables that fit one GPU): replicated table,
    test triples split over the ranks, rank vectors all-gathered."""
    from torchkge_b200.engine import QueryShard
    n_ent, n_rel, d = 150, 4, 16
    kg, dh, dt = helpers.make_kg(n_ent, n_rel, n_facts=1200, n_test=n_test, seed=33)
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=33)
    spec = ModelSpec.from_model(model)
    n = kg.n_facts
    csr_t = filter_csr(dt, kg.head_idx, kg.relations, kg.tail_idx)
    csr_h = filter_csr(dh, kg.tail_idx, kg.relations, kg.head_idx)
    qs = QueryShard.from_group(n)
    h, t, r = qs.slice(kg.head_idx, kg.tail_idx, kg.relations)
    local = rank_link_prediction(spec, h, t, r, qs.csr(csr_t), qs.csr(csr_h), engine=OracleEngine(),
                                 chunk=16)
    assert all(x.shape[0] == qs.hi - qs.lo for x in local)
    full = qs.all_gather(local)
    P = helpers.oracle_params(kind, model)
    ref = oracle.link_prediction(kind, P, kg.head_idx, kg.tail_idx, kg.relations, dh, dt, 30)
    return all(torch.equal(a, b) for a, b in zip(full, ref))


@pytest.mark.parametrize("kind,n_test,world", [("distmult", 75, 2), ("transe_l1", 1, 2), ("complex", 50, 3)])
def test_query_sharded_ranking_equals_single_process(kind, n_test, world):
    assert gloo.spawn(world, _worker_queries, kind, n_test) == {i: True for i in range(world)}


def test_query_shard_bounds():
    from torchkge_b200.engine import QueryShard
    for n, world in ((20466, 8), (5, 8), (0, 2), (7, 1)):
        shards = [QueryShard(n, r, world) for r in range(world)]
        assert shards[0].lo == 0 and shards[-1].hi == n
        assert all(a.hi == b.lo for a, b in zip(shards, shards[1:]))
        assert all(s.hi - s.lo <= s.per for s in shards)
