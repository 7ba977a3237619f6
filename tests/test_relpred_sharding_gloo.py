"""Multi-process (gloo, CPU) tests of the sharded relation-prediction host logic in
torchkge_b200.engine.rank_relation_prediction (and of score_triples_entity_sharded, the scoring of
sharded triplet classification): EntityShard with full and local storage, an empty shard, QueryShard
with fewer facts than ranks, chunk boundaries inside rank slices.  The CUDA engine is replaced by an
oracle-backed stand-in with the same interface -- this tests the plumbing (row exchange, the fact
split, the all-gathers, argument errors before any collective), not the kernels;
tests/test_relpred_shard_gpu.py runs the kernels."""
import pytest
import torch
import torch.distributed as dist

from oracle import kge_oracle as oracle
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import (EntityShard, ModelSpec, QueryShard, rank_relation_prediction,
                                  score_triples_entity_sharded)

_KIND_OF_CODE = {_lib.TRANSE_L1: "transe_l1", _lib.TRANSE_L2: "transe_l2", _lib.DISTMULT: "distmult",
                 _lib.COMPLEX: "complex", _lib.RESCAL: "rescal"}


class OracleRelEngine:
    """CPU stand-in for CudaEngine's relation-prediction methods (tests only).  Counting convention:
    raw_count += #{candidates scoring >= the true score}, filt_sub += #{filtered ids scoring >= it};
    finalize gives (raw, raw - sub)."""

    def pack(self, spec):
        return torch.zeros(1)

    def gather_rows(self, spec, idx):
        planes = [spec.ent0] + ([spec.ent1] if spec.ent1 is not None else [])
        out = torch.zeros(idx.shape[0], len(planes), spec.dim)
        own = (idx >= spec.ent_lo) & (idx < spec.ent_lo + spec.n_rows)
        for p, tab in enumerate(planes):
            out[own, p] = tab[idx[own] - spec.ent_lo]
        return out

    @staticmethod
    def _count(scores, true_idx, filt, raw, sub, true_score, true_score_in):
        ar = torch.arange(scores.shape[0])
        s_true = true_score_in if true_score_in is not None else scores[ar, true_idx]
        if true_score is not None:
            true_score.copy_(s_true)
        ge = scores >= s_true.view(-1, 1)
        raw += ge.sum(1).to(raw.dtype)
        if filt is not None:
            offs, ids = filt[0], filt[1]
            for i in range(scores.shape[0]):
                sub[i] += int(ge[i, ids[offs[i]:offs[i + 1]]].sum())

    def rank_side(self, spec, packed, side, hrows, trows, r_idx, true_idx, filt, raw_count, filt_sub,
                  true_score=None, true_rows=None, true_score_in=None, **kw):
        assert side == _lib.SIDE_REL
        n = hrows.shape[0]
        ar = torch.arange(n)
        kind = _KIND_OF_CODE[spec.code]
        if spec.ent1 is None:
            P = {"ent": torch.cat([hrows[:, 0], trows[:, 0]]), "rel": spec.ent0}
        else:
            P = {"re_ent": torch.cat([hrows[:, 0], trows[:, 0]]), "im_ent": torch.cat([hrows[:, 1], trows[:, 1]]),
                 "re_rel": spec.ent0, "im_rel": spec.ent1}
        scores = oracle.relation_scores_all(kind, P, ar, n + ar)
        self._count(scores, true_idx, filt, raw_count, filt_sub, true_score, true_score_in)
        return None

    def rescal_rel_scores(self, spec, hrows, trows):
        n = hrows.shape[0]
        ar = torch.arange(n)
        return oracle.relation_scores_all("rescal", {"ent": torch.cat([hrows, trows]), "rel_mat": spec.rel0}, ar, n + ar)

    def rank_dense(self, scores, true_idx, filt, raw_count, filt_sub, true_score=None, true_score_in=None):
        self._count(scores, true_idx, filt, raw_count, filt_sub, true_score, true_score_in)

    def finalize(self, raw, sub):
        return raw.long(), (raw - sub).long()

    def score_triples(self, code, dim, ent, rel0, rel1, h, t, r):
        kind = _KIND_OF_CODE[code]
        if ent.shape[0] == 1:
            P = {"ent": ent[0], "rel": rel0}
        else:
            P = {"re_ent": ent[0], "im_ent": ent[1], "re_rel": rel0, "im_rel": rel1}
        return oracle.score_triples(kind, P, h, t, r)


class Counting:
    """Counts this process's calls of the collectives the sharded paths use."""

    def __init__(self):
        self.calls = 0
        self._reduce, self._gather = dist.all_reduce, dist.all_gather
        dist.all_reduce, dist.all_gather = self.reduce, self.gather

    def reduce(self, *a, **k):
        self.calls += 1
        return self._reduce(*a, **k)

    def gather(self, *a, **k):
        self.calls += 1
        return self._gather(*a, **k)


def _graph(n_ent, n_rel, n_facts, seed):
    h, t, r = helpers.random_graph(n_ent, n_rel, n_facts, seed=seed, skew=False)
    h[:3], t[:3] = h[0], h[0]                 # self loops
    dr = oracle.build_rel_dict(h, t, r)
    return h, t, r, dr


def _shard_and_spec(storage, spec, n_ent, n):
    if storage == "query":
        return QueryShard.from_group(n), spec
    shard = EntityShard.from_group(n_ent, local_storage=storage == "local")
    if storage == "local":
        spec = spec.narrowed(shard.lo, shard.hi)
    return shard, spec


def _run_ranks(kind, storage, n_ent, n_facts, directed, chunk):
    n_rel, d = 6, 8
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=19)
    h, t, r, dr = _graph(n_ent, n_rel, n_facts, seed=19)
    csr = filter_csr(dr, h, t, r)
    shard, spec = _shard_and_spec(storage, ModelSpec.from_model(model), n_ent, h.shape[0])
    count = Counting()
    got = rank_relation_prediction(spec, h, t, r, csr, directed=directed, engine=OracleRelEngine(), chunk=chunk,
                                   shard=shard)
    want = oracle.relation_prediction(kind, helpers.oracle_params(kind, model), h, t, r, dr, 64, directed=directed)
    calls = torch.tensor([count.calls])
    everyone = [torch.zeros(1, dtype=torch.int64) for _ in range(dist.get_world_size())]
    dist.all_gather(everyone, calls)
    same_calls = len({int(x) for x in everyone}) == 1        # an empty shard joins every collective
    return torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]) and same_calls


def _run_scores(kind, n_ent, n_facts):
    model = helpers.make_model(kind, 8, n_ent, 4, seed=23)
    h, t, r, _ = _graph(n_ent, 4, n_facts, seed=23)
    spec = ModelSpec.from_model(model)
    shard = EntityShard.from_group(n_ent, local_storage=True)
    spec = spec.narrowed(shard.lo, shard.hi)
    got = score_triples_entity_sharded(spec, h, t, r, shard, engine=OracleRelEngine(), batch=5)
    want = oracle.score_triples(kind, helpers.oracle_params(kind, model), h, t, r)
    return torch.equal(got.view(torch.int32), want.view(torch.int32))


def _run_errors(case):
    """Every rank gets the same bad arguments: each must raise before any collective."""
    n_ent, n_rel, d = 30, 4, 8
    model = helpers.make_model("rotate" if case == "model" else "distmult", d, n_ent, n_rel, seed=29)
    h, t, r, dr = _graph(n_ent, n_rel, 20, seed=29)
    csr = filter_csr(dr, h, t, r)
    spec = ModelSpec.from_model(model)
    if case == "query_length":
        shard = QueryShard.from_group(h.shape[0] - 1)
    elif case == "rows":           # the whole table under local storage
        shard = EntityShard.from_group(n_ent, local_storage=True)
    elif case == "full_rows":      # only the local rows under full storage
        shard = EntityShard.from_group(n_ent)
        spec = spec.narrowed(shard.lo, shard.hi)
    else:
        shard = QueryShard.from_group(h.shape[0])
    count = Counting()
    try:
        rank_relation_prediction(spec, h, t, r, csr, engine=OracleRelEngine(), shard=shard)
    except (ValueError, NotImplementedError):
        return count.calls == 0
    return False


def _worker(rank, world, case):
    run = {"rank": _run_ranks, "scores": _run_scores, "errors": _run_errors}[case[0]]
    return bool(run(*case[1:]))


def _spawn(world, case):
    assert gloo.spawn(world, _worker, case) == {i: True for i in range(world)}


# (world, kind, storage, n_ent, n_facts, directed, chunk)
CASES = [
    (2, "transe_l2", "local", 31, 23, True, 7),
    (3, "complex", "local", 40, 29, False, 5),       # chunk boundaries inside rank slices
    (3, "distmult", "full", 40, 17, True, 64),
    (3, "transe_l1", "local", 2, 9, False, 4),       # n_ent < world: rank 2 holds nothing
    (3, "distmult", "query", 40, 2, True, 64),       # fewer facts than ranks
    (2, "rescal", "local", 25, 19, False, 6),
    (3, "rescal", "query", 25, 11, True, 64),
]


@pytest.mark.parametrize("case", CASES, ids=["%s-%s-w%d-%s" % (c[1], c[2], c[0], "dir" if c[5] else "undir")
                                             for c in CASES])
def test_sharded_relation_prediction_equals_oracle(case):
    _spawn(case[0], ("rank",) + case[1:])


@pytest.mark.parametrize("world,kind,n_ent", [(2, "distmult", 21), (3, "complex", 2), (3, "transe_l2", 30)])
def test_sharded_triple_scores_equal_oracle(world, kind, n_ent):
    _spawn(world, ("scores", kind, n_ent, 13))


@pytest.mark.parametrize("case", ["query_length", "rows", "full_rows", "model"])
@pytest.mark.parametrize("world", [2, 3])
def test_argument_errors_before_any_collective(case, world):
    _spawn(world, ("errors", case))
