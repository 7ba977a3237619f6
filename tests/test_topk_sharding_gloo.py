"""Multi-process (gloo, CPU) tests of the sharded top-k host logic in torchkge_b200.engine:
topk_entity_inference / topk_relation_inference under EntityShard (full and local storage, an
empty shard) and QueryShard (fewer queries than ranks).  The CUDA engine is replaced by an
oracle-backed stand-in with the same interface -- this tests the sharding plumbing (row exchange,
padding, the all-gathers, the merge), not the kernels; tests/test_topk_shard_gpu.py runs the kernels."""
import pytest
import torch

from oracle import kge_oracle as oracle
from tests import gloo, helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import (EntityShard, ModelSpec, QueryShard, topk_entity_inference,
                                  topk_relation_inference)
from torchkge_b200.inference import _mask_csr

_KIND_OF_CODE = {_lib.TRANSE_L1: "transe_l1", _lib.TRANSE_L2: "transe_l2",
                 _lib.DISTMULT: "distmult", _lib.COMPLEX: "complex"}


def key_order(scores, ids):
    """Column order of every row under the key order of csrc/topk.cu: NaN first, then scores
    descending (+0.0 above -0.0), ties by ascending id; empty slots (id < 0) last."""
    by_id = torch.sort(ids, dim=1, stable=True).indices
    s = scores.gather(1, by_id)
    key = s.double()
    key[(s == 0) & torch.signbit(s)] = -1e-300
    key[torch.isnan(s)] = float("nan")
    by_key = torch.sort(key, dim=1, descending=True, stable=True).indices
    order = by_id.gather(1, by_key)
    empty = (ids.gather(1, order) < 0).to(torch.int8)
    return order.gather(1, torch.sort(empty, dim=1, stable=True).indices)


class OracleTopkEngine:
    """CPU stand-in for CudaEngine's top-k methods (tests only)."""

    def pack(self, spec):
        return torch.zeros(1)

    def gather_rows(self, spec, idx):
        planes = [spec.ent0] + ([spec.ent1] if spec.ent1 is not None else [])
        out = torch.zeros(idx.shape[0], len(planes), spec.dim)
        own = (idx >= spec.ent_lo) & (idx < spec.ent_lo + spec.n_rows)
        for p, tab in enumerate(planes):
            out[own, p] = tab[idx[own] - spec.ent_lo]
        return out

    def topk_side(self, spec, packed, side, hrows, trows, r_idx, k, mask=None):
        kind = _KIND_OF_CODE[spec.code]
        n, rows = hrows.shape[0], spec.n_rows
        ar = torch.arange(n)
        if side == _lib.SIDE_REL:      # candidates: the relation rows of relation_spec
            if spec.ent1 is None:
                P = {"ent": torch.cat([hrows[:, 0], trows[:, 0]]), "rel": spec.ent0}
            else:
                P = {"re_ent": torch.cat([hrows[:, 0], trows[:, 0]]), "im_ent": torch.cat([hrows[:, 1], trows[:, 1]]),
                     "re_rel": spec.ent0, "im_rel": spec.ent1}
            s = oracle.relation_scores_all(kind, P, ar, n + ar)
        else:
            if spec.ent1 is None:
                P = {"ent": torch.cat([spec.ent0, hrows[:, 0]]), "rel": spec.rel0}
            else:
                P = {"re_ent": torch.cat([spec.ent0, hrows[:, 0]]), "im_ent": torch.cat([spec.ent1, hrows[:, 1]]),
                     "re_rel": spec.rel0, "im_rel": spec.rel1}
            s = oracle.scores_all(kind, P, rows + ar, rows + ar, r_idx,
                                  "tail" if side == _lib.SIDE_TAIL else "head")[:, :rows]
        s = s.clone()
        if mask is not None:
            offs, ids = mask
            for i in range(n):
                for c in ids[offs[i]:offs[i + 1]].tolist():
                    if spec.ent_lo <= c < spec.ent_lo + rows:
                        s[i, c - spec.ent_lo] = float("-inf")
        ids = (spec.ent_lo + torch.arange(rows)).expand(n, rows)
        order = key_order(s, ids)[:, :k]
        return ids.gather(1, order), s.gather(1, order)

    def topk_merge(self, pred_in, scores_in, k):
        n = pred_in.shape[1]
        ids = pred_in.permute(1, 0, 2).reshape(n, -1)
        s = scores_in.permute(1, 0, 2).reshape(n, -1)
        order = key_order(s, ids)[:, :k]
        pred, vals = ids.gather(1, order), s.gather(1, order).clone()
        vals[pred < 0] = float("-inf")
        return pred, vals


def _reference(kind, model, task, q1, q2, k, dictionary, side):
    """The oracle's dense scores, masked with -inf, then sort(descending=True)[:, :k]."""
    P = helpers.oracle_params(kind, model)
    if task == "entity":
        s = oracle.scores_all(kind, P, q1, q1, q2, side)
    else:
        s = oracle.relation_scores_all(kind, P, q1, q2)
    for i, (a, b) in enumerate(zip(q1.tolist(), q2.tolist())):
        m = dictionary.get((a, b))
        if m:
            s[i, sorted(m)] = float("-inf")
    vals, ids = s.sort(descending=True, stable=True)   # masked -inf entries in id order
    return ids[:, :k], vals[:, :k]


def _run(rank, world, task, kind, storage, n_ent, n_queries, k, side):
    n_rel, d = 5, 12
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=17)
    g = torch.Generator().manual_seed(17)
    q1 = torch.randint(0, n_ent, (n_queries,), generator=g)
    q2 = torch.randint(0, n_rel if task == "entity" else n_ent, (n_queries,), generator=g)
    # a dictionary with sets on some keys: masked ids in several shards
    dictionary = {}
    for i in range(0, n_queries, 2):
        cand = n_ent if task == "entity" else n_rel
        dictionary[(int(q1[i]), int(q2[i]))] = set(torch.randint(0, cand, (3,), generator=g).tolist())
    mask = _mask_csr(dictionary, q1, q2)
    spec = ModelSpec.from_model(model)
    if storage == "query":
        shard = QueryShard.from_group(n_queries)
    else:
        shard = EntityShard.from_group(n_ent, local_storage=storage == "local")
        if storage == "local":      # each rank HOLDS only its rows
            spec = spec.narrowed(shard.lo, shard.hi)
    eng = OracleTopkEngine()
    if task == "entity":
        s = _lib.SIDE_TAIL if side == "tail" else _lib.SIDE_HEAD
        pred, vals = topk_entity_inference(spec, q1, q2, s, k, mask, shard=shard, engine=eng, chunk=7)
    else:
        pred, vals = topk_relation_inference(spec, q1, q2, k, mask, shard=shard, engine=eng, chunk=7)
    want_ids, want_vals = _reference(kind, model, task, q1, q2, k, dictionary, side)
    return bool(pred.shape == (n_queries, k) and torch.equal(pred, want_ids)
                and torch.equal(vals.view(torch.int32), want_vals.view(torch.int32)))


# (world, task, kind, storage, n_ent, n_queries, k, side)
CASES = [
    (2, "entity", "transe_l2", "local", 61, 23, 7, "tail"),
    (3, "entity", "complex", "full", 50, 19, 10, "head"),
    (3, "entity", "distmult", "local", 40, 16, 21, "tail"),    # k above one shard's 14 rows
    (3, "entity", "transe_l1", "local", 2, 5, 2, "tail"),      # n_ent < world: rank 2 holds nothing
    (3, "entity", "distmult", "query", 40, 2, 5, "head"),      # fewer queries than ranks
    (2, "relation", "distmult", "local", 30, 17, 3, None),
    (3, "relation", "complex", "full", 30, 11, 4, None),
    (3, "relation", "transe_l2", "query", 30, 2, 2, None),
]


@pytest.mark.parametrize("case", CASES, ids=["%s-%s-%s-w%d" % (c[1], c[2], c[3], c[0]) for c in CASES])
def test_sharded_topk_equals_oracle(case):
    world = case[0]
    assert gloo.spawn(world, _run, *case[1:]) == {i: True for i in range(world)}


def test_key_order_of_the_stand_in():
    """NaN first, +0.0 above -0.0, ties by ascending id, empty slots last."""
    s = torch.tensor([[1.0, float("nan"), -0.0, 0.0, 1.0, float("-inf"), 5.0]])
    ids = torch.tensor([[9, 4, 2, 3, 1, 8, -1]])
    assert ids.gather(1, key_order(s, ids)).tolist() == [[4, 1, 9, 3, 2, 8, -1]]


def test_query_shard_all_gather_keeps_trailing_dims():
    """world 1: the results come back as given (the multi-rank form runs in the cases above)."""
    qs = QueryShard(5, 0, 1)
    x = torch.arange(30).view(5, 2, 3)
    out, = qs.all_gather([x])
    assert torch.equal(out, x)
