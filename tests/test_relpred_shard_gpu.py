"""Relation prediction over a sharded model (RelationPredictionEvaluator(..., shard=)): the rank
vectors of every rank must equal the unsharded evaluator's exactly, and the oracle's.  Shards are
emulated on one device by W threads whose collectives meet in process (tests/shard_threads.py); the
public API then runs in two processes (gloo on one GPU; NCCL when two GPUs are present)."""

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import gloo, helpers
from tests.shard_threads import run_ranks, thread_collectives
from torchkge_b200.engine import CudaEngine, EntityShard, ModelSpec, QueryShard, rank_relation_prediction

DEV = "cuda:0"
REL_KINDS = ["transe_l1", "transe_l2", "distmult", "rescal", "complex", "analogy"]
STORAGES = ["local", "full", "query"]


# ------------------------------------------------------------------ helpers
def make_shard(storage, rank, world, group, n_ent, n_facts):
    if storage == "query":
        return QueryShard(n_facts, rank, world, group)
    return EntityShard(n_ent, rank, world, group, local_storage=storage == "local")


def sharded_evaluator(kind, model, kg, dim, directed, storage, world):
    """[(rank_true_rels, filt_rank_true_rels)] of every emulated rank."""
    n_ent, n_rel = kg.n_ent, kg.n_rel

    def rank_fn(rank, group):
        shard = make_shard(storage, rank, world, group, n_ent, kg.n_facts)
        m = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim) if storage == "local" else model
        ev = tk.RelationPredictionEvaluator(m, kg, directed, shard=shard)
        ev.evaluate(b_size=64, verbose=False)
        return ev.rank_true_rels, ev.filt_rank_true_rels

    return run_ranks(world, rank_fn)


def unsharded(model, kg, directed):
    ev = tk.RelationPredictionEvaluator(model, kg, directed=directed)
    ev.evaluate(b_size=64, verbose=False)
    return ev.rank_true_rels, ev.filt_rank_true_rels


def assert_all_equal(per_rank, want, what):
    for rank, got in enumerate(per_rank):
        for g, w, name in zip(got, want, ("raw", "filtered")):
            bad = (g != w).nonzero().flatten()
            assert bad.numel() == 0, "%s rank %d: %d %s ranks differ, first at fact %d: %d != %d" % (
                what, rank, bad.numel(), name, bad[0], g[bad[0]], w[bad[0]])


def graph(n_ent, n_rel, n_facts, n_test, seed):
    h, t, r = helpers.random_graph(n_ent, n_rel, n_facts, seed=seed)
    dr = oracle.build_rel_dict(h, t, r)
    n_test = min(n_test, h.shape[0])
    kg = tk.KnowledgeGraph(h[:n_test], t[:n_test], r[:n_test], n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    kg.dict_of_rels = dr
    return kg, dr


def oracle_ranks(kind, model, kg, dr, dim, directed):
    if kind == "rescal" and not helpers.rescal_order_matches_here(dim):
        return None      # oneMKL on this CPU sums RESCAL's matmul in another order than the kernel replays
    P = helpers.oracle_params(kind, model)
    return oracle.relation_prediction(kind, P, kg.head_idx, kg.tail_idx, kg.relations, dr, 64, directed=directed)


# ------------------------------------------------------------------ 1. every model, every shard form
@pytest.mark.gpu
@pytest.mark.parametrize("directed", [True, False])
@pytest.mark.parametrize("kind", REL_KINDS)
def test_sharded_evaluator_equals_unsharded_and_oracle(kind, directed, monkeypatch):
    thread_collectives(monkeypatch)
    n_ent, n_rel, dim = 400, 300, 24       # more relations than one candidate tile (128)
    kg, dr = graph(n_ent, n_rel, 6000, 500, seed=31)
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=32).to(DEV)
    want = unsharded(model, kg, directed)
    ref = oracle_ranks(kind, model, kg, dr, dim, directed)
    if ref is not None:
        assert torch.equal(want[0], ref[0]) and torch.equal(want[1], ref[1])
    for world in (1, 2, 3, 8):
        for storage in STORAGES:
            got = sharded_evaluator(kind, model, kg, dim, directed, storage, world)
            assert_all_equal(got, want, "%s W=%d" % (storage, world))


# ------------------------------------------------------------------ 2. hard cases
def hard_graph(n_ent, n_rel, seed):
    """Facts over every pair of ranks, self loops, and repeated (h, t) pairs with several relations."""
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, n_ent, (300,), generator=g)
    t = torch.randint(0, n_ent, (300,), generator=g)
    h[:n_ent], t[:n_ent] = torch.arange(n_ent), torch.arange(n_ent)          # self loops
    h[n_ent:2 * n_ent], t[n_ent:2 * n_ent] = torch.arange(n_ent), n_ent - 1 - torch.arange(n_ent)
    r = torch.randint(0, n_rel, (300,), generator=g)
    trip = torch.unique(torch.stack([h, t, r], 1), dim=0)
    trip = trip[torch.randperm(trip.shape[0], generator=g)]
    h, t, r = trip[:, 0].contiguous(), trip[:, 1].contiguous(), trip[:, 2].contiguous()
    kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    kg.dict_of_rels = oracle.build_rel_dict(h, t, r)
    return kg


def tie_model(kind, dim, n_ent, n_rel, seed):
    """Rows of -0.0 and duplicated relation rows: exact ties between candidates."""
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=seed)
    with torch.no_grad():
        for name, w in model.state_dict().items():
            if "ent_emb" in name:
                w[[2, 9]] = -0.0
            else:
                w[n_rel // 2:n_rel // 2 + 5] = w[0:5].clone()
    return model.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", REL_KINDS)
def test_hard_cases_17_entities_over_8_ranks(kind, monkeypatch):
    """17 entities over 8 ranks (ranks 6 and 7 hold nothing), facts whose h and t live on different
    ranks, self loops, -0.0 rows, duplicated relations; the engine function with chunks of 7 facts,
    so chunk boundaries fall inside rank slices and some ranks get no facts in a chunk."""
    thread_collectives(monkeypatch)
    n_ent, n_rel, dim = 17, 40, 12
    kg = hard_graph(n_ent, n_rel, seed=41)
    model = tie_model(kind, dim, n_ent, n_rel, seed=42)
    per = (n_ent + 7) // 8
    assert (kg.head_idx // per != kg.tail_idx // per).any() and (kg.head_idx == kg.tail_idx).any()
    spec = ModelSpec.from_model(model)
    h, t, r = (x.to(DEV) for x in (kg.head_idx, kg.tail_idx, kg.relations))
    from torchkge_b200.data import filter_csr
    csr = tuple(x.to(DEV) for x in filter_csr(kg.dict_of_rels, kg.head_idx, kg.tail_idx, kg.relations))
    for directed in (True, False):
        want = unsharded(model, kg, directed)
        ref = oracle_ranks(kind, model, kg, kg.dict_of_rels, dim, directed)
        if ref is not None:
            assert torch.equal(want[0], ref[0]) and torch.equal(want[1], ref[1])
        for world in (2, 3, 8):
            for storage in STORAGES:
                def rank_fn(rank, group):
                    shard = make_shard(storage, rank, world, group, n_ent, kg.n_facts)
                    s = spec.narrowed(shard.lo, shard.hi) if storage == "local" else spec
                    out = rank_relation_prediction(s, h, t, r, csr, directed=directed, engine=CudaEngine(),
                                                   chunk=7, shard=shard)
                    return tuple(x.cpu() for x in out)

                assert_all_equal(run_ranks(world, rank_fn), want, "%s W=%d" % (storage, world))
                got = sharded_evaluator(kind, model, kg, dim, directed, storage, world)
                assert_all_equal(got, want, "evaluator %s W=%d" % (storage, world))


@pytest.mark.gpu
def test_rescal_dense_branch_several_chunks(monkeypatch):
    """More than 4,096 facts: the dense RESCAL branch runs several chunks, each split over the ranks."""
    thread_collectives(monkeypatch)
    n_ent, n_rel, dim = 300, 20, 16
    kg, dr = graph(n_ent, n_rel, 9000, 5000, seed=51)
    assert kg.n_facts > 4096
    model = helpers.make_model("rescal", dim, n_ent, n_rel, seed=52).to(DEV)
    for directed in (True, False):
        want = unsharded(model, kg, directed)
        for world in (3, 8):
            for storage in STORAGES:
                got = sharded_evaluator("rescal", model, kg, dim, directed, storage, world)
                assert_all_equal(got, want, "%s W=%d" % (storage, world))


@pytest.mark.gpu
def test_argument_errors():
    n_ent, n_rel, dim = 40, 5, 8
    kg, _ = graph(n_ent, n_rel, 200, 50, seed=61)
    model = helpers.make_model("distmult", dim, n_ent, n_rel, seed=62).to(DEV)
    with pytest.raises(ValueError, match="QueryShard covers"):
        tk.RelationPredictionEvaluator(model, kg, shard=QueryShard(kg.n_facts + 1, 0, 2)).evaluate(b_size=8)
    with pytest.raises(ValueError, match="local_storage=True"):     # the whole table, not rows [0, 20)
        tk.RelationPredictionEvaluator(model, kg, shard=EntityShard(n_ent, 0, 2, local_storage=True)).evaluate(8)
    with pytest.raises(ValueError, match="partitions 40 entities, the model has 20"):
        part = helpers.local_model("distmult", model, 0, 20, n_rel, dim)
        tk.RelationPredictionEvaluator(part, kg, shard=EntityShard(n_ent, 0, 2)).evaluate(8)
    rot = helpers.make_model("rotate", dim, n_ent, n_rel).to(DEV)
    with pytest.raises(NotImplementedError):
        tk.RelationPredictionEvaluator(rot, kg, shard=QueryShard(kg.n_facts, 0, 2)).evaluate(8)
    # the index check uses the global entity count: a local model of 20 rows takes ids up to 39 ...
    part = helpers.local_model("distmult", model, 20, 40, n_rel, dim)
    shard = EntityShard(n_ent, 1, 2, local_storage=True)
    bad = tk.KnowledgeGraph(torch.tensor([39]), torch.tensor([40]), torch.tensor([0]), n_ent + 1, n_rel,
                            dict_of_heads={}, dict_of_tails={})
    bad.dict_of_rels = {}
    # ... and refuses 40
    with pytest.raises(IndexError):
        tk.RelationPredictionEvaluator(part, bad, shard=shard).evaluate(8)


# ------------------------------------------------------------------ 3. public API, two processes
def _api_worker(rank, world, backend):
    dev = torch.device("cuda:%d" % (rank if backend == "nccl" else 0))
    torch.cuda.set_device(dev)
    try:
        results = {}
        n_ent, n_rel, dim = 1100, 9, 16
        h, t, r = helpers.random_graph(n_ent, n_rel, 4000, seed=71)
        mk = lambda a, b: tk.KnowledgeGraph(h[a:b], t[a:b], r[a:b], n_ent, n_rel,  # noqa: E731
                                            dict_of_heads={}, dict_of_tails={})
        kg, kg_val, kg_test = mk(0, 2000), mk(2000, 3000), mk(3000, 4000)
        kg_test.dict_of_rels = oracle.build_rel_dict(h, t, r)
        for kind in ("distmult", "complex"):
            model = helpers.make_model(kind, dim, n_ent, n_rel, seed=72).to(dev)
            ref_r = tk.RelationPredictionEvaluator(model, kg_test, directed=False)
            ref_r.evaluate(b_size=64, verbose=False)
            ref_c = tk.TripletClassificationEvaluator(model, kg_val, kg_test)
            ref_c.sampler = tk.PositionalNegativeSampler(kg_val, kg_test=kg_test, seed=500)
            ref_c.evaluate(b_size=128)
            ref_acc = ref_c.accuracy(b_size=128)
            full = EntityShard.from_group(n_ent)
            for name, shard, m in (
                    ("entity-local", EntityShard.from_group(n_ent, local_storage=True),
                     helpers.local_model(kind, model, full.lo, full.hi, n_rel, dim)),
                    ("query", QueryShard.from_group(kg_test.n_facts), model)):
                got_r = tk.RelationPredictionEvaluator(m, kg_test, directed=False, shard=shard)
                got_r.evaluate(b_size=64, verbose=False)
                results["%s/%s/relation" % (kind, name)] = (
                    torch.equal(got_r.rank_true_rels, ref_r.rank_true_rels)
                    and torch.equal(got_r.filt_rank_true_rels, ref_r.filt_rank_true_rels))
                got_c = tk.TripletClassificationEvaluator(m, kg_val, kg_test, shard=shard)
                # ranks seeded differently: rank 0's draws are used everywhere
                got_c.sampler = tk.PositionalNegativeSampler(kg_val, kg_test=kg_test, seed=500 + 7 * rank)
                got_c.evaluate(b_size=128)
                acc = got_c.accuracy(b_size=128)
                results["%s/%s/triplet" % (kind, name)] = (
                    torch.equal(got_c.thresholds.cpu().view(torch.int32), ref_c.thresholds.cpu().view(torch.int32))
                    and acc == ref_acc)
        return results
    except Exception as e:          # reported by the parent
        return {"error": "%s: %s" % (type(e).__name__, e)}


def _run_two_ranks(backend):
    ret = gloo.spawn(2, _api_worker, backend, backend=backend)
    for rank in (0, 1):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        assert all(res.values()) and len(res) == 8, "rank %d: %s" % (rank, res)


@pytest.mark.gpu
def test_public_api_two_processes_gloo_one_gpu():
    _run_two_ranks("gloo")


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_public_api_two_processes_nccl():
    _run_two_ranks("nccl")
