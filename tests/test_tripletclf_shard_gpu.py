"""Triplet classification over a sharded model (TripletClassificationEvaluator(..., shard=)): per-fact
scores bit-equal to the unsharded ``get_scores`` for all nine scoring kinds, and thresholds / accuracy
equal to an unsharded evaluator whose sampler draws what rank 0's draws -- also when the ranks'
samplers are seeded differently.  Ranks are emulated on one device by threads (tests/shard_threads.py);
the two-process form runs in tests/test_relpred_shard_gpu.py."""
import pytest
import torch

import torchkge_b200 as tk
from tests import helpers
from tests.shard_threads import run_ranks, thread_collectives
from tests.test_relpred_shard_gpu import STORAGES, make_shard
from torchkge_b200.engine import EntityShard

DEV = "cuda:0"
ALL_KINDS = ["transe_l1", "transe_l2", "toruse_l1", "toruse_l2", "distmult", "rescal", "complex",
             "analogy", "rotate"]


def graphs(n_ent, n_rel, seed):
    h, t, r = helpers.random_graph(n_ent, n_rel, 3000, seed=seed)
    mk = lambda a, b: tk.KnowledgeGraph(h[a:b], t[a:b], r[a:b], n_ent, n_rel,  # noqa: E731
                                        dict_of_heads={}, dict_of_tails={})
    return mk(0, 1200), mk(1200, 1900)


def sampler(kg_val, kg_test, seed):
    return tk.PositionalNegativeSampler(kg_val, kg_test=kg_test, seed=seed)


def bits(x):
    return x.detach().cpu().contiguous().view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ALL_KINDS)
def test_scores_thresholds_accuracy_equal_unsharded(kind, monkeypatch):
    thread_collectives(monkeypatch)
    n_ent, n_rel, dim = 300, 7, 16
    kg_val, kg_test = graphs(n_ent, n_rel, seed=81)
    model = helpers.make_model(kind, dim, n_ent, n_rel, seed=82).to(DEV)
    ref = tk.TripletClassificationEvaluator(model, kg_val, kg_test)
    ref.sampler = sampler(kg_val, kg_test, 900)          # what rank 0 will draw
    g = torch.Generator().manual_seed(83)
    nh = torch.randint(0, n_ent, (kg_test.n_facts,), generator=g)
    want_pos = ref.get_scores(kg_test.head_idx, kg_test.tail_idx, kg_test.relations, 100)
    want_neg = ref.get_scores(nh, kg_test.tail_idx, kg_test.relations, 100)
    ref.evaluate(b_size=100)
    want_acc = ref.accuracy(b_size=100)
    for world in (1, 2, 3, 8):
        for storage in STORAGES:
            def rank_fn(rank, group):
                shard = make_shard(storage, rank, world, group, n_ent, kg_test.n_facts)
                m = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim) if storage == "local" else model
                ev = tk.TripletClassificationEvaluator(m, kg_val, kg_test, shard=shard)
                ev.sampler = sampler(kg_val, kg_test, 900 + 13 * rank)      # seeded differently
                pos = ev.get_scores(kg_test.head_idx, kg_test.tail_idx, kg_test.relations, 100)
                neg = ev.get_scores(nh, kg_test.tail_idx, kg_test.relations, 37)
                ev.evaluate(b_size=100)
                return pos, neg, ev.thresholds, ev.accuracy(b_size=100)

            for rank, (pos, neg, thr, acc) in enumerate(run_ranks(world, rank_fn)):
                what = "%s W=%d rank %d" % (storage, world, rank)
                assert torch.equal(bits(pos), bits(want_pos)), what
                assert torch.equal(bits(neg), bits(want_neg)), what
                assert torch.equal(bits(thr), bits(ref.thresholds)), what
                assert acc == want_acc, what


@pytest.mark.gpu
def test_empty_shards_and_fewer_facts_than_ranks(monkeypatch):
    """5 entities over 8 ranks (three ranks hold nothing) and score vectors shorter than the world."""
    thread_collectives(monkeypatch)
    n_ent, n_rel, dim = 5, 2, 8
    h = torch.tensor([0, 1, 2, 3, 4, 4, 0, 2])
    t = torch.tensor([4, 3, 2, 1, 0, 4, 1, 0])
    r = torch.tensor([0, 1, 0, 1, 0, 1, 1, 0])
    kg_val = tk.KnowledgeGraph(h[:5], t[:5], r[:5], n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    kg_test = tk.KnowledgeGraph(h[5:], t[5:], r[5:], n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    for kind in ("complex", "analogy", "toruse_l2"):
        model = helpers.make_model(kind, dim, n_ent, n_rel, seed=84).to(DEV)
        ref = tk.TripletClassificationEvaluator(model, kg_val, kg_test)
        ref.sampler = sampler(kg_val, kg_test, 5)
        want = ref.get_scores(h, t, r, 3)
        ref.evaluate(b_size=2)
        want_acc = ref.accuracy(b_size=2)
        for storage in STORAGES:
            def rank_fn(rank, group):
                shard = make_shard(storage, rank, 8, group, n_ent, kg_test.n_facts)
                m = helpers.local_model(kind, model, shard.lo, shard.hi, n_rel, dim) if storage == "local" else model
                ev = tk.TripletClassificationEvaluator(m, kg_val, kg_test, shard=shard)
                ev.sampler = sampler(kg_val, kg_test, 5 + rank)
                s = ev.get_scores(h, t, r, 3)
                ev.evaluate(b_size=2)
                return s, ev.thresholds, ev.accuracy(b_size=2)

            for s, thr, acc in run_ranks(8, rank_fn):
                assert torch.equal(bits(s), bits(want)) and torch.equal(bits(thr), bits(ref.thresholds))
                assert acc == want_acc


@pytest.mark.gpu
def test_argument_errors_before_any_collective(monkeypatch):
    thread_collectives(monkeypatch)
    kg_val, kg_test = graphs(40, 3, seed=85)
    model = helpers.make_model("distmult", 8, 40, 3, seed=86).to(DEV)
    ev = tk.TripletClassificationEvaluator(model, kg_val, kg_test, shard=EntityShard(40, 0, 2, local_storage=True))
    with pytest.raises(ValueError, match="should hold 20 entity rows"):
        ev.evaluate(b_size=64)
    part = helpers.local_model("distmult", model, 0, 20, 3, 8)
    ev = tk.TripletClassificationEvaluator(part, kg_val, kg_test, shard=EntityShard(40, 0, 2))
    with pytest.raises(ValueError, match="should hold 40 entity rows"):
        ev.accuracy(b_size=64)
    tor = helpers.make_model("toruse_l1", 8, 40, 3)
    from torchkge_b200.models import l1_dissimilarity
    tor.dissimilarity = l1_dissimilarity            # plain L1 on fractional parts: no per-triple kernel
    tor = tor.to(DEV)
    part = helpers.local_model("toruse_l1", tor, 0, 20, 3, 8)
    part.dissimilarity = l1_dissimilarity
    ev = tk.TripletClassificationEvaluator(part, kg_val, kg_test, shard=EntityShard(40, 0, 2, local_storage=True))
    with pytest.raises(NotImplementedError):
        ev.evaluate(b_size=64)

