"""Host-side logic of the shim: filter CSR construction, shard ranges, loud failure on CPU."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import EntityShard, ModelSpec


def test_filter_csr_matches_get_true_targets_semantics():
    h, t, r = helpers.random_graph(60, 4, 900, seed=3)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    # quirk 1: true entity missing from its set -> row unfiltered
    for i in range(0, 50, 5):
        dt[(h[i].item(), r[i].item())].discard(t[i].item())
    # quirk 2: unknown key
    hq = torch.cat([h[:200], torch.tensor([59])])
    rq = torch.cat([r[:200], torch.tensor([3])])
    tq = torch.cat([t[:200], torch.tensor([0])])
    dt.pop((59, 3), None)
    offs, ids = filter_csr(dt, hq, rq, tq)
    assert offs.dtype == torch.int64 and offs.shape == (202,)
    for i in range(201):
        want = oracle.filter_targets(dt, hq[i].item(), rq[i].item(), tq[i].item())
        got = ids[offs[i]:offs[i + 1]].tolist()
        assert sorted(got) == sorted(want or [])
        assert tq[i].item() not in got


def test_filter_csr_accepts_list_valued_dicts():
    # the reference's own fixture uses lists (tests/test_utils.py:57)
    d = {(0, 0): [0, 1, 2], (0, 1): [1]}
    offs, ids = filter_csr(d, torch.tensor([0, 0, 0]), torch.tensor([0, 0, 1]), torch.tensor([1, 2, 1]))
    assert offs.tolist() == [0, 2, 4, 4]
    assert sorted(ids[:2].tolist()) == [0, 2] and sorted(ids[2:4].tolist()) == [0, 1]


@pytest.mark.parametrize("n_ent,world", [(10, 1), (10, 3), (1000000, 8), (7, 8), (5000000, 8)])
def test_entity_shard_ranges_partition_the_table(n_ent, world):
    shards = [EntityShard(n_ent, g, world) for g in range(world)]
    assert shards[0].lo == 0 and shards[-1].hi == n_ent
    for a, b in zip(shards, shards[1:]):
        assert a.hi == b.lo
    assert sum(s.hi - s.lo for s in shards) == n_ent


def test_model_spec_reads_reference_parameter_names():
    m = tk.ComplExModel(8, 12, 3)
    s = ModelSpec.from_model(m)
    assert s.code == _lib.COMPLEX and s.n_rows == 12 and s.cand_planes == 2
    assert s.ent0.data_ptr() == m.re_ent_emb.weight.data_ptr()  # no copy
    sub = s.narrowed(4, 9)
    assert sub.ent_lo == 4 and sub.n_rows == 5 and sub.n_ent == 12
    assert ModelSpec.from_model(tk.TransEModel(8, 12, 3, "L1")).code == _lib.TRANSE_L1
    assert ModelSpec.from_model(tk.TransEModel(8, 12, 3)).code == _lib.TRANSE_L2


def test_model_spec_of_a_three_plane_model():
    """Analogy (bilinear.py:559-763): the three planes of a table are equally spaced views of one
    stacked copy -- the C ABI takes planes 0 and 1 and finds plane 2 at the same spacing -- and stay
    so under narrowing to a shard; the plane width is scalar_dim, not emb_dim."""
    from torchkge_b200.engine import _equally_spaced, relation_spec
    m = tk.AnalogyModel(16, 12, 3)
    assert (m.scalar_dim, m.complex_dim) == (8, 8)
    assert set(m.state_dict()) == {"sc_ent_emb.weight", "re_ent_emb.weight", "im_ent_emb.weight",
                                   "sc_rel_emb.weight", "re_rel_emb.weight", "im_rel_emb.weight"}
    s = ModelSpec.from_model(m)
    assert s.code == _lib.ANALOGY and s.dim == 8 and s.n_rows == 12 and s.cand_planes == 3
    assert torch.equal(s.ent0, m.sc_ent_emb.weight) and torch.equal(s.ent1, m.re_ent_emb.weight)
    assert torch.equal(s.ent2, m.im_ent_emb.weight) and torch.equal(s.rel2, m.im_rel_emb.weight)
    assert _equally_spaced(s.ent0, s.ent1, s.ent2) and _equally_spaced(s.rel0, s.rel1, s.rel2)
    sub = s.narrowed(4, 9)
    assert sub.ent_lo == 4 and sub.n_rows == 5 and _equally_spaced(sub.ent0, sub.ent1, sub.ent2)
    assert torch.equal(sub.ent2, m.im_ent_emb.weight[4:9])
    r = relation_spec(s)
    assert r.n_rows == 3 and r.cand_planes == 3 and torch.equal(r.ent2, m.im_rel_emb.weight)
    with pytest.raises(ValueError):      # planes that are not views of one stacked tensor
        ModelSpec(_lib.ANALOGY, 8, 12, 3, s.ent0, s.ent1.clone(), s.rel0, s.rel1, ent2=s.ent2, rel2=s.rel2)
    with pytest.raises(NotImplementedError):   # odd emb_dim: the reference's inference fails on it too
        ModelSpec.from_model(tk.AnalogyModel(7, 12, 3))
    lib = _lib.load()
    assert lib.kge_cand_planes(_lib.ANALOGY) == 3
    assert [lib.kge_query_planes(_lib.ANALOGY, side) for side in (0, 1, 2)] == [3, 3, 3]
    # tensor-core image: one K = 3 x 64 contraction, the size of ComplEx's at 2 x 96
    assert lib.kge_tc_packed_bytes(_lib.ANALOGY, 1000, 64) == lib.kge_tc_packed_bytes(_lib.COMPLEX, 1000, 96) > 0
    assert lib.kge_packed_table_floats(_lib.ANALOGY, 1000, 64) == 8 * 64 * 3 * 128


def test_analogy_constructor_draws_the_reference_weights():
    """Same RNG calls in the same order as bilinear.py:620-631: replaying the fixture's recipe
    (tests/golden/make_golden.py: seed, constructor, row-wise perturbation) with THIS package's class
    reproduces the weights the unmodified reference drew, bit for bit."""
    from tests import helpers
    g = helpers.load_golden("toy_analogy")
    torch.manual_seed(7)
    m = tk.AnalogyModel(g["dim"], g["n_ent"], g["n_rel"])
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.0 + 0.5 * torch.rand(p.shape[0], 1))
    assert list(m.state_dict()) == list(g["state"])
    for k, v in m.state_dict().items():
        assert torch.equal(v, g["state"][k]), k
    # unequal widths (scalar_share != 0.5) are scored with torch ops: the reference's expression
    m = tk.AnalogyModel(10, 7, 2, scalar_share=0.3)
    assert (m.scalar_dim, m.complex_dim) == (3, 7)
    h, t, r = torch.tensor([0, 1, 2]), torch.tensor([3, 4, 5]), torch.tensor([0, 1, 0])
    re_h, im_h, re_t, im_t = m.re_ent_emb(h), m.im_ent_emb(h), m.re_ent_emb(t), m.im_ent_emb(t)
    re_r, im_r = m.re_rel_emb(r), m.im_rel_emb(r)
    want = ((m.sc_ent_emb(h) * m.sc_rel_emb(r) * m.sc_ent_emb(t)).sum(dim=1) +
            (re_h * (re_r * re_t + im_r * im_t) + im_h * (re_r * im_t - im_r * re_t)).sum(dim=1))
    assert torch.equal(m.scoring_function(h, t, r), want)


def test_state_dict_keys_match_reference_contract():
    assert set(tk.TransEModel(4, 5, 2).state_dict()) == {"ent_emb.weight", "rel_emb.weight"}
    assert set(tk.RESCALModel(4, 5, 2).state_dict()) == {"ent_emb.weight", "rel_mat.weight"}
    assert set(tk.ComplExModel(4, 5, 2).state_dict()) == {
        "re_ent_emb.weight", "im_ent_emb.weight", "re_rel_emb.weight", "im_rel_emb.weight"}
    assert tk.RESCALModel(4, 5, 2).rel_mat.weight.shape == (2, 16)


def test_constructor_weights_equal_reference_distribution():
    """Entity rows are unit-norm for TransE / DistMult / RESCAL; ComplEx is raw Xavier."""
    torch.manual_seed(0)
    m = tk.TransEModel(50, 40, 6)
    assert torch.allclose(m.ent_emb.weight.norm(dim=1), torch.ones(40), atol=1e-6)
    assert torch.allclose(m.rel_emb.weight.norm(dim=1), torch.ones(6), atol=1e-6)
    c = tk.ComplExModel(50, 40, 6)
    bound = (6.0 / (40 + 50)) ** 0.5
    assert c.re_ent_emb.weight.abs().max() <= bound


def test_evaluator_refuses_cpu_models_loudly():
    kg, _, _ = helpers.make_kg(30, 3, 100, 10)
    ev = tk.LinkPredictionEvaluator(tk.DistMultModel(8, 30, 3), kg)
    with pytest.raises(_lib.KgeLibraryError, match="no CPU"):
        ev.evaluate(b_size=4, verbose=False)
    with pytest.raises(tk.NotYetEvaluatedError):
        ev.mrr()


@pytest.mark.parametrize("case", ["toy_distmult", "syn_transe_l2"])
def test_bernoulli_probs_match_golden(case):
    """get_bernoulli_probs / evaluate_probabilities (host side) against the reference's values."""
    import numpy as np
    from torchkge_b200.sampling import BernoulliNegativeSampler
    g = helpers.load_golden(case)
    kg = tk.KnowledgeGraph(g["all_heads"], g["all_tails"], g["all_rels"], g["n_ent"], g["n_rel"],
                           dict_of_heads={}, dict_of_tails={})
    s = BernoulliNegativeSampler(kg, n_neg=3, seed=0)
    assert s.bern_probs.dtype == torch.float32 and s.bern_probs.shape == (g["n_rel"],)
    assert np.allclose(s.bern_probs.numpy(), g["raw"]["bern_probs"], rtol=0, atol=1e-7)
    assert s.n_ent == g["n_ent"] and s.n_neg == 3


def test_sampler_and_training_refuse_cpu_tensors():
    h, t, r = helpers.random_graph(50, 3, 200, seed=1)
    kg = tk.KnowledgeGraph(h, t, r, 50, 3, dict_of_heads={}, dict_of_tails={})
    s = tk.BernoulliNegativeSampler(kg, seed=0)
    with pytest.raises(_lib.KgeLibraryError):
        s.corrupt_batch(h[:10], t[:10], r[:10])
    for m in (tk.DistMultModel(8, 50, 3), tk.AnalogyModel(8, 50, 3), tk.TorusEModel(8, 50, 3, "torus_L2"),
              tk.ComplExModel(8, 50, 3)):
        with pytest.raises(_lib.KgeLibraryError):      # no CPU execution path for a kernel configuration
            m.scoring_function(h[:10], t[:10], r[:10])


def test_filter_index_equals_dictionary_semantics():
    """FilterIndex.csr == filter_csr on the reference's dictionaries, quirks included."""
    from torchkge_b200.data import FilterIndex
    h, t, r = helpers.random_graph(300, 6, 4000, seed=2)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    idx = FilterIndex(h, t, r, 300, 6)
    g = torch.Generator().manual_seed(0)
    # facts, plus random triples (true entity usually NOT in the set, some keys unknown)
    qh = torch.cat([h[:300], torch.randint(0, 300, (150,), generator=g)])
    qt = torch.cat([t[:300], torch.randint(0, 300, (150,), generator=g)])
    qr = torch.cat([r[:300], torch.randint(0, 6, (150,), generator=g)])
    for which, d, k1, k2, tr in (("tail", dt, qh, qr, qt), ("head", dh, qt, qr, qh)):
        o1, i1 = filter_csr(d, k1, k2, tr)
        o2, i2, q2 = idx.csr(which, k1, k2, tr)
        assert torch.equal(o1, o2)
        assert torch.equal(q2.long(), torch.repeat_interleave(torch.arange(450), o2[1:] - o2[:-1]))
        for q in range(450):
            assert sorted(i1[o1[q]:o1[q + 1]].tolist()) == sorted(i2[o2[q]:o2[q + 1]].tolist())
    kg = tk.KnowledgeGraph(h[:40], t[:40], r[:40], 300, 6, filter_facts=(h, t, r))
    assert kg.filter_index is not None
    assert all(kg.dict_of_tails[k] == v for k, v in dt.items())   # lazily materialised dicts
    assert all(kg.dict_of_heads[k] == v for k, v in dh.items())


def test_positional_sampler_candidate_sets_match_reference_definition():
    """possible_heads / possible_tails (sampling.py:371-409, operations.py get_possible_heads_tails):
    entities seen at that position with that relation in kg and kg_val, not kg_test."""
    h, t, r = helpers.random_graph(60, 4, 400, seed=2)
    mk = lambda a, b: tk.KnowledgeGraph(h[a:b], t[a:b], r[a:b], 60, 4, dict_of_heads={}, dict_of_tails={})  # noqa: E731
    kg, kg_val, kg_test = mk(0, 250), mk(250, 330), mk(330, 400)
    s = tk.PositionalNegativeSampler(kg, kg_val=kg_val, kg_test=kg_test, seed=1)
    hh, tt, rr = (torch.cat([kg.head_idx, kg_val.head_idx]), torch.cat([kg.tail_idx, kg_val.tail_idx]),
                  torch.cat([kg.relations, kg_val.relations]))
    for rel in range(4):
        assert s.possible_heads[rel] == sorted(set(hh[rr == rel].tolist()))
        assert s.possible_tails[rel] == sorted(set(tt[rr == rel].tolist()))
    assert s.n_poss_heads.tolist() == [len(s.possible_heads[i]) for i in range(4)]
    assert s.n_neg == 1 and s.bern_probs.shape == (4,)
    with pytest.raises(_lib.KgeLibraryError):
        s.corrupt_batch(kg.head_idx, kg.tail_idx, kg.relations)   # CPU tensors: no CPU path


def test_inference_mask_csr_and_arguments():
    from torchkge_b200.inference import _mask_csr
    d = {(1, 0): {5, 7}, (2, 1): set(), (3, 0): {9}}
    offs, ids = _mask_csr(d, torch.tensor([1, 2, 4, 3]), torch.tensor([0, 1, 0, 0]))
    assert offs.tolist() == [0, 2, 2, 2, 3]
    assert sorted(ids[:2].tolist()) == [5, 7] and ids[2].item() == 9
    model = helpers.make_model("distmult", 8, 20, 3)
    with pytest.raises(tk.WrongArgumentsError):
        tk.EntityInference(model, torch.arange(4), torch.zeros(4, dtype=torch.long), missing="neither")
    inf = tk.EntityInference(model, torch.arange(4), torch.zeros(4, dtype=torch.long), top_k=3)
    assert inf.predictions.shape == (4, 3) and inf.scores.shape == (4, 3)
    with pytest.raises(_lib.KgeLibraryError):
        inf.evaluate(b_size=2)        # CPU model: refused loudly


def test_relation_evaluator_and_knowledge_graph_dict_of_rels():
    h = torch.tensor([0, 0, 1, 2]); t = torch.tensor([1, 1, 2, 0]); r = torch.tensor([0, 1, 0, 2])
    kg = tk.KnowledgeGraph(h, t, r, 3, 3)
    assert kg.dict_of_rels[(0, 1)] == {0, 1} and kg.dict_of_rels[(2, 0)] == {2}
    kg.dict_of_rels = {(0, 1): {0}}
    assert kg.dict_of_rels == {(0, 1): {0}}
    ev = tk.RelationPredictionEvaluator(helpers.make_model("distmult", 8, 3, 3), kg, directed=False)
    assert ev.rank_true_rels.shape == (4,) and not ev.evaluated and ev.directed is False
    with pytest.raises(tk.NotYetEvaluatedError):
        ev.hit_at_k(1)
    with pytest.raises(_lib.KgeLibraryError):
        ev.evaluate(b_size=2)


def test_relation_side_element_kinds_and_flags():
    lib = _lib.load()
    assert lib.kge_query_planes(_lib.DISTMULT, _lib.SIDE_REL) == 2      # (h, t) around the candidate
    assert lib.kge_query_planes(_lib.TRANSE_L2, _lib.SIDE_REL) == 2
    assert lib.kge_query_planes(_lib.COMPLEX, _lib.SIDE_REL) == 2
    assert lib.kge_query_planes(_lib.RESCAL, _lib.SIDE_REL) == 0         # not on the relation path
    assert lib.kge_query_planes(_lib.ROTATE, _lib.SIDE_REL) == 0
    # the bound-and-refine flags only change the workspace of the models that have such a path
    base = lib.kge_rank_workspace_bytes(_lib.ROTATE, _lib.SIDE_TAIL, 64, 256, 50000, 0)
    assert lib.kge_rank_workspace_bytes(_lib.ROTATE, _lib.SIDE_TAIL, 64, 256, 50000, _lib.FLAG_APPROX_SCAN) > base
    assert lib.kge_rank_workspace_bytes(_lib.ROTATE, _lib.SIDE_TAIL, 64, 256, 50000, _lib.FLAG_TENSOR_CORE) == base
    l1 = lib.kge_rank_workspace_bytes(_lib.TRANSE_L1, _lib.SIDE_TAIL, 64, 256, 50000, 0)
    assert lib.kge_rank_workspace_bytes(_lib.TRANSE_L1, _lib.SIDE_TAIL, 64, 256, 50000, 3) == l1


def test_reference_import_paths_resolve():
    """`s/torchkge/torchkge_b200/` on the imports of a script that uses the hot path keeps working."""
    from torchkge_b200 import (KnowledgeGraph, LinkPredictionEvaluator, LogisticLoss, MarginLoss,  # noqa: F401
                               NotYetEvaluatedError, TorusEModel, TripletClassificationEvaluator)
    from torchkge_b200.data_structures import KnowledgeGraph as KG2
    from torchkge_b200.evaluation import LinkPredictionEvaluator as E2, RelationPredictionEvaluator  # noqa: F401
    from torchkge_b200.exceptions import NotYetEvaluatedError as N2
    from torchkge_b200.inference import EntityInference, RelationInference  # noqa: F401
    from torchkge_b200.models import ComplExModel, DistMultModel, RESCALModel, TransEModel  # noqa: F401
    from torchkge_b200.sampling import (BernoulliNegativeSampler, PositionalNegativeSampler,  # noqa: F401
                                        UniformNegativeSampler)
    from torchkge_b200.utils import (BinaryCrossEntropyLoss, MarginLoss as M2, get_bernoulli_probs,  # noqa: F401
                                     init_embedding, l1_dissimilarity, l2_dissimilarity)
    assert KG2 is KnowledgeGraph and E2 is LinkPredictionEvaluator and N2 is NotYetEvaluatedError and M2 is MarginLoss


def test_dict_filter_csr_equals_filter_csr_and_caches():
    """The fast route from the reference's dictionaries (distinct keys flattened once, rows
    expanded with tensor ops, cached on the graph) gives filter_csr's rows, quirks included."""
    from torchkge_b200.data import dict_filter_csr
    h, t, r = helpers.random_graph(200, 5, 3000, seed=4)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    g = torch.Generator().manual_seed(1)
    qh = torch.cat([h[:250], h[:50], torch.randint(0, 200, (120,), generator=g)])   # repeated keys too
    qt = torch.cat([t[:250], t[:50], torch.randint(0, 200, (120,), generator=g)])
    qr = torch.cat([r[:250], r[:50], torch.randint(0, 5, (120,), generator=g)])
    kg = tk.KnowledgeGraph(qh, qt, qr, 200, 5, dict_of_heads=dh, dict_of_tails=dt)
    for which, d, k1, k2, tr in (("tail", dt, qh, qr, qt), ("head", dh, qt, qr, qh)):
        o1, i1 = filter_csr(d, k1, k2, tr)
        (o2, i2, q2), nbytes = dict_filter_csr(kg, which, k1, k2, tr, torch.device("cpu"))
        assert torch.equal(o1, o2) and nbytes > 0
        assert torch.equal(q2.long(), torch.repeat_interleave(torch.arange(k1.shape[0]), o2[1:] - o2[:-1]))
        for q in range(k1.shape[0]):
            assert sorted(i1[o1[q]:o1[q + 1]].tolist()) == sorted(i2[o2[q]:o2[q + 1]].tolist())
        again = dict_filter_csr(kg, which, k1, k2, tr, torch.device("cpu"))
        assert again[0][0] is o2 and again[0][1] is i2    # served from the cache on the graph
    # editing a dictionary (its size changes) invalidates the cached rows
    dt[(999, 0)] = {1, 2}
    (o3, i3, _), _ = dict_filter_csr(kg, "tail", qh, qr, qt, torch.device("cpu"))
    assert torch.equal(o3, filter_csr(dt, qh, qr, qt)[0])


def test_csr_cut_carries_the_row_of_entry_array():
    """engine._csr_cut on (offs, ids, rows) triples: offsets and row ids are rebased to each piece."""
    from torchkge_b200.engine import _csr_cut
    offs = torch.tensor([0, 2, 2, 5, 6, 9])
    ids = torch.arange(100, 109)
    rows = torch.repeat_interleave(torch.arange(5), offs[1:] - offs[:-1]).to(torch.int32)
    whole, = _csr_cut((offs, ids, rows), [(0, 5)])
    assert whole[0] is offs and whole[2] is rows
    (o, i, q), = _csr_cut((offs, ids, rows), [(2, 5)])
    assert o.tolist() == [0, 3, 4, 7] and i.tolist() == list(range(102, 109))
    assert q.tolist() == [0, 0, 0, 1, 2, 2, 2]
    (o2, i2), = _csr_cut((offs, ids), [(1, 3)])
    assert o2.tolist() == [0, 0, 3] and i2.tolist() == [102, 103, 104]
    # several pieces from one cut, an empty one among them; no CSR, no pieces
    pieces = _csr_cut((offs, ids, rows), [(0, 2), (2, 2), (3, 5)])
    assert [p[0].tolist() for p in pieces] == [[0, 2, 2], [0], [0, 1, 4]]
    assert [p[2].tolist() for p in pieces] == [[0, 0], [], [0, 1, 1, 1]]
    assert _csr_cut(None, [(0, 1), (1, 2)]) == [None, None] and _csr_cut((offs, ids), []) == []


def test_data_loader_batches_in_fact_order():
    """utils.DataLoader (torchkge/utils/data.py:83-151): consecutive slices of the three index tensors,
    a partial last batch, len() = number of batches."""
    from torchkge_b200.utils import DataLoader
    h, t, r = helpers.random_graph(40, 3, 100, seed=0)
    kg = tk.KnowledgeGraph(h, t, r, 40, 3)
    dl = DataLoader(kg, batch_size=32)
    batches = list(dl)
    assert len(dl) == len(batches) == -(-kg.n_facts // 32)
    assert torch.equal(torch.cat([b[0] for b in batches]), kg.head_idx)
    assert torch.equal(torch.cat([b[1] for b in batches]), kg.tail_idx)
    assert torch.equal(torch.cat([b[2] for b in batches]), kg.relations)
    assert all(b[0].shape[0] == 32 for b in batches[:-1]) and 1 <= batches[-1][0].shape[0] <= 32
    assert list(dl)[0][0].data_ptr() == batches[0][0].data_ptr()      # a second pass starts over
    with pytest.raises(ValueError):
        DataLoader(kg, batch_size=8, use_cuda="sometimes")
