"""TransD on the GPU: link prediction (exact and tensor-core scans on the per-relation projected tables),
relation prediction, top-k inference, scoring_function with its gradients and triplet classification,
against the unmodified reference's outputs (tests/golden/transd_*.npz) and the CPU oracle
(oracle/transd_oracle.py)."""
import os
import sys

import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle, transd_oracle
from tests import helpers, transd_kit
from tests.train_kit import close_grad
from torchkge_b200 import engine as engine_mod

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LP_NAMES = ("rank_true_heads", "rank_true_tails", "filt_rank_true_heads", "filt_rank_true_tails")


@pytest.fixture(params=[True, False], ids=["tensor_core", "exact"])
def engine(request, monkeypatch):
    eng = engine_mod.CudaEngine(tensor_core=request.param)
    monkeypatch.setattr(engine_mod, "_default_engine", eng)
    return eng


@pytest.fixture(scope="module", params=transd_kit.CASES)
def golden(request):
    return transd_kit.load(request.param)


@pytest.fixture(scope="module")
def wide():
    """A graph with 150 relations (more than one 128-wide tile of them), 40 of them without test facts, widths
    50 / 37 (not multiples of 8), two entities duplicated three times in both entity tables and two ent_emb
    rows of -0.0: exact ties in every projected table."""
    n_ent, n_rel, d, rd = 1500, 150, 50, 37
    h, t, r = helpers.random_graph(n_ent, n_rel, 12000, seed=23)
    dh, dt = kge_oracle.build_filter_dicts(h, t, r)
    dr = kge_oracle.build_rel_dict(h, t, r)
    keep = r < 110                       # relations 110.. keep their facts in the filters, get no test facts
    th, tt, tr = h[keep][:500], t[keep][:500], r[keep][:500]
    kg = tk.KnowledgeGraph(th, tt, tr, n_ent, n_rel, dict_of_heads=dh, dict_of_tails=dt)
    kg.dict_of_rels = dr
    torch.manual_seed(23)
    model = tk.TransDModel(d, rd, n_ent, n_rel)
    with torch.no_grad():
        for table in (model.ent_emb.weight, model.ent_proj_vect.weight):
            for src, dst in ((int(th[0]), (5, 700)), (int(tt[1]), (6, 1499))):
                for x in dst:
                    table[x] = table[src]
        model.ent_emb.weight[9] = -0.0
        model.ent_emb.weight[int(th[2])] = -0.0
    P = transd_kit.params(model.state_dict())
    return {"kg": kg, "model": model, "P": P, "s": transd_oracle.scalars(P), "dh": dh, "dt": dt, "dr": dr,
            "h": th, "t": tt, "r": tr, "n_rel": n_rel}


def _lp(model, kg):
    ev = tk.LinkPredictionEvaluator(model, kg)
    ev.evaluate(b_size=64, verbose=False)
    return ev.rank_true_heads, ev.rank_true_tails, ev.filt_rank_true_heads, ev.filt_rank_true_tails


def test_link_prediction_equals_the_reference(golden, engine):
    model = transd_kit.model_from(golden).to(DEV)
    got = _lp(model, transd_kit.graph_of(golden))
    for name, x in zip(LP_NAMES, got):
        assert torch.equal(x, torch.from_numpy(golden["raw"][name]).long()), name
    if engine.tensor_core:
        assert engine.tc_stats, "the tensor-core scan did not run"


def test_link_prediction_equals_the_oracle_on_many_relations(wide, engine):
    w = wide
    got = _lp(w["model"].to(DEV), w["kg"])
    want = transd_oracle.link_prediction(w["P"], w["h"], w["t"], w["r"], w["dh"], w["dt"], 64, s=w["s"])
    for name, a, b in zip(LP_NAMES, got, want):
        assert torch.equal(a, b), "%s: %d facts differ" % (name, int((a != b).sum()))
    if engine.tensor_core:
        assert engine.tc_stats


def test_a_reference_model_object_ranks_as_this_package_s(golden):
    """A reference TransDModel (duck-typed by class name) gives the ranks of this package's model."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchkge")):
        pytest.skip("the reference package (oracle/_ref) is not built here")
    sys.path.insert(0, ref)
    try:
        from torchkge.models import TransDModel
    finally:
        sys.path.remove(ref)
    g = golden
    theirs = TransDModel(g["ent_dim"], g["rel_dim"], g["n_ent"], g["n_rel"])
    theirs.load_state_dict(dict(g["state"], projected_entities=torch.zeros(g["n_rel"], g["n_ent"], g["rel_dim"])))
    kg = transd_kit.graph_of(g)
    got = _lp(theirs.to(DEV), kg)
    want = _lp(transd_kit.model_from(g).to(DEV), kg)
    for name, a, b in zip(LP_NAMES, got, want):
        assert torch.equal(a, b), name
    ev = tk.RelationPredictionEvaluator(theirs, kg)
    ev.evaluate(b_size=64)
    assert torch.equal(ev.rank_true_rels, torch.from_numpy(g["raw"]["rank_true_rels_dir"]).long())


@pytest.mark.parametrize("directed", [True, False])
def test_relation_prediction_equals_the_reference_and_the_oracle(golden, wide, directed):
    tag = "dir" if directed else "undir"
    ev = tk.RelationPredictionEvaluator(transd_kit.model_from(golden).to(DEV), transd_kit.graph_of(golden),
                                        directed=directed)
    ev.evaluate(b_size=64)
    assert torch.equal(ev.rank_true_rels, torch.from_numpy(golden["raw"]["rank_true_rels_" + tag]).long())
    assert torch.equal(ev.filt_rank_true_rels, torch.from_numpy(golden["raw"]["filt_rank_true_rels_" + tag]).long())
    w = wide
    ev = tk.RelationPredictionEvaluator(w["model"].to(DEV), w["kg"], directed=directed)
    ev.evaluate(b_size=64)
    want = transd_oracle.relation_prediction(w["P"], w["h"], w["t"], w["r"], w["dr"], 64, directed, s=w["s"])
    assert torch.equal(ev.rank_true_rels, want[0])
    assert torch.equal(ev.filt_rank_true_rels, want[1])


def _exact_topk(scores, k, mask=None):
    """Best first; ties by ascending id (sort is stable); masked entries scored -inf."""
    scores = scores.clone()
    if mask is not None:
        for i, ids in enumerate(mask):
            if ids:
                scores[i, torch.tensor(sorted(ids))] = -float("inf")
    vals, idx = torch.sort(scores, dim=1, descending=True, stable=True)
    return idx[:, :k], vals[:, :k]


@pytest.mark.parametrize("missing", ["tails", "heads"])
@pytest.mark.parametrize("masked", [False, True])
def test_entity_inference_equals_an_exact_topk_of_the_oracle(wide, missing, masked):
    w, k = wide, 15
    ents = torch.cat([w["h"], w["t"][:40]]) if missing == "tails" else torch.cat([w["t"], w["h"][:40]])
    rels = torch.cat([w["r"], w["r"][:40].flip(0)])
    dic = (w["dt"] if missing == "tails" else w["dh"]) if masked else None
    ev = tk.EntityInference(w["model"].to(DEV), ents, rels, top_k=k, missing=missing, dictionary=dic)
    ev.evaluate(b_size=64)
    side = "tail" if missing == "tails" else "head"
    scores = transd_oracle.scores_all(w["P"], ents, ents, rels, side, s=w["s"])
    mask = [dic.get((int(e), int(r)), set()) for e, r in zip(ents, rels)] if masked else None
    pred, vals = _exact_topk(scores, k, mask)
    assert helpers.bits_equal(ev.scores, vals).all()
    assert torch.equal(ev.predictions, pred)


@pytest.mark.parametrize("masked", [False, True])
def test_relation_inference_equals_an_exact_topk_of_the_oracle(wide, masked):
    w, k = wide, 10
    dic = w["dr"] if masked else None
    ev = tk.RelationInference(w["model"].to(DEV), w["h"], w["t"], top_k=k, dictionary=dic)
    ev.evaluate(b_size=64)
    scores = transd_oracle.relation_scores_all(w["P"], w["h"], w["t"], s=w["s"])
    mask = [dic.get((int(a), int(b)), set()) for a, b in zip(w["h"], w["t"])] if masked else None
    pred, vals = _exact_topk(scores, k, mask)
    assert helpers.bits_equal(ev.scores, vals).all()
    assert torch.equal(ev.predictions, pred)


@pytest.mark.parametrize("ent_dim,rel_dim", [(5, 5), (9, 3), (40, 40), (50, 37), (200, 120)])
def test_scoring_function_and_gradients_against_float64_autograd(ent_dim, rel_dim):
    torch.manual_seed(ent_dim + rel_dim)
    n_ent, n_rel, b = 300, 7, 257
    model = tk.TransDModel(ent_dim, rel_dim, n_ent, n_rel).to(DEV)
    with torch.no_grad():        # away from the normalised state, so the normalisations' gradients matter
        for p in model.parameters():
            p.mul_(torch.rand_like(p) + 0.5)
    g = torch.Generator().manual_seed(ent_dim * 7 + rel_dim)
    h, t, nh, nt = (torch.randint(0, n_ent, (b,), generator=g) for _ in range(4))
    h[:9] = t[:9]                # h == t: both rows' gradients land on one row
    r = torch.randint(0, n_rel, (b,), generator=g)
    pos, neg = model(h.to(DEV), t.to(DEV), r.to(DEV), nh.to(DEV), nt.to(DEV))
    loss = tk.MarginLoss(margin=0.5)(pos, neg)
    loss.backward()
    P = {k: v.detach().cpu().double().requires_grad_(True) for k, v in transd_kit.params(model.state_dict()).items()}
    rpos = transd_oracle.score_triples(P, h, t, r)
    rneg = transd_oracle.score_triples(P, nh, nt, r)
    torch.testing.assert_close(pos.detach().cpu().double(), rpos.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(neg.detach().cpu().double(), rneg.detach(), rtol=1e-5, atol=1e-6)
    torch.nn.functional.relu(0.5 - rpos + rneg).sum().backward()
    for key, name in transd_kit.KEYS.items():
        close_grad(getattr(model, name).weight.grad, P[key].grad)


def test_margin_gradients_equal_the_reference_within_tolerance(golden):
    model = transd_kit.model_from(golden).to(DEV)
    h, t, r, nh, nt = (golden[k].to(DEV) for k in ("heads", "tails", "rels", "neg_heads", "neg_tails"))
    pos, neg = model(h, t, r, nh, nt)
    torch.testing.assert_close(pos.cpu(), torch.from_numpy(golden["raw"]["scores"]), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(neg.cpu(), torch.from_numpy(golden["raw"]["neg_scores"]), rtol=1e-5, atol=1e-6)
    tk.MarginLoss(margin=1.0)(pos, neg).backward()
    for name in transd_kit.GRAD_NAMES:
        close_grad(getattr(model, name).weight.grad, torch.from_numpy(golden["raw"]["grad:" + name]))
    assert model.evaluated_projections is False


def test_triplet_classification_agrees_with_the_oracle(wide):
    w = wide
    model = w["model"].to(DEV)
    kg_val = tk.KnowledgeGraph(w["h"][:250], w["t"][:250], w["r"][:250], 1500, w["n_rel"])
    kg_test = tk.KnowledgeGraph(w["h"][250:], w["t"][250:], w["r"][250:], 1500, w["n_rel"])
    ev = tk.TripletClassificationEvaluator(model, kg_val, kg_test)
    g = torch.Generator().manual_seed(3)
    draws = {which: (torch.randint(0, 1500, (250,), generator=g), torch.randint(0, 1500, (250,), generator=g))
             for which in ("main", "test")}
    ev.sampler.corrupt_kg = lambda b, cuda, which: draws[which]
    acc = ev.accuracy(64)
    P = w["P"]
    neg_val = transd_oracle.score_triples(P, *draws["main"], kg_val.relations)
    thr = torch.full((w["n_rel"],), -float("inf")).scatter_reduce(0, kg_val.relations, neg_val, "amax")
    present = torch.bincount(kg_val.relations, minlength=w["n_rel"]) > 0
    thr = torch.where(present, thr, neg_val.max())
    torch.testing.assert_close(ev.thresholds.cpu(), thr, rtol=1e-5, atol=1e-6)
    pos = transd_oracle.score_triples(P, kg_test.head_idx, kg_test.tail_idx, kg_test.relations)
    neg = transd_oracle.score_triples(P, *draws["test"], kg_test.relations)
    t_ = thr[kg_test.relations]
    want = ((pos > t_).sum().item() + (neg < t_).sum().item()) / (2 * kg_test.n_facts)
    assert abs(acc - want) <= 1.0 / kg_test.n_facts     # a score within float rounding of its threshold at most
