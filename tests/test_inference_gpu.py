"""EntityInference / RelationInference (torchkge/inference.py:78-250) on the GPU: the top-k scores
must equal, bit for bit, the k largest of the oracle's dense scores after masking the known
facts; the predicted indices must carry exactly those scores (order among exact ties is free)."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers

pytestmark = pytest.mark.gpu


def _check(pred, vals, dense, k):
    want_v, _ = torch.sort(dense, dim=1, descending=True)
    want_v = want_v[:, :k]
    assert helpers.bits_equal(vals, want_v).all()
    assert helpers.bits_equal(dense.gather(1, pred), vals).all()      # indices carry their scores
    for row in pred.tolist():
        assert len(set(row)) == len(row)                              # no candidate twice


@pytest.mark.parametrize("kind,d", [("transe_l2", 50), ("transe_l1", 33), ("distmult", 64),
                                    ("complex", 24), ("rescal", 12), ("rotate", 16)])
@pytest.mark.parametrize("missing", ["tails", "heads"])
def test_entity_inference_topk(kind, d, missing, cuda_device):
    n_ent, n_rel, n, k = 700, 6, 150, 7
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=2).to(cuda_device)
    P = helpers.oracle_params(kind, model)
    h, t, r = helpers.random_graph(n_ent, n_rel, 4000, seed=12)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    known = (h if missing == "tails" else t)[:n]
    rels = r[:n]
    dictionary = dt if missing == "tails" else dh
    inf = tk.EntityInference(model, known, rels, top_k=k, missing=missing, dictionary=dictionary)
    inf.evaluate(b_size=32, verbose=False)
    assert inf.predictions.shape == (n, k) and inf.predictions.dtype == torch.int64
    side = "tail" if missing == "tails" else "head"
    dense = (oracle.scores_all(kind, P, known, known, rels, side) if kind != "rotate"
             else oracle.rotate_scores_all(P, known, known, rels, side))
    for i in range(n):
        s = dictionary.get((known[i].item(), rels[i].item()))
        if s:
            dense[i][torch.tensor(list(s))] = -float("inf")
    if kind == "rescal" and not helpers.rescal_order_matches_here(d):   # this CPU's MKL sums differently
        want_v = torch.sort(dense, dim=1, descending=True)[0][:, :k]
        torch.testing.assert_close(inf.scores, want_v, rtol=1e-5, atol=1e-6)
    else:
        _check(inf.predictions, inf.scores, dense, k)
    # without a dictionary the known facts are allowed
    inf2 = tk.EntityInference(model, known, rels, top_k=1, missing=missing)
    inf2.evaluate(b_size=32, verbose=False)
    assert inf2.predictions.shape == (n, 1)


@pytest.mark.parametrize("kind,d", [("transe_l2", 40), ("distmult", 36), ("complex", 20), ("rescal", 12)])
def test_relation_inference_topk(kind, d, cuda_device):
    """RESCAL: dense relation scores (kge_rescal_rel_scores), then kge_topk_dense"""
    if kind == "rescal" and not helpers.rescal_order_matches_here(d):
        pytest.skip("oneMKL on this CPU sums RESCAL's batched matmul in another order than the authoring machine")
    n_ent, n_rel, n, k = 300, 40, 120, 5
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=3).to(cuda_device)
    P = helpers.oracle_params(kind, model)
    h, t, r = helpers.random_graph(n_ent, n_rel, 3000, seed=13)
    dr = oracle.build_rel_dict(h, t, r)
    inf = tk.RelationInference(model, h[:n], t[:n], top_k=k, dictionary=dr)
    inf.evaluate(b_size=16, verbose=False)
    dense = oracle.relation_scores_all(kind, P, h[:n], t[:n])
    for i in range(n):
        s = dr.get((h[i].item(), t[i].item()))
        if s:
            dense[i][torch.tensor(list(s))] = -float("inf")
    _check(inf.predictions, inf.scores, dense, k)


def test_wrong_arguments(cuda_device):
    model = helpers.make_model("distmult", 8, 20, 3).to(cuda_device)
    e, r = torch.arange(5), torch.zeros(5, dtype=torch.long)
    with pytest.raises(tk.WrongArgumentsError):
        tk.EntityInference(model, e, r, missing="both")
    with pytest.raises(tk.WrongArgumentsError):
        tk.EntityInference(model, e, r, top_k=21).evaluate(b_size=4)
