"""The TransD oracle (oracle/transd_oracle.py), which projects relation by relation, reproduces the unmodified
reference's outputs stored in tests/golden/transd_*.npz: link-prediction and relation-prediction ranks,
scoring_function values and the gradients of a margin loss."""
import pytest
import torch

from oracle import kge_oracle, transd_oracle
from tests import transd_kit
from tests.helpers import bits_equal


@pytest.fixture(scope="module", params=transd_kit.CASES)
def golden(request):
    return transd_kit.load(request.param)


def test_link_prediction_ranks(golden):
    g = golden
    got = transd_oracle.link_prediction(g["P"], g["heads"], g["tails"], g["rels"], g["dh"], g["dt"], g["b_size"])
    for name, x in zip(("rank_true_heads", "rank_true_tails", "filt_rank_true_heads", "filt_rank_true_tails"), got):
        assert torch.equal(x, torch.from_numpy(g["raw"][name]).long()), name


@pytest.mark.parametrize("directed", [True, False])
def test_relation_prediction_ranks(golden, directed):
    g = golden
    tag = "dir" if directed else "undir"
    rr, frr = transd_oracle.relation_prediction(g["P"], g["heads"], g["tails"], g["rels"], g["dr"], g["b_size"],
                                                directed=directed)
    assert torch.equal(rr, torch.from_numpy(g["raw"]["rank_true_rels_" + tag]).long())
    assert torch.equal(frr, torch.from_numpy(g["raw"]["filt_rank_true_rels_" + tag]).long())


def test_scoring_function_and_margin_gradients(golden):
    g = golden
    P = {k: v.clone().requires_grad_(True) for k, v in g["P"].items()}
    pos = transd_oracle.score_triples(P, g["heads"], g["tails"], g["rels"])
    neg = transd_oracle.score_triples(P, g["neg_heads"], g["neg_tails"], g["rels"])
    assert bits_equal(pos, torch.from_numpy(g["raw"]["scores"])).all()
    assert bits_equal(neg, torch.from_numpy(g["raw"]["neg_scores"])).all()
    loss = kge_oracle.margin_loss(pos, neg, 1.0)
    assert loss.item() == float(g["raw"]["loss"])
    loss.backward()
    for key, name in transd_kit.KEYS.items():
        want = torch.from_numpy(g["raw"]["grad:" + name])
        assert torch.allclose(P[key].grad, want, rtol=1e-6, atol=1e-7), name
