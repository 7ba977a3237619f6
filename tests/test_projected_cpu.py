"""The relation-grouped loops of TransH and TransD without a GPU: link prediction and entity top-k through CPU
stand-ins for the engine (the oracle-backed ones of the sharding tests, plus the per-relation projections of
oracle/transh_oracle.py and oracle/transd_oracle.py), against the oracles' ranks and scores.  This tests the host
loop -- grouping, one projection per relation, the filter and mask rows of each group, the way back to query
order -- not the kernels; tests/test_transh_gpu.py and tests/test_transd_gpu.py run those."""
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle, transd_oracle, transh_oracle
from tests import helpers, transd_kit, transh_kit
from tests.test_sharding_gloo import OracleEngine
from tests.test_topk_sharding_gloo import OracleTopkEngine, key_order
from torchkge_b200 import _lib
from torchkge_b200.data import filter_csr
from torchkge_b200.engine import (TransDSpec, TransHSpec, rank_link_prediction_projected, relation_groups,
                                  topk_entity_inference)
from torchkge_b200.inference import _mask_csr

N_ENT, N_REL, EMPTY_REL = 70, 6, 2


class ProjectingEngine(OracleEngine, OracleTopkEngine):
    """The stand-ins' scans, with the projections taken from the oracles; records every projected relation."""

    def __init__(self):
        self.projected = []

    def transh_project(self, spec, rel, out):
        self.projected.append(rel)
        out[:] = transh_oracle.projections({"ent": spec.ent0, "norm": spec.norm_vect})[rel]
        return out

    def transd_project(self, spec, rel, out):
        self.projected.append(rel)
        P = {"ent": spec.ent_full, "rel": spec.rel0, "rel_proj": spec.rel_proj}
        out[:] = transd_oracle.projection(P, spec.scalars, rel)
        return out


@pytest.fixture(scope="module", params=["transh", "transd"])
def case(request):
    """A model, its spec and oracle tables, and test facts spread over several relations, none of them of
    relation EMPTY_REL (whose facts still fill the filter sets)."""
    h, t, r = helpers.random_graph(N_ENT, N_REL, 900, seed=31)
    dh, dt = kge_oracle.build_filter_dicts(h, t, r)
    keep = r != EMPTY_REL
    h, t, r = h[keep][:90], t[keep][:90], r[keep][:90]
    torch.manual_seed(31)
    if request.param == "transh":
        model = tk.TransHModel(8, N_ENT, N_REL)
        P = transh_kit.params(model.state_dict())
        spec = TransHSpec(model)
    else:
        model = tk.TransDModel(10, 7, N_ENT, N_REL)
        P = transd_kit.params(model.state_dict())
        spec = TransDSpec(model)
        spec.scalars = transd_oracle.scalars(P)     # a host model gets none from the engine
    return {"kind": request.param, "P": P, "spec": spec, "h": h, "t": t, "r": r, "dh": dh, "dt": dt}


def _relations_with(r):
    return sorted(set(r.tolist()))


def test_link_prediction_equals_the_oracle(case):
    h, t, r = case["h"], case["t"], case["r"]
    order, order_host, groups = relation_groups(r, N_REL)
    hs, ts, rs = h[order], t[order], r[order]
    csr_t, csr_h = filter_csr(case["dt"], hs, rs, ts), filter_csr(case["dh"], ts, rs, hs)
    assert csr_t[1].numel() > 0 and csr_h[1].numel() > 0
    eng = ProjectingEngine()
    got = rank_link_prediction_projected(case["spec"], hs, ts, rs, groups, csr_t, csr_h, engine=eng, chunk=16)
    assert eng.projected == [rel for rel, _, _ in groups] == _relations_with(r)
    assert len(groups) > 2 and EMPTY_REL not in eng.projected and eng.projected[-1] > EMPTY_REL
    if case["kind"] == "transh":
        want = transh_oracle.link_prediction(case["P"], h, t, r, case["dh"], case["dt"], 32)
    else:
        want = transd_oracle.link_prediction(case["P"], h, t, r, case["dh"], case["dt"], 32)
    for g, w in zip(got, want):
        back = torch.empty_like(g)
        back[order] = g
        assert torch.equal(back, w)


@pytest.mark.parametrize("side", [_lib.SIDE_TAIL, _lib.SIDE_HEAD], ids=["tail", "head"])
def test_masked_entity_topk_equals_the_oracle(case, side):
    k = 6
    ents, rels = (case["h"], case["r"]) if side == _lib.SIDE_TAIL else (case["t"], case["r"])
    known = case["dt"] if side == _lib.SIDE_TAIL else case["dh"]
    mask = _mask_csr(known, ents, rels)
    assert mask[1].numel() > 0
    eng = ProjectingEngine()
    pred, vals = topk_entity_inference(case["spec"], ents, rels, side, k, mask=mask, engine=eng, chunk=8)
    assert eng.projected == _relations_with(rels)
    P, which = case["P"], "tail" if side == _lib.SIDE_TAIL else "head"
    if case["kind"] == "transh":
        s = transh_oracle.scores_all(P, transh_oracle.projections(P), ents, ents, rels, which)
    else:
        s = transd_oracle.scores_all(P, ents, ents, rels, which, case["spec"].scalars)
    s = s.clone()
    offs, ids = mask
    for i in range(ents.shape[0]):
        s[i, ids[offs[i]:offs[i + 1]]] = float("-inf")
    cand = torch.arange(N_ENT).expand(ents.shape[0], N_ENT)
    order = key_order(s, cand)[:, :k]
    assert torch.equal(pred, cand.gather(1, order))
    assert torch.equal(vals.view(torch.int32), s.gather(1, order).view(torch.int32))
