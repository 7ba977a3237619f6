"""TransH without a GPU: the projection arithmetic the kernels are made of against ATen, bit for bit; state_dict
compatibility with the reference's TransHModel; and every unsupported call raising before any device work."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import torchkge_b200 as tk
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard, ModelSpec, QueryShard

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    out = str(tmp_path_factory.mktemp("host_transh") / "host_transh.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I",
                           os.path.join(ROOT, "tests", "host_shim"), os.path.join(ROOT, "tests", "host_transh.cpp"),
                           "-o", out])
    return ctypes.CDLL(out)


@pytest.mark.parametrize("n_rel", [1, 3, 7, 300])
def test_projection_equals_aten_for_every_dim(n_rel, host_lib):
    """evaluate_projections (translation.py:279-281) sums (1, d) x (n_rel, d) over d: the device function must
    give its bits for every dim 1..1001, whatever the number of relations (the outer size of the sum)."""
    g = torch.Generator().manual_seed(n_rel)
    P = ctypes.c_void_p
    for d in range(1, 1002):
        ent = torch.rand(1, d, generator=g) * 2 - 1
        W = torch.nn.functional.normalize(torch.rand(n_rel, d, generator=g) * 2 - 1, p=2, dim=1)
        if d > 2:
            W[0, : d // 2] = 0.0
        nc = (ent.view(1, -1) * W).sum(dim=1)
        want = ent.view(1, -1) - nc.view(-1, 1) * W
        en, Wn = ent.numpy().copy(), W.numpy().copy()
        out = np.full((n_rel, d), np.nan, dtype=np.float32)
        assert host_lib.host_transh_project(d, n_rel, P(en.ctypes.data), P(Wn.ctypes.data), P(out.ctypes.data)) == 0
        got = torch.from_numpy(out)
        same = (got.view(torch.int32) == want.view(torch.int32)) | (got == want)
        assert same.all(), "n_rel=%d d=%d: %d of %d components differ" % (n_rel, d, int((~same).sum()), same.numel())


def test_same_seed_same_weights_and_state_dict_keys():
    torch.manual_seed(5)
    a = tk.TransHModel(12, 30, 4)
    torch.manual_seed(5)
    b = tk.TransHModel(12, 30, 4)
    assert list(a.state_dict()) == ["ent_emb.weight", "rel_emb.weight", "norm_vect.weight"]
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k])
    assert a.evaluated_projections is False


def test_loads_a_checkpoint_with_projected_entities_strictly():
    src = tk.TransHModel(8, 20, 3)
    state = dict(src.state_dict())
    state["projected_entities"] = torch.empty(3, 20, 8)
    dst = tk.TransHModel(8, 20, 3)
    dst.load_state_dict(state)            # strict=True
    for k in ("ent_emb.weight", "rel_emb.weight", "norm_vect.weight"):
        assert torch.equal(dst.state_dict()[k], src.state_dict()[k])
    assert "projected_entities" in state  # load_state_dict discards it from its own copy


def _reference_transh():
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchkge")):
        pytest.skip("the reference package (oracle/_ref) is not built here")
    sys.path.insert(0, ref)
    try:
        from torchkge.models import TransHModel
    finally:
        sys.path.remove(ref)
    return TransHModel


def test_state_dict_round_trip_with_the_reference():
    RefTransH = _reference_transh()
    torch.manual_seed(9)
    ref = RefTransH(10, 25, 4)
    torch.manual_seed(9)
    ours = tk.TransHModel(10, 25, 4)
    for k, v in ours.state_dict().items():      # same RNG calls in the same order
        assert torch.equal(v, ref.state_dict()[k]), k
    mine = tk.TransHModel(10, 25, 4)
    mine.load_state_dict(ref.state_dict())      # strict in
    back = RefTransH(10, 25, 4)
    res = back.load_state_dict(mine.state_dict(), strict=False)   # strict=False out
    assert list(res.missing_keys) == ["projected_entities"] and not res.unexpected_keys
    for k, v in mine.state_dict().items():
        assert torch.equal(back.state_dict()[k], v)


def test_project_and_normalize_keep_the_reference_bodies():
    m = tk.TransHModel(6, 9, 2)
    e, w = torch.rand(4, 6), torch.rand(4, 6)
    assert torch.equal(m.project(e, w), e - (e * w).sum(dim=1).view(-1, 1) * w)
    m.rel_emb.weight.data += 1.0
    ent, rel, nv = m.get_embeddings()
    assert torch.allclose(nv.norm(dim=1), torch.ones(2))
    assert torch.allclose((rel * nv).sum(dim=1), torch.zeros(2), atol=1e-6)


# ---------------------------------------------------------------------------- out of scope
def _kg():
    h, t, r = torch.tensor([0, 1, 2]), torch.tensor([1, 2, 3]), torch.tensor([0, 1, 0])
    return tk.KnowledgeGraph(h, t, r, 5, 2)


def _no_cuda(monkeypatch):
    """Any attempt to reach a device fails the test instead of raising the expected error."""
    def boom(*a, **k):
        raise AssertionError("a device was touched")
    monkeypatch.setattr(torch.cuda, "current_stream", boom)
    monkeypatch.setattr(torch.cuda, "synchronize", boom)


@pytest.mark.parametrize("shard", [QueryShard(3, 0, 2), EntityShard(5, 0, 2), EntityShard(5, 0, 1)])
def test_sharded_calls_raise_before_any_collective(shard, monkeypatch):
    _no_cuda(monkeypatch)
    import torch.distributed as dist
    monkeypatch.setattr(dist, "all_reduce", lambda *a, **k: pytest.fail("collective reached"))
    monkeypatch.setattr(dist, "all_gather", lambda *a, **k: pytest.fail("collective reached"))
    m, kg = tk.TransHModel(4, 5, 2), _kg()
    ents, rels = torch.tensor([0, 1]), torch.tensor([0, 1])
    calls = [lambda: tk.LinkPredictionEvaluator(m, kg, shard=shard).evaluate(8),
             lambda: tk.RelationPredictionEvaluator(m, kg, shard=shard).evaluate(8),
             lambda: tk.EntityInference(m, ents, rels, top_k=1, shard=shard).evaluate(8),
             lambda: tk.RelationInference(m, ents, rels, top_k=1, shard=shard).evaluate(8),
             lambda: tk.TripletClassificationEvaluator(m, kg, kg, shard=shard)]
    for call in calls:
        with pytest.raises(NotImplementedError, match="shard"):
            call()


def test_fused_step_raises_before_any_kernel(monkeypatch):
    _no_cuda(monkeypatch)
    m, kg = tk.TransHModel(4, 5, 2), _kg()
    h, t, r = kg.head_idx, kg.tail_idx, kg.relations
    for sampler in (tk.BernoulliNegativeSampler(kg), tk.UniformNegativeSampler(kg), tk.PositionalNegativeSampler(kg)):
        calls = sampler._calls if hasattr(sampler, "_calls") else None
        with pytest.raises(NotImplementedError, match="fused training step"):
            sampler.fused_step(m, h, t, r, margin=1.0)
        with pytest.raises(NotImplementedError, match="fused training step"):
            sampler.fused_step(m, h, t, r, criterion=tk.LogisticLoss())
        if calls is not None:
            assert sampler._calls == calls       # no draw was consumed
    from torchkge_b200.training import fused_margin_step
    with pytest.raises(NotImplementedError, match="fused training step"):
        fused_margin_step(m, h, t, r, 1.0)


def test_candidate_tensors_and_other_model_paths_raise():
    m = tk.TransHModel(4, 5, 2)
    idx = torch.tensor([0, 1])
    with pytest.raises(NotImplementedError, match="EntityInference"):
        m.inference_prepare_candidates(idx, idx, idx)
    with pytest.raises(NotImplementedError, match="EntityInference"):
        m.lp_prep_cands(idx, idx, idx, entities=False)
    with pytest.raises(NotImplementedError):
        m.inference_scoring_function(None, None, None)
    with pytest.raises(NotImplementedError, match="fused training step or shard"):
        ModelSpec.from_model(m)


def test_scoring_function_has_no_cpu_fallback():
    m = tk.TransHModel(4, 5, 2)
    idx = torch.tensor([0, 1])
    with pytest.raises(_lib.KgeLibraryError, match="CPU fallback"):
        m.scoring_function(idx, idx, idx)
