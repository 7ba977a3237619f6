"""TransD without a GPU: the projection arithmetic the kernels are made of against ATen, bit for bit; RNG and
state_dict compatibility with the reference's TransDModel; and every unsupported call raising before any
device work."""
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
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    out = str(tmp_path_factory.mktemp("host_transd") / "host_transd.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I",
                           os.path.join(ROOT, "tests", "host_shim"), os.path.join(ROOT, "tests", "host_transd.cpp"),
                           "-o", out])
    lib = ctypes.CDLL(out)
    lib.host_transd_project.argtypes = [ctypes.c_int, ctypes.c_int, P, ctypes.c_float, P, P]
    return lib


def _same_bits(got, want):
    return (got.view(torch.int32) == want.view(torch.int32)) | (got == want)


@pytest.mark.parametrize("dims", [range(1, 1002), [1024, 2048, 4095, 4096, 6000, 8191, 8192]],
                         ids=["1-1001", "up_to_8192"])
def test_entity_scalar_equals_aten(dims, host_lib):
    """evaluate_projectionss (translation.py:645) sums one entity's (ent_proj_vect * ent) over ent_emb_dim as a
    1-D tensor: the device function must give those bits for every width."""
    g = torch.Generator().manual_seed(17)
    for d in dims:
        ent = torch.rand(3, d, generator=g) * 2 - 1
        ep = torch.rand(3, d, generator=g) * 2 - 1
        ep[1, : d // 2] = 0.0
        want = torch.stack([(ep[i] * ent[i]).sum(dim=0) for i in range(3)])
        en, epn = ent.numpy().copy(), ep.numpy().copy()
        out = np.full(3, np.nan, dtype=np.float32)
        assert host_lib.host_transd_scalars(d, 3, P(en.ctypes.data), P(epn.ctypes.data), P(out.ctypes.data)) == 0
        same = _same_bits(torch.from_numpy(out), want)
        assert same.all(), "ent_dim=%d: %d of 3 scalars differ" % (d, int((~same).sum()))


@pytest.mark.parametrize("n_rel", [1, 3, 300])
@pytest.mark.parametrize("ent_dim,rel_dim", [(1, 1), (9, 1), (8, 8), (37, 37), (50, 37), (100, 100), (200, 64)])
def test_projection_equals_the_reference_expression(n_rel, ent_dim, rel_dim, host_lib):
    """sc_prod * rel_proj_vects + ent[:rel_emb_dim].view(1, -1) (translation.py:646), bit for bit."""
    g = torch.Generator().manual_seed(n_rel * 1000 + ent_dim * 10 + rel_dim)
    ent = torch.rand(ent_dim, generator=g) * 2 - 1
    ep = torch.rand(ent_dim, generator=g) * 2 - 1
    rel_proj_vects = torch.nn.functional.normalize(torch.rand(n_rel, rel_dim, generator=g) * 2 - 1, p=2, dim=1)
    sc_prod = (ep * ent).sum(dim=0)
    want = sc_prod * rel_proj_vects + ent[:rel_dim].view(1, -1)
    en, rp = ent.numpy().copy(), rel_proj_vects.numpy().copy()
    out = np.full((n_rel, rel_dim), np.nan, dtype=np.float32)
    assert host_lib.host_transd_project(rel_dim, n_rel, P(en.ctypes.data), float(sc_prod), P(rp.ctypes.data),
                                       P(out.ctypes.data)) == 0
    same = _same_bits(torch.from_numpy(out), want)
    assert same.all(), "%d of %d components differ" % (int((~same).sum()), same.numel())


def test_same_seed_same_weights_and_state_dict_keys():
    torch.manual_seed(5)
    a = tk.TransDModel(12, 7, 30, 4)
    torch.manual_seed(5)
    b = tk.TransDModel(12, 7, 30, 4)
    assert list(a.state_dict()) == ["ent_emb.weight", "rel_emb.weight", "ent_proj_vect.weight",
                                    "rel_proj_vect.weight"]
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k])
    assert a.evaluated_projections is False
    assert (a.ent_emb_dim, a.rel_emb_dim) == (12, 7)


def test_loads_a_checkpoint_with_projected_entities_strictly():
    src = tk.TransDModel(8, 6, 20, 3)
    state = dict(src.state_dict())
    state["projected_entities"] = torch.empty(3, 20, 6)
    dst = tk.TransDModel(8, 6, 20, 3)
    dst.load_state_dict(state)            # strict=True
    for k in src.state_dict():
        assert torch.equal(dst.state_dict()[k], src.state_dict()[k])


def _reference_transd():
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchkge")):
        pytest.skip("the reference package (oracle/_ref) is not built here")
    sys.path.insert(0, ref)
    try:
        from torchkge.models import TransDModel
    finally:
        sys.path.remove(ref)
    return TransDModel


@pytest.mark.parametrize("ent_dim,rel_dim", [(10, 10), (10, 4)])
def test_rng_parity_and_state_dict_round_trip_with_the_reference(ent_dim, rel_dim):
    RefTransD = _reference_transd()
    torch.manual_seed(9)
    ref = RefTransD(ent_dim, rel_dim, 25, 4)
    torch.manual_seed(9)
    ours = tk.TransDModel(ent_dim, rel_dim, 25, 4)
    for k, v in ours.state_dict().items():      # same RNG calls in the same order
        assert torch.equal(v, ref.state_dict()[k]), k
    mine = tk.TransDModel(ent_dim, rel_dim, 25, 4)
    mine.load_state_dict(ref.state_dict())      # strict in
    back = RefTransD(ent_dim, rel_dim, 25, 4)
    res = back.load_state_dict(mine.state_dict(), strict=False)   # strict=False out
    assert list(res.missing_keys) == ["projected_entities"] and not res.unexpected_keys
    for k, v in mine.state_dict().items():
        assert torch.equal(back.state_dict()[k], v)


def test_project_normalize_and_get_embeddings_keep_the_reference_bodies():
    m = tk.TransDModel(6, 4, 9, 2)
    e, ep, rp = torch.rand(5, 6), torch.rand(5, 6), torch.rand(5, 4)
    assert torch.equal(m.project(e, ep, rp), rp * (e * ep).sum(dim=1).view(5, 1) + e[:, :4])
    m.rel_proj_vect.weight.data *= 3.0
    ent, rel, ent_proj, rel_proj = m.get_embeddings()
    for x in (ent, rel, ent_proj, rel_proj):
        assert torch.allclose(x.norm(dim=1), torch.ones(x.shape[0]))


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


def test_rel_dim_above_ent_dim_raises_before_any_device_work(monkeypatch):
    _no_cuda(monkeypatch)
    m, kg = tk.TransDModel(4, 6, 5, 2), _kg()
    ents, rels = torch.tensor([0, 1]), torch.tensor([0, 1])
    calls = [lambda: tk.LinkPredictionEvaluator(m, kg).evaluate(8),
             lambda: tk.RelationPredictionEvaluator(m, kg).evaluate(8),
             lambda: tk.EntityInference(m, ents, rels, top_k=1).evaluate(8),
             lambda: tk.RelationInference(m, ents, rels, top_k=1).evaluate(8),
             lambda: m.scoring_function(ents, ents, rels)]
    for call in calls:
        with pytest.raises(ValueError, match="rel_emb_dim <= ent_emb_dim"):
            call()


@pytest.mark.parametrize("shard", [QueryShard(3, 0, 2), EntityShard(5, 0, 2), EntityShard(5, 0, 1)])
def test_sharded_calls_raise_before_any_collective(shard, monkeypatch):
    _no_cuda(monkeypatch)
    import torch.distributed as dist
    monkeypatch.setattr(dist, "all_reduce", lambda *a, **k: pytest.fail("collective reached"))
    monkeypatch.setattr(dist, "all_gather", lambda *a, **k: pytest.fail("collective reached"))
    m, kg = tk.TransDModel(4, 3, 5, 2), _kg()
    ents, rels = torch.tensor([0, 1]), torch.tensor([0, 1])
    calls = [lambda: tk.LinkPredictionEvaluator(m, kg, shard=shard).evaluate(8),
             lambda: tk.RelationPredictionEvaluator(m, kg, shard=shard).evaluate(8),
             lambda: tk.EntityInference(m, ents, rels, top_k=1, shard=shard).evaluate(8),
             lambda: tk.RelationInference(m, ents, rels, top_k=1, shard=shard).evaluate(8),
             lambda: tk.TripletClassificationEvaluator(m, kg, kg, shard=shard)]
    for call in calls:
        with pytest.raises(NotImplementedError, match="TransDModel does not support shard"):
            call()


def test_fused_step_raises_before_any_kernel_or_draw(monkeypatch):
    _no_cuda(monkeypatch)
    m, kg = tk.TransDModel(4, 3, 5, 2), _kg()
    h, t, r = kg.head_idx, kg.tail_idx, kg.relations
    for sampler in (tk.BernoulliNegativeSampler(kg), tk.UniformNegativeSampler(kg), tk.PositionalNegativeSampler(kg)):
        calls = sampler._calls if hasattr(sampler, "_calls") else None
        with pytest.raises(NotImplementedError, match="TransDModel has no fused training step"):
            sampler.fused_step(m, h, t, r, margin=1.0)
        with pytest.raises(NotImplementedError, match="TransDModel has no fused training step"):
            sampler.fused_step(m, h, t, r, criterion=tk.LogisticLoss())
        if calls is not None:
            assert sampler._calls == calls       # no draw was consumed
    from torchkge_b200.training import fused_margin_step
    with pytest.raises(NotImplementedError, match="TransDModel has no fused training step"):
        fused_margin_step(m, h, t, r, 1.0)


def test_candidate_tensors_and_other_model_paths_raise():
    m = tk.TransDModel(4, 3, 5, 2)
    idx = torch.tensor([0, 1])
    with pytest.raises(NotImplementedError, match="EntityInference"):
        m.inference_prepare_candidates(idx, idx, idx)
    with pytest.raises(NotImplementedError, match="EntityInference"):
        m.lp_prep_cands(idx, idx, idx, entities=False)
    with pytest.raises(NotImplementedError):
        m.inference_scoring_function(None, None, None)
    with pytest.raises(NotImplementedError, match="fused training step or shard"):
        ModelSpec.from_model(m)


def test_host_model_has_no_cpu_fallback():
    m, kg = tk.TransDModel(4, 3, 5, 2), _kg()
    idx = torch.tensor([0, 1])
    with pytest.raises(_lib.KgeLibraryError, match="CPU fallback"):
        m.scoring_function(idx, idx, idx)
    with pytest.raises(_lib.KgeLibraryError, match="CUDA device"):
        tk.LinkPredictionEvaluator(m, kg).evaluate(8)
