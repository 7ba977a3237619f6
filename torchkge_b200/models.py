"""Embedding models with the reference's class names, constructor arguments, parameter names
and method signatures (torchkge/models/interfaces.py, translation.py:18-125,
bilinear.py:14-267, 414-556), whose scoring bodies are calls into the CUDA engine.

Only what lies on the hot path is here: TransE (L1 / L2), TransH, TransD, TorusE, DistMult, RESCAL,
ComplEx, Analogy and the RotatE addition.  ``state_dict`` keys equal the reference's, so weights move freely between
the two packages.  The pre-0.17 method names ``lp_prep_cands`` / ``lp_scoring_function``
(docs/history.rst:37-42) are kept as aliases.
"""
import math

import torch
from torch import nn
from torch.nn.functional import normalize

from . import _lib
from .engine import ModelSpec, _device_guard, default_engine


def init_embedding(n_vectors, dim):
    """nn.Embedding with Xavier-uniform weights (torchkge/utils/modeling.py:21-28).  Same RNG
    calls in the same order as the reference, so equal seeds give equal weights."""
    emb = nn.Embedding(n_vectors, dim)
    nn.init.xavier_uniform_(emb.weight.data)
    return emb


def l1_dissimilarity(a, b):
    """torchkge/utils/dissimilarities.py:11-16.  The models use the function's IDENTITY to select
    the L1 kernels (interfaces.py:205-208 does the same); calling it evaluates the reference's
    expression with tensor ops on the tensors' device, for user code that does
    ``model.dissimilarity(x, y)``."""
    assert len(a.shape) == len(b.shape)
    return (a - b).norm(p=1, dim=-1)


def l2_dissimilarity(a, b):
    """torchkge/utils/dissimilarities.py:19-25 (2-norm first, then squared); see l1_dissimilarity."""
    assert len(a.shape) == len(b.shape)
    return (a - b).norm(p=2, dim=-1) ** 2


class Model(nn.Module):
    """Interface of every model (torchkge/models/interfaces.py:13-174)."""

    def __init__(self, n_entities, n_relations):
        super().__init__()
        self.n_ent = n_entities
        self.n_rel = n_relations

    # ---- training-side API -------------------------------------------------------------
    def forward(self, heads, tails, relations, negative_heads, negative_tails,
                negative_relations=None):
        """(pos, neg) scores; several negatives per fact are laid out as n_neg blocks of the
        batch (interfaces.py:39-82)."""
        pos = self.scoring_function(heads, tails, relations)
        if negative_relations is None:
            negative_relations = relations
        if negative_heads.shape[0] > negative_relations.shape[0]:
            n_neg = int(negative_heads.shape[0] / negative_relations.shape[0])
            pos = pos.repeat(n_neg)
            neg = self.scoring_function(negative_heads, negative_tails,
                                        negative_relations.repeat(n_neg))
        else:
            neg = self.scoring_function(negative_heads, negative_tails, negative_relations)
        return pos, neg

    def scoring_function(self, h_idx, t_idx, r_idx):
        raise NotImplementedError

    def normalize_parameters(self):
        raise NotImplementedError

    def get_embeddings(self):
        raise NotImplementedError

    # ---- inference-side API ------------------------------------------------------------
    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        raise NotImplementedError

    def inference_scoring_function(self, h, t, r):
        """Scores of (h, r, c) or (c, r, t) for every candidate c, shape (b, n_candidates).

        Exactly one of ``h`` / ``t`` is the 3-D candidates tensor returned by
        ``inference_prepare_candidates`` (a stride-0 expansion of the entity table); the
        scores come from the same CUDA scan the evaluator uses, written out densely.
        """
        return _dense_scores(self, h, t, r)

    # pre-0.17 names
    def lp_prep_cands(self, h_idx, t_idx, r_idx, entities=True):
        return self.inference_prepare_candidates(h_idx, t_idx, r_idx, entities=entities)

    def lp_scoring_function(self, h, t, r):
        return self.inference_scoring_function(h, t, r)

    # ---- helpers -----------------------------------------------------------------------
    def _kernel_code(self):
        return ModelSpec.from_model(self).code

    def _expand(self, weight, b_size):
        n, d = weight.shape
        return weight.data.view(1, n, d).expand(b_size, n, d)


def _as_planes(x):
    """Tensor or (re, im) tuple -> list of tensors."""
    return list(x) if isinstance(x, (tuple, list)) else [x]


def _dense_scores(model, h, t, r):
    hp, tp, rp = _as_planes(h), _as_planes(t), _as_planes(r)
    if (rp[0].dim() == 3 and hp[0].dim() == 2 and tp[0].dim() == 2
            and type(model).__name__ != "RESCALModel"):
        return _dense_relation_scores(model, hp, tp, rp)
    if type(model).__name__ == "RESCALModel" and rp[0].dim() == 4 and hp[0].dim() == 2 and tp[0].dim() == 2:
        return _rescal_relation_scores(model, hp[0], tp[0], rp[0])
    if rp[0].dim() != 2 and not (type(model).__name__ == "RESCALModel" and rp[0].dim() == 3):
        raise NotImplementedError("relation-prediction scoring (candidate relations) is not on "
                                  "the CUDA path for this model")
    if tp[0].dim() == 3 and hp[0].dim() == 2:
        side, cand, ent = _lib.SIDE_TAIL, tp, hp
    elif hp[0].dim() == 3 and tp[0].dim() == 2:
        side, cand, ent = _lib.SIDE_HEAD, hp, tp
    else:
        raise ValueError("exactly one of h / t must be the 3-D candidates tensor")
    for c in cand:
        if c.shape[0] > 1 and c.stride(0) != 0:
            raise NotImplementedError("per-row candidate tensors are not supported: pass the "
                                      "tensor returned by inference_prepare_candidates")
    if not ent[0].is_cuda:
        raise _lib.KgeLibraryError("inference_scoring_function needs CUDA tensors; there is no "
                                   "CPU fallback")
    b, n_cand, d = cand[0].shape
    tables = [c[0].detach().contiguous() for c in cand]
    code = model._kernel_code()
    rel = [x.detach().contiguous().view(b, -1) for x in rp]
    if code == _lib.ROTATE:
        # inference_prepare_candidates hands out (cos, sin) planes for RotatE
        pass
    if code == _lib.ANALOGY:    # three planes: equally spaced views of one stacked copy
        tables, rel = list(ModelSpec.stacked(tables)), list(ModelSpec.stacked(rel))
    spec = ModelSpec(code, d, n_cand, b, tables[0], tables[1] if len(tables) > 1 else None,
                     rel[0], rel[1] if len(rel) > 1 else None,
                     ent2=tables[2] if len(tables) > 2 else None, rel2=rel[2] if len(rel) > 2 else None)
    eng = default_engine()
    rows = torch.stack([x.detach().contiguous() for x in ent], dim=1).contiguous()  # (b, planes, d)
    with _device_guard(rows.device):
        # the scan layout is rebuilt on every call (2 x table bytes of traffic, small next to the
        # b x n_cand scan): a cache keyed on data_ptr / _version would go stale under in-place
        # updates through ``.data`` (optimizer steps on .data, ``weight.data.frac_()``)
        packed = eng.pack(spec)
        return eng.score_all(spec, packed, side, rows, rows, None)


def _dense_relation_scores(model, hp, tp, rp):
    """The relation case of ``inference_scoring_function`` (interfaces.py:261-272,
    bilinear.py:241-245, 524-528): ``r`` is the (b, n_rel, d) candidates tensor returned by
    ``inference_prepare_candidates(..., entities=False)``; scores of (h, c, t) for every relation c,
    from ``kge_score_all`` with ``KGE_SIDE_REL`` (same arithmetic as RelationPredictionEvaluator)."""
    from .engine import relation_spec
    for c in rp:
        if c.shape[0] > 1 and c.stride(0) != 0:
            raise NotImplementedError("per-row candidate tensors are not supported: pass the "
                                      "tensor returned by inference_prepare_candidates")
    if not hp[0].is_cuda:
        raise _lib.KgeLibraryError("inference_scoring_function needs CUDA tensors; there is no "
                                   "CPU fallback")
    b, n_rel, d = rp[0].shape
    tables = [c[0].detach().contiguous() for c in rp]
    code = model._kernel_code()
    if code == _lib.ANALOGY:
        cands = ModelSpec.stacked(tables)
        rspec = ModelSpec(code, d, n_rel, n_rel, cands[0], cands[1], None, None, ent2=cands[2])
    else:
        rspec = relation_spec(ModelSpec(code, d, model.n_ent, n_rel, tables[0], None, tables[0],
                                        tables[1] if len(tables) > 1 else None))
    eng = default_engine()
    hrows = torch.stack([x.detach().contiguous() for x in hp], dim=1).contiguous()  # (b, planes, d)
    trows = torch.stack([x.detach().contiguous() for x in tp], dim=1).contiguous()
    with _device_guard(hrows.device):
        packed = eng.pack(rspec)       # rebuilt per call, see _dense_scores
        return eng.score_all(rspec, packed, _lib.SIDE_REL, hrows, trows, None)


def _rescal_relation_scores(model, h, t, cands):
    """RESCAL's relation case of ``inference_scoring_function`` (bilinear.py:115-121): ``cands`` is
    the (b, n_rel, d, d) expansion of ``rel_mat`` returned by ``inference_prepare_candidates(...,
    entities=False)``; scores ((h^T M_c) * t).sum() for every relation c (kge_rescal_rel_scores)."""
    if cands.shape[0] > 1 and cands.stride(0) != 0:
        raise NotImplementedError("per-row candidate tensors are not supported: pass the tensor returned by "
                                  "inference_prepare_candidates")
    if not h.is_cuda:
        raise _lib.KgeLibraryError("inference_scoring_function needs CUDA tensors; there is no CPU fallback")
    b, n_rel, d, _ = cands.shape
    mats = cands[0].detach().contiguous().view(n_rel, d * d)
    spec = ModelSpec(_lib.RESCAL, d, model.n_ent, n_rel, h.detach(), None, mats, None)
    with _device_guard(h.device):
        return default_engine().rescal_rel_scores(spec, h.detach().contiguous(), t.detach().contiguous())


def l1_torus_dissimilarity(a, b):
    """torchkge/utils/dissimilarities.py:28-34 (also the selector of the torus-L1 kernels)."""
    return 2 * torch.min(torch.abs(a - b), 1 - torch.abs(a - b)).sum(dim=-1)


def l2_torus_dissimilarity(a, b):
    """torchkge/utils/dissimilarities.py:37-43 (also the selector of the torus-L2 kernels)."""
    return 4 * torch.min((a - b) ** 2, 1 - (a - b) ** 2).sum(dim=-1)


class TranslationModel(Model):
    """torchkge/models/interfaces.py:177-272; 'L1', 'L2', 'torus_L1' and 'torus_L2' have kernels
    ('torus_eL2' goes through a cosine and is not on the CUDA path)."""

    def __init__(self, n_entities, n_relations, dissimilarity_type):
        super().__init__(n_entities, n_relations)
        assert dissimilarity_type in ['L1', 'L2', 'torus_L1', 'torus_L2', 'torus_eL2']
        if dissimilarity_type == 'L1':
            self.dissimilarity = l1_dissimilarity
        elif dissimilarity_type == 'L2':
            self.dissimilarity = l2_dissimilarity
        elif dissimilarity_type == 'torus_L1':
            self.dissimilarity = l1_torus_dissimilarity
        elif dissimilarity_type == 'torus_L2':
            self.dissimilarity = l2_torus_dissimilarity
        else:
            raise NotImplementedError("torus_eL2 (cosine-based) is outside the CUDA path")


class BilinearModel(Model):
    """torchkge/models/interfaces.py:275-330"""

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(n_entities, n_relations)
        self.emb_dim = emb_dim


class TransEModel(TranslationModel):
    """TransE (Bordes et al. 2013) -- torchkge/models/translation.py:18-125."""

    def __init__(self, emb_dim, n_entities, n_relations, dissimilarity_type='L2'):
        super().__init__(n_entities, n_relations, dissimilarity_type)
        self.emb_dim = emb_dim
        self.ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_emb = init_embedding(self.n_rel, self.emb_dim)
        self.normalize_parameters()
        self.rel_emb.weight.data = normalize(self.rel_emb.weight.data, p=2, dim=1)

    def scoring_function(self, h_idx, t_idx, r_idx):
        from .training import score_triples
        return score_triples(self, h_idx, t_idx, r_idx)

    def normalize_parameters(self):
        self.ent_emb.weight.data = normalize(self.ent_emb.weight.data, p=2, dim=1)

    def get_embeddings(self):
        self.normalize_parameters()
        return self.ent_emb.weight.data, self.rel_emb.weight.data

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        h, t, r = self.ent_emb(h_idx), self.ent_emb(t_idx), self.rel_emb(r_idx)
        cands = self._expand(self.ent_emb.weight if entities else self.rel_emb.weight, b)
        return h, t, r, cands


class ProjectedTranslationModel(TranslationModel):
    """TransH and TransD: TransE-L2 between per-relation projections of h and t, ranked here without the
    reference's (n_rel, n_ent, width) ``projected_entities`` cache.  A subclass names that width in
    ``cand_width``, for the error messages."""

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        raise NotImplementedError(
            "%s has no inference_prepare_candidates: the reference's candidates are a per-row "
            "(b, n_ent, %s) tensor of projected entities.  Use LinkPredictionEvaluator, "
            "RelationPredictionEvaluator, EntityInference or RelationInference, which project on the GPU."
            % (type(self).__name__, self.cand_width))

    def inference_scoring_function(self, h, t, r):
        raise NotImplementedError(
            "%s has no inference_scoring_function: use LinkPredictionEvaluator, "
            "RelationPredictionEvaluator, EntityInference or RelationInference." % type(self).__name__)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        # a reference checkpoint carries its projection cache: not a parameter here
        state_dict.pop(prefix + "projected_entities", None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)


class TransHModel(ProjectedTranslationModel):
    """TransH (Wang et al. 2014) -- torchkge/models/translation.py:128-284: TransE-L2 between the
    projections of h and t on a relation-specific hyperplane of normal vector ``norm_vect``.

    There is no ``projected_entities`` cache: the reference fills an (n_rel, n_ent, emb_dim) tensor
    (translation.py:179-181, 270-284), 8 GB at FB15k's size.  Link prediction and ``EntityInference``
    project the entity table on the GPU for one relation at a time, on every call; relation prediction
    and ``RelationInference`` project the two rows of each fact on the fly.  A reference checkpoint
    loads here with the default ``strict=True`` (its ``projected_entities`` entry is discarded); this
    model's ``state_dict`` loads into the reference with ``strict=False``.

    ``inference_prepare_candidates`` / ``inference_scoring_function`` are not available: the
    reference's entity candidates are a per-row (b, n_ent, emb_dim) tensor.  Use
    ``LinkPredictionEvaluator``, ``RelationPredictionEvaluator``, ``EntityInference`` or
    ``RelationInference``.  Out of scope: the fused training step and ``shard=``.
    """

    cand_width = "emb_dim"

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(n_entities, n_relations, dissimilarity_type='L2')
        self.emb_dim = emb_dim
        self.ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_emb = init_embedding(self.n_rel, self.emb_dim)
        self.norm_vect = init_embedding(self.n_rel, self.emb_dim)
        self.normalize_parameters()
        self.evaluated_projections = False

    def scoring_function(self, h_idx, t_idx, r_idx):
        """-||P(h~) + r - P(t~)||^2 with h, t and the normal vector L2-normalised (translation.py:183-198),
        on the per-triple kernels kge_transh_score_triples_fwd / _bwd."""
        self.evaluated_projections = False
        from .training import score_triples_transh
        return score_triples_transh(self, h_idx, t_idx, r_idx)

    @staticmethod
    def project(ent, norm_vect):
        return ent - (ent * norm_vect).sum(dim=1).view(-1, 1) * norm_vect

    def normalize_parameters(self):
        self.ent_emb.weight.data = normalize(self.ent_emb.weight.data, p=2, dim=1)
        self.norm_vect.weight.data = normalize(self.norm_vect.weight.data, p=2, dim=1)
        self.rel_emb.weight.data = self.project(self.rel_emb.weight.data, self.norm_vect.weight.data)

    def get_embeddings(self):
        self.normalize_parameters()
        return self.ent_emb.weight.data, self.rel_emb.weight.data, self.norm_vect.weight.data


class TransDModel(ProjectedTranslationModel):
    """TransD (Ji et al. 2015) -- torchkge/models/translation.py:461-652: TransE-L2 between the projections
    P_r(e) = (e . e_p) r_p + e[:rel_emb_dim] of h and t, with an entity projection vector e_p
    (``ent_proj_vect``, ent_emb_dim) and a relation projection vector r_p (``rel_proj_vect``, rel_emb_dim).

    There is no ``projected_entities`` cache: the reference fills an (n_rel, n_ent, rel_emb_dim) tensor
    (translation.py:533-536, 629-652), 8 GB at FB15k's size.  Link prediction and ``EntityInference``
    compute every entity's scalar e . e_p once per call and project the entity table on the GPU for one
    relation at a time; relation prediction and ``RelationInference`` project the two rows of each fact on
    the fly.  Unlike the reference, which ranks on projections cached until the next ``scoring_function``
    call, every call projects the current weights.  A reference checkpoint loads here with the default
    ``strict=True`` (its ``projected_entities`` entry is discarded); this model's ``state_dict`` loads into
    the reference with ``strict=False``.  ``rel_emb_dim`` may not exceed ``ent_emb_dim``.

    ``inference_prepare_candidates`` / ``inference_scoring_function`` are not available: the
    reference's entity candidates are a per-row (b, n_ent, rel_emb_dim) tensor.  Use
    ``LinkPredictionEvaluator``, ``RelationPredictionEvaluator``, ``EntityInference`` or
    ``RelationInference``.  Out of scope: the fused training step and ``shard=``.
    """

    cand_width = "rel_emb_dim"

    def __init__(self, ent_emb_dim, rel_emb_dim, n_entities, n_relations):
        super().__init__(n_entities, n_relations, dissimilarity_type='L2')
        self.ent_emb_dim = ent_emb_dim
        self.rel_emb_dim = rel_emb_dim
        self.ent_emb = init_embedding(self.n_ent, self.ent_emb_dim)
        self.rel_emb = init_embedding(self.n_rel, self.rel_emb_dim)
        self.ent_proj_vect = init_embedding(self.n_ent, self.ent_emb_dim)
        self.rel_proj_vect = init_embedding(self.n_rel, self.rel_emb_dim)
        self.normalize_parameters()
        self.evaluated_projections = False

    def scoring_function(self, h_idx, t_idx, r_idx):
        """-||P(h~) + r~ - P(t~)||^2 with h, t, r and the three projection vectors L2-normalised
        (translation.py:538-556), on the per-triple kernels kge_transd_score_triples_fwd / _bwd."""
        self.evaluated_projections = False
        from .training import score_triples_transd
        return score_triples_transd(self, h_idx, t_idx, r_idx)

    def project(self, ent, e_proj_vect, r_proj_vect):
        b_size = ent.shape[0]
        scalar_product = (ent * e_proj_vect).sum(dim=1)
        proj_e = (r_proj_vect * scalar_product.view(b_size, 1))
        return proj_e + ent[:, :self.rel_emb_dim]

    def normalize_parameters(self):
        self.ent_emb.weight.data = normalize(self.ent_emb.weight.data, p=2, dim=1)
        self.rel_emb.weight.data = normalize(self.rel_emb.weight.data, p=2, dim=1)
        self.ent_proj_vect.weight.data = normalize(self.ent_proj_vect.weight.data, p=2, dim=1)
        self.rel_proj_vect.weight.data = normalize(self.rel_proj_vect.weight.data, p=2, dim=1)

    def get_embeddings(self):
        self.normalize_parameters()
        return self.ent_emb.weight.data, self.rel_emb.weight.data, \
            self.ent_proj_vect.weight.data, self.rel_proj_vect.weight.data


class DistMultModel(BilinearModel):
    """DistMult (Yang et al. 2014) -- torchkge/models/bilinear.py:146-267."""

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(emb_dim, n_entities, n_relations)
        self.ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_emb = init_embedding(self.n_rel, self.emb_dim)
        self.normalize_parameters()

    def scoring_function(self, h_idx, t_idx, r_idx):
        from .training import score_triples
        return score_triples(self, h_idx, t_idx, r_idx)

    def normalize_parameters(self):
        self.ent_emb.weight.data = normalize(self.ent_emb.weight.data, p=2, dim=1)

    def get_embeddings(self):
        self.normalize_parameters()
        return self.ent_emb.weight.data, self.rel_emb.weight.data

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        h, t, r = self.ent_emb(h_idx), self.ent_emb(t_idx), self.rel_emb(r_idx)
        cands = self._expand(self.ent_emb.weight if entities else self.rel_emb.weight, b)
        return h, t, r, cands


class RESCALModel(BilinearModel):
    """RESCAL (Nickel et al. 2011) -- torchkge/models/bilinear.py:14-143."""

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(emb_dim, n_entities, n_relations)
        self.ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_mat = init_embedding(self.n_rel, self.emb_dim * self.emb_dim)
        self.normalize_parameters()

    def scoring_function(self, h_idx, t_idx, r_idx):
        from .training import score_triples
        return score_triples(self, h_idx, t_idx, r_idx)

    def normalize_parameters(self):
        self.ent_emb.weight.data = normalize(self.ent_emb.weight.data, p=2, dim=1)

    def get_embeddings(self):
        self.normalize_parameters()
        return (self.ent_emb.weight.data,
                self.rel_mat.weight.data.view(-1, self.emb_dim, self.emb_dim))

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        h, t = self.ent_emb(h_idx), self.ent_emb(t_idx)
        r_mat = self.rel_mat(r_idx).view(-1, self.emb_dim, self.emb_dim)
        if entities:
            cands = self._expand(self.ent_emb.weight, b)
        else:
            cands = self.rel_mat.weight.data.view(1, self.n_rel, self.emb_dim, self.emb_dim)
            cands = cands.expand(b, self.n_rel, self.emb_dim, self.emb_dim)
        return h, t, r_mat, cands


class ComplExModel(BilinearModel):
    """ComplEx (Trouillon et al. 2016) -- torchkge/models/bilinear.py:414-556."""

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(emb_dim, n_entities, n_relations)
        self.re_ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.im_ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.re_rel_emb = init_embedding(self.n_rel, self.emb_dim)
        self.im_rel_emb = init_embedding(self.n_rel, self.emb_dim)

    def scoring_function(self, h_idx, t_idx, r_idx):
        from .training import score_triples
        return score_triples(self, h_idx, t_idx, r_idx)

    def normalize_parameters(self):
        pass

    def get_embeddings(self):
        return (self.re_ent_emb.weight.data, self.im_ent_emb.weight.data,
                self.re_rel_emb.weight.data, self.im_rel_emb.weight.data)

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        h = (self.re_ent_emb(h_idx), self.im_ent_emb(h_idx))
        t = (self.re_ent_emb(t_idx), self.im_ent_emb(t_idx))
        r = (self.re_rel_emb(r_idx), self.im_rel_emb(r_idx))
        if entities:
            cands = (self._expand(self.re_ent_emb.weight, b), self._expand(self.im_ent_emb.weight, b))
        else:
            cands = (self._expand(self.re_rel_emb.weight, b), self._expand(self.im_rel_emb.weight, b))
        return h, t, r, cands


class AnalogyModel(BilinearModel):
    """ANALOGY (Liu et al. 2017) -- torchkge/models/bilinear.py:559-763: DistMult on ``scalar_dim``
    coordinates plus ComplEx on ``complex_dim`` coordinates (scalar_share of emb_dim, half by default).

    Link prediction (tensor-core bound-and-refine over the concatenated planes, or the exact scalar
    scan), relation prediction and top-k inference run on the scan kernels with the
    three-plane element (csrc/reduce.cuh: EL_DOT3) and need scalar_dim == complex_dim -- as does the
    reference's own ``inference_scoring_function``, which adds the (b, n, scalar_dim) and
    (b, n, complex_dim) products element-wise (bilinear.py:695-698).  ``scoring_function`` runs on the
    per-triple kernels of csrc/train.cu under the same condition and is composed from torch ops
    otherwise.
    """

    def __init__(self, emb_dim, n_entities, n_relations, scalar_share=0.5):
        super().__init__(emb_dim, n_entities, n_relations)
        self.scalar_dim = int(self.emb_dim * scalar_share)
        self.complex_dim = int((self.emb_dim - self.scalar_dim))
        self.sc_ent_emb = init_embedding(self.n_ent, self.scalar_dim)
        self.re_ent_emb = init_embedding(self.n_ent, self.complex_dim)
        self.im_ent_emb = init_embedding(self.n_ent, self.complex_dim)
        self.sc_rel_emb = init_embedding(self.n_rel, self.scalar_dim)
        self.re_rel_emb = init_embedding(self.n_rel, self.complex_dim)
        self.im_rel_emb = init_embedding(self.n_rel, self.complex_dim)

    def scoring_function(self, h_idx, t_idx, r_idx):
        """(sc_h * sc_r * sc_t).sum(1) + Re(<h, r, conj(t)>) on the complex part (bilinear.py:634-650)."""
        if self.scalar_dim == self.complex_dim:
            from .training import score_triples     # kge_score_triples_fwd / _bwd (train.cu); CPU tensors raise
            return score_triples(self, h_idx, t_idx, r_idx)
        # unequal widths (scalar_share != 0.5 or an odd emb_dim): not a kernel configuration; the
        # reference's expression in torch ops on the model's device
        sc_h, re_h, im_h = self.sc_ent_emb(h_idx), self.re_ent_emb(h_idx), self.im_ent_emb(h_idx)
        sc_t, re_t, im_t = self.sc_ent_emb(t_idx), self.re_ent_emb(t_idx), self.im_ent_emb(t_idx)
        sc_r, re_r, im_r = self.sc_rel_emb(r_idx), self.re_rel_emb(r_idx), self.im_rel_emb(r_idx)
        return ((sc_h * sc_r * sc_t).sum(dim=1) +
                (re_h * (re_r * re_t + im_r * im_t) + im_h * (re_r * im_t - im_r * re_t)).sum(dim=1))

    def _kernel_code(self):
        if self.scalar_dim != self.complex_dim:
            raise NotImplementedError("Analogy on the CUDA path needs scalar_dim == complex_dim (got %d and %d)"
                                      % (self.scalar_dim, self.complex_dim))
        return _lib.ANALOGY

    def normalize_parameters(self):
        pass

    def get_embeddings(self):
        return (self.sc_ent_emb.weight.data, self.re_ent_emb.weight.data, self.im_ent_emb.weight.data,
                self.sc_rel_emb.weight.data, self.re_rel_emb.weight.data, self.im_rel_emb.weight.data)

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        h = (self.sc_ent_emb(h_idx), self.re_ent_emb(h_idx), self.im_ent_emb(h_idx))
        t = (self.sc_ent_emb(t_idx), self.re_ent_emb(t_idx), self.im_ent_emb(t_idx))
        r = (self.sc_rel_emb(r_idx), self.re_rel_emb(r_idx), self.im_rel_emb(r_idx))
        if entities:
            cands = tuple(self._expand(e.weight, b) for e in (self.sc_ent_emb, self.re_ent_emb, self.im_ent_emb))
        else:
            cands = tuple(self._expand(e.weight, b) for e in (self.sc_rel_emb, self.re_rel_emb, self.im_rel_emb))
        return h, t, r, cands


class RotatEModel(BilinearModel):
    """RotatE (Sun et al. 2019): score = -sum_k |h_k r_k - t_k|, r_k = exp(i theta_k).

    Not part of the reference; laid out like ``ComplExModel`` (separate real / imaginary
    entity tables, tuple-returning ``inference_prepare_candidates``) with relation phases in
    ``rel_emb``.  The oracle for it is oracle/kge_oracle.py:rotate_scores_all.
    """

    def __init__(self, emb_dim, n_entities, n_relations):
        super().__init__(emb_dim, n_entities, n_relations)
        self.re_ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.im_ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_emb = nn.Embedding(self.n_rel, self.emb_dim)
        nn.init.uniform_(self.rel_emb.weight.data, -math.pi, math.pi)

    def relation_planes(self):
        """(cos theta, sin theta) tables, shape (n_rel, emb_dim)."""
        ph = self.rel_emb.weight.detach()
        return torch.cos(ph), torch.sin(ph)

    def scoring_function(self, h_idx, t_idx, r_idx):
        from .training import score_triples
        return score_triples(self, h_idx, t_idx, r_idx)

    def normalize_parameters(self):
        pass

    def get_embeddings(self):
        return self.re_ent_emb.weight.data, self.im_ent_emb.weight.data, self.rel_emb.weight.data

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        if not entities:
            raise NotImplementedError("RotatE relation prediction is not implemented")
        b = h_idx.shape[0]
        h = (self.re_ent_emb(h_idx), self.im_ent_emb(h_idx))
        t = (self.re_ent_emb(t_idx), self.im_ent_emb(t_idx))
        ph = self.rel_emb(r_idx)
        r = (torch.cos(ph), torch.sin(ph))
        cands = (self._expand(self.re_ent_emb.weight, b), self._expand(self.im_ent_emb.weight, b))
        return h, t, r, cands


class TorusEModel(TranslationModel):
    """TorusE (Ebisu & Ichise 2018) -- torchkge/models/translation.py:655-767: TransE on the torus
    [0, 1)^d (all parameters are kept as their fractional parts) with the torus dissimilarities.

    ``dissimilarity_type`` is 'torus_L1' or 'torus_L2' ('L1' on fractional parts is accepted too;
    'torus_eL2' is not on the CUDA path).  Link prediction (``LinkPredictionEvaluator``,
    ``inference_scoring_function``, ``EntityInference``) runs on the scan kernels with their own
    element kinds; ``scoring_function`` (training) with the torus dissimilarities runs on the per-triple
    kernels of csrc/train.cu (forward and backward; the fused margin step too), the plain 'L1' variant is
    composed from torch ops.
    """

    def __init__(self, emb_dim, n_entities, n_relations, dissimilarity_type):
        assert dissimilarity_type in ['L1', 'torus_L1', 'torus_L2', 'torus_eL2']
        super().__init__(n_entities, n_relations, dissimilarity_type)
        self.emb_dim = emb_dim
        self.ent_emb = init_embedding(self.n_ent, self.emb_dim)
        self.rel_emb = init_embedding(self.n_rel, self.emb_dim)
        self.normalized = False
        self.normalize_parameters()

    def scoring_function(self, h_idx, t_idx, r_idx):
        """-dissimilarity(frac(h) + frac(r), frac(t)) (translation.py:706-720)."""
        self.normalized = False
        if self.dissimilarity in (l1_torus_dissimilarity, l2_torus_dissimilarity):
            from .training import score_triples     # kge_score_triples_fwd / _bwd (train.cu); CPU tensors raise
            return score_triples(self, h_idx, t_idx, r_idx)
        # plain 'L1' on fractional parts: not a kernel configuration (the TransE-L1 kernels normalise rows)
        h, t, r = self.ent_emb(h_idx), self.ent_emb(t_idx), self.rel_emb(r_idx)
        h.data.frac_()
        t.data.frac_()
        r.data.frac_()
        if self.dissimilarity is l1_dissimilarity:
            return -(h + r - t).norm(p=1, dim=-1)
        return -self.dissimilarity(h + r, t)

    def normalize_parameters(self):
        self.ent_emb.weight.data.frac_()
        self.rel_emb.weight.data.frac_()
        self.normalized = True

    def get_embeddings(self):
        self.normalize_parameters()
        return self.ent_emb.weight.data, self.rel_emb.weight.data

    def inference_prepare_candidates(self, h_idx, t_idx, r_idx, entities=True):
        b = h_idx.shape[0]
        if not self.normalized:
            self.normalize_parameters()
        h, t, r = self.ent_emb(h_idx), self.ent_emb(t_idx), self.rel_emb(r_idx)
        cands = self._expand(self.ent_emb.weight if entities else self.rel_emb.weight, b)
        return h, t, r, cands

