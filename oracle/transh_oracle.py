"""CPU oracle for TransH (torchkge v0.17.7, models/translation.py:128-284) -- TEST INFRASTRUCTURE ONLY.

The reference's own operations, in the same order, in plain PyTorch CPU tensor ops, so that it produces the
reference's bits on the same machine:
  * projections          evaluate_projections (translation.py:270-284): for every entity e, one
                         (n_rel, dim) product with the normal vectors summed over dim, then e - nc * w
  * all-entity scores    inference_prepare_candidates (translation.py:237-256) + the translation-model
                         inference_scoring_function (interfaces.py:240-272) with the L2 dissimilarity
  * per-triple scores    scoring_function (translation.py:183-202)
The filter, rank and evaluator loops are those of ``kge_oracle``.  ``P`` holds the raw tables: ``ent``
(ent_emb.weight), ``rel`` (rel_emb.weight), ``norm`` (norm_vect.weight).  ``tests/test_oracle_transh_cpu.py``
requires this module to reproduce the reference's outputs stored in ``tests/golden/transh_*.npz``.
"""
import torch

from oracle.kge_oracle import filtered_scores, l2_diss, rank_of_true


def projections(P):
    """(n_rel, n_ent, dim) projected entities, entity by entity as evaluate_projections builds them."""
    E, W = P["ent"], P["norm"]
    n_rel, d = W.shape
    out = torch.empty((n_rel, E.shape[0], d), dtype=E.dtype)
    for i in range(E.shape[0]):
        ent = E[i:i + 1]
        nc = (ent.view(1, -1) * W).sum(dim=1)
        out[:, i, :] = ent.view(1, -1) - nc.view(-1, 1) * W
    return out


def scores_all(P, proj, h_idx, t_idx, r_idx, side):
    """(b, n_ent) scores of every entity as tail (side='tail') or head (side='head') of the facts."""
    b = h_idx.shape[0]
    d = P["ent"].shape[1]
    r = P["rel"][r_idx]
    cand = proj[r_idx]                          # (b, n_ent, d)
    if side == "tail":                          # interfaces.py:249-254
        hr = (proj[r_idx, h_idx] + r).view(b, 1, d)
        return -l2_diss(hr, cand)
    t_ = proj[r_idx, t_idx].view(b, 1, d)       # interfaces.py:256-260
    return -l2_diss(cand + r.view(b, 1, d), t_)


def link_prediction(P, heads, tails, rels, dict_of_heads, dict_of_tails, b_size, proj=None):
    """LinkPredictionEvaluator.evaluate (evaluation.py:263-308) on TransH: (rank_true_heads,
    rank_true_tails, filt_rank_true_heads, filt_rank_true_tails)."""
    proj = projections(P) if proj is None else proj
    n = heads.shape[0]
    out = [torch.empty(n, dtype=torch.long) for _ in range(4)]
    for lo in range(0, n, b_size):
        hi = min(n, lo + b_size)
        h, t, r = heads[lo:hi], tails[lo:hi], rels[lo:hi]
        s = scores_all(P, proj, h, t, r, "tail")
        out[1][lo:hi] = rank_of_true(s, t)
        out[3][lo:hi] = rank_of_true(filtered_scores(s, dict_of_tails, h, r, t), t)
        s = scores_all(P, proj, h, t, r, "head")
        out[0][lo:hi] = rank_of_true(s, h)
        out[2][lo:hi] = rank_of_true(filtered_scores(s, dict_of_heads, t, r, h), h)
    return tuple(out)


def relation_scores_all(P, proj, h_idx, t_idx):
    """(b, n_rel) scores of every relation for the pairs (h, t): the relation case of
    inference_prepare_candidates (translation.py:252-256) and inference_scoring_function
    (interfaces.py:261-272)."""
    b = h_idx.shape[0]
    d = P["ent"].shape[1]
    n_rel = P["rel"].shape[0]
    proj_h = proj[:, h_idx].transpose(0, 1).view(b, -1, d)
    proj_t = proj[:, t_idx].transpose(0, 1).view(b, -1, d)
    cands = P["rel"].view(1, n_rel, d).expand(b, n_rel, d)
    return -l2_diss(proj_h + cands, proj_t)


def relation_prediction(P, heads, tails, rels, dict_of_rels, b_size, directed=True, proj=None):
    """RelationPredictionEvaluator.evaluate (evaluation.py:64-112) on TransH: (rank_true_rels,
    filt_rank_true_rels); undirected as kge_oracle.relation_prediction."""
    proj = projections(P) if proj is None else proj
    n = heads.shape[0]
    out = [torch.empty(n, dtype=torch.long) for _ in range(2)]
    for lo in range(0, n, b_size):
        hi = min(n, lo + b_size)
        h, t, r = heads[lo:hi], tails[lo:hi], rels[lo:hi]
        s = relation_scores_all(P, proj, h, t)
        fs = filtered_scores(s, dict_of_rels, h, t, r)
        if not directed:
            s2 = relation_scores_all(P, proj, t, h)
            fs2 = filtered_scores(s2, dict_of_rels, h, t, r)
            s, fs = torch.cat((s, s2), dim=1), torch.cat((fs, fs2), dim=1)
        out[0][lo:hi] = rank_of_true(s, r)
        out[1][lo:hi] = rank_of_true(fs, r)
    return tuple(out)


def score_triples(P, h_idx, t_idx, r_idx):
    """scoring_function (translation.py:183-202); differentiable when the tables require grad."""
    nrm = torch.nn.functional.normalize
    h = nrm(P["ent"][h_idx], p=2, dim=1)
    t = nrm(P["ent"][t_idx], p=2, dim=1)
    r = P["rel"][r_idx]
    w = nrm(P["norm"][r_idx], p=2, dim=1)

    def project(e):
        return e - (e * w).sum(dim=1).view(-1, 1) * w
    return -l2_diss(project(h) + r, project(t))
