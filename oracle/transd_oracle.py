"""CPU oracle for TransD (torchkge v0.17.7, models/translation.py:461-652) -- TEST INFRASTRUCTURE ONLY.

The reference's own operations, in plain PyTorch CPU tensor ops, so that it produces the reference's bits on
the same machine, but relation by relation: it never builds the reference's (n_rel, n_ent, rel_emb_dim)
``projected_entities`` cache.
  * scalars              evaluate_projectionss (translation.py:645): s_e = (ent_proj_vect[e] * ent[e]).sum(dim=0),
                         one 1-D sum per entity as the reference's loop computes it
  * projections          translation.py:646: s_e * rel_proj_vect[r] + ent[e][:rel_emb_dim], element-wise, so one
                         relation's table (``projection``) has the bits of the reference's slice for it
  * all-entity scores    inference_prepare_candidates (translation.py:603-627) + the translation-model
                         inference_scoring_function (interfaces.py:240-272) with the L2 dissimilarity
  * per-triple scores    scoring_function (translation.py:538-568)
The filter, rank and evaluator loops are those of ``kge_oracle``; every row's rank depends on that row only, so
the facts are scored grouped by relation.  ``P`` holds the raw tables: ``ent`` (ent_emb.weight), ``rel``
(rel_emb.weight), ``ent_proj`` (ent_proj_vect.weight), ``rel_proj`` (rel_proj_vect.weight).
``tests/test_oracle_transd_cpu.py`` requires this module to reproduce the reference's outputs stored in
``tests/golden/transd_*.npz``.
"""
import torch

from oracle.kge_oracle import filtered_scores, l2_diss, rank_of_true


def scalars(P):
    """(n_ent,) s_e, each a 1-D sum over ent_emb_dim as evaluate_projectionss computes it."""
    E, EP = P["ent"], P["ent_proj"]
    return torch.stack([(EP[i] * E[i]).sum(dim=0) for i in range(E.shape[0])])


def projection(P, s, rel):
    """(n_ent, rel_emb_dim) entities projected for relation ``rel``: the reference's projected_entities[rel]."""
    d = P["rel"].shape[1]
    return s.view(-1, 1) * P["rel_proj"][rel].view(1, -1) + P["ent"][:, :d]


def _by_relation(rels):
    """[(relation, positions of the facts with that relation)]"""
    return [(int(r), (rels == r).nonzero().view(-1)) for r in torch.unique(rels)]


def scores_all(P, h_idx, t_idx, r_idx, side, s=None):
    """(b, n_ent) scores of every entity as tail (side='tail') or head (side='head') of the facts."""
    s = scalars(P) if s is None else s
    b, d = h_idx.shape[0], P["rel"].shape[1]
    out = torch.empty((b, P["ent"].shape[0]), dtype=P["ent"].dtype)
    for rel, pos in _by_relation(r_idx):
        proj = projection(P, s, rel)
        m = pos.shape[0]
        r = P["rel"][rel].view(1, d).expand(m, d)
        cand = proj.view(1, -1, d)
        if side == "tail":                                   # interfaces.py:249-254
            hr = (proj[h_idx[pos]] + r).view(m, 1, d)
            out[pos] = -l2_diss(hr, cand)
        else:                                                # interfaces.py:256-260
            t_ = proj[t_idx[pos]].view(m, 1, d)
            out[pos] = -l2_diss(cand + r.reshape(m, 1, d), t_)
    return out


def link_prediction(P, heads, tails, rels, dict_of_heads, dict_of_tails, b_size, s=None):
    """LinkPredictionEvaluator.evaluate (evaluation.py:263-308) on TransD: (rank_true_heads,
    rank_true_tails, filt_rank_true_heads, filt_rank_true_tails)."""
    s = scalars(P) if s is None else s
    n = heads.shape[0]
    out = [torch.empty(n, dtype=torch.long) for _ in range(4)]
    for lo in range(0, n, b_size):
        hi = min(n, lo + b_size)
        h, t, r = heads[lo:hi], tails[lo:hi], rels[lo:hi]
        sc = scores_all(P, h, t, r, "tail", s)
        out[1][lo:hi] = rank_of_true(sc, t)
        out[3][lo:hi] = rank_of_true(filtered_scores(sc, dict_of_tails, h, r, t), t)
        sc = scores_all(P, h, t, r, "head", s)
        out[0][lo:hi] = rank_of_true(sc, h)
        out[2][lo:hi] = rank_of_true(filtered_scores(sc, dict_of_heads, t, r, h), h)
    return tuple(out)


def relation_scores_all(P, h_idx, t_idx, s=None):
    """(b, n_rel) scores of every relation for the pairs (h, t): the relation case of
    inference_prepare_candidates (translation.py:621-625) and inference_scoring_function
    (interfaces.py:261-272), the (b, n_rel, rel_emb_dim) projections built for the batch only."""
    s = scalars(P) if s is None else s
    b = h_idx.shape[0]
    n_rel, d = P["rel"].shape
    rp = P["rel_proj"].view(1, n_rel, d)
    proj_h = s[h_idx].view(b, 1, 1) * rp + P["ent"][h_idx, :d].view(b, 1, d)
    proj_t = s[t_idx].view(b, 1, 1) * rp + P["ent"][t_idx, :d].view(b, 1, d)
    cands = P["rel"].view(1, n_rel, d).expand(b, n_rel, d)
    return -l2_diss(proj_h + cands, proj_t)


def relation_prediction(P, heads, tails, rels, dict_of_rels, b_size, directed=True, s=None):
    """RelationPredictionEvaluator.evaluate (evaluation.py:64-112) on TransD: (rank_true_rels,
    filt_rank_true_rels); undirected as kge_oracle.relation_prediction."""
    s = scalars(P) if s is None else s
    n = heads.shape[0]
    out = [torch.empty(n, dtype=torch.long) for _ in range(2)]
    for lo in range(0, n, b_size):
        hi = min(n, lo + b_size)
        h, t, r = heads[lo:hi], tails[lo:hi], rels[lo:hi]
        sc = relation_scores_all(P, h, t, s)
        fs = filtered_scores(sc, dict_of_rels, h, t, r)
        if not directed:
            s2 = relation_scores_all(P, t, h, s)
            fs2 = filtered_scores(s2, dict_of_rels, h, t, r)
            sc, fs = torch.cat((sc, s2), dim=1), torch.cat((fs, fs2), dim=1)
        out[0][lo:hi] = rank_of_true(sc, r)
        out[1][lo:hi] = rank_of_true(fs, r)
    return tuple(out)


def score_triples(P, h_idx, t_idx, r_idx):
    """scoring_function (translation.py:538-568); differentiable when the tables require grad."""
    nrm = torch.nn.functional.normalize
    d = P["rel"].shape[1]
    h = nrm(P["ent"][h_idx], p=2, dim=1)
    t = nrm(P["ent"][t_idx], p=2, dim=1)
    r = nrm(P["rel"][r_idx], p=2, dim=1)
    hp = nrm(P["ent_proj"][h_idx], p=2, dim=1)
    tp = nrm(P["ent_proj"][t_idx], p=2, dim=1)
    rp = nrm(P["rel_proj"][r_idx], p=2, dim=1)

    def project(e, ep):
        return rp * (e * ep).sum(dim=1).view(-1, 1) + e[:, :d]
    return -l2_diss(project(h, hp) + r, project(t, tp))
