"""TransD fixtures and graphs shared by the TransD test modules (tests/golden/make_golden_transd.py writes the
fixtures from the unmodified reference)."""
import os

import numpy as np
import torch

import torchkge_b200 as tk
from tests import helpers

CASES = ["transd_toy", "transd_syn"]
GRAD_NAMES = ("ent_emb", "rel_emb", "ent_proj_vect", "rel_proj_vect")
KEYS = {"ent": "ent_emb", "rel": "rel_emb", "ent_proj": "ent_proj_vect", "rel_proj": "rel_proj_vect"}


def load(name):
    """dict with ent_dim, rel_dim, n_ent, n_rel, b_size, state (state_dict tensors), P (oracle tables), the test
    facts, their negatives, the filter dicts dh / dt / dr and every reference output array (``raw``)."""
    z = np.load(os.path.join(helpers.GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    g = {k: z[k] for k in z.files}
    out = {k: int(g[k]) for k in ("ent_dim", "rel_dim", "n_ent", "n_rel", "b_size")}
    out["raw"] = g
    out["state"] = {k[2:]: torch.from_numpy(v.copy()) for k, v in g.items() if k.startswith("w:")}
    out["P"] = params(out["state"])
    for k in ("heads", "tails", "rels", "neg_heads", "neg_tails"):
        out[k] = torch.from_numpy(g[k].copy()).long()
    for k in ("dh", "dt", "dr"):
        out[k] = helpers._arrays_to_dict(g[k + "_keys"], g[k + "_offs"], g[k + "_vals"])
    return out


def params(state):
    """state_dict of a TransD model -> the oracle's tables (CPU)."""
    return {k: state[v + ".weight"].detach().cpu() for k, v in KEYS.items()}


def model_from(g):
    model = tk.TransDModel(g["ent_dim"], g["rel_dim"], g["n_ent"], g["n_rel"])
    model.load_state_dict(g["state"])
    return model


def graph_of(g):
    """The fixture's test facts as a KnowledgeGraph with the full graph's filter dicts."""
    kg = tk.KnowledgeGraph(g["heads"], g["tails"], g["rels"], g["n_ent"], g["n_rel"], dict_of_heads=g["dh"],
                           dict_of_tails=g["dt"])
    kg.dict_of_rels = g["dr"]
    return kg
