"""Shared test utilities: synthetic graphs, model <-> oracle parameter mapping."""
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle

KIND_TO_CLASS = {
    "transe_l1": lambda d, ne, nr: tk.TransEModel(d, ne, nr, dissimilarity_type="L1"),
    "transe_l2": lambda d, ne, nr: tk.TransEModel(d, ne, nr, dissimilarity_type="L2"),
    "distmult": lambda d, ne, nr: tk.DistMultModel(d, ne, nr),
    "rescal": lambda d, ne, nr: tk.RESCALModel(d, ne, nr),
    "complex": lambda d, ne, nr: tk.ComplExModel(d, ne, nr),
    "rotate": lambda d, ne, nr: tk.RotatEModel(d, ne, nr),
    "toruse_l1": lambda d, ne, nr: tk.TorusEModel(d, ne, nr, dissimilarity_type="torus_L1"),
    "toruse_l2": lambda d, ne, nr: tk.TorusEModel(d, ne, nr, dissimilarity_type="torus_L2"),
    "analogy": lambda d, ne, nr: tk.AnalogyModel(d, ne, nr),     # d = emb_dim: two halves
}


def make_model(kind, d, n_ent, n_rel, seed=0):
    torch.manual_seed(seed)
    return KIND_TO_CLASS[kind](d, n_ent, n_rel)


def oracle_params(kind, model):
    """CPU fp32 copies of the model's tables under the oracle's key names.

    For RotatE call this AFTER moving the model to its final device: the (cos, sin) relation
    planes are computed there, and libm results differ between CPU and GPU in the last ulp."""
    g = lambda w: w.detach().cpu().clone()  # noqa: E731
    if kind in ("transe_l1", "transe_l2", "distmult"):
        return {"ent": g(model.ent_emb.weight), "rel": g(model.rel_emb.weight)}
    if kind in ("toruse_l1", "toruse_l2"):
        model.normalize_parameters()      # the tables the evaluator reads hold fractional parts
        return {"ent": g(model.ent_emb.weight), "rel": g(model.rel_emb.weight)}
    if kind == "rescal":
        return {"ent": g(model.ent_emb.weight), "rel_mat": g(model.rel_mat.weight)}
    if kind == "complex":
        return {"re_ent": g(model.re_ent_emb.weight), "im_ent": g(model.im_ent_emb.weight),
                "re_rel": g(model.re_rel_emb.weight), "im_rel": g(model.im_rel_emb.weight)}
    if kind == "analogy":
        return {"sc_ent": g(model.sc_ent_emb.weight), "re_ent": g(model.re_ent_emb.weight),
                "im_ent": g(model.im_ent_emb.weight), "sc_rel": g(model.sc_rel_emb.weight),
                "re_rel": g(model.re_rel_emb.weight), "im_rel": g(model.im_rel_emb.weight)}
    if kind == "rotate":
        re_r, im_r = model.relation_planes()  # computed on the model's device: same bits for both
        return {"re_ent": g(model.re_ent_emb.weight), "im_ent": g(model.im_ent_emb.weight),
                "re_rel": g(re_r), "im_rel": g(im_r)}
    raise ValueError(kind)


def random_graph(n_ent, n_rel, n_facts, seed=0, skew=True):
    """Deduplicated random facts; with skew, a few (h, r) / (t, r) keys get large filter sets."""
    g = torch.Generator().manual_seed(seed)
    if skew:
        w_e = 1.0 / torch.arange(1, n_ent + 1, dtype=torch.float64) ** 0.8
        w_r = 1.0 / torch.arange(1, n_rel + 1, dtype=torch.float64)
        h = torch.multinomial(w_e, n_facts, replacement=True, generator=g)
        t = torch.multinomial(w_e, n_facts, replacement=True, generator=g)
        r = torch.multinomial(w_r, n_facts, replacement=True, generator=g)
    else:
        h = torch.randint(0, n_ent, (n_facts,), generator=g)
        t = torch.randint(0, n_ent, (n_facts,), generator=g)
        r = torch.randint(0, n_rel, (n_facts,), generator=g)
    trip = torch.unique(torch.stack([h, t, r], 1), dim=0)
    perm = torch.randperm(trip.shape[0], generator=g)
    trip = trip[perm]
    return trip[:, 0].contiguous(), trip[:, 1].contiguous(), trip[:, 2].contiguous()


def make_kg(n_ent, n_rel, n_facts, n_test, seed=0):
    """(test KnowledgeGraph carrying full-graph filter dicts, (dict_of_heads, dict_of_tails))."""
    h, t, r = random_graph(n_ent, n_rel, n_facts, seed)
    dh, dt = oracle.build_filter_dicts(h, t, r)
    n_test = min(n_test, h.shape[0])
    kg = tk.KnowledgeGraph(h[:n_test], t[:n_test], r[:n_test], n_ent, n_rel,
                           dict_of_heads=dh, dict_of_tails=dt)
    return kg, dh, dt


# ---------------------------------------------------------------------------- golden fixtures
import os  # noqa: E402
from collections import defaultdict  # noqa: E402

import numpy as np  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_CASES = ["toy_transe_l1", "toy_transe_l2", "toy_distmult", "toy_rescal", "toy_complex",
                "syn_transe_l1", "syn_transe_l2", "syn_distmult", "syn_rescal", "syn_complex"]
#: same layout, from tests/golden/make_golden_analogy.py (AnalogyModel, models/bilinear.py:559-763)
ANALOGY_CASES = ["toy_analogy", "syn_analogy"]

_STATE_TO_ORACLE = {
    "ent_emb.weight": "ent", "rel_emb.weight": "rel", "rel_mat.weight": "rel_mat",
    "re_ent_emb.weight": "re_ent", "im_ent_emb.weight": "im_ent",
    "re_rel_emb.weight": "re_rel", "im_rel_emb.weight": "im_rel",
    "sc_ent_emb.weight": "sc_ent", "sc_rel_emb.weight": "sc_rel",
}


def _arrays_to_dict(keys, offs, vals):
    d = defaultdict(set)
    for i, (a, b) in enumerate(keys.tolist()):
        d[(a, b)] = set(vals[offs[i]:offs[i + 1]].tolist())
    return d


def load_golden(name):
    """dict with: kind, dim, n_ent, n_rel, b_size, P (oracle params), state (state_dict arrays),
    heads/tails/rels (test facts), dh/dt (filter dicts) and every reference output array."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    g = {k: z[k] for k in z.files}
    out = {"kind": str(g["kind"]), "dim": int(g["dim"]), "n_ent": int(g["n_ent"]),
           "n_rel": int(g["n_rel"]), "b_size": int(g["b_size"]), "raw": g}
    out["state"] = {k[2:]: torch.from_numpy(v.copy()) for k, v in g.items() if k.startswith("w:")}
    out["grads"] = {k[2:]: torch.from_numpy(v.copy()) for k, v in g.items() if k.startswith("g:")}
    out["P"] = {_STATE_TO_ORACLE[k]: v for k, v in out["state"].items()}
    for k in ("heads", "tails", "rels", "all_heads", "all_tails", "all_rels", "neg_heads", "neg_tails"):
        out[k] = torch.from_numpy(g[k].copy()).long()
    out["dh"] = _arrays_to_dict(g["dh_keys"], g["dh_offs"], g["dh_vals"])
    out["dt"] = _arrays_to_dict(g["dt_keys"], g["dt_offs"], g["dt_vals"])
    return out


def load_golden_rel(name):
    """Relation-prediction outputs of the reference for fixture `name` (rel_<name>.npz) plus the
    dict_of_rels it used (key "dr")."""
    z = np.load(os.path.join(GOLDEN_DIR, "rel_" + name + ".npz"), allow_pickle=False)
    out = {k: z[k] for k in z.files}
    out["dr"] = _arrays_to_dict(z["dr_keys"], z["dr_offs"], z["dr_vals"])
    return out


TORUS_CASES = ["torus_l1", "torus_l2"]


def load_golden_torus(name):
    """TorusE fixture (tests/golden/make_golden_torus.py): same layout as load_golden, without the
    training-side arrays."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    g = {k: z[k] for k in z.files}
    out = {"kind": str(g["kind"]), "dim": int(g["dim"]), "n_ent": int(g["n_ent"]),
           "n_rel": int(g["n_rel"]), "b_size": int(g["b_size"]), "raw": g}
    out["state"] = {k[2:]: torch.from_numpy(v.copy()) for k, v in g.items() if k.startswith("w:")}
    out["P"] = {_STATE_TO_ORACLE[k]: v for k, v in out["state"].items()}
    for k in ("heads", "tails", "rels"):
        out[k] = torch.from_numpy(g[k].copy()).long()
    out["dh"] = _arrays_to_dict(g["dh_keys"], g["dh_offs"], g["dh_vals"])
    out["dt"] = _arrays_to_dict(g["dt_keys"], g["dt_offs"], g["dt_vals"])
    return out


def model_from_golden(g):
    model = KIND_TO_CLASS[g["kind"]](g["dim"], g["n_ent"], g["n_rel"])
    model.load_state_dict(g["state"])
    return model


def bits_equal(a, b):
    """Element-wise: same fp32 bit pattern, or numerically equal (+0 == -0)."""
    a = a.detach().cpu().float().contiguous()
    b = b.detach().cpu().float().contiguous()
    return (a.numpy().view(np.uint32) == b.numpy().view(np.uint32)) | (a == b).numpy()


# ---------------------------------------------------------------------------- RESCAL query prep
def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def rescal_prep_emulated(side, vec, M):
    """numpy restatement of the summation order of `matmul(h.view(b, 1, d), M)` (side 'tail') /
    `matmul(M, t.view(b, d, 1))` (side 'head') as oneMKL 2024.2 (AVX-512 path) + ATen execute it
    for batches of >= 2 facts -- the order csrc/reduce.cuh:rescal_query_component replays.
    vec (d,), M (d, d) float32 numpy; returns (d,).  Used to tell whether THIS machine's MKL takes
    the same code path as the authoring machine (rescal_order_matches_here)."""
    d = vec.shape[0]
    vec, M = vec.astype(np.float32), M.astype(np.float32)
    y = np.zeros(d, np.float32)
    if side == "tail":
        H = lambda k: np.full(d, vec[k], np.float32)   # noqa: E731
        if d < 20:
            for k in range(d):
                y = y + H(k) * M[k]
            return y
        k = 0
        while k + 8 <= d:
            y = _fma32(H(k + 6), M[k + 6], y)
            y = _fma32(H(k + 4), M[k + 4], y)
            y = y + _fma32(H(k + 5), M[k + 5], H(k + 7) * M[k + 7])
            y = y + (_fma32(H(k), M[k], H(k + 2) * M[k + 2]) + _fma32(H(k + 1), M[k + 1], H(k + 3) * M[k + 3]))
            k += 8
        while k < d:
            y = _fma32(H(k), M[k], y)
            k += 1
        jm = 16 * (d // 16)
        if jm < d:
            yy = np.zeros(d, np.float32)
            for k in range(d):
                yy = _fma32(H(k), M[k], yy)
            y[jm:] = yy[jm:]
        return y
    T = lambda k: np.full(d, vec[k], np.float32)   # noqa: E731
    if d < 20:
        for k in range(d):
            y = y + M[:, k] * T(k)
        return y
    bounds = [0]                       # K-blocks of 384 while more than 768 terms remain ...
    while d > 384 and d - bounds[-1] > 768:
        bounds.append(bounds[-1] + 384)
    if d > 384:                        # ... then the last 385..768 terms as two chains
        bounds.append(bounds[-1] + (d - bounds[-1] + 1) // 2)
    bounds.append(d)
    parts = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        acc = np.zeros(d, np.float32)
        for k in range(a, b):
            acc = _fma32(M[:, k], T(k), acc)
        parts.append(acc)
    y = parts[0]
    for p in parts[1:]:
        y = y + p
    return y


_RESCAL_ORDER = {}


def rescal_order_matches_here(d):
    """True when torch.matmul on THIS machine sums RESCAL's query preparation in the order the CUDA
    kernel replays (it does on the authoring machine: tests/test_host_arith.py).  oneMKL picks its
    kernels by CPU: on a machine where this is False the reference's own RESCAL bits differ from the
    committed golden fixtures, and oracle-vs-GPU rank equality cannot be expected there."""
    if d not in _RESCAL_ORDER:
        g = torch.Generator().manual_seed(d)
        v, M = torch.randn(3, d, generator=g), torch.randn(3, d, d, generator=g)
        wt = torch.matmul(v.view(3, 1, d), M).view(3, d).numpy()
        wh = torch.matmul(M, v.view(3, d, 1)).view(3, d).numpy()
        ok = True
        for i in range(3):
            ok &= bool((rescal_prep_emulated("tail", v[i].numpy(), M[i].numpy()) == wt[i]).all())
            ok &= bool((rescal_prep_emulated("head", v[i].numpy(), M[i].numpy()) == wh[i]).all())
        _RESCAL_ORDER[d] = ok
    return _RESCAL_ORDER[d]


# ---------------------------------------------------------------------------- entity-sharded models
def local_model(kind, model, lo, hi, n_rel, dim):
    """The same model holding only entity rows [lo, hi), on the model's device."""
    part = make_model(kind, dim, hi - lo, n_rel, seed=0)
    part.load_state_dict({name: w[lo:hi] if "ent_emb" in name else w for name, w in model.state_dict().items()})
    return part.to(next(model.parameters()).device)
