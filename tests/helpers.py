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


# ---------------------------------------------------------------------------- fused training step
from torchkge_b200 import _lib  # noqa: E402
from torchkge_b200.engine import EntityShard, _exchanged_rows  # noqa: E402
from torchkge_b200.training import (ShardedStep, _kernel_dim, _MarginStep, _param_tensors, _row_spec,  # noqa: E402
                                    _training_code)

DEV = "cuda:0"
LOSS_KINDS = {"margin": _lib.LOSS_MARGIN, "logistic": _lib.LOSS_LOGISTIC, "bce": _lib.LOSS_BCE}


def close_grad(a, b, rtol=1e-4):
    """Gradient tables are sums of many signed terms accumulated by atomics in arbitrary order: rtol on
    the element plus an absolute floor of 1e-5 of the table's largest entry (tests/test_train_gpu.py)."""
    b = b.detach().cpu().float()
    torch.testing.assert_close(a.detach().cpu().float(), b, rtol=rtol, atol=1e-5 * float(b.abs().max()) + 1e-9)


def train_leaves(model):
    """The model's tables in ModelSpec order as fresh leaves (RotatE: the (cos, sin) planes; Analogy:
    stacked (3, n, dim) tables)."""
    code = _training_code(model)
    ts = [None if x is None else x.detach().clone().contiguous().requires_grad_(True)
          for x in _param_tensors(model, code)]
    return code, _kernel_dim(model, code), ts


def train_model(kind, d, n_ent, n_rel, seed):
    """A model on cuda:0 whose entity rows are not unit rows where the model normalises them."""
    model = make_model(kind, d, n_ent, n_rel, seed=seed)
    if kind in ("transe_l1", "transe_l2", "distmult", "rescal"):
        with torch.no_grad():
            model.ent_emb.weight.mul_(1.0 + torch.rand(n_ent, 1))   # un-normalised rows
    if kind.startswith("toruse"):
        model.normalize_parameters()
    return model.to(DEV)


def negatives(h, t, n_ent, n_neg, gen):
    """Head and tail corruption mixed, a negative equal to its positive, a few with both ends replaced."""
    b = h.shape[0]
    nh, nt = h.repeat(n_neg), t.repeat(n_neg)
    which = torch.rand(b * n_neg, generator=gen) < 0.45
    rnd = torch.randint(1, n_ent, (b * n_neg,), generator=gen)
    nh = torch.where(which, rnd, nh)
    nt = torch.where(~which, rnd, nt)
    nt[0], nh[0] = t[0], h[0]
    both = torch.arange(7, b * n_neg, 97)
    nh[both] = (h.repeat(n_neg)[both] + 3) % n_ent
    nt[both] = (t.repeat(n_neg)[both] + 5) % n_ent
    return nh, nt


def torch_loss(loss, pos, neg, margin=0.0):
    """utils/losses.py restated with torch's own modules (pos already repeated n_neg times).
    "logistic_stable": the same loss through softplus -- SoftMarginLoss evaluates log(1 + exp(-y x)) as
    written and overflows to inf beyond |x| ~ 88, where the package's LogisticLoss, fused or not, is finite."""
    if loss == "margin":
        return torch.nn.MarginRankingLoss(margin=margin, reduction="sum")(pos, neg, torch.ones_like(pos))
    if loss == "logistic_stable":
        return torch.nn.functional.softplus(-pos).sum() + torch.nn.functional.softplus(neg).sum()
    if loss == "logistic":
        crit = torch.nn.SoftMarginLoss(reduction="sum")
        return crit(pos, torch.ones_like(pos)) + crit(neg, -torch.ones_like(neg))
    crit = torch.nn.BCELoss(reduction="sum")
    return crit(torch.sigmoid(pos), torch.ones_like(pos)) + crit(torch.sigmoid(neg), torch.zeros_like(neg))


def _torus_scores(kind, ent, rel, h, t, r):
    """translation.py:706-720 with dissimilarities.py:28-43 (torus L1 / L2)."""
    x = (torch.frac(ent[h]) + torch.frac(rel[r])) - torch.frac(ent[t])
    if kind == "toruse_l1":
        ax = x.abs()
        return -(2 * torch.minimum(ax, 1 - ax)).sum(dim=1)
    x2 = x * x
    return -(4 * torch.minimum(x2, 1 - x2)).sum(dim=1)


def cpu_pos_neg(kind, leaves, h, t, r, nh, nt):
    """oracle.forward_pos_neg over CPU copies of the kernel's leaves (TorusE restated above)."""
    e0, e1, r0, r1 = leaves
    if kind.startswith("toruse"):
        n_neg = nh.shape[0] // h.shape[0]
        return (_torus_scores(kind, e0, r0, h, t, r).repeat(n_neg),
                _torus_scores(kind, e0, r0, nh, nt, r.repeat(n_neg)))
    if kind in ("transe_l1", "transe_l2", "distmult"):
        P = {"ent": e0, "rel": r0}
    elif kind == "rescal":
        P = {"ent": e0, "rel_mat": r0}
    elif kind == "analogy":
        P = {"sc_ent": e0[0], "re_ent": e0[1], "im_ent": e0[2], "sc_rel": r0[0], "re_rel": r0[1], "im_rel": r0[2]}
    else:
        P = {"re_ent": e0, "im_ent": e1, "re_rel": r0, "im_rel": r1}
    return oracle.forward_pos_neg(kind, P, h, t, r, nh, nt)


def cpu_leaves(ts, dtype=torch.float32):
    """CPU copies of the kernel's leaves, as fresh leaves of `dtype`."""
    return [None if x is None else x.detach().cpu().to(dtype).clone().requires_grad_(True) for x in ts]


def check_against_cpu(model, kind, loss, h, t, r, nh, nt, rtol=2e-4, ref=None):
    """fused step on the GPU (external negatives) vs torch autograd on the CPU (torch_loss(ref or loss)),
    same leaf tables."""
    code, dim, ts = train_leaves(model)
    got = _MarginStep.apply(code, dim, model.n_ent, 0.0, nh.shape[0] // h.shape[0], h.to(DEV), t.to(DEV),
                            r.to(DEV), nh.to(DEV), nt.to(DEV), None, 0, 0, *ts, LOSS_KINDS[loss])
    got.backward()
    cpu = cpu_leaves(ts)
    pos, neg = cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    want = torch_loss(ref or loss, pos, neg)
    want.backward()
    assert abs(got.item() - want.item()) <= 2e-5 * abs(want.item()) + 1e-12, (got.item(), want.item())
    for a, b in zip(ts, cpu):
        if a is not None:
            close_grad(a.grad, b.grad, rtol)
    return ts, cpu


def unsharded(model, h, t, r, probs, margin, n_neg, seed, offset, loss_kind=_lib.LOSS_MARGIN):
    """(loss, [grad tables]) of the fused step on the whole table, Philox negatives."""
    code, dim, ts = train_leaves(model)
    loss = _MarginStep.apply(code, dim, model.n_ent, margin, n_neg, h, t, r, None, None, probs, seed, offset, *ts,
                             loss_kind)
    loss.backward()
    return loss.item(), [None if x is None else x.grad for x in ts]


def emulated(model, h, t, r, probs, margin, n_neg, seed, offset, world, eng, loss_kind=_lib.LOSS_MARGIN):
    """What `world` ranks compute, one rank range after the other on one device: the loss, the
    relation gradients and grad_hrows / grad_trows summed over the ranks (the all-reduces), then
    every rank's scatter into its own rows."""
    code, dim, ts = train_leaves(model)
    tabs = [None if x is None else x.detach() for x in ts]
    n_ent, b = model.n_ent, h.shape[0]
    full = ShardedStep(code, dim, n_ent, 0, n_ent, n_neg, float(margin), seed, offset, loss_kind)
    rows = _exchanged_rows(_row_spec(full, tabs), torch.cat([h, t]), EntityShard(n_ent), eng)
    hrows, trows = rows[:b], rows[b:]
    loss = torch.zeros((), dtype=torch.float32, device=DEV)
    grad_rows = torch.zeros_like(rows)
    grel = [None if x is None else torch.zeros_like(x) for x in tabs[2:]]
    gent = [None if x is None else torch.zeros_like(x) for x in tabs[:2]]
    parts = []
    for rank in range(world):
        sh = EntityShard(n_ent, rank, world, local_storage=True)
        n = sh.hi - sh.lo
        # every rank's entity rows and entity gradient are views of rows [lo, hi) of one table (a
        # three-plane table keeps its planes equally spaced)
        local = [None if x is None else x.narrow(-2, sh.lo, n) for x in tabs[:2]] + tabs[2:]
        lg = [None if x is None else x.narrow(-2, sh.lo, n) for x in gent]
        parts.append((sh, lg))
        if n == 0:
            continue
        step = ShardedStep(code, dim, n_ent, sh.lo, n, n_neg, float(margin), seed, offset, loss_kind)
        loss += eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
        g_rows = torch.zeros_like(rows)
        g_rel = [None if x is None else torch.zeros_like(x) for x in tabs[2:]]
        gl = torch.ones((), dtype=torch.float32, device=DEV)
        eng.margin_step_bwd(step, local, lg + g_rel, h, t, r, probs, gl, hrows, trows, g_rows[:b], g_rows[b:])
        grad_rows += g_rows
        for a, c in zip(grel, g_rel):
            if a is not None:
                a += c
    for sh, lg in parts:          # after the all-reduce: every rank adds the rows it holds
        if sh.hi > sh.lo:
            eng.scatter_rows_add(code, dim, lg[0], lg[1], sh.lo, torch.cat([h, t]), grad_rows)
    return loss.item(), gent + grel
