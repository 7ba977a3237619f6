"""The fused training step's test kit: models and their leaves, the float64 reference, the calls into the
step (whole table, one shard, emulated ranks), the draw statements, the launch rule of csrc/train.cu, the
child-process re-run under an environment switch, the CPU stand-in engine of the sharded host logic, the
two-process public-API run and the ABI checks.  The tests of the step call the package's private training
layer (_MarginStep, ShardedStep) through this module only."""
import ctypes
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import torchkge_b200 as tk
from oracle import kge_oracle as oracle
from tests import helpers
from torchkge_b200 import _lib
from torchkge_b200.engine import EntityShard, _exchanged_rows, _ptr, _stream
from torchkge_b200.training import ShardedStep, _kernel_dim, _MarginStep, _param_tensors, _row_spec, _training_code

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN_CU = os.path.join(ROOT, "torchkge_b200", "csrc", "train.cu")
DEV = "cuda:0"
LOSS_KINDS = {"margin": _lib.LOSS_MARGIN, "logistic": _lib.LOSS_LOGISTIC, "bce": _lib.LOSS_BCE}


# ---------------------------------------------------------------------------- models and the float64 reference
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
    model = helpers.make_model(kind, d, n_ent, n_rel, seed=seed)
    if kind in ("transe_l1", "transe_l2", "distmult", "rescal"):
        with torch.no_grad():
            model.ent_emb.weight.mul_(1.0 + torch.rand(n_ent, 1))   # un-normalised rows
    if kind.startswith("toruse"):
        model.normalize_parameters()
    return model.to(DEV)


def batch(n_ent, n_rel, b, gen):
    """b positives and Bernoulli probabilities on the GPU, drawn from `gen` (a generator or a seed)."""
    if not isinstance(gen, torch.Generator):
        gen = torch.Generator().manual_seed(gen)
    h, t = torch.randint(0, n_ent, (b,), generator=gen), torch.randint(0, n_ent, (b,), generator=gen)
    r = torch.randint(0, n_rel, (b,), generator=gen)
    probs = torch.rand(n_rel, generator=gen)
    return h.to(DEV), t.to(DEV), r.to(DEV), probs.to(DEV)


def problem(kind, d, n_neg, seed, n_ent, n_rel, b=23):
    """A model and a batch of b positives (23: the last block holds three warps) with Bernoulli
    probabilities, all on the GPU."""
    return (train_model(kind, d, n_ent, n_rel, seed=seed),) + batch(n_ent, n_rel, b, seed + n_neg)


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


def cpu_scores(kind, leaves, h, t, r):
    """oracle.score_triples over CPU copies of the kernel's leaves (TorusE restated above)."""
    e0, e1, r0, r1 = leaves
    if kind.startswith("toruse"):
        return _torus_scores(kind, e0, r0, h, t, r)
    if kind in ("transe_l1", "transe_l2", "distmult"):
        P = {"ent": e0, "rel": r0}
    elif kind == "rescal":
        P = {"ent": e0, "rel_mat": r0}
    elif kind == "analogy":
        P = {"sc_ent": e0[0], "re_ent": e0[1], "im_ent": e0[2], "sc_rel": r0[0], "re_rel": r0[1], "im_rel": r0[2]}
    else:
        P = {"re_ent": e0, "im_ent": e1, "re_rel": r0, "im_rel": r1}
    return oracle.score_triples(kind, P, h, t, r)


def cpu_pos_neg(kind, leaves, h, t, r, nh, nt, nr=None):
    """The positives' scores repeated once per negative, and the negatives' (relation nr, or the positive's)."""
    n_neg = nh.shape[0] // h.shape[0]
    pos = cpu_scores(kind, leaves, h, t, r).repeat(n_neg)
    return pos, cpu_scores(kind, leaves, nh, nt, r.repeat(n_neg) if nr is None else nr)


def cpu_leaves(ts, dtype=torch.float32):
    """CPU copies of the kernel's leaves, as fresh leaves of `dtype`."""
    return [None if x is None else x.detach().cpu().to(dtype).clone().requires_grad_(True) for x in ts]


def reference(kind, leaves, h, t, r, nh, nt, loss, margin, nr=None):
    """float64 CPU autograd of the oracle's scores on copies of the kernel's leaves: (loss, [grads], pos, neg)."""
    cpu = cpu_leaves(leaves, torch.float64)
    pos, neg = cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu(), None if nr is None else nr.cpu())
    want = torch_loss(loss, pos, neg, margin)
    want.backward()
    return want.item(), [None if x is None else x.grad for x in cpu], pos.detach(), neg.detach()


def margin_between(diff, q=0.5):
    """A float32 margin m in the widest gap between neighbouring values of pos - neg near its q-quantile:
    about half the hinges are active, and none lies so close to its kink that float32 and float64 could
    disagree on whether it is."""
    s = torch.sort(diff.detach().flatten()).values
    k = int(q * (s.shape[0] - 1))
    w = min(200, s.shape[0] // 4)
    if w == 0:
        return float(torch.tensor(float(s[0]) + 0.5, dtype=torch.float32))
    lo, hi = k - w, k + w
    i = lo + int(torch.argmax(s[lo + 1:hi + 1] - s[lo:hi]))
    return float(torch.tensor(float(s[i] + s[i + 1]) / 2, dtype=torch.float32))


def check_against_cpu(model, kind, loss, h, t, r, nh, nt, rtol=2e-4, ref=None):
    """fused step on the GPU (external negatives) vs torch autograd on the CPU (torch_loss(ref or loss)),
    same leaf tables: (the step's gradients, the CPU leaves)."""
    got, grads = whole_table_step(model, h, t, r, loss=loss, negatives=(nh, nt))
    cpu = cpu_leaves(train_leaves(model)[2])
    pos, neg = cpu_pos_neg(kind, cpu, h.cpu(), t.cpu(), r.cpu(), nh.cpu(), nt.cpu())
    want = torch_loss(ref or loss, pos, neg)
    want.backward()
    assert abs(got - want.item()) <= 2e-5 * abs(want.item()) + 1e-12, (got, want.item())
    for a, b in zip(grads, cpu):
        if a is not None:
            close_grad(a, b.grad, rtol)
    return grads, cpu


# ---------------------------------------------------------------------------- calls into the step
# Every call takes the negatives as keywords: caller negatives=(nh, nt) or (nh, nt, nr); else the step's
# own draws from probs at (seed, offset) -- the entity step, with rel_share the relation-corrupting step
# over the model's relations, with positional=(head_offs, head_ents, tail_offs, tail_ents) the positional
# step.  loss names a LOSS_KINDS entry; the margin is read by the margin loss only.
def corrupt_batch(h, t, r, probs, n_neg, n_ent, seed, offset):
    """kge_corrupt_batch's negatives: the ones the entity step draws at (seed, offset)."""
    nh = torch.empty(h.shape[0] * n_neg, dtype=torch.int64, device=DEV)
    nt = torch.empty_like(nh)
    _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), h.shape[0], n_neg, _ptr(probs), n_ent, seed,
                                             offset, _ptr(nh), _ptr(nt), _stream(h.device)), "kge_corrupt_batch")
    return nh, nt


def _step_args(model, h, t, r, n_neg, loss, margin, probs, seed, offset, negatives, rel_share, positional):
    """(code, dim, h, t, r, the arguments of _MarginStep after the tables)."""
    code = _training_code(model)
    nh, nt, nr = (tuple(negatives) + (None,))[:3] if negatives is not None else (None, None, None)
    if n_neg is None:
        n_neg = nh.shape[0] // h.shape[0]
    rel = None if rel_share is None else (model.n_rel, rel_share)
    pos = None if positional is None else tuple(x.to(DEV) for x in positional)
    head = (code, _kernel_dim(model, code), model.n_ent, margin, n_neg, h.to(DEV), t.to(DEV), r.to(DEV), nh, nt,
            probs, seed, offset)
    return head, (LOSS_KINDS[loss], nr, rel, pos)


def whole_table_step(model, h, t, r, *, n_neg=None, loss="margin", margin=0.0, probs=None, seed=0, offset=0,
                     negatives=None, rel_share=None, positional=None, outputs=False):
    """The fused step on the whole table, forward and backward: (loss, [gradient tables]); with outputs, also
    forward_outputs() of the same step."""
    head, tail = _step_args(model, h, t, r, n_neg, loss, margin, probs, seed, offset, negatives, rel_share,
                            positional)
    ts = train_leaves(model)[2]
    got = _MarginStep.apply(*head, *ts, *tail)
    got.backward()
    res = got.item(), [None if x is None else x.grad for x in ts]
    if outputs:
        res += (forward_outputs(model, h, t, r, n_neg=n_neg, loss=loss, margin=margin, probs=probs, seed=seed,
                                offset=offset, negatives=negatives, rel_share=rel_share, positional=positional),)
    return res


def forward_outputs(model, h, t, r, *, n_neg=None, loss="margin", margin=0.0, probs=None, seed=0, offset=0,
                    negatives=None, rel_share=None, positional=None):
    """One forward of the step through its C entry point (kge_margin_step_fwd, kge_rel_step_fwd or
    kge_pos_step_fwd) with every optional output set: {"loss", "pos", "neg", "nh", "nt"} and, for a
    relation-corrupting step, "nr".  The outputs start as NaN / -1, so an output left unwritten shows."""
    head, tail = _step_args(model, h, t, r, n_neg, loss, margin, probs, seed, offset, negatives, rel_share,
                            positional)
    b, n = h.shape[0], h.shape[0] * head[4]
    out = {"loss": torch.zeros((), device=DEV), "pos": torch.full((b,), float("nan"), device=DEV),
           "neg": torch.full((n,), float("nan"), device=DEV)}
    for k in ("nh", "nt") + (("nr",) if rel_share is not None else ()):
        out[k] = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    tabs = [None if x is None else x.detach() for x in train_leaves(model)[2]]
    a = _MarginStep._args(*head, tabs, out["loss"], torch.device(DEV), *tail)
    base = a if isinstance(a, _lib.MarginStepArgs) else a.base
    base.pos_out, base.neg_out, base.nh_out, base.nt_out = (_ptr(out[k]) for k in ("pos", "neg", "nh", "nt"))
    if "nr" in out:
        a.nr_out = _ptr(out["nr"])
    name = _MarginStep._entry(a, "fwd")
    assert getattr(_lib.load(), name)(ctypes.byref(a)) == 0, name
    torch.cuda.synchronize()
    return out


def sharded_step(model, lo, n, *, n_neg, loss="margin", margin=0.0, seed=0, offset=0, rel_share=None,
                 positional=None):
    """What the kernels of the rank holding entity rows [lo, lo + n) are told (ShardedStep)."""
    code = _training_code(model)
    return ShardedStep(code, _kernel_dim(model, code), model.n_ent, lo, n, n_neg, float(margin), seed, offset,
                       LOSS_KINDS[loss], 0 if rel_share is None else model.n_rel,
                       1.0 if rel_share is None else rel_share,
                       None if positional is None else tuple(x.to(DEV) for x in positional))


def emulated(model, h, t, r, world, eng, *, probs, n_neg, loss="margin", margin=0.0, seed=0, offset=0,
             rel_share=None, positional=None):
    """What `world` ranks compute, one rank range after the other on one device: the loss, the
    relation gradients and grad_hrows / grad_trows summed over the ranks (the all-reduces), then
    every rank's scatter into its own rows.  (loss, [gradient tables]) as whole_table_step."""
    code, dim, ts = train_leaves(model)
    tabs = [None if x is None else x.detach() for x in ts]
    n_ent, b = model.n_ent, h.shape[0]
    kw = dict(n_neg=n_neg, loss=loss, margin=margin, seed=seed, offset=offset, rel_share=rel_share,
              positional=positional)
    rows = _exchanged_rows(_row_spec(sharded_step(model, 0, n_ent, **kw), tabs), torch.cat([h, t]),
                           EntityShard(n_ent), eng)
    hrows, trows = rows[:b], rows[b:]
    total = torch.zeros((), dtype=torch.float32, device=DEV)
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
        step = sharded_step(model, sh.lo, n, **kw)
        total += eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
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
    return total.item(), gent + grel


def compare(got, want, rtol=1e-4):
    """Two (loss, [gradient tables]) of the same step: the loss within 1e-5, gradients under close_grad."""
    (gl, gg), (wl, wg) = got, want
    assert gl == pytest.approx(wl, rel=1e-5, abs=1e-6)
    for a, b in zip(gg, wg):
        if b is not None:
            close_grad(a, b, rtol)


# ---------------------------------------------------------------------------- the draw statements
# The numpy Philox statements say what the kernels draw, bit for bit (csrc/train.cu: draw_one, draw_rel,
# draw_pos).  Negative j of fact i is drawn at counter index j b + i; every function returns numpy-built
# torch tensors over those indices.
def philox_words(seed, offset, idx):
    """Philox4x32-10 with counter (idx, offset) and key seed, in numpy (csrc/train.cu: philox4x32)."""
    M = np.uint64(0xFFFFFFFF)
    idx = idx.astype(np.uint64)
    c0, c1 = idx & M, idx >> np.uint64(32)
    c2 = np.full_like(c0, offset & 0xFFFFFFFF)
    c3 = np.full_like(c0, offset >> 32)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & M
        hi1, lo1 = p1 >> np.uint64(32), p1 & M
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def _unit(w):
    """(w >> 8) / 2^24 in float32."""
    return (w >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def _below(w, n):
    """(w n) >> 32: uniform on [0, n)."""
    return ((w * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def philox_draws(seed, offset, r, n_neg, probs, n_ent):
    """draw_one: (head?, replacement) -- head iff (x >> 8) / 2^24 < p_r, entity 1 + (y (n_ent - 1)) >> 32."""
    R = np.tile(r.cpu().numpy(), n_neg)
    x, y, _, _ = philox_words(seed, offset, np.arange(R.shape[0]))
    head = _unit(x) < probs.cpu().numpy().astype(np.float32)[R]
    return torch.from_numpy(head), torch.from_numpy(1 + _below(y, n_ent - 1))


def philox_rel_draws(seed, offset, r, n_neg, probs, n_ent, n_rel, rel_share):
    """draw_rel: (relation?, new relation) -- an entity negative iff (z >> 8) / 2^24 < rel_share, drawn as
    draw_one from words x and y; else relation 1 + (w (n_rel - 1)) >> 32 -- and draw_one's (head?, entity)."""
    _, _, z, w = philox_words(seed, offset, np.arange(r.shape[0] * n_neg))
    is_rel = torch.from_numpy(~(_unit(z) < np.float32(rel_share)))
    return (is_rel, torch.from_numpy(1 + _below(w, n_rel - 1))) + philox_draws(seed, offset, r, n_neg, probs, n_ent)


def philox_pos_draws(seed, offset, r, n_neg, probs, n_ent, pos):
    """draw_pos: (head?, replacement) -- the side as draw_one, then entry (y n) >> 32 of relation r's n
    candidates on that side, or (y n_ent) >> 32 where it has none."""
    ho, he, to, te = (x.cpu().numpy().astype(np.int64) for x in pos)
    R = np.tile(r.cpu().numpy(), n_neg)
    x, y, _, _ = philox_words(seed, offset, np.arange(R.shape[0]))
    head = _unit(x) < probs.cpu().numpy().astype(np.float32)[R]
    lo = np.where(head, ho[R], to[R])
    n = np.where(head, ho[R + 1] - ho[R], to[R + 1] - to[R])
    pick = np.where(n > 0, lo + _below(y, n.astype(np.uint64)), 0)
    e = np.where(n > 0, np.where(head, he[np.minimum(pick, max(he.size - 1, 0))] if he.size else 0,
                                 te[np.minimum(pick, max(te.size - 1, 0))] if te.size else 0), _below(y, n_ent))
    return torch.from_numpy(head), torch.from_numpy(e)


def csr(rel, ent, n_rel, n_ent):
    """Sorted CSR of the distinct (relation, entity) pairs, as PositionalNegativeSampler builds it."""
    key = torch.unique(rel * n_ent + ent)
    offs = torch.zeros(n_rel + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.bincount(key // n_ent, minlength=n_rel), 0)
    return offs, key % n_ent


# The stand-in engine's laws: functions of (seed, offset) and the global sizes only, from a torch generator.
# They serve the sharding plumbing; the kernels draw by the Philox statements above.
def _stand_in_generator(seed, offset):
    return torch.Generator().manual_seed((seed * 1000003 + offset) % (1 << 62))


def stand_in_draws(seed, offset, r, n_neg, probs, n_ent):
    """The entity step: (head?, replacement on [1, n_ent))."""
    g = _stand_in_generator(seed, offset)
    b = r.shape[0]
    u = torch.rand(n_neg * b, generator=g)
    e = torch.randint(1, max(n_ent, 2), (n_neg * b,), generator=g)
    return u < probs[r.repeat(n_neg)], e


def stand_in_rel_draws(seed, offset, h, r, n_neg, probs, n_ent, n_rel, rel_share):
    """The relation-corrupting step: (kind 0 tail, 1 head, 2 relation; replacement)."""
    g = _stand_in_generator(seed, offset)
    n = n_neg * h.shape[0]
    u, z = torch.rand(n, generator=g), torch.rand(n, generator=g)
    e = torch.randint(1, max(n_ent, 2), (n,), generator=g)
    q = torch.randint(1, max(n_rel, 2), (n,), generator=g)
    kind = torch.where(z < rel_share, (u < probs[r.repeat(n_neg)]).long(), torch.full_like(e, 2))
    return kind, torch.where(kind == 2, q, e)


def stand_in_pos_draws(seed, offset, r, n_neg, probs, n_ent, pos):
    """The positional step: (head?, replacement from relation r's candidates on that side, or on
    [0, n_ent) where it has none)."""
    g = _stand_in_generator(seed, offset)
    n = n_neg * r.shape[0]
    u, v = torch.rand(n, generator=g), torch.rand(n, generator=g)
    R = r.repeat(n_neg)
    head = u < probs[R]
    ho, he, to, te = pos
    lo = torch.where(head, ho[R], to[R])
    cnt = torch.where(head, ho[R + 1] - ho[R], to[R + 1] - to[R])
    k = (v * cnt).long().clamp(max=(cnt - 1).clamp(min=0))
    pick = lo + k
    hv = he[pick.clamp(max=max(he.numel() - 1, 0))] if he.numel() else torch.zeros_like(pick)
    tv = te[pick.clamp(max=max(te.numel() - 1, 0))] if te.numel() else torch.zeros_like(pick)
    e = torch.where(cnt > 0, torch.where(head, hv, tv), (v * n_ent).long().clamp(max=n_ent - 1))
    return head, e


# ---------------------------------------------------------------------------- the launch rule, restated
# test_train_paths_gpu.py::test_launch_rule_mirrors_train_cu pins every constant and branch below to train.cu.
RING_SLOTS = 8                 # RING: rows in flight per warp
WARPS_PER_BLOCK = 4
FAST_MAX_DIM = 256             # 4 floats x 32 lanes x FAST_NCH chunks
SMEM_DEFAULT = 48 * 1024       # dynamic shared memory without cudaFuncSetAttribute
SMEM_MAX = 96 * 1024           # what launch_ring_variant raises the limit to
RING_MAX_NEG = 8192
FAST_KINDS = {"transe_l1": _lib.TRANSE_L1, "transe_l2": _lib.TRANSE_L2, "distmult": _lib.DISTMULT}


def _pad(x, m):
    return (x + m - 1) // m * m


def ring_smem_bytes(dim, n_neg):
    """Dynamic shared memory of one ring block: per warp RING rows, the codes of every negative and
    one mbarrier per slot, each warp's part rounded up to 128 bytes."""
    per_warp = RING_SLOTS * dim * 4 + _pad(n_neg, 4) * 4 + RING_SLOTS * 8
    return WARPS_PER_BLOCK * _pad(per_warp, 128)


def last_n_neg_within(dim, limit):
    """The largest n_neg whose ring block fits in `limit` bytes."""
    n = 1
    while ring_smem_bytes(dim, n + 1) <= limit:
        n += 1
    return n


def expected_kernels(kind, dim, n_neg, loss, shard, negatives="entity", env=None):
    """Signatures (see kernel_signature) of the forward and backward kernels one step launches.
    negatives: "entity", "relation" (a relation-corrupting step at rel_share < 1, or with caller negatives or
    nr_out; at rel_share >= 1 it is the entity step) or "positional".  The ring takes TransE-L1 / L2 and
    DistMult where it fits; else only the unsharded entity step with the margin loss has the register form;
    everything else takes the generic kernels."""
    env = os.environ if env is None else env
    ring_on = env.get("KGE_TRAIN_RING", "")[:1] != "0"
    tight = env.get("KGE_TRAIN_BWD_BLOCKS", "")[:1] == "5"
    fast = kind in FAST_KINDS and dim % 4 == 0 and dim <= FAST_MAX_DIM
    lk = LOSS_KINDS[loss]
    if fast and ring_on and n_neg <= RING_MAX_NEG and ring_smem_bytes(dim, n_neg) <= SMEM_MAX:
        if negatives != "entity":
            name = {"relation": "ring_rel", "positional": "ring_pos"}[negatives]
            return {(name, FAST_KINDS[kind], False, shard, lk), (name, FAST_KINDS[kind], True, shard, lk)}
        minb = 5 if tight and not shard and loss == "margin" else 0
        return {("ring", FAST_KINDS[kind], False, 0, shard, lk), ("ring", FAST_KINDS[kind], True, minb, shard, lk)}
    if fast and negatives == "entity" and not shard and loss == "margin":
        return {("fast", FAST_KINDS[kind], False), ("fast", FAST_KINDS[kind], True)}
    return {("shard_fwd",), ("shard_bwd",)} if shard else {("fwd",), ("bwd",)}


_KERNEL = r"margin_step_(ring_rel|ring_pos|ring|fast|shard_fwd|shard_bwd|fwd|bwd)_kernel"
_DEMANGLED = re.compile(r"(?<![\w])" + _KERNEL + r"(?:<([^<>]*)>)?\(")
_MANGLED = re.compile(r"\d" + _KERNEL + r"(?:I((?:L[ib]\d+E)+)E)?")


def kernel_signature(name):
    """("ring", model, bwd, minb, shard, loss), ("ring_rel" or "ring_pos", model, bwd, shard, loss),
    ("fast", model, bwd), ("fwd",), ("bwd",), ("shard_fwd",) or ("shard_bwd",) for a fused-step kernel's
    (demangled or mangled) name; None for any other kernel."""
    m = _DEMANGLED.search(name)
    if m:
        args = [] if m.group(2) is None else [a.strip() for a in m.group(2).split(",")]
        args = [a == "true" if a in ("true", "false") else int(re.sub(r"^\(\w+\)", "", a)) for a in args]
    else:
        m = _MANGLED.search(name)
        if not m:
            return None
        args = [bool(int(v)) if k == "b" else int(v) for k, v in re.findall(r"L([ib])(\d+)E", m.group(2) or "")]
    return (m.group(1),) + tuple(args)


def _cuda_kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def launched(fn, expected, tries=4):
    """The set of fused-step kernel signatures that ran on the GPU while fn() ran.  torch.profiler now and
    then leaves a kernel out of its record, so fn (which must be repeatable) runs up to `tries` times
    under it until every expected kernel has been seen; the union is returned, so a kernel that should
    not run still shows."""
    ran, names = set(), []
    for _ in range(tries):
        names = _cuda_kernel_names(fn)
        ran |= {s for s in map(kernel_signature, names) if s is not None}
        if ran >= expected:
            break
    if not ran:
        control = _cuda_kernel_names(lambda: torch.ones(4, device=DEV).add_(1))
        if not control:
            pytest.fail("torch.profiler records no CUDA kernels here, not even torch's own: the kernel each "
                        "step runs cannot be checked")
        if not names:
            pytest.fail("torch.profiler recorded a torch kernel but none while the fused step ran")
    return ran


# ---------------------------------------------------------------------------- the child-process re-run
def rerun(module_file, switch, k=None):
    """pytest over module_file (with -k k when given) in a fresh process with the environment switch
    "NAME=value" set -- the switches are read once per process; asserts that it passed and returns its
    output."""
    name, value = switch.split("=")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(module_file)] + (["-k", k] if k else [])
    start = time.time()
    proc = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **{name: value}), capture_output=True, text=True,
                          timeout=1200)
    print("%s: %.0f s\n%s" % (switch, time.time() - start, proc.stdout[-600:]))
    assert proc.returncode == 0, "%s\n%s\n%s" % (switch, proc.stdout[-6000:], proc.stderr[-3000:])
    assert " passed" in proc.stdout, proc.stdout[-2000:]
    return proc.stdout


# ---------------------------------------------------------------------------- the CPU stand-in engine
_KIND_OF_CODE = {_lib.TRANSE_L2: "transe_l2", _lib.DISTMULT: "distmult", _lib.COMPLEX: "complex"}
_ENT_KEYS = {"transe_l2": ("ent",), "distmult": ("ent",), "complex": ("re_ent", "im_ent")}
_REL_KEYS = {"transe_l2": ("rel",), "distmult": ("rel",), "complex": ("re_rel", "im_rel")}


def pair_loss(kind, pos, neg, margin=0.0):
    """utils/losses.py:12-112 with torch's modules, summed over the pairs."""
    if kind == _lib.LOSS_MARGIN:
        return torch.relu(margin - pos + neg).sum()
    if kind == _lib.LOSS_LOGISTIC:
        crit = torch.nn.SoftMarginLoss(reduction="sum")
        return crit(pos, torch.ones_like(pos)) + crit(neg, -torch.ones_like(neg))
    crit = torch.nn.BCELoss(reduction="sum")
    return crit(torch.sigmoid(pos), torch.ones_like(pos)) + crit(torch.sigmoid(neg), torch.zeros_like(neg))


class OracleStepEngine:
    """CPU stand-in for CudaEngine's sharded-step methods (tests only).  The draw law follows the step:
    positional (step.pos), relation-corrupting (step.n_rel > 0) or the entity step; the loss follows
    step.loss_kind."""

    def __init__(self):
        self.calls = []

    def gather_rows(self, spec, idx):
        planes = [spec.ent0] + ([spec.ent1] if spec.ent1 is not None else [])
        out = torch.zeros(idx.shape[0], len(planes), spec.dim)
        own = (idx >= spec.ent_lo) & (idx < spec.ent_lo + spec.n_rows)
        for p, tab in enumerate(planes):
            out[own, p] = tab[idx[own] - spec.ent_lo]
        return out

    def _partial(self, step, tables, h, t, r, probs, hrows, trows, grad):
        """Loss of the negatives this shard owns, from a table [local rows | hrows | trows]: an entity
        negative on the rank holding its replacement, a relation negative on the rank holding the
        positive's head; the positive's term once per owned negative."""
        kind = _KIND_OF_CODE[step.code]
        b, n = h.shape[0], step.n_rows
        ent = [x for x in tables[:2] if x is not None]
        P = {}
        for p, key in enumerate(_ENT_KEYS[kind]):
            P[key] = torch.cat([ent[p], hrows[:, p], trows[:, p]]).clone().requires_grad_(grad)
        for p, key in enumerate(_REL_KEYS[kind]):
            P[key] = tables[2 + p].clone().requires_grad_(grad)
        if step.pos is not None:            # k: 0 tail, 1 head, 2 relation replaced
            head, e = stand_in_pos_draws(step.seed, step.offset, r, step.n_neg, probs, step.n_ent, step.pos)
            k = head.long()
        elif step.n_rel > 0:
            k, e = stand_in_rel_draws(step.seed, step.offset, h, r, step.n_neg, probs, step.n_ent, step.n_rel,
                                      step.rel_share)
        else:
            head, e = stand_in_draws(step.seed, step.offset, r, step.n_neg, probs, step.n_ent)
            k = head.long()
        holder = torch.where(k == 2, h.repeat(step.n_neg), e)
        own = (holder >= step.ent_lo) & (holder < step.ent_lo + n)
        i = torch.arange(b).repeat(step.n_neg)[own]
        k, e = k[own], e[own]
        loc = e - step.ent_lo
        nh = torch.where(k == 1, loc, n + i)
        nt = torch.where(k == 0, loc, n + b + i)
        nr = torch.where(k == 2, e, r[i])
        pos = oracle.score_triples(kind, P, n + i, n + b + i, r[i])
        neg = oracle.score_triples(kind, P, nh, nt, nr)
        return pair_loss(step.loss_kind, pos, neg, step.margin), P

    def margin_step_fwd(self, step, tables, h, t, r, probs, hrows, trows):
        self.calls.append("fwd")
        with torch.no_grad():
            return self._partial(step, tables, h, t, r, probs, hrows, trows, False)[0].float()

    def margin_step_bwd(self, step, tables, grads, h, t, r, probs, gloss, hrows, trows, grad_hrows, grad_trows):
        self.calls.append("bwd")
        kind = _KIND_OF_CODE[step.code]
        with torch.enable_grad():          # autograd's backward runs with grad mode off
            loss, P = self._partial(step, tables, h, t, r, probs, hrows, trows, True)
            (loss * gloss).backward()
        n, b = step.n_rows, h.shape[0]
        for p, key in enumerate(_ENT_KEYS[kind]):
            gx = P[key].grad
            grads[p] += gx[:n]
            grad_hrows[:, p] += gx[n:n + b]
            grad_trows[:, p] += gx[n + b:]
        for p, key in enumerate(_REL_KEYS[kind]):
            grads[2 + p] += P[key].grad

    def scatter_rows_add(self, code, dim, grad0, grad1, ent_lo, idx, rows):
        self.calls.append("scatter")
        own = (idx >= ent_lo) & (idx < ent_lo + grad0.shape[0])
        for p, g in enumerate(x for x in (grad0, grad1) if x is not None):
            g.index_add_(0, idx[own] - ent_lo, rows[own, p])


class CountingShard(EntityShard):
    """EntityShard that counts its collectives."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.collectives = []

    def all_reduce_sum(self, t):
        self.collectives.append(("all_reduce", t.numel()))
        return super().all_reduce_sum(t)

    def stack_all(self, t):
        self.collectives.append(("stack_all", t.numel()))
        return super().stack_all(t)


class NoCollectiveShard(EntityShard):
    """An EntityShard whose collectives fail: argument errors must come before any of them."""

    def all_reduce_sum(self, t):
        raise AssertionError("collective reached")

    stack_all = all_reduce_sum


def oracle_loss(kind, loss_kind, model, h, t, r, nh, nt, nr=None, margin=0.0):
    """pair_loss of the whole model on the given negatives by the oracle's CPU autograd: (loss, {oracle
    key: gradient})."""
    P = {k: v.requires_grad_(True) for k, v in helpers.oracle_params(kind, model).items()}
    n_neg = nh.shape[0] // h.shape[0]
    pos = oracle.score_triples(kind, P, h, t, r).repeat(n_neg)
    neg = oracle.score_triples(kind, P, nh, nt, r.repeat(n_neg) if nr is None else nr)
    loss = pair_loss(loss_kind, pos, neg, margin)
    loss.backward()
    return loss.item(), {k: v.grad for k, v in P.items()}


def param_names(kind):
    """{oracle key: parameter name} of the stand-in's models."""
    names = ("ent_emb.weight", "rel_emb.weight") if kind != "complex" else \
        ("re_ent_emb.weight", "im_ent_emb.weight", "re_rel_emb.weight", "im_rel_emb.weight")
    return dict(zip(_ENT_KEYS[kind] + _REL_KEYS[kind], names))


def grads_match(kind, local, want, shard, suffix=""):
    """{oracle key + suffix: whether the local model's gradient is the oracle's} -- entity tables on the
    shard's rows."""
    params = dict(local.named_parameters())
    return {key + suffix: torch.allclose(params[name].grad, want[key][shard.lo:shard.hi] if "ent" in key else
                                         want[key], rtol=1e-4, atol=1e-6)
            for key, name in param_names(kind).items()}


def every_rank_ok(ret, world, min_checks=0):
    """Every rank of gloo.spawn reported no error, at least min_checks checks, and every check true."""
    for rank in range(world):
        res = ret[rank]
        assert "error" not in res, "rank %d: %s" % (rank, res.get("error"))
        bad = [k for k, v in res.items() if not v]
        assert not bad and len(res) >= min_checks, "rank %d: %s" % (rank, res)


# ---------------------------------------------------------------------------- the public API, two processes
def train_with(sampler, model, batches, shard, crit, n_neg=None):
    """SGD(lr 0.05) through sampler.fused_step over the batches: the losses.  crit: a margin (float) or a
    criterion."""
    margin, crit = (crit, None) if isinstance(crit, float) else (None, crit)
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    losses = []
    for h, t, r in batches:
        opt.zero_grad()
        loss = sampler.fused_step(model, h, t, r, margin, n_neg, criterion=crit, shard=shard)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    return losses


def whole_against_shard(runs, new_sampler, dev, n_batches, n_neg=None, on_ranks=False, loss_atol=0.0):
    """One rank of the two-process public-API run: for each (kind, dim, crit) of runs, the whole model and
    the model holding this rank's entity rows trained side by side from fresh samplers (new_sampler(kg)) over
    n_batches batches of 512 facts of one graph, then the losses and parameters compared.  on_ranks: the
    losses and relation tables are also the same on every rank.  Returns ({check: bool}, kg, batches, the
    last local model, its shard)."""
    res = {}
    n_ent, n_rel = 3001, 7
    hh, tt, rr = helpers.random_graph(n_ent, n_rel, 6000, seed=5)
    kg = tk.KnowledgeGraph(hh, tt, rr, n_ent, n_rel, dict_of_heads={}, dict_of_tails={})
    batches = [(hh[i:i + 512].to(dev), tt[i:i + 512].to(dev), rr[i:i + 512].to(dev))
               for i in range(0, 512 * n_batches, 512)]
    for kind, dim, crit in runs:
        full = helpers.make_model(kind, dim, n_ent, n_rel, seed=21).to(dev)
        shard = EntityShard.from_group(n_ent, local_storage=True)
        local = helpers.local_model(kind, full, shard.lo, shard.hi, n_rel, dim)
        want = train_with(new_sampler(kg), full, batches, None, crit, n_neg)
        got = train_with(new_sampler(kg), local, batches, shard, crit, n_neg)
        if on_ranks:
            everyone = shard.stack_all(torch.tensor(got, dtype=torch.float64, device=dev))
            res[kind + "/losses_equal_on_ranks"] = bool((everyone == everyone[0]).all())
        res[kind + "/losses_close"] = all(abs(a - b) <= 1e-5 * abs(b) + loss_atol for a, b in zip(got, want))
        for name, p in local.named_parameters():
            ref = dict(full.named_parameters())[name]
            if "ent_emb" in name:
                ref = ref[shard.lo:shard.hi]
            elif on_ranks:
                allp = shard.stack_all(p.detach())
                res[kind + "/" + name + "/bitwise_on_ranks"] = bool((allp == allp[0]).all())
            res[kind + "/" + name] = torch.allclose(p, ref, rtol=1e-4, atol=1e-5)
    return res, kg, batches, local, shard


# ---------------------------------------------------------------------------- the ABI
def header():
    """include/kge_b200.h without its comments."""
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "kge_b200.h")).read(), flags=re.S)


def header_fields(typedef):
    """Field names of `typedef` in include/kge_b200.h, in order."""
    body = re.search(r"typedef struct \{([^{}]*)\}\s*%s\s*;" % typedef, header(), flags=re.S).group(1)
    return [re.findall(r"[A-Za-z_][A-Za-z0-9_]*", part)[-1]
            for decl in body.split(";") if decl.strip() for part in decl.split(",")]


_ABI_CHILD = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from torchkge_b200 import _lib
lib = _lib.load()
F = 8   # a non-NULL stand-in pointer: every call below fails its checks before touching memory
res = {}
g = _lib.Grads(F, None, F, None)


def ok_args(cls, fields):
    a = cls()
    b = a.base
    b.tb.model, b.tb.dim, b.tb.ent0, b.tb.rel0 = _lib.DISTMULT, 8, F, F
    b.n_neg, b.b, b.n_ent, b.h, b.t, b.r, b.bern_probs, b.loss = 2, 4, 10, F, F, F, F, F
    for k, v in fields.items():
        setattr(a, k, v)
    return a


def step_cases(cls, fields, fwd, bwd, cases):
    for name, edit in cases.items():
        a = ok_args(cls, fields)
        edit(a)
        p = None if name == "null" else ctypes.byref(a)
        res["fwd_" + name] = fwd(p)
        res["bwd_" + name] = bwd(p, ctypes.byref(g), F)
    a = ok_args(cls, fields)
    res["bwd_no_grad_loss"] = bwd(ctypes.byref(a), ctypes.byref(g), None)
    res["bwd_no_grads"] = bwd(ctypes.byref(a), None, F)
    a.base.hrows, a.base.trows, a.base.n_rows = F, F, 10
    res["bwd_sharded_no_grad_rows"] = bwd(ctypes.byref(a), ctypes.byref(g), F)
"""


def malformed_calls(body):
    """{name: return code} that `body` records in `res` in a child process that sees no GPU.  The child
    defines F (a non-NULL pointer no call may touch), g (Grads over F), ok_args(cls, fields) (a well-formed
    cls -- RelStepArgs or PosStepArgs -- over F, with `fields` set beside its base) and
    step_cases(cls, fields, fwd, bwd, cases): each case's edit of ok_args through fwd and bwd, then bwd
    without its loss gradient, without its gradients, and sharded without row gradients."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _ABI_CHILD + body + "\nprint(json.dumps(res))\n", ROOT], env=env,
                          capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, proc.stderr[-3000:]
    return json.loads(proc.stdout.strip().splitlines()[-1])
