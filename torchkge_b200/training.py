"""Training-side entry points: differentiable per-triple scoring (``Model.scoring_function``),
the three losses and the fused sample + score + loss step, as autograd Functions over the CUDA
kernels of csrc/train.cu.  Gradients are dense tables (what ``nn.Embedding`` yields in the
reference), accumulated with atomics.
"""
import collections
import ctypes
import struct

import torch

from . import _lib
from .engine import (PROJECTED_SPECS, EntityShard, ModelSpec, QueryShard, _check_table, _device_guard,
                     _exchanged_rows, _plane_ptrs, _ptr, _stream, check_transd_widths, default_engine)


def _param_tensors(model, code):
    """Parameters in ModelSpec order (ent0, ent1, rel0, rel1); RotatE's relation planes are
    differentiable functions (cos, sin) of its phase parameter."""
    if code in (_lib.TRANSE_L1, _lib.TRANSE_L2, _lib.DISTMULT, _lib.TORUSE_L1, _lib.TORUSE_L2):
        return model.ent_emb.weight, None, model.rel_emb.weight, None
    if code == _lib.RESCAL:
        return model.ent_emb.weight, None, model.rel_mat.weight, None
    if code == _lib.COMPLEX:
        return (model.re_ent_emb.weight, model.im_ent_emb.weight, model.re_rel_emb.weight,
                model.im_rel_emb.weight)
    if code == _lib.ROTATE:
        ph = model.rel_emb.weight
        return model.re_ent_emb.weight, model.im_ent_emb.weight, torch.cos(ph), torch.sin(ph)
    if code == _lib.ANALOGY:
        # three planes per table: one stacked (3, n, dim) tensor in the ent0 / rel0 slot (autograd
        # splits its gradient back onto the three embeddings); see _plane_ptrs
        return (torch.stack([model.sc_ent_emb.weight, model.re_ent_emb.weight, model.im_ent_emb.weight]), None,
                torch.stack([model.sc_rel_emb.weight, model.re_rel_emb.weight, model.im_rel_emb.weight]), None)
    raise NotImplementedError(code)


def _kernel_dim(model, code):
    """Width of one plane: emb_dim, or Analogy's scalar_dim (= complex_dim on this path)."""
    return model.scalar_dim if code == _lib.ANALOGY else model.emb_dim


def _tables(code, dim, tensors):
    tb = _lib.Tables()
    tb.model, tb.dim = code, dim
    tb.ent0, tb.ent1 = _plane_ptrs(tensors[0], tensors[1])
    tb.rel0, tb.rel1 = _plane_ptrs(tensors[2], tensors[3])
    return tb


def _check_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.KgeLibraryError("training kernels need CUDA tensors (got %s); there is no "
                                       "CPU fallback" % t.device)


def _idx(t, dev):
    return t.to(device=dev, dtype=torch.int64).contiguous()


def _zero_grads(tensors):
    gs = [None if x is None else torch.zeros_like(x, dtype=torch.float32) for x in tensors]
    g = _lib.Grads()
    g.ent0, g.ent1 = _plane_ptrs(gs[0], gs[1])
    g.rel0, g.rel1 = _plane_ptrs(gs[2], gs[3])
    return gs, g


class _ScoreTriples(torch.autograd.Function):
    @staticmethod
    def forward(ctx, code, dim, h, t, r, ent0, ent1, rel0, rel1):
        tensors = [None if x is None else x.detach().contiguous() for x in (ent0, ent1, rel0, rel1)]
        _check_cuda(tensors[0], h, t, r)
        dev = tensors[0].device
        h, t, r = _idx(h, dev), _idx(t, dev), _idx(r, dev)
        n = h.shape[0]
        out = torch.empty(n, dtype=torch.float32, device=dev)
        tb = _tables(code, dim, tensors)
        _lib.check(_lib.load().kge_score_triples_fwd(ctypes.byref(tb), _ptr(h), _ptr(t), _ptr(r), n,
                                                     _ptr(out), _stream(dev)), "kge_score_triples_fwd")
        ctx.code, ctx.dim = code, dim
        ctx.save_for_backward(h, t, r, *[x for x in tensors if x is not None])
        ctx.present = [x is not None for x in tensors]
        return out

    @staticmethod
    def backward(ctx, gout):
        saved = list(ctx.saved_tensors)
        h, t, r = saved[:3]
        it = iter(saved[3:])
        tensors = [next(it) if p else None for p in ctx.present]
        dev = h.device
        gout = gout.contiguous().float()
        tb = _tables(ctx.code, ctx.dim, tensors)
        gs, g = _zero_grads(tensors)
        _lib.check(_lib.load().kge_score_triples_bwd(ctypes.byref(tb), ctypes.byref(g), _ptr(h), _ptr(t),
                                                     _ptr(r), h.shape[0], _ptr(gout), _stream(dev)),
                   "kge_score_triples_bwd")
        return (None, None, None, None, None, *gs)


def _training_code(model):
    """Kernel selector of the training-side kernels.  TorusE: the torus dissimilarities have their own
    per-triple kernels (no row normalisation, fractional parts taken on the fly, translation.py:706-720);
    its plain-'L1' variant is not on the CUDA path (the TransE-L1 kernels L2-normalise the entity rows)."""
    if type(model).__name__ == "TorusEModel":
        dname = getattr(model.dissimilarity, "__name__", str(model.dissimilarity))
        code = {"l1_torus_dissimilarity": _lib.TORUSE_L1, "l2_torus_dissimilarity": _lib.TORUSE_L2}.get(dname)
        if code is None:
            raise NotImplementedError("TorusE with dissimilarity %s has no training kernel" % dname)
        return code
    if type(model).__name__ == "AnalogyModel":
        if model.scalar_dim != model.complex_dim:
            raise NotImplementedError("the Analogy training kernels need scalar_dim == complex_dim")
        return _lib.ANALOGY
    return ModelSpec.from_model(model).code


def score_triples(model, h_idx, t_idx, r_idx):
    """``model.scoring_function(h_idx, t_idx, r_idx)`` -> (n,) float scores, differentiable with
    respect to the model's embedding tables."""
    code = _training_code(model)
    ent0, ent1, rel0, rel1 = _param_tensors(model, code)
    return _ScoreTriples.apply(code, _kernel_dim(model, code), h_idx, t_idx, r_idx, ent0, ent1, rel0, rel1)


class _ProjectedScoreTriples(torch.autograd.Function):
    """TransH's or TransD's scoring_function on kge_<prefix>_score_triples_fwd / _bwd (translation.py:183-202,
    538-568): ``prefix`` "transh" or "transd", ``dims`` the widths and ``tables`` the raw tables, in the order of
    the C entry points."""

    @staticmethod
    def forward(ctx, prefix, dims, h, t, r, *tables):
        tables = [x.detach().contiguous() for x in tables]
        for x in tables:
            if x.dtype != torch.float32:
                raise TypeError("embedding tables must be float32, got %s" % x.dtype)
        _check_cuda(tables[0], h, t, r)
        dev = tables[0].device
        h, t, r = _idx(h, dev), _idx(t, dev), _idx(r, dev)
        out = torch.empty(h.shape[0], dtype=torch.float32, device=dev)
        name = "kge_%s_score_triples_fwd" % prefix
        _lib.check(getattr(_lib.load(), name)(*(_ptr(x) for x in tables), *dims, _ptr(h), _ptr(t), _ptr(r),
                                              h.shape[0], _ptr(out), _stream(dev)), name)
        ctx.prefix, ctx.dims = prefix, dims
        ctx.save_for_backward(h, t, r, *tables)
        return out

    @staticmethod
    def backward(ctx, gout):
        h, t, r, *tables = ctx.saved_tensors
        grads = [torch.zeros_like(x) for x in tables]
        gout = gout.contiguous().float()
        name = "kge_%s_score_triples_bwd" % ctx.prefix
        _lib.check(getattr(_lib.load(), name)(*(_ptr(x) for x in tables), *(_ptr(g) for g in grads), *ctx.dims,
                                              _ptr(h), _ptr(t), _ptr(r), h.shape[0], _ptr(gout), _stream(h.device)),
                   name)
        return (None, None, None, None, None, *grads)


def score_triples_transh(model, h_idx, t_idx, r_idx):
    """TransH's ``scoring_function(h_idx, t_idx, r_idx)`` -> (n,) float scores, differentiable with respect
    to ent_emb, rel_emb and norm_vect."""
    return _ProjectedScoreTriples.apply("transh", (model.emb_dim,), h_idx, t_idx, r_idx, model.ent_emb.weight,
                                        model.rel_emb.weight, model.norm_vect.weight)


def score_triples_transd(model, h_idx, t_idx, r_idx):
    """TransD's ``scoring_function(h_idx, t_idx, r_idx)`` -> (n,) float scores, differentiable with respect
    to ent_emb, rel_emb, ent_proj_vect and rel_proj_vect."""
    check_transd_widths(model.ent_emb_dim, model.rel_emb_dim)
    return _ProjectedScoreTriples.apply("transd", (model.ent_emb_dim, model.rel_emb_dim), h_idx, t_idx, r_idx,
                                        model.ent_emb.weight, model.rel_emb.weight, model.ent_proj_vect.weight,
                                        model.rel_proj_vect.weight)


class _MarginLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, neg, margin):
        _check_cuda(pos, neg)
        pos, neg = pos.detach().contiguous().float(), neg.detach().contiguous().float()
        if pos.shape != neg.shape:
            raise ValueError("positive and negative score tensors must have the same shape")
        loss = torch.zeros((), dtype=torch.float32, device=pos.device)
        _lib.check(_lib.load().kge_margin_loss_fwd(_ptr(pos), _ptr(neg), pos.numel(), float(margin),
                                                   _ptr(loss), _stream(pos.device)), "kge_margin_loss_fwd")
        ctx.margin = float(margin)
        ctx.save_for_backward(pos, neg)
        return loss

    @staticmethod
    def backward(ctx, gl):
        pos, neg = ctx.saved_tensors
        gl = gl.contiguous().float()
        gp, gn = torch.empty_like(pos), torch.empty_like(neg)
        _lib.check(_lib.load().kge_margin_loss_bwd(_ptr(pos), _ptr(neg), pos.numel(), ctx.margin,
                                                   _ptr(gl), _ptr(gp), _ptr(gn), _stream(pos.device)),
                   "kge_margin_loss_bwd")
        return gp, gn, None


def margin_loss(pos, neg, margin):
    return _MarginLoss.apply(pos, neg, margin)


class _PairLoss(torch.autograd.Function):
    """LogisticLoss / BinaryCrossEntropyLoss (kge_pair_loss_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, pos, neg, kind):
        _check_cuda(pos, neg)
        pos, neg = pos.detach().contiguous().float(), neg.detach().contiguous().float()
        if pos.shape != neg.shape:
            raise ValueError("positive and negative score tensors must have the same shape")
        loss = torch.zeros((), dtype=torch.float32, device=pos.device)
        _lib.check(_lib.load().kge_pair_loss_fwd(kind, _ptr(pos), _ptr(neg), pos.numel(), _ptr(loss),
                                                 _stream(pos.device)), "kge_pair_loss_fwd")
        ctx.kind = kind
        ctx.save_for_backward(pos, neg)
        return loss

    @staticmethod
    def backward(ctx, gl):
        pos, neg = ctx.saved_tensors
        gl = gl.contiguous().float()
        gp, gn = torch.empty_like(pos), torch.empty_like(neg)
        _lib.check(_lib.load().kge_pair_loss_bwd(ctx.kind, _ptr(pos), _ptr(neg), pos.numel(), _ptr(gl),
                                                 _ptr(gp), _ptr(gn), _stream(pos.device)),
                   "kge_pair_loss_bwd")
        return gp, gn, None


def pair_loss(pos, neg, kind):
    return _PairLoss.apply(pos, neg, kind)


def loss_kind_of(criterion):
    """(loss kind, margin) of the fused step for ``criterion``: a ``MarginLoss``, ``LogisticLoss`` or
    ``BinaryCrossEntropyLoss`` of this package or of torchkge, recognised by class name as models are
    (torchkge's ``MarginLoss`` keeps its margin in ``criterion.loss.margin``).  The margin is 0.0 for
    the losses that have none.  Anything else raises TypeError."""
    name = type(criterion).__name__
    if name == "MarginLoss":
        margin = getattr(criterion, "margin", None)
        if margin is None:
            margin = getattr(getattr(criterion, "loss", None), "margin", None)
        if margin is None:
            raise TypeError("MarginLoss without a margin attribute")
        return _lib.LOSS_MARGIN, float(margin)
    if name == "LogisticLoss":
        return _lib.LOSS_LOGISTIC, 0.0
    if name == "BinaryCrossEntropyLoss":
        return _lib.LOSS_BCE, 0.0
    raise TypeError("the fused training step supports MarginLoss, LogisticLoss and BinaryCrossEntropyLoss, "
                    "not %s" % name)


class _MarginStep(torch.autograd.Function):
    """The fused step on the whole table; loss_kind: _lib.LOSS_* (margin is used by the margin loss only)."""

    @staticmethod
    def forward(ctx, code, dim, n_ent, margin, n_neg, h, t, r, nh, nt, probs, seed, offset,
                ent0, ent1, rel0, rel1, loss_kind=_lib.LOSS_MARGIN, nr=None, rel=None, pos=None):
        # rel: (n_rel, rel_share) for a relation-corrupting step (kge_rel_step_*; external negatives then
        # come with nr), None for the entity step (kge_margin_step_*)
        # pos: (head_offs, head_ents, tail_offs, tail_ents) for a positional step (kge_pos_step_*)
        tensors = [None if x is None else x.detach().contiguous() for x in (ent0, ent1, rel0, rel1)]
        _check_cuda(tensors[0], h, t, r)
        dev = tensors[0].device
        h, t, r = _idx(h, dev), _idx(t, dev), _idx(r, dev)
        if nh is not None:
            nh, nt = _idx(nh, dev), _idx(nt, dev)
        if nr is not None:
            nr = _idx(nr, dev)
        if probs is not None:
            probs = probs.to(device=dev, dtype=torch.float32).contiguous()
        if pos is not None:
            pos = tuple(_idx(x, dev) for x in pos)
        loss = torch.zeros((), dtype=torch.float32, device=dev)
        a = _MarginStep._args(code, dim, n_ent, margin, n_neg, h, t, r, nh, nt, probs, seed, offset,
                              tensors, loss, dev, loss_kind, nr, rel, pos)
        name = _MarginStep._entry(a, "fwd")
        _lib.check(getattr(_lib.load(), name)(ctypes.byref(a)), name)
        ctx.meta = (code, dim, n_ent, margin, n_neg, seed, offset, loss_kind, rel)
        ctx.present = [x is not None for x in tensors]
        ctx.has_neg, ctx.has_nr, ctx.has_probs = nh is not None, nr is not None, probs is not None
        ctx.has_pos = pos is not None
        extra = (([nh, nt] if nh is not None else []) + ([nr] if nr is not None else []) +
                 ([probs] if probs is not None else []) + (list(pos) if pos is not None else []))
        ctx.save_for_backward(h, t, r, *extra, *[x for x in tensors if x is not None])
        return loss

    @staticmethod
    def _entry(a, which):
        """The entry point for ``a``: kge_margin_step_<which>, kge_rel_step_<which> or kge_pos_step_<which>."""
        return {_lib.RelStepArgs: "kge_rel_step_", _lib.PosStepArgs: "kge_pos_step_"}.get(
            type(a), "kge_margin_step_") + which

    @staticmethod
    def _args(code, dim, n_ent, margin, n_neg, h, t, r, nh, nt, probs, seed, offset, tensors, loss, dev,
              loss_kind=_lib.LOSS_MARGIN, nr=None, rel=None, pos=None):
        """kge_margin_step_args_t, or with rel = (n_rel, rel_share) kge_rel_step_args_t around it, or with
        pos = (head_offs, head_ents, tail_offs, tail_ents) kge_pos_step_args_t around it."""
        a = _lib.MarginStepArgs()
        a.tb = _tables(code, dim, tensors)
        a.n_neg, a.margin, a.b, a.n_ent = n_neg, float(margin), h.shape[0], n_ent
        a.h, a.t, a.r, a.nh, a.nt, a.bern_probs = (_ptr(x) for x in (h, t, r, nh, nt, probs))
        a.seed, a.offset = int(seed), int(offset)
        a.loss, a.stream = _ptr(loss), _stream(dev)
        a.loss_kind = int(loss_kind)
        if pos is not None:
            pa = _lib.PosStepArgs()
            pa.base, pa.n_rel = a, int(pos[0].shape[0]) - 1
            pa.head_offs, pa.head_ents, pa.tail_offs, pa.tail_ents = (_ptr(x) for x in pos)
            return pa
        if rel is None:
            return a
        ra = _lib.RelStepArgs()
        ra.base = a
        ra.n_rel, ra.rel_share, ra.nr = int(rel[0]), float(rel[1]), _ptr(nr)
        return ra

    @staticmethod
    def backward(ctx, gl):
        code, dim, n_ent, margin, n_neg, seed, offset, loss_kind, rel = ctx.meta
        saved = list(ctx.saved_tensors)
        h, t, r = saved[:3]
        k = 3
        nh = nt = nr = probs = None
        if ctx.has_neg:
            nh, nt = saved[k], saved[k + 1]
            k += 2
        if ctx.has_nr:
            nr = saved[k]
            k += 1
        if ctx.has_probs:
            probs = saved[k]
            k += 1
        pos = None
        if ctx.has_pos:
            pos = tuple(saved[k:k + 4])
            k += 4
        it = iter(saved[k:])
        tensors = [next(it) if p else None for p in ctx.present]
        dev = h.device
        gl = gl.contiguous().float()
        dummy = torch.zeros((), dtype=torch.float32, device=dev)
        a = _MarginStep._args(code, dim, n_ent, margin, n_neg, h, t, r, nh, nt, probs, seed, offset,
                              tensors, dummy, dev, loss_kind, nr, rel, pos)
        gs, g = _zero_grads(tensors)
        name = _MarginStep._entry(a, "bwd")
        _lib.check(getattr(_lib.load(), name)(ctypes.byref(a), ctypes.byref(g), _ptr(gl)), name)
        return (None,) * 13 + tuple(gs) + (None,) * 4


#: what every rank's kernels of one sharded step are told (engine.margin_step_fwd / _bwd)
#: loss_kind: _lib.LOSS_* (default the margin loss); n_rel > 0: a relation-corrupting step that replaces an
#: entity with probability rel_share (kge_rel_step_*), n_rel = 0 the entity step; pos = (head_offs, head_ents,
#: tail_offs, tail_ents): the positional step (kge_pos_step_*), every rank holding the whole CSR
ShardedStep = collections.namedtuple("ShardedStep",
                                     "code dim n_ent ent_lo n_rows n_neg margin seed offset loss_kind n_rel rel_share "
                                     "pos", defaults=(_lib.LOSS_MARGIN, 0, 1.0, None))


class _ShardedMarginStep(torch.autograd.Function):
    """The fused step (any loss kind) on a range-partitioned entity table (EntityShard, local storage):
      1. the positives' h / t rows: each rank gathers the rows it holds, one sum-all-reduce;
      2. every rank draws all negatives with the global n_ent and scores those whose replaced entity
         it holds (the intact entity's row comes from step 1, the relation table is replicated);
      3. one all-reduce of the scalar loss.
    Backward: replaced rows go straight into the local gradient; the gradients of the positives' rows
    (grad_hrows / grad_trows) and of the relations are summed over the ranks by ONE all-reduce, after
    which every rank adds the rows it holds into its entity gradient.  Communication per step:
    2 b planes dim floats forward, the same plus the relation table backward -- independent of n_neg."""

    @staticmethod
    def forward(ctx, step, shard, engine, h, t, r, probs, ent0, ent1, rel0, rel1):
        tensors = [None if x is None else x.detach().contiguous() for x in (ent0, ent1, rel0, rel1)]
        dev = tensors[2].device
        h, t, r = _idx(h, dev), _idx(t, dev), _idx(r, dev)
        probs = probs.to(device=dev, dtype=torch.float32).contiguous()
        b = h.shape[0]
        with _device_guard(dev):
            spec = _row_spec(step, tensors)
            rows = _exchanged_rows(spec, torch.cat([h, t]), shard, engine)   # (2b, planes, dim)
            hrows, trows = rows[:b], rows[b:]
            if step.n_rows > 0:
                loss = engine.margin_step_fwd(step, tensors, h, t, r, probs, hrows, trows)
            else:             # holds no entity: scores no negative, still joins every collective
                loss = torch.zeros((), dtype=torch.float32, device=dev)
            shard.all_reduce_sum(loss)
        ctx.step, ctx.shard, ctx.engine = step, shard, engine
        ctx.present = [x is not None for x in tensors]
        ctx.save_for_backward(h, t, r, probs, rows, *[x for x in tensors if x is not None])
        return loss

    @staticmethod
    def backward(ctx, gl):
        step, shard, engine = ctx.step, ctx.shard, ctx.engine
        saved = list(ctx.saved_tensors)
        h, t, r, probs, rows = saved[:5]
        it = iter(saved[5:])
        tensors = [next(it) if p else None for p in ctx.present]
        dev = h.device
        b = h.shape[0]
        gl = gl.detach().to(device=dev, dtype=torch.float32).contiguous()
        # grad_hrows, grad_trows and the relation gradients are views of ONE buffer: one all-reduce
        sizes = [rows.numel()] + [0 if x is None else x.numel() for x in tensors[2:]]
        flat = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        grad_rows = flat[:sizes[0]].view(rows.shape)
        grel = [None if x is None else part.view(x.shape)
                for x, part in zip(tensors[2:], flat[sizes[0]:].split(sizes[1:]))]
        gent = [None if x is None else torch.zeros_like(x, dtype=torch.float32) for x in tensors[:2]]
        grads = gent + grel
        with _device_guard(dev):
            if step.n_rows > 0:
                engine.margin_step_bwd(step, tensors, grads, h, t, r, probs, gl, rows[:b], rows[b:],
                                       grad_rows[:b], grad_rows[b:])
            shard.all_reduce_sum(flat)
            if step.n_rows > 0:
                engine.scatter_rows_add(step.code, step.dim, gent[0], gent[1], step.ent_lo, torch.cat([h, t]),
                                        grad_rows)
        return (None,) * 7 + tuple(grads)


def _row_spec(step, tensors):
    """ModelSpec over this shard's entity rows, for the positive-row gather (engine.gather_rows)."""
    e0, e1, r0, r1 = tensors
    e2 = r2 = None
    if e0.dim() == 3:            # Analogy: stacked (3, n, dim) planes
        e0, e1, e2 = e0[0], e0[1], e0[2]
        r0, r1, r2 = r0[0], r0[1], r0[2]
    return ModelSpec(step.code, step.dim, step.n_ent, r0.shape[0], e0, e1, r0, r1, ent_lo=step.ent_lo,
                     ent2=e2, rel2=r2)


def _signed64(x):
    x = int(x) & 0xFFFFFFFFFFFFFFFF
    return x - (1 << 64) if x >= (1 << 63) else x


def sharded_margin_step(model, heads, tails, relations, margin, n_neg, bern_probs, seed, offset, shard,
                        engine=None, loss_kind=_lib.LOSS_MARGIN, rel_share=None, positional=None):
    """``fused_margin_step(..., shard=shard)`` (``fused_loss_step`` with ``loss_kind``) for a model that
    holds only the entity rows [shard.lo, shard.hi) of an EntityShard with local storage; the same
    (heads, tails, relations), seed, offset, n_neg, margin and loss kind on every rank.  Returns the full
    loss on every rank; its backward leaves every rank with the gradient of its own rows and the
    (identical) relation gradient.  Every rank counts the positive's term of a pair only for the
    negatives it scores, so the ranks' sums are the unsharded loss and gradients.
    ``engine``: CudaEngine or a stand-in with margin_step_fwd / margin_step_bwd / scatter_rows_add /
    gather_rows.
    ``rel_share``: a relation-corrupting step (``BernoulliRelationNegativeSampler``): each negative replaces
    an entity with probability rel_share, else the relation; the rank that holds a positive's head scores
    its relation negatives.  Every rank must pass the same rel_share (None: the entity step).
    ``positional``: (head_offs, head_ents, tail_offs, tail_ents), the whole candidate CSR on every rank (see
    ``fused_margin_step``); a negative is scored by the rank holding the entity it draws."""
    # argument errors first, on every rank: none of them may leave the others waiting in a collective
    if isinstance(shard, QueryShard):
        raise ValueError("the fused training step takes an EntityShard; QueryShard (data-parallel "
                         "replicas) is not supported")
    if not isinstance(shard, EntityShard):
        raise ValueError("shard must be an EntityShard, got %s" % type(shard).__name__)
    if not shard.local_storage:
        raise ValueError("the sharded training step needs EntityShard(local_storage=True): the model "
                         "holds only rows [lo, hi)")
    if bern_probs is None:
        raise ValueError("bern_probs must be given (a sharded step draws its own negatives)")
    code = _training_code(model)
    ent0, ent1, rel0, rel1 = _param_tensors(model, code)
    b = int(heads.shape[0])
    n_rel, share = (0, 1.0) if rel_share is None else (int(rel0.shape[-2]), float(rel_share))
    if rel_share is not None:
        _check_rel_share(n_rel, share)
    if positional is not None:
        if rel_share is not None:
            raise ValueError("positional negatives replace an entity: they take no rel_share")
        positional = _positional_csr(positional, int(rel0.shape[-2]), rel0.device)
    step = ShardedStep(code, _kernel_dim(model, code), shard.n_ent, shard.lo, int(ent0.shape[-2]), int(n_neg),
                       float(margin), int(seed) & 0xFFFFFFFFFFFFFFFF, int(offset) & 0xFFFFFFFFFFFFFFFF,
                       int(loss_kind), n_rel, share, positional)
    _check_table(step, shard)
    # one small collective: every rank must draw the same negatives for the same batch and loss.  The last
    # field holds the loss kind and, above it, the float32 bits of 1 - rel_share: 0 for the entity step,
    # whose draws are those of rel_share = 1; bit 40 marks the positional step
    kind_share = step.loss_kind | struct.unpack("<I", struct.pack("<f", 1.0 - share))[0] << 8
    if positional is not None:
        kind_share |= 1 << 40
    mine = torch.tensor([_signed64(step.seed), _signed64(step.offset), b, step.n_neg,
                         struct.unpack("<q", struct.pack("<d", step.margin))[0], kind_share],
                        dtype=torch.int64, device=rel0.device)
    everyone = shard.stack_all(mine)
    if not bool((everyone == mine).all()):
        raise ValueError("the ranks of a sharded step disagree on (seed, offset, batch size, n_neg, margin, "
                         "loss kind, rel_share and positional or not): %s" % everyone.tolist())
    if positional is not None:
        # every rank is positional here (the check above): a second collective of the CSR's sizes, so ranks
        # whose samplers were built on different graphs raise on every rank
        sizes = torch.tensor([int(x.shape[0]) for x in positional], dtype=torch.int64, device=rel0.device)
        every_size = shard.stack_all(sizes)
        if not bool((every_size == sizes).all()):
            raise ValueError("the ranks of a positional sharded step hold different candidate CSRs (sizes of "
                             "head_offs, head_ents, tail_offs, tail_ents per rank: %s)" % every_size.tolist())
    return _ShardedMarginStep.apply(step, shard, engine or default_engine(), heads, tails, relations,
                                    bern_probs, ent0, ent1, rel0, rel1)


def _check_rel_share(n_rel, rel_share):
    """The relation draw is uniform on [1, n_rel): it needs two relations unless it never happens."""
    if not 0.0 <= rel_share <= 1.0:
        raise ValueError("rel_share must lie in [0, 1], got %r" % (rel_share,))
    if n_rel < 2 and rel_share < 1.0:
        raise ValueError("relation corruption draws from [1, n_rel) and needs n_rel >= 2 (n_rel = %d); "
                         "use rel_share = 1" % n_rel)


def _positional_csr(positional, n_rel, dev):
    """The positional step's (head_offs, head_ents, tail_offs, tail_ents) as int64 tensors on dev, after
    checking that they are two CSRs over the model's n_rel relations."""
    if len(positional) != 4:
        raise ValueError("positional must be (head_offs, head_ents, tail_offs, tail_ents)")
    for name, x in zip(("head_offs", "head_ents", "tail_offs", "tail_ents"), positional):
        if not isinstance(x, torch.Tensor) or x.dim() != 1:
            raise ValueError("positional: %s must be a 1-D tensor" % name)
    for name, offs in (("head_offs", positional[0]), ("tail_offs", positional[2])):
        if offs.shape[0] != n_rel + 1:
            raise ValueError("positional: %s covers %d relations, the model has %d" % (name, offs.shape[0] - 1, n_rel))
    return tuple(_idx(x, dev) for x in positional)


def refuse_projected_fused_step(model):
    """TransH and TransD have per-triple kernels (score_triples_transh / _transd) but no fused training step."""
    name = type(model).__name__
    if name in PROJECTED_SPECS:
        raise NotImplementedError("%s has no fused training step: train it with model(h, t, r, nh, nt), "
                                  "a loss and backward()" % name)


def _fused_step(model, heads, tails, relations, loss_kind, margin, n_neg, negatives, bern_probs, seed, offset,
                shard, rel_share=None, positional=None):
    refuse_projected_fused_step(model)
    if negatives is not None and len(negatives) not in (2, 3):
        raise ValueError("negatives must be (neg_heads, neg_tails) or (neg_heads, neg_tails, neg_rels)")
    if positional is not None and negatives is not None:
        raise ValueError("positional sets how negatives are drawn; it takes no caller negatives")
    if positional is not None and rel_share is not None:
        raise ValueError("positional negatives replace an entity: they take no rel_share")
    if shard is not None:
        if negatives is not None:
            raise ValueError("external negatives are not supported by the sharded training step")
        return sharded_margin_step(model, heads, tails, relations, margin, n_neg, bern_probs, seed, offset,
                                   shard, loss_kind=loss_kind, rel_share=rel_share, positional=positional)
    spec_code = _training_code(model)
    ent0, ent1, rel0, rel1 = _param_tensors(model, spec_code)
    nh = nt = nr = None
    rel = None
    if positional is not None:
        positional = _positional_csr(positional, int(rel0.shape[-2]), rel0.device)
        if bern_probs is None:
            raise ValueError("a positional step needs bern_probs")
    if negatives is not None and rel_share is not None:
        raise ValueError("rel_share sets how negatives are drawn; with caller negatives give (neg_heads, "
                         "neg_tails, neg_rels) and no rel_share")
    if rel_share is not None:
        rel = (int(rel0.shape[-2]), float(rel_share))
        _check_rel_share(*rel)
    if negatives is not None:
        nh, nt = negatives[:2]
        if len(negatives) == 3:      # any positions may change: the draw parameters play no part
            nr = negatives[2]
            rel = (int(rel0.shape[-2]), 1.0)
        lengths = {int(x.shape[0]) for x in negatives}
        if len(lengths) != 1 or nh.shape[0] % max(int(heads.shape[0]), 1) != 0:
            raise ValueError("the negatives must have one common length, a multiple of the batch size (got %s "
                             "for a batch of %d)" % ([int(x.shape[0]) for x in negatives], heads.shape[0]))
        n_neg = int(nh.shape[0] // heads.shape[0])
    elif bern_probs is None:
        raise ValueError("either negatives or bern_probs must be given")
    return _MarginStep.apply(spec_code, _kernel_dim(model, spec_code), model.n_ent, margin, n_neg, heads, tails,
                             relations, nh, nt, bern_probs, seed, offset, ent0, ent1, rel0, rel1, loss_kind, nr, rel,
                             positional)


def fused_loss_step(model, heads, tails, relations, criterion, n_neg=1, negatives=None, bern_probs=None,
                    seed=0, offset=0, *, shard=None, rel_share=None, positional=None):
    """``fused_margin_step`` for any of the three losses: Bernoulli corruption (or the given
    ``negatives``), ``model(h, t, r, nh, nt)`` and ``criterion(pos, neg)`` in a single kernel,
    differentiable with respect to the embedding tables.

    criterion: ``MarginLoss(margin)``, ``LogisticLoss()`` or ``BinaryCrossEntropyLoss()``, of this
        package or of torchkge; anything else raises TypeError (on every rank, before any collective).
        The loss is summed over every (positive i, negative j) pair, the positive's score repeated
        n_neg times as in ``Model.forward``:
          logistic: softplus(-pos_i) + softplus(neg_ij)
          BCE     : -max(log sig(pos_i), -100) - max(log(1 - sig(neg_ij)), -100)
        and its gradients are those torch's SoftMarginLoss / BCELoss backward give.
    shard, rel_share, negatives, positional: as in ``fused_margin_step``; every rank must pass the same kind of
    loss.
    """
    kind, margin = loss_kind_of(criterion)
    return _fused_step(model, heads, tails, relations, kind, margin, n_neg, negatives, bern_probs, seed, offset,
                       shard, rel_share, positional)


def fused_margin_step(model, heads, tails, relations, margin, n_neg=1, negatives=None,
                      bern_probs=None, seed=0, offset=0, *, shard=None, rel_share=None, positional=None):
    """Loss of one training step, fused: Bernoulli corruption (or the given ``negatives =
    (neg_heads, neg_tails)``), ``model(h, t, r, nh, nt)`` and ``MarginLoss(margin)`` in a
    single kernel, differentiable with respect to the embedding tables.

    Equivalent to the tutorial loop body (docs/tutorials/transe.rst:47-57)
        nh, nt = sampler.corrupt_batch(h, t, r); pos, neg = model(h, t, r, nh, nt)
        loss = criterion(pos, neg)
    without materialising nh, nt, pos, neg.

    shard: ``EntityShard(local_storage=True)`` when the model holds only the entity rows [lo, hi) of
        a table range-partitioned over a process group (sharded_margin_step).  Every rank passes the
        same batch, seed, offset, n_neg and margin -- the batch contents are not checked -- and gets
        the full loss; the negatives are drawn on [1, shard.n_ent).  External negatives are not
        supported in this mode.

    rel_share: relation-corrupting negatives (``BernoulliRelationNegativeSampler``): each negative replaces
        an entity (head with probability bern_probs[r], else tail) with probability rel_share, else the
        relation, uniform on [1, n_rel) -- the draws of ``kge_corrupt_batch_rel``.  None: the entity step.
    negatives: also ``(neg_heads, neg_tails, neg_rels)``; a negative is then scored as
        ``model.scoring_function(nh, nt, nr)`` and any of its positions may differ from the positive's.

    positional: ``(head_offs, head_ents, tail_offs, tail_ents)``, positional negatives
        (``PositionalNegativeSampler``): the head (probability bern_probs[r]) or the tail is replaced by an
        entity drawn uniformly from relation r's sorted candidates on that side, ents[offs[r]:offs[r + 1]], or
        uniformly from [0, n_ent) when there are none -- the draws of ``kge_pos_step_fwd``.  Both CSRs cover the
        model's relations; their entities must be ids of the model's table (the sampler checks this).  Not with
        ``negatives`` or ``rel_share``.  With ``shard`` every rank passes the whole CSR.

    ``fused_loss_step`` takes a criterion instead of a margin (LogisticLoss, BinaryCrossEntropyLoss).
    """
    return _fused_step(model, heads, tails, relations, _lib.LOSS_MARGIN, margin, n_neg, negatives, bern_probs,
                       seed, offset, shard, rel_share, positional)
