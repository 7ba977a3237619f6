"""Host-side driver of the CUDA engine: turns torch tensors into C-ABI calls.

Nothing here computes scores: torch is used for device memory, streams and (when the entity
table is range-partitioned) the collectives of the sharded paths.  The only engine is the CUDA one; tests
may substitute an object with the same methods (``pack``, ``gather_rows``, ``rank_side``,
``score_all``; ``topk_side`` / ``topk_merge`` for top-k inference; ``margin_step_fwd`` /
``margin_step_bwd`` / ``scatter_rows_add`` for the sharded training step; ``finalize`` /
``rescal_rel_scores`` / ``rank_dense`` for relation prediction; ``score_triples`` for triplet
classification; ``transh_project`` / ``transd_project`` for the relation-grouped loops of TransH and
TransD) to exercise the sharding and grouping logic on CPU.
"""
import ctypes
import os

import torch

from . import _lib

#: default number of test triples ranked per kernel launch (bounds workspace memory only;
#: results never depend on it)
DEFAULT_CHUNK = 65536


class ModelSpec:
    """What the kernels read from a model: which score function, and raw fp32 tables.

    Mirrors the state_dict contract of the reference models (SURVEY.md section 5):
    ``ent_emb.weight`` / ``rel_emb.weight`` (TransE models/translation.py:63-64, DistMult
    models/bilinear.py:183-184), ``ent_emb.weight`` / ``rel_mat.weight`` (RESCAL
    models/bilinear.py:55-56), ``re_/im_ent_emb.weight`` + ``re_/im_rel_emb.weight``
    (ComplEx models/bilinear.py:455-458); Analogy (models/bilinear.py:623-631) has three planes per
    table -- ``sc_/re_/im_ent_emb.weight``, ``sc_/re_/im_rel_emb.weight`` -- handed over as views of one
    stacked (3, n, dim) copy (``stacked``): the C ABI takes planes 0 and 1 and finds plane 2 at the
    same spacing (include/kge_b200.h, "three-plane tables").
    """

    def __init__(self, code, dim, n_ent, n_rel, ent0, ent1, rel0, rel1, ent_lo=0, ent2=None, rel2=None):
        self.code = code
        self.dim = int(dim)
        self.n_ent = int(n_ent)      # global number of entities
        self.n_rel = int(n_rel)
        self.ent0, self.ent1, self.rel0, self.rel1 = ent0, ent1, rel0, rel1
        self.ent2, self.rel2 = ent2, rel2
        self.ent_lo = int(ent_lo)    # global id of row 0 of ent0/ent1
        self.n_rows = int(ent0.shape[0])
        if code == _lib.ANALOGY:
            for name, planes in (("entity", (ent0, ent1, ent2)), ("relation", (rel0, rel1, rel2))):
                if planes[0] is None and name == "relation":
                    continue         # relation prediction: the candidates are the relation rows
                if any(x is None for x in planes) or not _equally_spaced(*planes):
                    raise ValueError("Analogy %s planes must be equally spaced views of one stacked "
                                     "tensor (ModelSpec.stacked)" % name)

    @property
    def cand_planes(self):
        return 3 if self.code == _lib.ANALOGY else (2 if self.code in (_lib.COMPLEX, _lib.ROTATE) else 1)

    @staticmethod
    def stacked(planes):
        """[plane tensors (n, d)] -> the views (p0, p1, p2) of one contiguous (3, n, d) copy."""
        s = torch.stack([ModelSpec._f32(x) for x in planes])
        return s[0], s[1], s[2]

    def narrowed(self, lo, hi):
        """Same model restricted to entity rows [lo, hi) (views, no copy)."""
        a, b = lo - self.ent_lo, hi - self.ent_lo
        if a < 0 or b > self.n_rows:
            raise ValueError("shard [%d,%d) outside held rows" % (lo, hi))
        e1 = None if self.ent1 is None else self.ent1[a:b]
        e2 = None if self.ent2 is None else self.ent2[a:b]
        return ModelSpec(self.code, self.dim, self.n_ent, self.n_rel, self.ent0[a:b], e1,
                         self.rel0, self.rel1, ent_lo=lo, ent2=e2, rel2=self.rel2)

    @staticmethod
    def _f32(t):
        t = t.detach()
        if t.dtype != torch.float32:
            raise TypeError("embedding tables must be float32, got %s" % t.dtype)
        return t.contiguous()

    @classmethod
    def from_model(cls, model):
        """Accepts torchkge_b200 models and (duck-typed) the reference's own model classes."""
        name = type(model).__name__
        f = cls._f32
        if name == "TransEModel":
            dname = getattr(model.dissimilarity, "__name__", str(model.dissimilarity))
            if dname == "l1_dissimilarity":
                code = _lib.TRANSE_L1
            elif dname == "l2_dissimilarity":
                code = _lib.TRANSE_L2
            else:
                raise NotImplementedError("TransE dissimilarity %s is not on the CUDA path" % dname)
            return cls(code, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.ent_emb.weight), None, f(model.rel_emb.weight), None)
        if name == "TorusEModel":
            dname = getattr(model.dissimilarity, "__name__", str(model.dissimilarity))
            code = {"l1_torus_dissimilarity": _lib.TORUSE_L1, "l2_torus_dissimilarity": _lib.TORUSE_L2,
                    "l1_dissimilarity": _lib.TRANSE_L1}.get(dname)
            if code is None:
                raise NotImplementedError("TorusE dissimilarity %s is not on the CUDA path" % dname)
            if not getattr(model, "normalized", False):
                model.normalize_parameters()   # as inference_prepare_candidates does (translation.py:745-746)
            return cls(code, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.ent_emb.weight), None, f(model.rel_emb.weight), None)
        if name == "DistMultModel":
            return cls(_lib.DISTMULT, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.ent_emb.weight), None, f(model.rel_emb.weight), None)
        if name == "RESCALModel":
            return cls(_lib.RESCAL, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.ent_emb.weight), None, f(model.rel_mat.weight), None)
        if name == "ComplExModel":
            return cls(_lib.COMPLEX, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.re_ent_emb.weight), f(model.im_ent_emb.weight),
                       f(model.re_rel_emb.weight), f(model.im_rel_emb.weight))
        if name == "RotatEModel":
            re_r, im_r = model.relation_planes()
            return cls(_lib.ROTATE, model.emb_dim, model.n_ent, model.n_rel,
                       f(model.re_ent_emb.weight), f(model.im_ent_emb.weight), f(re_r), f(im_r))
        if name == "AnalogyModel":
            if model.scalar_dim != model.complex_dim:
                # the reference's own inference_scoring_function adds (b, n, scalar_dim) and
                # (b, n, complex_dim) tensors (bilinear.py:695-698): it needs equal widths too
                raise NotImplementedError("Analogy link prediction needs scalar_dim == complex_dim "
                                          "(got %d and %d)" % (model.scalar_dim, model.complex_dim))
            e = cls.stacked([model.sc_ent_emb.weight, model.re_ent_emb.weight, model.im_ent_emb.weight])
            r = cls.stacked([model.sc_rel_emb.weight, model.re_rel_emb.weight, model.im_rel_emb.weight])
            return cls(_lib.ANALOGY, model.scalar_dim, model.n_ent, model.n_rel, e[0], e[1], r[0], r[1],
                       ent2=e[2], rel2=r[2])
        if name in PROJECTED_SPECS:
            # every entry point that supports TransH / TransD builds its spec from PROJECTED_SPECS; the others
            # (the fused training step, sharded calls) end here
            raise NotImplementedError(
                "%s is supported by the unsharded LinkPredictionEvaluator, RelationPredictionEvaluator, "
                "TripletClassificationEvaluator, EntityInference, RelationInference and scoring_function only "
                "(not by the fused training step or shard=)" % name)
        raise NotImplementedError(
            "%s has no CUDA link-prediction path (supported: TransE L1/L2, TransH, TransD, TorusE "
            "torus_L1/torus_L2, DistMult, RESCAL, ComplEx, Analogy, RotatE)" % name)


#: widest embedding the kernels take (csrc/kernels.h: SCAN_MAX_DIM)
MAX_DIM = 8192


class ProjectedSpec(ModelSpec):
    """A TransH or TransD model read as TransE-L2, whose entity rows are ranked only after a per-relation
    projection: ``project(engine, rel, out)`` writes the (n_rows, dim) table of relation ``rel`` into ``out``
    (the relation-grouped loops of rank_link_prediction_projected and topk_entity_inference), and
    ``rel_scores(engine, hrows, trows, h_idx, t_idx)`` gives the dense (n, n_rel) relation scores of the facts
    (_dense_rel_scores).  ``name``: the model's class name, for error messages."""

    def __init__(self, model, dim, ent0, rel0):
        super().__init__(_lib.TRANSE_L2, dim, model.n_ent, model.n_rel, ent0, None, rel0, None)
        self.name = type(model).__name__


class TransHSpec(ProjectedSpec):
    """TransH (translation.py:168-181): ent_emb and rel_emb read as a TransE-L2 model's, plus the raw normal
    vectors (``norm_vect``)."""

    def __init__(self, model):
        f = ModelSpec._f32
        super().__init__(model, model.emb_dim, f(model.ent_emb.weight), f(model.rel_emb.weight))
        self.norm_vect = f(model.norm_vect.weight)

    def project(self, engine, rel, out):
        return engine.transh_project(self, rel, out)

    def rel_scores(self, engine, hrows, trows, h_idx, t_idx):
        return engine.transh_rel_scores(self, hrows, trows)


def check_transd_widths(ent_dim, rel_dim):
    """TransD's widths, checked before any device work: the reference's projection adds a rel_emb_dim vector to
    ent[:rel_emb_dim] (translation.py:568, 646) and fails on a broadcast when rel_emb_dim > ent_emb_dim."""
    if not 1 <= rel_dim <= ent_dim:
        raise ValueError("TransDModel needs 1 <= rel_emb_dim <= ent_emb_dim (got rel_emb_dim = %d, ent_emb_dim = %d)"
                         % (rel_dim, ent_dim))
    if ent_dim > MAX_DIM:
        raise ValueError("TransDModel: ent_emb_dim = %d exceeds %d" % (ent_dim, MAX_DIM))


class TransDSpec(ProjectedSpec):
    """TransD (translation.py:518-536), read at width rel_emb_dim: ent0 holds the first rel_emb_dim coordinates
    of the raw ent_emb rows (the rows relation prediction projects on the fly), rel0 the raw rel_emb table.  It
    also holds the raw ent_emb table (``ent_full``, its width ``ent_dim``), the raw rel_proj_vect table
    (``rel_proj``) and every entity's scalar s_e = (ent_proj_vect[e] * ent_emb[e]).sum() (``scalars``), computed
    once here: it does not depend on the relation."""

    def __init__(self, model):
        check_transd_widths(model.ent_emb_dim, model.rel_emb_dim)
        f = ModelSpec._f32
        ent, rel_dim = f(model.ent_emb.weight), model.rel_emb_dim
        super().__init__(model, rel_dim, ent[:, :rel_dim].contiguous(), f(model.rel_emb.weight))
        self.ent_full, self.ent_dim = ent, model.ent_emb_dim
        self.rel_proj = f(model.rel_proj_vect.weight)
        # a model on the host has none: shard_spec refuses it next
        self.scalars = (default_engine().transd_entity_scalars(ent, f(model.ent_proj_vect.weight))
                        if ent.is_cuda else None)

    def project(self, engine, rel, out):
        return engine.transd_project(self, rel, out)

    def rel_scores(self, engine, hrows, trows, h_idx, t_idx):
        return engine.transd_rel_scores(self, hrows, trows, self.scalars[h_idx], self.scalars[t_idx])


#: the models ranked on per-relation projected entity tables: class name (this package's or, duck-typed, the
#: reference's) -> spec
PROJECTED_SPECS = {"TransHModel": TransHSpec, "TransDModel": TransDSpec}


def refuse_projected_shard(name, shard):
    """A TransH / TransD model (``name``: its class name) takes no shard=: raised on every rank, before any
    device work or collective."""
    if shard is not None and name in PROJECTED_SPECS:
        raise NotImplementedError("%s does not support shard= (EntityShard / QueryShard)" % name)


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _plane_ptrs(x0, x1):
    """(plane 0, plane 1) pointers of a table: a stacked (3, n, dim) tensor stands for three equally
    spaced planes, of which the C ABI takes the first two (include/kge_b200.h, "three-plane tables")."""
    if x0 is not None and x0.dim() == 3:
        return _ptr(x0[0]), _ptr(x0[1])
    return _ptr(x0), _ptr(x1)


def _equally_spaced(p0, p1, p2):
    """planes of a three-plane table as the C ABI expects them: plane 2 at p1 + (p1 - p0)"""
    return (p0.shape == p1.shape == p2.shape and p0.is_contiguous() and p1.is_contiguous() and p2.is_contiguous()
            and p2.data_ptr() - p1.data_ptr() == p1.data_ptr() - p0.data_ptr())


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _lib.KgeLibraryError(
                "the link-prediction engine runs on CUDA tensors only (got a %s tensor); "
                "move the model to a GPU -- there is no CPU fallback" % t.device)


def _device_guard(device):
    """The library launches on the CURRENT device (cudaGetDevice) with the stream it is handed:
    every public entry point runs its calls under the device of the tensors it was given."""
    if getattr(device, "type", None) == "cuda":
        return torch.cuda.device(device)
    import contextlib
    return contextlib.nullcontext()


class CudaEngine:
    """Direct calls into libkge_b200.so on the current CUDA stream."""

    def __init__(self, tensor_core=None):
        self.lib = _lib.load()
        self.launches = 0  # kernels launched through this engine (bench.py reports it)
        if tensor_core is None:
            tensor_core = os.environ.get("KGE_TENSOR_CORE", "1") != "0"
        #: use the tensor-core (wgmma) bound-and-refine scan for models that have one (ranks unchanged)
        self.tensor_core = bool(tensor_core)
        self.tc_stats = []  # (device tensor [found, capacity]) per tensor-core call, for checks
        #: tensor-core operand images kept between evaluations, each with a device-side content
        #: checksum of the table it was built from (kge_tc_pack_table_cached): an unchanged table
        #: costs one read instead of a rebuild, a changed one is always rebuilt.  KGE_TC_CACHE=0 or
        #: ``tc_cache_entries = 0`` disables it; ``clear_cache()`` frees the images.
        self.tc_cache_entries = 0 if os.environ.get("KGE_TC_CACHE", "1") == "0" else 2
        self._tc_cache = {}
        #: KGE_TRACE=1: rank_link_prediction appends (label, host seconds, CUDA event) marks here
        self.trace = [] if os.environ.get("KGE_TRACE") else None

    def mark(self, label):
        """Debug aid (KGE_TRACE=1): a host timestamp and a CUDA event on the current stream."""
        if self.trace is None:
            return
        import time
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self.trace.append((label, time.perf_counter(), ev))

    def trace_report(self):
        """[(label, host ms since first mark, device ms since first mark)] of the recorded marks."""
        if not self.trace:
            return []
        torch.cuda.synchronize()
        l0, t0, e0 = self.trace[0]
        out = [(lab, 1e3 * (t - t0), e0.elapsed_time(ev)) for lab, t, ev in self.trace]
        self.trace = []
        return out

    # ---- table packing: once per evaluate() ----
    def pack(self, spec):
        _need_cuda(spec.ent0, spec.ent1)
        n_floats = self.lib.kge_packed_table_floats(spec.code, spec.n_rows, spec.dim)
        packed = torch.empty(max(n_floats, 1), dtype=torch.float32, device=spec.ent0.device)
        if spec.n_rows > 0:
            _lib.check(self.lib.kge_pack_table(spec.code, _ptr(spec.ent0), _ptr(spec.ent1),
                                               spec.n_rows, spec.dim, _ptr(packed),
                                               _stream(packed.device)), "kge_pack_table")
            self.launches += 1
        return packed

    def clear_cache(self):
        self._tc_cache.clear()

    def pack_tc(self, spec, cache=True):
        """Tensor-core operand image of the shard, or None when the model has no such path.
        ``cache=False``: build it without the checksummed cache (a table rewritten in place for every call,
        such as TransH's per-relation projection buffer)."""
        if not self.tensor_core:
            return None
        nbytes = self.lib.kge_tc_packed_bytes(spec.code, spec.n_rows, spec.dim)
        if nbytes == 0:
            return None
        dev = spec.ent0.device
        # a three-plane spec reads a stacked COPY of the weights made for this call (ModelSpec.stacked):
        # its address changes every time, so there is nothing to cache an image under
        if not cache or self.tc_cache_entries <= 0 or getattr(spec, "ent2", None) is not None:
            out = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(self.lib.kge_tc_pack_table(spec.code, _ptr(spec.ent0), _ptr(spec.ent1), spec.n_rows,
                                                  spec.dim, _ptr(out), _stream(dev)), "kge_tc_pack_table")
            self.launches += 4
            return out
        key = (spec.code, spec.ent0.data_ptr(), None if spec.ent1 is None else spec.ent1.data_ptr(),
               spec.n_rows, spec.dim, self.lib.kge_tc_layout_id(), str(dev))
        hit = self._tc_cache.pop(key, None)
        if hit is None:
            while len(self._tc_cache) >= self.tc_cache_entries:
                self._tc_cache.pop(next(iter(self._tc_cache)))
            # the table tensors are kept too: their storage cannot be freed and re-used at the same
            # address by another table while the entry lives
            hit = (torch.empty(nbytes, dtype=torch.uint8, device=dev),
                   torch.zeros(4, dtype=torch.int64, device=dev), spec.ent0, spec.ent1)
        self._tc_cache[key] = hit        # most recently used last
        out, guard = hit[0], hit[1]
        _lib.check(self.lib.kge_tc_pack_table_cached(spec.code, _ptr(spec.ent0), _ptr(spec.ent1), spec.n_rows,
                                                     spec.dim, _ptr(out), _ptr(guard), _stream(dev)),
                   "kge_tc_pack_table_cached")
        self.launches += 8 if spec.ent1 is None else 9
        return out

    def gather_rows(self, spec, idx):
        _need_cuda(spec.ent0, idx)
        n = idx.shape[0]
        out = torch.empty((n, spec.cand_planes, spec.dim), dtype=torch.float32,
                          device=spec.ent0.device)
        _lib.check(self.lib.kge_gather_rows(spec.code, _ptr(spec.ent0), _ptr(spec.ent1),
                                            spec.ent_lo, spec.n_rows, spec.dim, _ptr(idx), n,
                                            _ptr(out), _stream(out.device)), "kge_gather_rows")
        self.launches += 1
        return out

    def rank_side(self, spec, packed, side, hrows, trows, r_idx, true_idx, filt, raw_count,
                  filt_sub, true_score=None, tc_packed=None, tc_dump=None, true_rows=None,
                  true_score_in=None, approx=False, stats=None):
        """Adds this shard's counts for one side into raw_count / filt_sub (int32, device).
        ``stats``: optional int64[2] device tensor receiving (near-ties found, capacity) of a
        bound-and-refine call (one is allocated when absent)."""
        n = r_idx.shape[0] if r_idx is not None else hrows.shape[0]
        dev = raw_count.device
        flags = _lib.FLAG_TENSOR_CORE if tc_packed is not None else 0
        if tc_packed is None and approx and spec.code == _lib.ROTATE:
            flags = _lib.FLAG_APPROX_SCAN
        ws_bytes = self.lib.kge_rank_workspace_bytes(spec.code, side, spec.dim, n, spec.n_rows, flags)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        a = _lib.RankArgs()
        a.model, a.side, a.dim, a.flags = spec.code, side, spec.dim, flags
        if flags:
            if stats is None:
                stats = torch.zeros(2, dtype=torch.int64, device=dev)
            a.tc_packed, a.tc_stats, a.tc_dump = _ptr(tc_packed), _ptr(stats), _ptr(tc_dump)
            self.tc_stats.append(stats)
            del self.tc_stats[:-256]
        else:
            stats = None
        a.n, a.n_ent, a.ent_lo, a.n_rows = n, spec.n_ent, spec.ent_lo, spec.n_rows
        a.packed, a.ent0, a.ent1 = _ptr(packed), _ptr(spec.ent0), _ptr(spec.ent1)
        a.rel0, a.rel1 = _ptr(spec.rel0), _ptr(spec.rel1)
        a.hrows, a.trows, a.r_idx, a.true_idx = _ptr(hrows), _ptr(trows), _ptr(r_idx), _ptr(true_idx)
        if filt is not None:
            offs, ids = filt[0], filt[1]
            a.filt_offs, a.filt_ids, a.n_filt = _ptr(offs), _ptr(ids), ids.shape[0]
            a.filt_qid = _ptr(filt[2]) if len(filt) > 2 else None
        a.raw_count, a.filt_sub, a.true_score = _ptr(raw_count), _ptr(filt_sub), _ptr(true_score)
        a.true_rows, a.true_score_in = _ptr(true_rows), _ptr(true_score_in)
        a.workspace, a.workspace_bytes, a.stream = _ptr(ws), ws_bytes, _stream(dev)
        _lib.check(self.lib.kge_rank_side(ctypes.byref(a)), "kge_rank_side")
        # prep, pack_queries, pad fill, true scores, scan (+ filter)
        self.launches += 5 + (1 if filt is not None and filt[1].shape[0] > 0 else 0)
        # handle for filter_side; keeps buffers alive
        return (a, ws, packed, hrows, trows, tc_packed, stats, true_rows, true_score_in)

    def filter_side(self, handle, filt, filt_sub):
        """Sparse filter pass for a side whose dense scan was enqueued earlier by rank_side
        (with filt=None); ``handle`` is what that call returned."""
        a = handle[0]
        offs, ids = filt[0], filt[1]
        if ids.shape[0] == 0:
            return
        a.filt_offs, a.filt_ids, a.n_filt = _ptr(offs), _ptr(ids), ids.shape[0]
        # optional third array: the CSR row of every entry (int32), spares the kernel a bisection per entry
        a.filt_qid = _ptr(filt[2]) if len(filt) > 2 and filt[2] is not None else None
        self._keep = filt
        a.filt_sub = _ptr(filt_sub)
        a.stream = _stream(filt_sub.device)
        _lib.check(self.lib.kge_filter_side(ctypes.byref(a)), "kge_filter_side")
        self.launches += 1

    def score_all(self, spec, packed, side, hrows, trows, r_idx):
        n = hrows.shape[0]
        dev = hrows.device
        scores = torch.empty((n, spec.n_rows), dtype=torch.float32, device=dev)
        ws_bytes = self.lib.kge_rank_workspace_bytes(spec.code, side, spec.dim, n, 0, 0)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        a = _lib.ScoreAllArgs()
        a.model, a.side, a.dim = spec.code, side, spec.dim
        a.n, a.n_rows = n, spec.n_rows
        a.packed, a.rel0, a.rel1 = _ptr(packed), _ptr(spec.rel0), _ptr(spec.rel1)
        a.hrows, a.trows, a.r_idx = _ptr(hrows), _ptr(trows), _ptr(r_idx)
        a.scores, a.workspace, a.workspace_bytes = _ptr(scores), _ptr(ws), ws_bytes
        a.stream = _stream(dev)
        _lib.check(self.lib.kge_score_all(ctypes.byref(a)), "kge_score_all")
        self.launches += 4
        return scores

    def topk_side(self, spec, packed, side, hrows, trows, r_idx, k, mask=None):
        """(pred int64 (n, k), scores float32 (n, k)) of the k best candidates per query, exact
        scores, best first; ``mask`` = device CSR (offs, ids ascending per row) of candidates to set to
        -inf.  No (n, n_rows) matrix is allocated (include/kge_b200.h: kge_topk_side)."""
        n = hrows.shape[0]
        dev = hrows.device
        pred = torch.empty((n, k), dtype=torch.int64, device=dev)
        scores = torch.empty((n, k), dtype=torch.float32, device=dev)
        ws_bytes = self.lib.kge_topk_workspace_bytes(spec.code, side, spec.dim, n, spec.n_rows, k)
        if ws_bytes == 0:
            raise _lib.KgeLibraryError("kge_topk_workspace_bytes: unsupported arguments (k must be in [1, 1024])")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        a = _lib.TopkArgs()
        a.model, a.side, a.dim, a.k = spec.code, side, spec.dim, k
        a.n, a.n_rows = n, spec.n_rows
        a.packed, a.rel0, a.rel1 = _ptr(packed), _ptr(spec.rel0), _ptr(spec.rel1)
        a.hrows, a.trows, a.r_idx = _ptr(hrows), _ptr(trows), _ptr(r_idx)
        if mask is not None and mask[1].numel() > 0:
            a.mask_offs, a.mask_ids = _ptr(mask[0]), _ptr(mask[1])
        a.pred, a.scores = _ptr(pred), _ptr(scores)
        a.workspace, a.workspace_bytes, a.stream = _ptr(ws), ws_bytes, _stream(dev)
        a.ent_lo = spec.ent_lo   # pred holds global ids; mask ids are global too
        _lib.check(self.lib.kge_topk_side(ctypes.byref(a)), "kge_topk_side")
        self.launches += 7   # prep, pack, fill, finish + at least one collect scan / merge pair
        return pred, scores

    def topk_merge(self, pred_in, scores_in, k):
        """(pred int64 (n, k), scores float32 (n, k)): the k best entries of the union of the lists
        pred_in int64 / scores_in float32 (n_lists, n, k_in), each sorted best first as topk_side
        returns them, pred = -1 marking an empty slot; same order as topk_side (kge_topk_merge)."""
        _need_cuda(pred_in, scores_in)
        pred_in, scores_in = pred_in.contiguous(), scores_in.contiguous()
        n_lists, n, k_in = pred_in.shape
        dev = pred_in.device
        pred = torch.empty((n, k), dtype=torch.int64, device=dev)
        scores = torch.empty((n, k), dtype=torch.float32, device=dev)
        _lib.check(self.lib.kge_topk_merge(_ptr(pred_in), _ptr(scores_in), n_lists, n, k_in, k, _ptr(pred),
                                           _ptr(scores), _stream(dev)), "kge_topk_merge")
        self.launches += 1
        return pred, scores

    def rescal_rel_scores(self, spec, hrows, trows):
        """(n, n_rel) scores ((h^T M_c) * t).sum() of every relation matrix c: RESCAL's relation case
        (bilinear.py:115-121), dense (the candidates are per-fact vectors, nothing to scan)."""
        n, dev = hrows.shape[0], hrows.device
        scores = torch.empty((n, spec.n_rel), dtype=torch.float32, device=dev)
        _lib.check(self.lib.kge_rescal_rel_scores(_ptr(hrows), _ptr(trows), _ptr(spec.rel0), spec.dim, n,
                                                  spec.n_rel, _ptr(scores), _stream(dev)), "kge_rescal_rel_scores")
        self.launches += 1
        return scores

    def transh_project(self, spec, rel, out):
        """out (n_rows, dim) <- the entity rows of ``spec`` (TransHSpec) projected on the hyperplane of
        relation ``rel`` (kge_transh_project, translation.py:279-281)."""
        _need_cuda(spec.ent0, out)
        _lib.check(self.lib.kge_transh_project(_ptr(spec.ent0), _ptr(spec.norm_vect[rel]), spec.n_rows, spec.dim,
                                               _ptr(out), _stream(out.device)), "kge_transh_project")
        self.launches += 1
        return out

    def transh_rel_scores(self, spec, hrows, trows):
        """(n, n_rel) scores -||(P_c(h) + r_c) - P_c(t)||^2 of every relation c: TransH's relation case
        (interfaces.py:261-272), dense like RESCAL's."""
        n, dev = hrows.shape[0], hrows.device
        scores = torch.empty((n, spec.n_rel), dtype=torch.float32, device=dev)
        _lib.check(self.lib.kge_transh_rel_scores(_ptr(hrows), _ptr(trows), _ptr(spec.rel0), _ptr(spec.norm_vect),
                                                  spec.dim, n, spec.n_rel, _ptr(scores), _stream(dev)),
                   "kge_transh_rel_scores")
        self.launches += 1
        return scores

    def transd_entity_scalars(self, ent, ent_proj):
        """(n_rows,) s_e = (ent_proj[e] * ent[e]).sum() of TransD's raw ent_emb / ent_proj_vect tables, in ATen's
        order (kge_transd_entity_scalars, translation.py:645)."""
        _need_cuda(ent, ent_proj)
        n, dim = ent.shape
        s = torch.empty(n, dtype=torch.float32, device=ent.device)
        _lib.check(self.lib.kge_transd_entity_scalars(_ptr(ent), _ptr(ent_proj), n, dim, _ptr(s),
                                                      _stream(ent.device)), "kge_transd_entity_scalars")
        self.launches += 1
        return s

    def transd_project(self, spec, rel, out):
        """out (n_rows, rel_dim) <- the entity rows of ``spec`` (TransDSpec) projected for relation ``rel``
        (kge_transd_project, translation.py:646)."""
        _need_cuda(spec.ent_full, out)
        _lib.check(self.lib.kge_transd_project(_ptr(spec.ent_full), spec.ent_dim, _ptr(spec.scalars),
                                               _ptr(spec.rel_proj[rel]), spec.n_rows, spec.dim, _ptr(out),
                                               _stream(out.device)), "kge_transd_project")
        self.launches += 1
        return out

    def transd_rel_scores(self, spec, hrows, trows, hs, ts):
        """(n, n_rel) scores -||(P_c(h) + r_c) - P_c(t)||^2 of every relation c: TransD's relation case
        (interfaces.py:261-272), dense like TransH's; hrows / trows (n, rel_dim), hs / ts (n,) their scalars."""
        n, dev = hrows.shape[0], hrows.device
        scores = torch.empty((n, spec.n_rel), dtype=torch.float32, device=dev)
        _lib.check(self.lib.kge_transd_rel_scores(_ptr(hrows), _ptr(hs), _ptr(trows), _ptr(ts), _ptr(spec.rel0),
                                                  _ptr(spec.rel_proj), spec.dim, n, spec.n_rel, _ptr(scores),
                                                  _stream(dev)), "kge_transd_rel_scores")
        self.launches += 1
        return scores

    def rank_dense(self, scores, true_idx, filt, raw_count, filt_sub, true_score=None, true_score_in=None):
        """get_rank + filter_scores on a dense (n, n_cand) matrix, counters added into."""
        n, n_c = scores.shape
        if filt is not None and filt[1].numel() == 0:
            filt = None      # nothing to discount (an empty tensor has no device pointer)
        offs, ids = filt if filt is not None else (None, None)
        _lib.check(self.lib.kge_rank_dense(_ptr(scores), n, n_c, _ptr(true_idx), _ptr(true_score_in), _ptr(offs),
                                           _ptr(ids), _ptr(raw_count), _ptr(filt_sub), _ptr(true_score),
                                           _stream(scores.device)), "kge_rank_dense")
        self.launches += 1

    def topk_dense(self, scores, k, mask=None):
        """(pred, scores) of the k best columns per row of a dense matrix (kge_topk_dense)."""
        n, n_c = scores.shape
        dev = scores.device
        pred = torch.empty((n, k), dtype=torch.int64, device=dev)
        vals = torch.empty((n, k), dtype=torch.float32, device=dev)
        ws_bytes = self.lib.kge_topk_dense_workspace_bytes(n, n_c, k)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        if mask is not None and mask[1].numel() == 0:
            mask = None
        offs, ids = mask if mask is not None else (None, None)
        _lib.check(self.lib.kge_topk_dense(_ptr(scores), n, n_c, k, _ptr(offs), _ptr(ids), _ptr(pred), _ptr(vals),
                                           _ptr(ws), ws_bytes, _stream(dev)), "kge_topk_dense")
        self.launches += 3
        return pred, vals

    def score_triples(self, code, dim, ent, rel0, rel1, h, t, r):
        """(n,) scores of the triples (h[i], r[i], t[i]) by the per-triple kernel of
        ``model.scoring_function`` (kge_score_triples_fwd), without autograd.  ``ent``: a plane-major
        (planes, rows, dim) entity table (three-plane models find plane 2 at the same spacing);
        rel0 / rel1 as in ModelSpec."""
        _need_cuda(ent, h, t, r)
        n = h.shape[0]
        out = torch.empty(n, dtype=torch.float32, device=ent.device)
        if n == 0:
            return out
        tb = _lib.Tables()
        tb.model, tb.dim = code, dim
        tb.ent0, tb.ent1 = _ptr(ent[0]), (_ptr(ent[1]) if ent.shape[0] > 1 else None)
        tb.rel0, tb.rel1 = _ptr(rel0), _ptr(rel1)
        _lib.check(self.lib.kge_score_triples_fwd(ctypes.byref(tb), _ptr(h), _ptr(t), _ptr(r), n, _ptr(out),
                                                  _stream(out.device)), "kge_score_triples_fwd")
        self.launches += 1
        return out

    def finalize(self, raw_count, filt_sub):
        n = raw_count.shape[0]
        ranks = torch.empty(n, dtype=torch.int64, device=raw_count.device)
        filt = torch.empty(n, dtype=torch.int64, device=raw_count.device)
        _lib.check(self.lib.kge_finalize_ranks(_ptr(raw_count), _ptr(filt_sub), n, _ptr(ranks),
                                               _ptr(filt), _stream(raw_count.device)),
                   "kge_finalize_ranks")
        self.launches += 1
        return ranks, filt

    # ---- entity-sharded fused training step (torchkge_b200.training.sharded_margin_step) ----
    @staticmethod
    def _shard_step_args(step, tables, h, t, r, probs, loss, hrows, trows):
        _need_cuda(tables[0], h, hrows, trows)
        a = _lib.MarginStepArgs()
        a.tb = _lib.Tables()
        a.tb.model, a.tb.dim = step.code, step.dim
        a.tb.ent0, a.tb.ent1 = _plane_ptrs(tables[0], tables[1])
        a.tb.rel0, a.tb.rel1 = _plane_ptrs(tables[2], tables[3])
        a.n_neg, a.margin, a.b, a.n_ent = step.n_neg, step.margin, h.shape[0], step.n_ent
        a.h, a.t, a.r, a.bern_probs = _ptr(h), _ptr(t), _ptr(r), _ptr(probs)
        a.seed, a.offset = step.seed, step.offset
        a.loss, a.stream = _ptr(loss), _stream(h.device)
        a.ent_lo, a.n_rows = step.ent_lo, step.n_rows
        a.hrows, a.trows = _ptr(hrows), _ptr(trows)
        a.loss_kind = step.loss_kind
        pos = getattr(step, "pos", None)
        if pos is not None:                # positional step: kge_pos_step_* around the same arguments
            pa = _lib.PosStepArgs()
            pa.base, pa.n_rel = a, pos[0].shape[0] - 1
            pa.head_offs, pa.head_ents, pa.tail_offs, pa.tail_ents = (_ptr(x) for x in pos)
            return pa
        if getattr(step, "n_rel", 0) == 0:
            return a
        ra = _lib.RelStepArgs()           # relation-corrupting step: kge_rel_step_* around the same arguments
        ra.base, ra.n_rel, ra.rel_share = a, step.n_rel, step.rel_share
        return ra

    def _step_call(self, a, which, *rest):
        name = {_lib.RelStepArgs: "kge_rel_step_", _lib.PosStepArgs: "kge_pos_step_"}.get(
            type(a), "kge_margin_step_") + which
        _lib.check(getattr(self.lib, name)(ctypes.byref(a), *rest), name)

    def margin_step_fwd(self, step, tables, h, t, r, probs, hrows, trows):
        """Sum of the loss terms (step.loss_kind: the hinge, logistic or BCE term of each pair) of the
        negatives this shard scores (float32 scalar tensor): the negatives whose replaced entity lies in
        [step.ent_lo, step.ent_lo + step.n_rows).  ``tables``:
        (ent0, ent1, rel0, rel1) with this shard's entity rows (a three-plane table as one stacked
        (3, n, dim) tensor in ent0 / rel0); hrows / trows: (b, planes, dim) rows of every positive.
        step.n_rel > 0: the relation-corrupting step (kge_rel_step_fwd), whose relation negatives this shard
        scores when it holds the positive's head.  step.pos = (head_offs, head_ents, tail_offs, tail_ents): the
        positional step (kge_pos_step_fwd), drawn from those candidate slices."""
        loss = torch.zeros((), dtype=torch.float32, device=h.device)
        a = self._shard_step_args(step, tables, h, t, r, probs, loss, hrows, trows)
        self._step_call(a, "fwd")
        self.launches += 1
        return loss

    def margin_step_bwd(self, step, tables, grads, h, t, r, probs, gloss, hrows, trows, grad_hrows, grad_trows):
        """Backward of margin_step_fwd, added into ``grads`` (gradient tensors shaped like ``tables``)
        and grad_hrows / grad_trows (b, planes, dim)."""
        dummy = torch.zeros((), dtype=torch.float32, device=h.device)   # the loss is not recomputed
        a = self._shard_step_args(step, tables, h, t, r, probs, dummy, hrows, trows)
        base = a if isinstance(a, _lib.MarginStepArgs) else a.base
        base.grad_hrows, base.grad_trows = _ptr(grad_hrows), _ptr(grad_trows)
        g = _lib.Grads()
        g.ent0, g.ent1 = _plane_ptrs(grads[0], grads[1])
        g.rel0, g.rel1 = _plane_ptrs(grads[2], grads[3])
        self._step_call(a, "bwd", ctypes.byref(g), _ptr(gloss))
        self.launches += 1

    def scatter_rows_add(self, code, dim, grad0, grad1, ent_lo, idx, rows):
        """grad[idx[i] - ent_lo] += rows[i] plane by plane for the ids this shard holds, others ignored
        (kge_scatter_rows_add); grad0 / grad1 as in _plane_ptrs, rows (n, planes, dim)."""
        _need_cuda(grad0, idx, rows)
        g0, g1 = _plane_ptrs(grad0, grad1)
        rows = rows.contiguous()
        _lib.check(self.lib.kge_scatter_rows_add(code, g0, g1, ent_lo, grad0.shape[-2], dim, _ptr(idx),
                                                 idx.shape[0], _ptr(rows), _stream(rows.device)),
                   "kge_scatter_rows_add")
        self.launches += 1


_default_engine = None


def default_engine():
    global _default_engine
    if _default_engine is None:
        _default_engine = CudaEngine()
    return _default_engine


class _RangeSplit:
    """n items split over the ranks of a process group: rank g gets [g*per, (g+1)*per), clipped to n,
    with per = ceil(n / world).  Every collective of a sharded call goes through ``all_reduce_sum`` /
    ``stack_all`` of the shard object the caller passed (tests substitute them)."""

    def __init__(self, n, rank, world, group):
        self.rank, self.world, self.group = rank, world, group
        self.per = (n + world - 1) // world
        self.lo = min(n, rank * self.per)
        self.hi = min(n, (rank + 1) * self.per)

    @classmethod
    def from_group(cls, n, group=None, *args, **kwargs):
        import torch.distributed as dist
        return cls(n, dist.get_rank(group), dist.get_world_size(group), group, *args, **kwargs)

    def all_reduce_sum(self, t):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    def stack_all(self, t):
        """(world, *t.shape): every rank's ``t`` (same shape on all ranks), in rank order."""
        if self.world == 1:
            return t.unsqueeze(0)
        import torch.distributed as dist
        everyone = torch.empty((self.world,) + tuple(t.shape), dtype=t.dtype, device=t.device)
        dist.all_gather(list(everyone.unbind(0)), t.contiguous(), group=self.group)
        return everyone

    def split(self, m):
        """The QueryShard of m items over the same ranks; its collectives go through this shard's."""
        part = QueryShard(m, self.rank, self.world, self.group)
        part.all_reduce_sum, part.stack_all = self.all_reduce_sum, self.stack_all
        return part


class EntityShard(_RangeSplit):
    """Range partition of the entity table over the ranks of a process group
    (SURVEY.md section 8e): rank g holds rows [g*ceil(nE/G), (g+1)*ceil(nE/G))."""

    def __init__(self, n_ent, rank=0, world=1, group=None, local_storage=False):
        super().__init__(n_ent, rank, world, group)
        self.n_ent = n_ent
        #: True when the model on this rank HOLDS only rows [lo, hi) (its row 0 is entity lo);
        #: False when every rank holds the full table and merely scans its own range (_check_table)
        self.local_storage = local_storage


class QueryShard(_RangeSplit):
    """Contiguous split of n test triples over the ranks of a process group, for tables that fit
    one GPU (SURVEY.md section 8e, second form): the entity table is replicated, every rank ranks
    ITS triples against all entities -- independent units, no collective on the data path -- and
    the rank vectors are all-gathered at the end."""

    def __init__(self, n, rank=0, world=1, group=None):
        self.n = int(n)
        super().__init__(self.n, rank, world, group)

    def slice(self, *tensors):
        """This rank's rows of each (n,) tensor."""
        return tuple(x[self.lo:self.hi].contiguous() for x in tensors)

    def csr(self, filt):
        """This rank's rows of a CSR over the n triples (offsets rebased)."""
        return _csr_cut(filt, [(self.lo, self.hi)])[0]

    def all_gather(self, parts):
        """Per-rank results (one row per local triple: vectors, or tensors with the same trailing
        dimensions, all of one dtype) -> full-length results on every rank, with ONE collective for
        all of them."""
        if self.world == 1:
            return list(parts)
        k = len(parts)
        trail = tuple(parts[0].shape[1:])
        mine = torch.zeros((k, self.per) + trail, dtype=parts[0].dtype, device=parts[0].device)
        for i, x in enumerate(parts):
            mine[i, :x.shape[0]] = x
        everyone = self.stack_all(mine)
        # rank-major slices of length `per` concatenate to the original order of the triples
        full = everyone.transpose(0, 1).reshape((k, self.world * self.per) + trail)[:, :self.n]
        return [full[i] for i in range(k)]


def _csr_cut(csr, ranges):
    """Rows [lo, hi) of a CSR (offs (n+1,), ids[, row ids]) for every (lo, hi) of ``ranges``, offsets
    rebased to 0 and row ids (when present) to lo; host or device tensors.  One device -> host read
    for all ranges, none when the only range is the whole CSR."""
    if csr is None:
        return [None] * len(ranges)
    offs, ids = csr[0], csr[1]
    if not ranges or ranges == [(0, offs.shape[0] - 1)]:
        return [csr] * len(ranges)
    qid = csr[2] if len(csr) > 2 else None
    at = offs[torch.tensor([x for r in ranges for x in r], device=offs.device)].tolist()
    out = []
    for (lo, hi), a, b in zip(ranges, at[0::2], at[1::2]):
        part = ((offs[lo:hi + 1] - a).contiguous(), ids[a:b].contiguous())
        out.append(part if qid is None else part + ((qid[a:b] - lo).contiguous(),))
    return out


def _check_table(spec, shard):
    """The table rule of an EntityShard (DESIGN.md section 6), checked on every rank before the first
    collective: under local storage the model holds exactly rows [lo, hi) (ent_lo == lo), under full
    storage the whole table (ent_lo == 0, n_rows == n_ent).  ``spec``: anything with n_ent, ent_lo
    and n_rows."""
    lo, rows = (shard.lo, shard.hi - shard.lo) if shard.local_storage else (0, shard.n_ent)
    if (spec.n_ent, spec.ent_lo, spec.n_rows) != (shard.n_ent, lo, rows):
        raise ValueError("EntityShard(local_storage=%s): rank %d should hold %d entity rows (entities [%d, %d)), "
                         "the model holds %d entity rows from entity %d (the shard partitions %d entities, the "
                         "model has %d)" % (shard.local_storage, shard.rank, rows, lo, lo + rows, spec.n_rows,
                                            spec.ent_lo, shard.n_ent, spec.n_ent))


def _scanned(spec, shard):
    """The rows [lo, hi) this rank scans (after _check_table): the model's own rows under local storage,
    views into the whole table under full storage."""
    if (spec.ent_lo, spec.n_rows) == (shard.lo, shard.hi - shard.lo):
        return spec
    return spec.narrowed(shard.lo, shard.hi)


def _check_queries(shard, n):
    """A QueryShard splits exactly the n facts or queries of the call."""
    if shard.n != n:
        raise ValueError("QueryShard covers %d facts or queries, got %d" % (shard.n, n))


def shard_spec(model, shard=None, who="evaluate", n=None, build=ModelSpec.from_model):
    """The ModelSpec the engine reads for ``model`` (``build(model)``) under ``shard``, after the shard's
    argument checks: under an EntityShard with local storage the model holds entity rows [lo, hi) and its
    row 0 is entity lo (_check_table); a QueryShard must cover ``n`` facts, when ``n`` is given.  The
    checks come first, then the model must be on a CUDA device.  TransH / TransD: no shard, and the spec of
    PROJECTED_SPECS."""
    name = type(model).__name__
    refuse_projected_shard(name, shard)
    spec = PROJECTED_SPECS.get(name, build)(model)
    if isinstance(shard, EntityShard):
        if shard.local_storage:
            spec = ModelSpec(spec.code, spec.dim, shard.n_ent, spec.n_rel, spec.ent0, spec.ent1, spec.rel0,
                             spec.rel1, ent_lo=shard.lo, ent2=spec.ent2, rel2=spec.rel2)
        _check_table(spec, shard)
    elif isinstance(shard, QueryShard) and n is not None:
        _check_queries(shard, n)
    if not spec.ent0.is_cuda:
        raise _lib.KgeLibraryError("%s needs the model on a CUDA device (model.cuda()); this package has no "
                                   "CPU execution path" % who)
    return spec


def _by_query_slices(shard, run, idx, csr=None):
    """``run(*this rank's slice of every tensor of idx, its rows of csr)`` -> (n_local, ...) results, then
    ONE all-gather: the full results on every rank."""
    return shard.all_gather(list(run(*shard.slice(*idx), shard.csr(csr))))


class LazyRanks:
    """Result of ``rank_link_prediction(..., sync=False)``: the four rank vectors are enqueued on
    the device but nothing has been synchronised yet.  ``overflow`` is a device scalar > 0 iff
    some bound-and-refine call ran out of room in its near-tie list (adversarial tables only);
    ``get()`` looks at it (one host sync) and, in that case, recomputes everything on the exact
    scalar scan.  Callers that copy the ranks to the host anyway pass the flag along in that copy
    (``get(flag_host=...)``)."""

    def __init__(self, ranks, overflow, redo):
        self.ranks, self.overflow, self._redo = ranks, overflow, redo

    def get(self, flag_host=None):
        if self.overflow is not None:
            flag = int(self.overflow.item()) if flag_host is None else int(flag_host)
            if flag > 0:
                import warnings
                warnings.warn("torchkge_b200: the near-tie list of %d bound-and-refine call(s) overflowed "
                              "(adversarial or degenerate embeddings?); recomputing the ranks on the exact "
                              "scalar scan" % flag, RuntimeWarning)
                self.ranks, self.overflow = self._redo(), None
        return self.ranks


def rank_link_prediction(spec, h_idx, t_idx, r_idx, filt_tail, filt_head, shard=None,
                         engine=None, chunk=DEFAULT_CHUNK, packed=None, exact=False, sync=True, tc_cache=True):
    """Rank every triple's true tail and head against all entities, raw and filtered.

    spec       ModelSpec holding either the full entity table or exactly this rank's shard
    h/t/r_idx  int64 device tensors (n,)
    filt_*     (offs int64 (n+1,), ids int64 (m,)) device CSR of entities to discount, None,
               or a zero-argument callable returning such a CSR -- callables are invoked only
               after every dense scan has been enqueued, so that building the CSR on the host
               overlaps with the scans on the device
    shard      EntityShard when the table is range-partitioned over a process group
    exact      True: scalar ATen-order scan only (no tensor-core / approximate bound-and-refine)
    sync       False: return a LazyRanks (no host synchronisation at all inside this call)
    tc_cache   False: build the tensor-core image without the engine's cache (CudaEngine.pack_tc)
    Returns (rank_heads, rank_tails, filt_rank_heads, filt_rank_tails), int64 device tensors.
    """
    engine = engine or default_engine()
    n = h_idx.shape[0]
    if isinstance(spec, ProjectedSpec):
        raise ValueError("a %s spec is ranked by rank_link_prediction_projected" % spec.name[:-len("Model")])
    table = spec
    if shard is not None:
        _check_table(spec, shard)
        spec = _scanned(spec, shard)
        if spec is not table:
            packed = None
    mark = getattr(engine, "mark", lambda label: None)
    mark("step begin")
    dev = spec.ent0.device
    with _device_guard(dev):
        tc_packed = None
        if hasattr(engine, "pack_tc") and not exact:
            tc_packed = engine.pack_tc(spec) if tc_cache else engine.pack_tc(spec, cache=False)
        mark("pack_tc")
        if packed is None and tc_packed is None:
            packed = engine.pack(spec)   # scalar-scan layout: only when there is no tensor-core path
        mark("pack")
        # RotatE has no tensor-core form; its bound-and-refine runs on the fp32 pipes (KGE_FLAG_APPROX_SCAN)
        refine = (not exact and tc_packed is None and spec.code == _lib.ROTATE
                  and getattr(engine, "tensor_core", False))
        if tc_packed is not None or refine:
            # the near-tie list of one call holds n * n_rows / 128 pairs at most 2^28 (2 GB): keep the
            # facts per call small enough for tables of many millions of rows, so that running out of
            # room stays the exception it is meant to be
            chunk = min(chunk, max(1024, ((1 << 35) // max(spec.n_rows, 1)) // 128 * 128))
        # counters raw_t, sub_t, raw_h, sub_h and, behind them, one slot for the overflow flag so
        # that a sharded run needs a single all-reduce
        buf = torch.zeros(4 * n + 1, dtype=torch.int32, device=dev)
        counters = buf[:4 * n].view(4, n)
        n_calls = 2 * ((n + chunk - 1) // chunk)
        stats_all = (torch.zeros((max(n_calls, 1), 2), dtype=torch.int64, device=dev)
                     if (tc_packed is not None or refine) else None)
        pending = []
        call = 0
        chunks = [(lo, min(n, lo + chunk)) for lo in range(0, n, chunk)]
        for c, (lo, hi) in enumerate(chunks):
            h, t, r = h_idx[lo:hi], t_idx[lo:hi], r_idx[lo:hi]
            hrows = engine.gather_rows(spec, h)
            trows = engine.gather_rows(spec, t)
            if shard is not None and shard.world > 1:
                # every row is owned by exactly one rank; the others contribute zeros
                shard.all_reduce_sum(hrows)
                shard.all_reduce_sum(trows)
            for side, true_idx, which, raw, sub in ((_lib.SIDE_TAIL, t, 0, counters[0], counters[1]),
                                                    (_lib.SIDE_HEAD, h, 1, counters[2], counters[3])):
                if tc_packed is not None:
                    handle = engine.rank_side(spec, packed, side, hrows, trows, r, true_idx, None,
                                              raw[lo:hi], sub[lo:hi], tc_packed=tc_packed,
                                              stats=stats_all[call])
                elif refine:
                    handle = engine.rank_side(spec, packed, side, hrows, trows, r, true_idx, None,
                                              raw[lo:hi], sub[lo:hi], approx=True, stats=stats_all[call])
                else:
                    handle = engine.rank_side(spec, packed, side, hrows, trows, r, true_idx, None,
                                              raw[lo:hi], sub[lo:hi])
                call += 1
                pending.append((handle, which, c, lo, hi, sub))
                mark("rank_side %d enqueued" % side)
        filts = [f() if callable(f) else f for f in (filt_tail, filt_head)]
        parts = [_csr_cut(f, chunks) for f in filts]   # one device -> host read per CSR, none for one chunk
        for handle, which, c, lo, hi, sub in pending:
            if filts[which] is not None:
                engine.filter_side(handle, parts[which][c], sub[lo:hi])
        mark("filters enqueued")
        del pending
        overflow = None
        if stats_all is not None:
            # the near-tie list of a bound-and-refine call is bounded; a call that ran out of room
            # (never seen on real or synthetic embeddings, possible on adversarial ones) reports
            # found = capacity + 1.  The flag travels with the counters; nobody waits for it here.
            buf[4 * n:] = (stats_all[:, 0] > stats_all[:, 1]).sum().to(torch.int32)
            overflow = buf[4 * n]
        if shard is not None and shard.world > 1:
            shard.all_reduce_sum(buf)  # the single collective on the rank counters (+ flag)
        mark("collective")
        rank_t, filt_t = engine.finalize(counters[0], counters[1])
        rank_h, filt_h = engine.finalize(counters[2], counters[3])
        mark("finalize")
    result = (rank_h, rank_t, filt_h, filt_t)

    def redo():
        return rank_link_prediction(table, h_idx, t_idx, r_idx, filts[0], filts[1], shard=shard,
                                    engine=engine, chunk=chunk, exact=True)

    lazy = LazyRanks(result, overflow, redo)
    return lazy.get() if sync else lazy


def relation_groups(r_idx, n_rel):
    """Facts grouped by relation: (order, order_host, groups) with ``order`` the device permutation that sorts
    r_idx (stable), ``order_host`` its host copy and ``groups`` the host list of (relation, lo, hi) of the
    sorted facts, relations without facts left out.  One device -> host copy."""
    order = torch.argsort(r_idx, stable=True)
    both = torch.cat([torch.bincount(r_idx, minlength=n_rel), order]).cpu()   # the one host synchronisation
    counts, order_host = both[:n_rel].tolist(), both[n_rel:]
    groups, lo = [], 0
    for rel, c in enumerate(counts):
        if c:
            groups.append((rel, lo, lo + c))
            lo += c
    return order, order_host, groups


def _projected_groups(spec, groups, engine):
    """The relation-grouped loop of a ProjectedSpec: for every (relation, lo, hi) of ``groups`` (relation_groups),
    the entity table projected for the relation (``spec.project``) into one (n_rows, dim) buffer, allocated once,
    then (relation, lo, hi, the buffer's TransE-L2 spec)."""
    proj = torch.empty((spec.n_rows, spec.dim), dtype=torch.float32, device=spec.ent0.device)
    table = ModelSpec(spec.code, spec.dim, spec.n_ent, spec.n_rel, proj, None, spec.rel0, None)
    for rel, lo, hi in groups:
        spec.project(engine, rel, proj)
        yield rel, lo, hi, table


def rank_link_prediction_projected(spec, h_idx, t_idx, r_idx, groups, filt_tail, filt_head, engine=None,
                                   chunk=DEFAULT_CHUNK, exact=False, sync=True):
    """rank_link_prediction for TransH and TransD (ProjectedSpec): the facts come sorted by relation, ``groups``
    the (relation, lo, hi) of relation_groups.  Per relation, the entity table is projected (_projected_groups)
    and the group is ranked on it as TransE-L2 -- tail queries fl(P_r(h) + r) against the projected candidates,
    head candidates (P_r(c) + r) - P_r(t), exactly the reference's arithmetic on its projected_entities
    (interfaces.py:249-260) -- with the filter CSR rows of the group.  The tensor-core image of the buffer is
    rebuilt per relation, without the cache.  Arguments and result as rank_link_prediction's (no shard)."""
    engine = engine or default_engine()
    n = h_idx.shape[0]
    dev = spec.ent0.device
    with _device_guard(dev):
        ranks = [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(4)]
        filts = [f() if callable(f) else f for f in (filt_tail, filt_head)]
        ranges = [(lo, hi) for _, lo, hi in groups]
        parts = [_csr_cut(f, ranges) for f in filts]    # one device -> host read per CSR
        flags = []
        for (_, lo, hi, table), ft, fh in zip(_projected_groups(spec, groups, engine), parts[0], parts[1]):
            lazy = rank_link_prediction(table, h_idx[lo:hi], t_idx[lo:hi], r_idx[lo:hi], ft, fh, engine=engine,
                                        chunk=chunk, exact=exact, sync=False, tc_cache=False)
            for out, x in zip(ranks, lazy.ranks):
                out[lo:hi] = x
            if lazy.overflow is not None:
                flags.append(lazy.overflow.view(1))
        overflow = torch.cat(flags).sum() if flags else None

    def redo():
        return rank_link_prediction_projected(spec, h_idx, t_idx, r_idx, groups, filts[0], filts[1], engine=engine,
                                              chunk=chunk, exact=True)

    lazy = LazyRanks(tuple(ranks), overflow, redo)
    return lazy.get() if sync else lazy


def relation_spec(spec):
    """The model seen from relation prediction: the candidate table is the RELATION table
    (``inference_prepare_candidates(..., entities=False)``: translation.py:118-121,
    bilinear.py:263-265, 551-554)."""
    cand2 = None
    if spec.code in (_lib.TRANSE_L1, _lib.TRANSE_L2, _lib.DISTMULT):
        cand0, cand1 = spec.rel0, None
    elif spec.code == _lib.COMPLEX:
        cand0, cand1 = spec.rel0, spec.rel1
    elif spec.code == _lib.ANALOGY:
        cand0, cand1, cand2 = spec.rel0, spec.rel1, spec.rel2
    else:
        raise NotImplementedError(
            "%s has no scan-based relation-prediction path (TransE L1/L2, DistMult, ComplEx, Analogy have; "
            "RESCAL goes through the dense kge_rescal_rel_scores)" % _lib.MODEL_NAMES.get(spec.code, spec.code))
    return ModelSpec(spec.code, spec.dim, spec.n_rel, spec.n_rel, cand0, cand1, None, None, ent2=cand2)


def _dense_relations(spec):
    """Models whose relation case is a dense (n, n_rel) score matrix rather than a scan over a candidate table:
    RESCAL (per-fact vectors h^T M_c, bilinear.py:115-121), TransH and TransD (rows projected per relation,
    interfaces.py:261-272)."""
    return spec.code == _lib.RESCAL or isinstance(spec, ProjectedSpec)


def _dense_rel_scores(engine, spec, hrows, trows, h_idx=None, t_idx=None):
    """(n, n_rel) relation scores of the facts (hrows, ?, trows), hrows / trows (n, dim), for _dense_relations.
    TransD also reads the scalars of the facts' entities h_idx / t_idx (unsharded calls only)."""
    if isinstance(spec, ProjectedSpec):
        return spec.rel_scores(engine, hrows, trows, h_idx, t_idx)
    return engine.rescal_rel_scores(spec, hrows, trows)


def rank_relation_prediction(spec, h_idx, t_idx, r_idx, filt, directed=True, engine=None,
                             chunk=DEFAULT_CHUNK, shard=None):
    """Rank every fact's true relation against all relations (RelationPredictionEvaluator,
    torchkge/evaluation.py:64-112).

    filt       device CSR (offs, ids) of the relations to discount per fact (dict_of_rels[(h, t)]
               minus the true one), or None
    directed   False: the scores of (t, ?, h) are ranked together with those of (h, ?, t), against
               the directed true score (evaluation.py:99-107)
    shard      None; QueryShard over the n facts: every rank ranks its slice of the facts (and of
               ``filt``) against the replicated table; EntityShard: the relations, the candidates, are
               on every rank, so the facts are split too -- under local storage the h / t rows of each
               chunk are first exchanged by one all-reduce, and the chunk's facts split as
               ``shard.split`` splits them (_exchanged_chunks); under full storage the facts are split
               as ``shard.split(n)`` splits them.  Either way one all-gather per split brings every
               rank the full rank vectors, equal to the unsharded call's.
    Returns (rank_true_rels, filt_rank_true_rels), int64 device tensors.
    """
    engine = engine or default_engine()
    n = h_idx.shape[0]
    dev = spec.ent0.device
    if isinstance(spec, ProjectedSpec):
        refuse_projected_shard(spec.name, shard)
    rspec = None if _dense_relations(spec) else relation_spec(spec)   # unsupported models raise here
    if isinstance(shard, EntityShard):
        _check_table(spec, shard)
        if not shard.local_storage:
            shard = shard.split(n)
    if isinstance(shard, QueryShard) and shard.world > 1:
        _check_queries(shard, n)
        return tuple(_by_query_slices(shard, lambda h, t, r, f: rank_relation_prediction(
            spec, h, t, r, f, directed, engine, chunk), (h_idx, t_idx, r_idx), filt))
    with _device_guard(dev):
        packed = None if rspec is None else engine.pack(rspec)
        keep = []

        def rank_rows(hrows, trows, r, f, raw, sub, h=None, t=None):
            """Adds the counts of facts (hrows, ?, trows) with true relations r into raw / sub; h / t: the
            facts' entities (unsharded calls)."""
            m = r.shape[0]
            s_true = torch.empty(m, dtype=torch.float32, device=dev)
            if rspec is None:
                # RESCAL, TransH, TransD: a dense (m, n_rel) score matrix (_dense_rel_scores) ranked by
                # kge_rank_dense
                hrows, trows = hrows.reshape(m, spec.dim), trows.reshape(m, spec.dim)
                engine.rank_dense(_dense_rel_scores(engine, spec, hrows, trows, h, t), r, f, raw, sub,
                                  true_score=s_true)
                if not directed:
                    engine.rank_dense(_dense_rel_scores(engine, spec, trows, hrows, t, h), r, f, raw, sub,
                                      true_score_in=s_true)
                return
            rrows = engine.gather_rows(rspec, r)
            keep.append(engine.rank_side(rspec, packed, _lib.SIDE_REL, hrows, trows, None, r, f, raw, sub,
                                         true_score=s_true, true_rows=rrows))
            if not directed:
                keep.append(engine.rank_side(rspec, packed, _lib.SIDE_REL, trows, hrows, None, r, f, raw, sub,
                                             true_rows=rrows, true_score_in=s_true))
            keep.append((s_true, f))

        # the dense branch holds (chunk, n_rel) scores: at most 4096 facts per call
        step = min(chunk, 4096) if rspec is None else chunk
        chunks = [(lo, min(n, lo + step)) for lo in range(0, n, step)]
        if shard is None or shard.world == 1:
            counters = torch.zeros((2, n), dtype=torch.int32, device=dev)
            for (lo, hi), f in zip(chunks, _csr_cut(filt, chunks)):
                h, t, r = h_idx[lo:hi], t_idx[lo:hi], r_idx[lo:hi].contiguous()
                rank_rows(engine.gather_rows(spec, h), engine.gather_rows(spec, t), r, f,
                          counters[0][lo:hi], counters[1][lo:hi], h, t)
            ranks, filt_ranks = engine.finalize(counters[0], counters[1])
            del keep
            return ranks, filt_ranks

        def run(lo, hi, hrows, trows, f):
            counters = torch.zeros((2, hi - lo), dtype=torch.int32, device=dev)
            if hi > lo:        # a rank with no facts in this chunk still joins the all-gather
                rank_rows(hrows, trows, r_idx[lo:hi].contiguous(), f, counters[0], counters[1])
            return engine.finalize(counters[0], counters[1])

        out = [torch.empty(n, dtype=torch.int64, device=dev) for _ in range(2)]
        ranks, filt_ranks = _exchanged_chunks(spec, shard, engine, h_idx, t_idx, chunks, filt, run, out)
        del keep
        return ranks, filt_ranks


def score_triples_entity_sharded(spec, h_idx, t_idx, r_idx, shard, engine=None, batch=DEFAULT_CHUNK):
    """(n,) scores of the triples (h_idx[i], r_idx[i], t_idx[i]) of a model whose entity rows are split
    over ``shard`` (EntityShard, local storage; spec.ent_lo / spec.n_ent set from it, spec over the
    tables the per-triple kernel reads).  Per batch of ``batch`` triples the h and t rows are exchanged
    by one all-reduce (_exchanged_rows), laid out plane-major and scored on every rank with h = i,
    t = b + i: the kernel reads the same bits as on the whole table, so every rank gets the scores of
    ``model.scoring_function``, bit for bit."""
    engine = engine or default_engine()
    _check_table(spec, shard)
    n = h_idx.shape[0]
    dev = spec.ent0.device
    out = torch.empty(n, dtype=torch.float32, device=dev)
    with _device_guard(dev):
        for lo in range(0, n, batch):
            hi = min(n, lo + batch)
            m = hi - lo
            rows = _exchanged_rows(spec, torch.cat([h_idx[lo:hi], t_idx[lo:hi]]), shard, engine)
            ent = rows.transpose(0, 1).contiguous()          # (planes, 2m, dim)
            ar = torch.arange(m, dtype=torch.int64, device=dev)
            out[lo:hi] = engine.score_triples(spec.code, spec.dim, ent, spec.rel0, spec.rel1, ar, ar + m,
                                              r_idx[lo:hi].contiguous())
    return out


# ------------------------------------------------------------------------------ top-k inference
#: queries per top-k call (bounds the collect lists of kge_topk_side; results never depend on it)
TOPK_CHUNK = 16384
TOPK_MAX_K = 1024          # csrc/kernels.h


def _check_k(k, n_cand):
    from .exceptions import WrongArgumentsError
    if k > n_cand:
        raise WrongArgumentsError("top_k = %d exceeds the %d candidates" % (k, n_cand))


def _on(csr, device):
    return None if csr is None else tuple(x.to(device) for x in csr)


def _topk_chunks(n, n_cand, k, topk_chunk, mask_csr, device, chunk):
    """Runs topk_chunk(lo, hi, mask) -> (pred, vals) over chunks of queries; ``mask_csr`` is a host
    CSR over all n queries, each chunk gets its rows (offsets rebased) on the device."""
    _check_k(k, n_cand)
    pred = torch.empty((n, k), dtype=torch.int64, device=device)
    vals = torch.empty((n, k), dtype=torch.float32, device=device)
    chunks = [(lo, min(n, lo + chunk)) for lo in range(0, n, chunk)]
    for (lo, hi), mask in zip(chunks, _csr_cut(mask_csr, chunks)):
        pred[lo:hi], vals[lo:hi] = topk_chunk(lo, hi, _on(mask, device))
    return pred, vals


def _pair_pack(pred, vals):
    """(n, k) int64 ids and (n, k) float32 scores -> one (n, 2, k) int64 tensor holding the score
    bits, so that one collective carries both."""
    return torch.stack([pred, vals.view(torch.int32).to(torch.int64)], 1)


def _pair_unpack(t):
    """(..., 2, k) int64 from _pair_pack -> (ids int64 (..., k), scores float32 (..., k)), contiguous."""
    return t[..., 0, :].contiguous(), t[..., 1, :].to(torch.int32).contiguous().view(torch.float32)


def _check_sharded_k(k, n_cand):
    """Argument errors of a sharded call, raised on every rank before the first collective (a rank
    with nothing to compute must not wait in a collective that the others never reach)."""
    _check_k(k, n_cand)
    if not 1 <= k <= TOPK_MAX_K:
        raise _lib.KgeLibraryError("top-k inference: k must be in [1, %d]" % TOPK_MAX_K)


def _exchanged_rows(spec, idx, shard, engine):
    """(n, planes, dim) rows of the entities ``idx`` on every rank: each rank fills the rows it holds,
    the others stay zero, one sum-all-reduce."""
    if spec.n_rows > 0:
        rows = engine.gather_rows(spec, idx)
    else:                  # an empty shard (n_ent < world) has no table to read
        rows = torch.zeros((idx.shape[0], spec.cand_planes, spec.dim), dtype=torch.float32, device=idx.device)
    return shard.all_reduce_sum(rows)


def _exchanged_chunks(spec, shard, engine, e1, e2, chunks, csr, run, out):
    """Facts or queries (e1[i], ?, e2[i]) under an EntityShard, for tasks whose candidates every rank
    holds, chunk by chunk: the rows of the chunk's e1 and e2 are exchanged by one all-reduce, this rank
    runs its part [lo, hi) of the chunk (as ``shard.split`` splits it) -- ``run(lo, hi, rows1, rows2,
    csr rows)`` -> (hi - lo, ...) results, as many as ``out`` has tensors -- and ONE all-gather brings
    every rank the chunk's results, written into ``out``."""
    parts = [shard.split(hi - lo) for lo, hi in chunks]
    mine = [(lo + p.lo, lo + p.hi) for (lo, _), p in zip(chunks, parts)]
    for (lo, hi), part, (a, b), f in zip(chunks, parts, mine, _csr_cut(csr, mine)):
        m = hi - lo
        rows = _exchanged_rows(spec, torch.cat([e1[lo:hi], e2[lo:hi]]), shard, engine)
        full = part.all_gather(list(run(a, b, rows[part.lo:part.hi], rows[m + part.lo:m + part.hi], f)))
        for o, x in zip(out, full):
            o[lo:hi] = x
    return out


def topk_entity_inference(spec, ents, rels, side, k, mask=None, shard=None, engine=None, chunk=TOPK_CHUNK):
    """The k best entities completing (ents[i], rels[i], ?) (side SIDE_TAIL) or (?, rels[i], ents[i])
    (SIDE_HEAD), best first (EntityInference).

    spec       ModelSpec holding the full entity table, or exactly this rank's rows under an
               EntityShard with local storage (spec.ent_lo / spec.n_ent set from the shard)
    ents/rels  int64 device tensors (n,)
    mask       host CSR (offs int64 (n+1,), ids int64) of GLOBAL entity ids to score -inf per query,
               ascending within a row, or None
    shard      None; EntityShard: every rank scans its rows for every query (query rows exchanged by
               one all-reduce per chunk), keeps its top min(k, rows) and the lists of all ranks are
               all-gathered and merged by kge_topk_merge; QueryShard: every rank answers its slice of
               the queries against the whole table and the results are all-gathered
    Returns (pred int64 (n, k), scores float32 (n, k)) on the device, the same on every rank and
    equal, bit for bit, to the unsharded call.
    """
    engine = engine or default_engine()
    n = ents.shape[0]
    dev = spec.ent0.device
    if isinstance(spec, ProjectedSpec):
        refuse_projected_shard(spec.name, shard)
        return _topk_entity_projected(spec, ents, rels, side, k, mask, engine, chunk)
    if shard is not None and shard.world > 1:
        _check_sharded_k(k, spec.n_ent)
    if isinstance(shard, EntityShard):
        _check_table(spec, shard)
    if isinstance(shard, QueryShard) and shard.world > 1:
        _check_queries(shard, n)
        full, = _by_query_slices(shard, lambda e, r, m: [_pair_pack(*topk_entity_inference(
            spec, e, r, side, k, m, engine=engine, chunk=chunk))], (ents, rels), mask)
        return _pair_unpack(full)
    with _device_guard(dev):
        if shard is None or shard.world == 1:
            packed = engine.pack(spec)

            def topk_chunk(lo, hi, m):
                rows = engine.gather_rows(spec, ents[lo:hi])
                return engine.topk_side(spec, packed, side, rows, rows, rels[lo:hi].contiguous(), k, m)

            return _topk_chunks(n, spec.n_rows, k, topk_chunk, mask, dev, chunk)
        spec = _scanned(spec, shard)
        k_loc = min(k, spec.n_rows)
        packed = engine.pack(spec) if k_loc > 0 else None

        def topk_chunk(lo, hi, m):
            rows = _exchanged_rows(spec, ents[lo:hi], shard, engine)
            pred = torch.full((hi - lo, k), -1, dtype=torch.int64, device=dev)
            vals = torch.full((hi - lo, k), float("-inf"), dtype=torch.float32, device=dev)
            if k_loc > 0:     # a shard with fewer rows than k pads its list with empty slots
                pred[:, :k_loc], vals[:, :k_loc] = engine.topk_side(spec, packed, side, rows, rows,
                                                                    rels[lo:hi].contiguous(), k_loc, m)
            pred_in, scores_in = _pair_unpack(shard.stack_all(_pair_pack(pred, vals)))
            return engine.topk_merge(pred_in, scores_in, k)

        return _topk_chunks(n, spec.n_ent, k, topk_chunk, mask, dev, chunk)


def _topk_entity_projected(spec, ents, rels, side, k, mask, engine, chunk):
    """topk_entity_inference for TransH and TransD: the queries grouped by relation (relation_groups), the entity
    table projected per relation (_projected_groups) and scanned as TransE-L2, as in
    rank_link_prediction_projected."""
    n = ents.shape[0]
    dev = spec.ent0.device
    _check_k(k, spec.n_rows)
    with _device_guard(dev):
        order, perm, groups = relation_groups(rels, spec.n_rel)
        ents_s, rels_s = ents[order].contiguous(), rels[order].contiguous()
        if mask is not None:        # host CSR over the queries -> rows in sorted order
            offs, ids = mask
            lens = offs[1:] - offs[:-1]
            new_offs = torch.zeros(n + 1, dtype=torch.int64)
            new_offs[1:] = torch.cumsum(lens[perm], 0)
            sel = torch.repeat_interleave(offs[:-1][perm], lens[perm]) + (
                torch.arange(int(new_offs[-1])) - torch.repeat_interleave(new_offs[:-1], lens[perm]))
            mask = (new_offs, ids[sel])
        pred = torch.empty((n, k), dtype=torch.int64, device=dev)
        vals = torch.empty((n, k), dtype=torch.float32, device=dev)
        masks = _csr_cut(mask, [(lo, hi) for _, lo, hi in groups])
        for (_, lo, hi, table), m in zip(_projected_groups(spec, groups, engine), masks):
            packed = engine.pack(table)

            def topk_chunk(a, b, mm):
                rows = engine.gather_rows(table, ents_s[lo + a:lo + b])
                return engine.topk_side(table, packed, side, rows, rows, rels_s[lo + a:lo + b], k, mm)

            pred[lo:hi], vals[lo:hi] = _topk_chunks(hi - lo, spec.n_rows, k, topk_chunk, m, dev, chunk)
        out_pred, out_vals = torch.empty_like(pred), torch.empty_like(vals)
        out_pred[order], out_vals[order] = pred, vals
        return out_pred, out_vals


def topk_relation_inference(spec, e1, e2, k, mask=None, shard=None, engine=None, chunk=TOPK_CHUNK):
    """The k best relations completing (e1[i], ?, e2[i]), best first (RelationInference).

    The candidates are the relations, which every rank holds, so both shard types split the queries
    over the ranks and all-gather the results; under an EntityShard the rows of e1 / e2 are first
    exchanged (one all-reduce per chunk), the queries of each chunk are split as QueryShard splits
    them.  Arguments and result as in topk_entity_inference; ``mask`` lists relation ids.
    """
    engine = engine or default_engine()
    n = e1.shape[0]
    dev = spec.ent0.device
    if isinstance(spec, ProjectedSpec):
        refuse_projected_shard(spec.name, shard)
    if isinstance(shard, QueryShard) and shard.world > 1:
        _check_sharded_k(k, spec.n_rel)
        _check_queries(shard, n)
        full, = _by_query_slices(shard, lambda a, b, m: [_pair_pack(*topk_relation_inference(
            spec, a, b, k, m, engine=engine, chunk=chunk))], (e1, e2), mask)
        return _pair_unpack(full)
    if _dense_relations(spec):
        # RESCAL, TransH, TransD: dense (n, n_rel) scores, then the same selection kernels
        rspec, packed, n_cand = None, None, spec.n_rel
    else:
        rspec = relation_spec(spec)
        packed, n_cand = engine.pack(rspec), rspec.n_rows

    def local_topk(hrows, trows, m, a=None, b=None):
        if rspec is None:
            m_rows = hrows.shape[0]
            scores = _dense_rel_scores(engine, spec, hrows.view(m_rows, spec.dim), trows.view(m_rows, spec.dim), a, b)
            return engine.topk_dense(scores, k, m)
        return engine.topk_side(rspec, packed, _lib.SIDE_REL, hrows, trows, None, k, m)

    if isinstance(shard, EntityShard):
        if shard.world > 1:
            _check_sharded_k(k, n_cand)
        _check_table(spec, shard)
    with _device_guard(dev):
        if shard is None or shard.world == 1:
            def topk_chunk(lo, hi, m):
                a, b = e1[lo:hi], e2[lo:hi]
                return local_topk(engine.gather_rows(spec, a), engine.gather_rows(spec, b), m, a, b)

            return _topk_chunks(n, n_cand, k, topk_chunk, mask, dev, chunk)

        def run(lo, hi, rows1, rows2, m):
            if hi > lo:
                return [_pair_pack(*local_topk(rows1, rows2, _on(m, dev)))]
            return [torch.empty((0, 2, k), dtype=torch.int64, device=dev)]

        chunks = [(lo, min(n, lo + chunk)) for lo in range(0, n, chunk)]
        full, = _exchanged_chunks(_scanned(spec, shard), shard, engine, e1, e2, chunks, mask, run,
                                  [torch.empty((n, 2, k), dtype=torch.int64, device=dev)])
        return _pair_unpack(full)
