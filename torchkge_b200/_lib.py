"""ctypes binding of libkge_b200.so (C ABI declared in include/kge_b200.h).

The product path has no CPU fallback: if the shared library is missing or a call fails,
``KgeLibraryError`` is raised.  Host-only entry points (schedule construction, size
queries) work without a GPU and are what the ``-m "not gpu"`` tests exercise.
"""
import ctypes
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libkge_b200.so")

# kge_model_t / kge_side_t (include/kge_b200.h)
TRANSE_L1, TRANSE_L2, DISTMULT, RESCAL, COMPLEX, ROTATE, TORUSE_L1, TORUSE_L2, ANALOGY = range(9)
SIDE_TAIL, SIDE_HEAD, SIDE_REL = 0, 1, 2
TILE_C, TILE_Q = 128, 64
ABI_VERSION = 11
FLAG_TENSOR_CORE = 1
FLAG_APPROX_SCAN = 2
LOSS_MARGIN, LOSS_LOGISTIC, LOSS_BCE = 0, 1, 2

MODEL_NAMES = {TRANSE_L1: "TransE-L1", TRANSE_L2: "TransE-L2", DISTMULT: "DistMult",
               RESCAL: "RESCAL", COMPLEX: "ComplEx", ROTATE: "RotatE",
               TORUSE_L1: "TorusE-L1", TORUSE_L2: "TorusE-L2", ANALOGY: "Analogy"}


class KgeLibraryError(RuntimeError):
    """libkge_b200.so is missing, stale or returned an error code."""


_c = ctypes
_p = ctypes.c_void_p


class RankArgs(ctypes.Structure):
    """kge_rank_args_t"""
    _fields_ = [
        ("model", _c.c_int32), ("side", _c.c_int32), ("dim", _c.c_int32), ("flags", _c.c_int32),
        ("n", _c.c_int64), ("n_ent", _c.c_int64), ("ent_lo", _c.c_int64), ("n_rows", _c.c_int64),
        ("packed", _p), ("ent0", _p), ("ent1", _p), ("rel0", _p), ("rel1", _p),
        ("hrows", _p), ("trows", _p), ("r_idx", _p), ("true_idx", _p),
        ("filt_offs", _p), ("filt_ids", _p), ("n_filt", _c.c_int64),
        ("raw_count", _p), ("filt_sub", _p), ("true_score", _p),
        ("workspace", _p), ("workspace_bytes", _c.c_size_t), ("stream", _p),
        ("tc_packed", _p), ("tc_stats", _p), ("tc_dump", _p),
        ("true_rows", _p), ("true_score_in", _p), ("filt_qid", _p),
    ]


class ScoreAllArgs(ctypes.Structure):
    """kge_score_all_args_t"""
    _fields_ = [
        ("model", _c.c_int32), ("side", _c.c_int32), ("dim", _c.c_int32), ("reserved0", _c.c_int32),
        ("n", _c.c_int64), ("n_rows", _c.c_int64),
        ("packed", _p), ("rel0", _p), ("rel1", _p), ("hrows", _p), ("trows", _p), ("r_idx", _p),
        ("scores", _p), ("workspace", _p), ("workspace_bytes", _c.c_size_t), ("stream", _p),
    ]


class TopkArgs(ctypes.Structure):
    """kge_topk_args_t"""
    _fields_ = [
        ("model", _c.c_int32), ("side", _c.c_int32), ("dim", _c.c_int32), ("k", _c.c_int32),
        ("n", _c.c_int64), ("n_rows", _c.c_int64),
        ("packed", _p), ("rel0", _p), ("rel1", _p), ("hrows", _p), ("trows", _p), ("r_idx", _p),
        ("mask_offs", _p), ("mask_ids", _p), ("pred", _p), ("scores", _p),
        ("workspace", _p), ("workspace_bytes", _c.c_size_t), ("stream", _p),
        ("ent_lo", _c.c_int64),
    ]


class Tables(ctypes.Structure):
    """kge_tables_t"""
    _fields_ = [("model", _c.c_int32), ("dim", _c.c_int32),
                ("ent0", _p), ("ent1", _p), ("rel0", _p), ("rel1", _p)]


class Grads(ctypes.Structure):
    """kge_grads_t"""
    _fields_ = [("ent0", _p), ("ent1", _p), ("rel0", _p), ("rel1", _p)]


class MarginStepArgs(ctypes.Structure):
    """kge_margin_step_args_t"""
    _fields_ = [
        ("tb", Tables), ("n_neg", _c.c_int32), ("margin", _c.c_float),
        ("b", _c.c_int64), ("n_ent", _c.c_int64),
        ("h", _p), ("t", _p), ("r", _p), ("nh", _p), ("nt", _p), ("bern_probs", _p),
        ("seed", _c.c_uint64), ("offset", _c.c_uint64),
        ("loss", _p), ("pos_out", _p), ("neg_out", _p), ("nh_out", _p), ("nt_out", _p),
        ("stream", _p),
        ("ent_lo", _c.c_int64), ("n_rows", _c.c_int64),
        ("hrows", _p), ("trows", _p), ("grad_hrows", _p), ("grad_trows", _p),
        ("loss_kind", _c.c_int32),
    ]


class RelStepArgs(ctypes.Structure):
    """kge_rel_step_args_t"""
    _fields_ = [
        ("base", MarginStepArgs), ("n_rel", _c.c_int64), ("rel_share", _c.c_float),
        ("nr", _p), ("nr_out", _p),
    ]


class PosStepArgs(ctypes.Structure):
    """kge_pos_step_args_t"""
    _fields_ = [
        ("base", MarginStepArgs), ("n_rel", _c.c_int64),
        ("head_offs", _p), ("head_ents", _p), ("tail_offs", _p), ("tail_ents", _p),
    ]


# name -> (restype, argtypes); every symbol include/kge_b200.h declares
SIGNATURES = {
    "kge_abi_version": (_c.c_int, []),
    "kge_last_error": (_c.c_char_p, []),
    "kge_cand_planes": (_c.c_int, [_c.c_int]),
    "kge_query_planes": (_c.c_int, [_c.c_int, _c.c_int]),
    "kge_build_schedule": (_c.c_int, [_c.c_int, _c.c_int, _p, _p]),
    "kge_packed_table_floats": (_c.c_size_t, [_c.c_int, _c.c_int64, _c.c_int]),
    "kge_pack_table": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _c.c_int, _p, _p]),
    "kge_gather_rows": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _c.c_int64, _c.c_int, _p,
                                   _c.c_int64, _p, _p]),
    "kge_rank_workspace_bytes": (_c.c_size_t, [_c.c_int, _c.c_int, _c.c_int, _c.c_int64, _c.c_int64,
                                               _c.c_int]),
    "kge_schedule_depth": (_c.c_int, [_c.c_int, _c.c_int]),
    "kge_tc_packed_bytes": (_c.c_size_t, [_c.c_int, _c.c_int64, _c.c_int]),
    "kge_tc_configure": (_c.c_int, [_c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "kge_tc_bound_constants": (_c.c_int, [_c.c_int, _c.c_int, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float),
                                          _c.POINTER(_c.c_float), _c.POINTER(_c.c_int)]),
    "kge_tc_layout_id": (_c.c_int, []),
    "kge_tc_pack_table": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _c.c_int, _p, _p]),
    "kge_tc_pack_table_cached": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _c.c_int, _p, _p, _p]),
    "kge_rank_side": (_c.c_int, [_c.POINTER(RankArgs)]),
    "kge_filter_side": (_c.c_int, [_c.POINTER(RankArgs)]),
    "kge_finalize_ranks": (_c.c_int, [_p, _p, _c.c_int64, _p, _p, _p]),
    "kge_score_all": (_c.c_int, [_c.POINTER(ScoreAllArgs)]),
    "kge_topk_workspace_bytes": (_c.c_size_t, [_c.c_int, _c.c_int, _c.c_int, _c.c_int64, _c.c_int64, _c.c_int]),
    "kge_topk_side": (_c.c_int, [_c.POINTER(TopkArgs)]),
    "kge_topk_merge": (_c.c_int, [_p, _p, _c.c_int, _c.c_int64, _c.c_int, _c.c_int, _p, _p, _p]),
    "kge_rescal_rel_scores": (_c.c_int, [_p, _p, _p, _c.c_int, _c.c_int64, _c.c_int64, _p, _p]),
    "kge_transh_rel_scores": (_c.c_int, [_p, _p, _p, _p, _c.c_int, _c.c_int64, _c.c_int64, _p, _p]),
    "kge_transh_project": (_c.c_int, [_p, _p, _c.c_int64, _c.c_int, _p, _p]),
    "kge_transd_entity_scalars": (_c.c_int, [_p, _p, _c.c_int64, _c.c_int, _p, _p]),
    "kge_transd_project": (_c.c_int, [_p, _c.c_int, _p, _p, _c.c_int64, _c.c_int, _p, _p]),
    "kge_transd_rel_scores": (_c.c_int, [_p, _p, _p, _p, _p, _p, _c.c_int, _c.c_int64, _c.c_int64, _p, _p]),
    "kge_rank_dense": (_c.c_int, [_p, _c.c_int64, _c.c_int64, _p, _p, _p, _p, _p, _p, _p, _p]),
    "kge_topk_dense_workspace_bytes": (_c.c_size_t, [_c.c_int64, _c.c_int64, _c.c_int]),
    "kge_topk_dense": (_c.c_int, [_p, _c.c_int64, _c.c_int64, _c.c_int, _p, _p, _p, _p, _p, _c.c_size_t, _p]),
    "kge_score_triples_fwd": (_c.c_int, [_c.POINTER(Tables), _p, _p, _p, _c.c_int64, _p, _p]),
    "kge_score_triples_bwd": (_c.c_int, [_c.POINTER(Tables), _c.POINTER(Grads), _p, _p, _p,
                                         _c.c_int64, _p, _p]),
    "kge_transh_score_triples_fwd": (_c.c_int, [_p, _p, _p, _c.c_int, _p, _p, _p, _c.c_int64, _p, _p]),
    "kge_transh_score_triples_bwd": (_c.c_int, [_p, _p, _p, _p, _p, _p, _c.c_int, _p, _p, _p, _c.c_int64, _p,
                                                _p]),
    "kge_transd_score_triples_fwd": (_c.c_int, [_p, _p, _p, _p, _c.c_int, _c.c_int, _p, _p, _p, _c.c_int64, _p,
                                                _p]),
    "kge_transd_score_triples_bwd": (_c.c_int, [_p, _p, _p, _p, _p, _p, _p, _p, _c.c_int, _c.c_int, _p, _p, _p,
                                                _c.c_int64, _p, _p]),
    "kge_corrupt_batch": (_c.c_int, [_p, _p, _p, _c.c_int64, _c.c_int32, _p, _c.c_int64,
                                     _c.c_uint64, _c.c_uint64, _p, _p, _p]),
    "kge_margin_loss_fwd": (_c.c_int, [_p, _p, _c.c_int64, _c.c_float, _p, _p]),
    "kge_margin_loss_bwd": (_c.c_int, [_p, _p, _c.c_int64, _c.c_float, _p, _p, _p, _p]),
    "kge_pair_loss_fwd": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _p, _p]),
    "kge_pair_loss_bwd": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _p, _p, _p, _p]),
    "kge_margin_step_fwd": (_c.c_int, [_c.POINTER(MarginStepArgs)]),
    "kge_margin_step_bwd": (_c.c_int, [_c.POINTER(MarginStepArgs), _c.POINTER(Grads), _p]),
    "kge_scatter_rows_add": (_c.c_int, [_c.c_int, _p, _p, _c.c_int64, _c.c_int64, _c.c_int, _p, _c.c_int64,
                                        _p, _p]),
    "kge_corrupt_batch_rel": (_c.c_int, [_p, _p, _p, _c.c_int64, _c.c_int32, _p, _c.c_int64, _c.c_int64,
                                         _c.c_float, _c.c_uint64, _c.c_uint64, _p, _p, _p, _p]),
    "kge_rel_step_fwd": (_c.c_int, [_c.POINTER(RelStepArgs)]),
    "kge_rel_step_bwd": (_c.c_int, [_c.POINTER(RelStepArgs), _c.POINTER(Grads), _p]),
    "kge_pos_step_fwd": (_c.c_int, [_c.POINTER(PosStepArgs)]),
    "kge_pos_step_bwd": (_c.c_int, [_c.POINTER(PosStepArgs), _c.POINTER(Grads), _p]),
    "kge_cooccurrence": (_c.c_int, [_p, _p, _p, _c.c_int64, _p, _p, _p, _c.c_int64, _c.c_int64, _c.c_int64,
                                    _c.c_int, _c.c_int, _p, _p]),
    "kge_scan_timing_enable": (_c.c_int, [_c.c_int]),
    "kge_scan_timing_read": (_c.c_int, [_c.c_int, _c.POINTER(_c.c_int64), _c.POINTER(_c.c_double)]),
}

_lock = threading.Lock()
_lib = None


def load():
    """Load (once) and return the ctypes handle; raises KgeLibraryError if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise KgeLibraryError(
                "%s not found: build it with `python -m torchkge_b200._build` "
                "(there is no CPU fallback)" % LIB_PATH)
        try:
            lib = ctypes.CDLL(LIB_PATH)
        except OSError as e:  # missing libcudart etc.
            raise KgeLibraryError("cannot load %s: %s" % (LIB_PATH, e)) from e
        for name, (res, args) in SIGNATURES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as e:
                raise KgeLibraryError("%s does not export %s (stale build?)" % (LIB_PATH, name)) from e
            fn.restype = res
            fn.argtypes = args
        if lib.kge_abi_version() != ABI_VERSION:
            raise KgeLibraryError("ABI mismatch: library %d, binding %d"
                                  % (lib.kge_abi_version(), ABI_VERSION))
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().kge_last_error().decode(errors="replace")
        raise KgeLibraryError("%s failed (code %d): %s" % (what, rc, msg))


def build_schedule(model, dim):
    """(perm, code) numpy arrays of the reduction schedule for (model, dim) -- host only."""
    import numpy as np
    lib = load()
    perm = np.zeros(dim, dtype=np.int32)
    code = np.zeros(dim, dtype=np.uint8)
    check(lib.kge_build_schedule(model, dim, perm.ctypes.data, code.ctypes.data), "kge_build_schedule")
    return perm, code


def tc_configure(bk=-1, resident=-1, ct_group=-1, max_ctas=-1, fp16=-1):
    """Tuning / test hook of the tensor-core scan (include/kge_b200.h: kge_tc_configure)."""
    check(load().kge_tc_configure(bk, resident, ct_group, max_ctas, fp16), "kge_tc_configure")


def tc_bound_constants(model, dim):
    """(gamma, gamma2, gamma_p, fp16) of the tensor-core scan's error bound for (model, dim) -- host only."""
    g, g2, gp, f = ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0), ctypes.c_int(0)
    check(load().kge_tc_bound_constants(model, dim, ctypes.byref(g), ctypes.byref(g2), ctypes.byref(gp),
                                        ctypes.byref(f)), "kge_tc_bound_constants")
    return g.value, g2.value, gp.value, bool(f.value)


def scan_timing_enable(on=True):
    check(load().kge_scan_timing_enable(1 if on else 0), "kge_scan_timing_enable")


def scan_timing_read(kind=0):
    """(launches, total_ms) since the last read for kind 0 = scalar dense scan, 1 = tensor-core
    scan, 2 = exact recheck of the near-tie list."""
    n, ms = ctypes.c_int64(0), ctypes.c_double(0.0)
    check(load().kge_scan_timing_read(kind, ctypes.byref(n), ctypes.byref(ms)), "kge_scan_timing_read")
    return n.value, ms.value
