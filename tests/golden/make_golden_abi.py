"""The host layer's answers to size queries and malformed calls: tests/golden/abi_answers.json.

    python tests/golden/make_golden_abi.py

Records, for libkge_b200.so as built in the tree:
  * the size queries (kge_rank_workspace_bytes, kge_topk_workspace_bytes, kge_topk_dense_workspace_bytes,
    kge_packed_table_floats, kge_tc_packed_bytes) over the grid below, the tensor-core ones under both
    k-block widths of kge_tc_configure.  Each answer list is stored as its length and SHA-256;
  * for every launching entry point, malformed calls (required pointers nulled in turn, negative sizes,
    unknown model / side / loss kind, missing second planes, k out of range, a workspace one byte too
    small, inconsistent sharded-step fields, empty calls, and pairs of bad arguments, which pin the order
    of the checks) and the (return code, kge_last_error()) of each.

The calls run in a child process started with CUDA_VISIBLE_DEVICES="": a call that gets past its
argument checks fails there with KGE_ERR_CUDA instead of launching on the dummy pointers.  Only calls
answered with KGE_ERR_ARG, KGE_ERR_UNSUPPORTED or an early KGE_OK go into the fixture.
tests/test_abi_answers.py replays them and compares.
"""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from torchkge_b200 import _lib  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "abi_answers.json")
OK, ERR_CUDA = 0, 2
L = _lib

MODELS, SIDES = range(10), range(4)   # model 9 and side 3 are unknown
DIMS = (1, 16, 200, 256, 1000)
NS = (0, 1, 129, 65536)
N_ROWS = (0, 1, 255, 256, 10 ** 6)
FLAGS = (0, L.FLAG_TENSOR_CORE, L.FLAG_APPROX_SCAN)
KS = (1, 1024)
DIM_UNSUPPORTED = 9000
BIG = 1 << 50                         # a workspace size that passes every size check


def ptr(i):
    """A fixed dummy device address, distinct per field."""
    return 0x7f0000000000 + (i + 1) * 0x100000


def digest(values):
    return {"n": len(values), "sha256": hashlib.sha256(json.dumps(values).encode()).hexdigest()}


def sizes(lib):
    grid = [(m, s, d, n, r) for m in MODELS for s in SIDES for d in DIMS for n in NS for r in N_ROWS]
    tables = [(m, r, d) for m in MODELS for r in N_ROWS for d in DIMS]
    out = {
        "kge_rank_workspace_bytes": [lib.kge_rank_workspace_bytes(*g, f) for g in grid for f in FLAGS[::2]],
        "kge_topk_workspace_bytes": [lib.kge_topk_workspace_bytes(*g, k) for g in grid for k in KS],
        "kge_topk_dense_workspace_bytes": [lib.kge_topk_dense_workspace_bytes(n, r, k)
                                           for n in NS for r in N_ROWS for k in KS],
        "kge_packed_table_floats": [lib.kge_packed_table_floats(*t) for t in tables],
    }
    bk0 = lib.kge_tc_layout_id() // 2
    for bk in (32, 64):   # the k-block width sizes both tensor-core images
        lib.kge_tc_configure(bk, -1, -1, -1, -1)
        out["kge_tc_packed_bytes/bk%d" % bk] = [lib.kge_tc_packed_bytes(*t) for t in tables]
        out["kge_rank_workspace_bytes/tensor_core/bk%d" % bk] = [
            lib.kge_rank_workspace_bytes(*g, L.FLAG_TENSOR_CORE) for g in grid]
    lib.kge_tc_configure(bk0, -1, -1, -1, -1)
    return {k: digest(v) for k, v in out.items()}


def struct(cls, values):
    s = cls()
    for name, v in values.items():
        setattr(s, name, struct(type(getattr(s, name)), v) if isinstance(v, dict) else v)
    return s


def pointers(cls):
    return [name for name, ty in cls._fields_ if ty is L._p]


def sweep(cases, group, call, base, variants, nulls):
    """cases[group][name] = thunk: the base arguments, each of `nulls` set to None in turn, each variant."""
    g = cases.setdefault(group, {})
    g["base"] = call(base)
    for f in nulls:
        g["null:" + f] = call(dict(base, **{f: None}))
    for name, over in variants.items():
        g[name] = call(dict(base, **over))


def by_struct(fn, cls, *extra):
    def call(values):
        s = struct(cls, values)
        return lambda: fn(ctypes.byref(s), *extra)
    return call


def by_args(fn, names):
    return lambda values: (lambda args: lambda: fn(*args))([values[n] for n in names])


def query_cases(lib, cases):
    none = {c: {f: None for f in pointers(c)} for c in (L.RankArgs, L.ScoreAllArgs, L.TopkArgs)}
    common = {"unknown_model": dict(model=42), "unknown_side": dict(side=3), "n_negative": dict(n=-1),
              "dim0": dict(dim=0), "dim_unsupported": dict(dim=DIM_UNSUPPORTED),
              "null_rel1_dim_unsupported": dict(rel1=None, dim=DIM_UNSUPPORTED),
              "dim_unsupported_workspace_short": dict(dim=DIM_UNSUPPORTED, workspace_bytes=0),
              "null_hrows_and_rel1": dict(hrows=None, rel1=None)}
    for model, side, flags in ((L.TRANSE_L1, L.SIDE_TAIL, 0), (L.TRANSE_L2, L.SIDE_HEAD, L.FLAG_TENSOR_CORE),
                               (L.DISTMULT, L.SIDE_REL, L.FLAG_TENSOR_CORE), (L.COMPLEX, L.SIDE_TAIL, L.FLAG_TENSOR_CORE),
                               (L.ROTATE, L.SIDE_HEAD, L.FLAG_APPROX_SCAN)):
        cfg = "m%d_s%d_f%d" % (model, side, flags)
        base = dict({f: ptr(i) for i, f in enumerate(pointers(L.RankArgs))}, model=model, side=side, dim=16,
                    flags=flags, n=5, n_ent=1000, n_rows=300, n_filt=7, workspace_bytes=BIG, stream=None,
                    tc_dump=None, tc_stats=None, true_score_in=None)
        short = lib.kge_rank_workspace_bytes(model, side, 16, 5, 300, flags) - 1
        rank = dict(common, n0_no_pointers=dict(none[L.RankArgs], n=0), n_rows_negative=dict(n_rows=-1),
                    workspace_short=dict(workspace_bytes=short), no_true_rows=dict(true_rows=None),
                    no_true_rows_with_score_in=dict(true_rows=None, true_score_in=ptr(60)),
                    filter_no_ids=dict(filt_ids=None), filter_no_ids_n_filt0=dict(filt_ids=None, n_filt=0),
                    null_ent1_and_rel1=dict(ent1=None, rel1=None),
                    null_rel1_and_true_rows=dict(rel1=None, true_rows=None),
                    null_true_rows_and_filt_ids=dict(true_rows=None, filt_ids=None),
                    null_filt_ids_dim_unsupported=dict(filt_ids=None, dim=DIM_UNSUPPORTED),
                    dim_unsupported_null_packed=dict(dim=DIM_UNSUPPORTED, packed=None, tc_packed=None),
                    null_packed_and_tc_packed=dict(packed=None, tc_packed=None),
                    tc_flag=dict(flags=L.FLAG_TENSOR_CORE), no_flags=dict(flags=0))
        sweep(cases, "kge_rank_side/" + cfg, by_struct(lib.kge_rank_side, L.RankArgs), base, rank,
              pointers(L.RankArgs))
        lead = lib.kge_rank_workspace_bytes(model, side, 16, 5, 0, 0)
        sweep(cases, "kge_filter_side/" + cfg, by_struct(lib.kge_filter_side, L.RankArgs), base,
              dict(common, n0=dict(n=0), n_filt0=dict(n_filt=0), n_rows0=dict(n_rows=0),
                   workspace_short=dict(workspace_bytes=lead - 1), null_ent1_dim_unsupported=dict(
                       ent1=None, dim=DIM_UNSUPPORTED)),
              ["ent0", "ent1", "filt_offs", "filt_ids", "filt_sub", "workspace"])
        base = dict({f: ptr(i) for i, f in enumerate(pointers(L.ScoreAllArgs))}, model=model, side=side, dim=16,
                    n=5, n_rows=300, workspace_bytes=BIG, stream=None)
        short = lib.kge_rank_workspace_bytes(model, side, 16, 5, 300, 0) - 1
        sweep(cases, "kge_score_all/" + cfg, by_struct(lib.kge_score_all, L.ScoreAllArgs), base,
              dict(common, n0_no_pointers=dict(none[L.ScoreAllArgs], n=0), n_rows0=dict(n_rows=0),
                   workspace_short=dict(workspace_bytes=short), null_scores_and_rel1=dict(scores=None, rel1=None)),
              pointers(L.ScoreAllArgs))
        base = dict({f: ptr(i) for i, f in enumerate(pointers(L.TopkArgs))}, model=model, side=side, dim=16, k=10,
                    n=5, n_rows=300, workspace_bytes=BIG, stream=None, ent_lo=0)
        short = lib.kge_topk_workspace_bytes(model, side, 16, 5, 300, 10) - 1
        sweep(cases, "kge_topk_side/" + cfg, by_struct(lib.kge_topk_side, L.TopkArgs), base,
              dict(common, n0_no_pointers=dict(none[L.TopkArgs], n=0), k0=dict(k=0), k1025=dict(k=1025),
                   k_above_n_rows=dict(k=301), n0_k_above_n_rows=dict(n=0, k=301), k0_dim0=dict(k=0, dim=0),
                   dim0_k_above_n_rows=dict(dim=0, k=301), n_rows_negative=dict(n_rows=-1),
                   ent_lo_negative=dict(ent_lo=-1), ent_lo_above_limit=dict(ent_lo=(1 << 31) - 300),
                   n0_ent_lo_negative=dict(n=0, ent_lo=-1), mask_ids_missing=dict(mask_ids=None),
                   null_rel1_and_mask_ids=dict(rel1=None, mask_ids=None),
                   mask_ids_missing_dim_unsupported=dict(mask_ids=None, dim=DIM_UNSUPPORTED),
                   workspace_short=dict(workspace_bytes=short)),
              pointers(L.TopkArgs))
    for fn in ("kge_rank_side", "kge_filter_side", "kge_score_all", "kge_topk_side"):
        cases[fn + "/null_args"] = {"call": (lambda f: lambda: f(None))(getattr(lib, fn))}


def table_cases(lib, cases):
    for model in (L.TRANSE_L2, L.COMPLEX, L.ROTATE, 9):
        base = dict(model=model, ent0=ptr(0), ent1=ptr(1), n_rows=300, dim=16, packed=ptr(2), tc_packed=ptr(2),
                    guard=ptr(3), ent_lo=0, idx=ptr(4), n=5, out=ptr(5), grad0=ptr(0), grad1=ptr(1), rows=ptr(5),
                    stream=None)
        names = ["model", "ent0", "ent1", "n_rows", "dim"]
        sweep(cases, "kge_pack_table/m%d" % model, by_args(lib.kge_pack_table, names + ["packed", "stream"]), base,
              {"dim_unsupported": dict(dim=DIM_UNSUPPORTED), "null_ent1_dim_unsupported": dict(ent1=None, dim=0)},
              ["ent0", "ent1", "packed"])
        tc = {"n_rows0_no_pointers": dict(n_rows=0, ent0=None, ent1=None, tc_packed=None)}
        sweep(cases, "kge_tc_pack_table/m%d" % model, by_args(lib.kge_tc_pack_table, names + ["tc_packed", "stream"]),
              base, tc, ["ent0", "ent1", "tc_packed"])
        sweep(cases, "kge_tc_pack_table_cached/m%d" % model,
              by_args(lib.kge_tc_pack_table_cached, names + ["tc_packed", "guard", "stream"]), base, tc,
              ["ent0", "tc_packed"])
        rows = ["ent_lo", "n_rows", "dim", "idx", "n"]
        sweep(cases, "kge_gather_rows/m%d" % model,
              by_args(lib.kge_gather_rows, ["model", "ent0", "ent1"] + rows + ["out", "stream"]), base,
              {"n0_no_pointers": dict(n=0, ent0=None, idx=None, out=None)}, ["ent0", "ent1", "idx", "out"])
        sweep(cases, "kge_scatter_rows_add/m%d" % model,
              by_args(lib.kge_scatter_rows_add, ["model", "grad0", "grad1"] + rows + ["rows", "stream"]), base,
              {"n_negative": dict(n=-1), "n_rows0": dict(n_rows=0), "dim0": dict(dim=0),
               "n0_no_pointers": dict(n=0, grad0=None, idx=None, rows=None)}, ["grad0", "grad1", "idx", "rows"])
    base = dict(pred_in=ptr(0), scores_in=ptr(1), n_lists=4, n=5, k_in=10, k=10, pred=ptr(2), scores=ptr(3),
                stream=None)
    sweep(cases, "kge_topk_merge", by_args(lib.kge_topk_merge, list(base)), base,
          {"n_lists0": dict(n_lists=0), "n_lists65": dict(n_lists=65), "k0": dict(k=0), "k_in1025": dict(k_in=1025),
           "n_negative": dict(n=-1), "n0_k0": dict(n=0, k=0), "n0_no_pointers": dict(n=0, pred=None, scores=None)},
          ["pred_in", "scores_in", "pred", "scores"])
    base = dict(scores=ptr(0), n=5, n_cand=300, k=10, mask_offs=ptr(1), mask_ids=ptr(2), pred=ptr(3),
                out_scores=ptr(4), workspace=ptr(5), workspace_bytes=BIG, stream=None)
    sweep(cases, "kge_topk_dense", by_args(lib.kge_topk_dense, list(base)), base,
          {"n0": dict(n=0), "n_cand0": dict(n_cand=0), "k1025": dict(k=1025), "k_above_n_cand": dict(k=301),
           "workspace_short": dict(workspace_bytes=lib.kge_topk_dense_workspace_bytes(5, 300, 10) - 1)},
          ["scores", "pred", "out_scores", "workspace"])


def train_cases(lib, cases):
    grads = dict(ent0=ptr(20), ent1=ptr(21), rel0=ptr(22), rel1=ptr(23))
    for model in (L.TRANSE_L2, L.COMPLEX, 9):
        tb = dict(model=model, dim=16, ent0=ptr(10), ent1=ptr(11), rel0=ptr(12), rel1=ptr(13))
        tables = dict({"tables_null:" + f: dict(tb=dict(tb, **{f: None})) for f in ("ent0", "ent1", "rel0", "rel1")},
                      tables_dim0=dict(tb=dict(tb, dim=0)))

        def triples(fn, *g):
            return lambda v: (lambda s: lambda: fn(ctypes.byref(s), *g, v["h"], v["t"], v["r"], v["n"], v["out"],
                                                   None))(struct(L.Tables, v["tb"]))
        base = dict(tb=tb, h=ptr(0), t=ptr(1), r=ptr(2), n=5, out=ptr(3))
        variants = dict(tables, n0=dict(n=0), n_negative=dict(n=-1), tables_null_n0=dict(tb=dict(tb, rel0=None), n=0))
        sweep(cases, "kge_score_triples_fwd/m%d" % model, triples(lib.kge_score_triples_fwd), base, variants,
              ["h", "t", "r", "out"])
        sweep(cases, "kge_score_triples_bwd/m%d" % model,
              triples(lib.kge_score_triples_bwd, ctypes.byref(struct(L.Grads, grads))), base, variants,
              ["h", "t", "r", "out"])
        for f in grads:
            sweep(cases, "kge_score_triples_bwd/m%d/grads_null:%s" % (model, f),
                  triples(lib.kge_score_triples_bwd, ctypes.byref(struct(L.Grads, dict(grads, **{f: None})))), base,
                  {"n0": dict(n=0)}, [])
        for sharded in (False, True):
            base = dict({f: ptr(30 + i) for i, f in enumerate(pointers(L.MarginStepArgs))}, tb=tb, n_neg=4,
                        margin=1.0, b=8, n_ent=1000, stream=None, nh=None, nt=None, pos_out=None, neg_out=None,
                        nh_out=None, nt_out=None, loss_kind=L.LOSS_BCE if sharded else L.LOSS_MARGIN,
                        ent_lo=100 if sharded else 0, n_rows=200 if sharded else 0)
            if not sharded:
                base.update(hrows=None, trows=None, grad_hrows=None, grad_trows=None)
            rows = dict(hrows=ptr(56), trows=ptr(57))
            variants = dict(
                tables, b0=dict(b=0), b_negative=dict(b=-1), n_neg0=dict(n_neg=0), loss_kind3=dict(loss_kind=3),
                loss_kind_negative=dict(loss_kind=-1), nh_only=dict(nh=ptr(50)), nh_out_only=dict(nh_out=ptr(52)),
                external_negatives_no_probs=dict(nh=ptr(50), nt=ptr(51), bern_probs=None),
                b0_null_h=dict(b=0, h=None, t=None, r=None), hrows_only=dict(hrows=ptr(56), trows=None),
                ent_lo_negative=dict(rows, ent_lo=-1), n_rows_negative=dict(rows, n_rows=-1),
                rows_past_n_ent=dict(rows, ent_lo=900, n_rows=101),
                empty_shard_no_tables=dict(rows, n_rows=0, tb=dict(tb, ent0=None, ent1=None)),
                shard_with_rows_no_tables=dict(rows, n_rows=5, tb=dict(tb, ent0=None, ent1=None)),
                shard_with_external_negatives=dict(rows, nh=ptr(50), nt=ptr(51)),
                shard_with_outputs=dict(rows, pos_out=ptr(54)))
            cfg = "m%d_%s" % (model, "shard" if sharded else "full")
            sweep(cases, "kge_margin_step_fwd/" + cfg, by_struct(lib.kge_margin_step_fwd, L.MarginStepArgs), base,
                  variants, [f for f in pointers(L.MarginStepArgs) if base.get(f)])
            sweep(cases, "kge_margin_step_bwd/" + cfg,
                  by_struct(lib.kge_margin_step_bwd, L.MarginStepArgs, ctypes.byref(struct(L.Grads, grads)), ptr(60)),
                  base, variants, ["grad_hrows", "grad_trows"] if sharded else [])
            for f, g, gl in [("grad_loss", grads, None), ("grads", None, ptr(60))] + [
                    ("grads:" + f, dict(grads, **{f: None}), ptr(60)) for f in grads]:
                gs = None if g is None else ctypes.byref(struct(L.Grads, g))
                sweep(cases, "kge_margin_step_bwd/%s/null:%s" % (cfg, f),
                      by_struct(lib.kge_margin_step_bwd, L.MarginStepArgs, gs, gl), base,
                      {"empty_shard": dict(rows, n_rows=0)}, [])
    cases["kge_margin_step_fwd/null_args"] = {"call": lambda: lib.kge_margin_step_fwd(None)}
    cases["kge_margin_step_bwd/null_args"] = {"call": lambda: lib.kge_margin_step_bwd(None, None, None)}


def loss_cases(lib, cases):
    p = dict(pos=ptr(0), neg=ptr(1), n=5, margin=1.0, loss=ptr(2), grad_loss=ptr(2), grad_pos=ptr(3), grad_neg=ptr(4),
             stream=None)
    bwd = ["pos", "neg", "n", "margin", "grad_loss", "grad_pos", "grad_neg", "stream"]
    sized = {"n0_no_pointers": dict(n=0, pos=None, neg=None, loss=None, grad_loss=None), "n_negative": dict(n=-1)}
    sweep(cases, "kge_margin_loss_fwd", by_args(lib.kge_margin_loss_fwd, ["pos", "neg", "n", "margin", "loss", "stream"]),
          p, sized, ["pos", "neg", "loss"])
    sweep(cases, "kge_margin_loss_bwd", by_args(lib.kge_margin_loss_bwd, bwd), p, sized, bwd[:2] + bwd[4:7])
    for kind in (-1, 0, 1, 2, 3):
        q = dict(p, kind=kind)
        sweep(cases, "kge_pair_loss_fwd/kind%d" % kind, by_args(lib.kge_pair_loss_fwd, ["kind", "pos", "neg", "n", "loss",
                                                                                       "stream"]),
              q, sized, ["pos", "neg", "loss"])
        sweep(cases, "kge_pair_loss_bwd/kind%d" % kind, by_args(lib.kge_pair_loss_bwd, ["kind"] + bwd[:3] + bwd[4:]),
              q, sized, bwd[:2] + bwd[4:7])


def calls(lib):
    """group -> case -> [return code, kge_last_error() or None for KGE_OK], every case."""
    cases = {}
    for add in (query_cases, table_cases, train_cases, loss_cases):
        add(lib, cases)
    out = {}
    for group, g in cases.items():
        for name, thunk in g.items():
            rc = thunk()
            out.setdefault(group, {})[name] = [rc, None if rc == OK else lib.kge_last_error().decode()]
    return out


def answers():
    """sizes() and calls(), run in a child process that sees no GPU."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "--child"]
    proc = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    if proc.returncode != 0:
        raise RuntimeError("answer child exited with %d:\n%s" % (proc.returncode, proc.stderr[-4000:]))
    return json.loads(proc.stdout)


def main():
    got = answers()
    kept = {}
    for group, g in got["calls"].items():
        g = {k: v for k, v in g.items() if v[0] != ERR_CUDA}
        if g:
            kept[group] = g
    with open(OUT, "w") as f:   # one line per size query and per group of calls
        f.write('{"sizes": {\n%s\n},\n"calls": {\n%s\n}}\n' % (
            ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in got["sizes"].items()),
            ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v)) for k, v in kept.items())))
    print("%s: %d size queries, %d calls" % (OUT, len(got["sizes"]), sum(len(g) for g in kept.values())))


if __name__ == "__main__":
    if "--child" in sys.argv:
        lib = _lib.load()
        json.dump({"sizes": sizes(lib), "calls": calls(lib)}, sys.stdout)
    else:
        main()
