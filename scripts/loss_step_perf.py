"""Single-GPU measurements of the fused training step with each loss (DESIGN.md section 4.4).

    python scripts/loss_step_perf.py [--out FILE.json] [--reps N] [--windows N] [--parent-lib PATH]

C5 shape (DistMult d=200, 1M entities, 1000 relations, B = 32,768, n_neg = 256), Philox negatives, timed
with CUDA events after warm-up; every figure is the median of --windows windows of --reps calls:
1. fused forward, and forward + backward, for MarginLoss(1.0), LogisticLoss and BinaryCrossEntropyLoss
   (kge_margin_step_fwd / _bwd with loss_kind, gradient buffers zeroed inside the timed call);
2. the three-call logistic path through the public API: kge_corrupt_batch, model(h, t, r, nh, nt),
   LogisticLoss, backward -- against fused_loss_step(..., LogisticLoss()).backward();
3. 8 emulated entity shards with the logistic loss, every rank's forward + backward + scatter one after
   another (the maximum over the ranks and the sum; collectives not run);
4. the fused and three-call losses at the same seed and offset, each also against a float64 sum of the
   per-pair terms of the three-call scores (both are fp32 sums of 8.4M terms in atomics order);
5. with --parent-lib (a libkge_b200.so built from the parent commit, same ABI): the margin forward +
   backward of both libraries on the same arguments, alternating window by window.
Records the GPU name, power limit and SM clock in the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torchkge_b200 as tk  # noqa: E402
from torchkge_b200 import _lib, synthetic as S  # noqa: E402
from torchkge_b200.engine import CudaEngine, EntityShard, _ptr, _stream  # noqa: E402
from torchkge_b200.training import ShardedStep, _MarginStep, fused_loss_step  # noqa: E402

SEED, OFFSET = 7, 1


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:      # measurement still valid, the facts are then missing
        return {"error": str(e)}


def window(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def timed(fns, reps, windows, warm=2):
    """{name: median ms per call}; the functions' windows alternate."""
    for fn in fns.values():
        for _ in range(warm):
            fn()
    torch.cuda.synchronize()
    got = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            got[k].append(window(fn, reps))
    return {k: statistics.median(v) for k, v in got.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--parent-lib", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("loss_step_perf.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_facts(), "torch_device": torch.cuda.get_device_name(dev)}
    c = S.C5
    dim, n_ent, n_rel, n_neg, b = c["dim"], c["n_ent"], c["n_rel"], c["n_neg"], 32768
    res["shape"] = "DistMult d=%d, %d entities, %d relations, B=%d, n_neg=%d" % (dim, n_ent, n_rel, b, n_neg)
    tabs = S.make_tables(_lib.DISTMULT, dim, n_ent, n_rel, 0, n_ent, 1, dev)
    ent, rel = tabs["ent0"].contiguous(), tabs["rel0"].contiguous()
    g = torch.Generator(device=dev).manual_seed(1)
    probs = torch.rand(n_rel, generator=g, device=dev) * 0.8 + 0.1
    h = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    t = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    r = torch.randint(0, n_rel, (b,), generator=g, device=dev)
    lib = _lib.load()

    # ---- 1. the fused step per loss, at the ABI (forward; forward + backward with zeroed gradients)
    gent, grel = torch.zeros_like(ent), torch.zeros_like(rel)
    gl = torch.ones((), device=dev)
    loss_buf = torch.zeros((), device=dev)

    def args_for(kind, margin=1.0):
        a = _MarginStep._args(_lib.DISTMULT, dim, n_ent, margin, n_neg, h, t, r, None, None, probs, SEED, OFFSET,
                              [ent, None, rel, None], loss_buf, dev, kind)
        gr = _lib.Grads()
        gr.ent0, gr.rel0 = _ptr(gent), _ptr(grel)
        return a, gr

    def fwd(lib_, a):
        return lambda: _lib.check(lib_.kge_margin_step_fwd(ctypes.byref(a)), "kge_margin_step_fwd")

    def fwd_bwd(lib_, a, gr):
        def run():
            gent.zero_()
            grel.zero_()
            _lib.check(lib_.kge_margin_step_fwd(ctypes.byref(a)), "kge_margin_step_fwd")
            _lib.check(lib_.kge_margin_step_bwd(ctypes.byref(a), ctypes.byref(gr), _ptr(gl)), "kge_margin_step_bwd")
        return run

    kinds = {"margin": _lib.LOSS_MARGIN, "logistic": _lib.LOSS_LOGISTIC, "bce": _lib.LOSS_BCE}
    built = {k: args_for(v) for k, v in kinds.items()}
    fns = {}
    for k, (a, gr) in built.items():
        fns[k + "_fwd"] = fwd(lib, a)
        fns[k + "_fwd_bwd"] = fwd_bwd(lib, a, gr)
    res["fused_ms"] = timed(fns, args.reps, args.windows)
    for k, (a, _) in built.items():     # the loss of one call, for the record
        loss_buf.zero_()
        fwd(lib, a)()
        torch.cuda.synchronize()
        res.setdefault("fused_loss", {})[k] = loss_buf.item()
    hinge_frac = None
    with torch.no_grad():              # the share of active hinges of the margin step (every negative's row is
        nh = torch.empty(b * n_neg, dtype=torch.int64, device=dev)      # scattered by the other losses)
        nt = torch.empty_like(nh)
        _lib.check(lib.kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), b, n_neg, _ptr(probs), n_ent, SEED, OFFSET,
                                         _ptr(nh), _ptr(nt), _stream(dev)), "kge_corrupt_batch")
        model = tk.DistMultModel(dim, n_ent, n_rel).to(dev)
        model.ent_emb.weight.data.copy_(ent)
        model.rel_emb.weight.data.copy_(rel)
        pos, neg = model(h, t, r, nh, nt)
        hinge_frac = ((1.0 - pos + neg) > 0).float().mean().item()
        del pos, neg
    res["margin_active_hinge_fraction"] = hinge_frac

    # ---- 2. + 4. the three-call logistic path vs fused_loss_step through the public API
    crit = {"logistic": tk.LogisticLoss(), "bce": tk.BinaryCrossEntropyLoss()}

    def three_call(name, backward=True):
        model.zero_grad(set_to_none=True)
        nh_ = torch.empty(b * n_neg, dtype=torch.int64, device=dev)
        nt_ = torch.empty_like(nh_)
        _lib.check(lib.kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), b, n_neg, _ptr(probs), n_ent, SEED, OFFSET,
                                         _ptr(nh_), _ptr(nt_), _stream(dev)), "kge_corrupt_batch")
        loss = crit[name](*model(h, t, r, nh_, nt_))
        if backward:
            loss.backward()
        return loss

    def fused(name, backward=True):
        model.zero_grad(set_to_none=True)
        loss = fused_loss_step(model, h, t, r, crit[name], n_neg=n_neg, bern_probs=probs, seed=SEED, offset=OFFSET)
        if backward:
            loss.backward()
        return loss

    res["public_api_fwd_bwd_ms"] = timed({"logistic_three_call": lambda: three_call("logistic"),
                                          "logistic_fused": lambda: fused("logistic")}, args.reps, args.windows)
    agree = {}
    with torch.no_grad():              # float64 sum of the per-pair terms of the three-call scores
        pos, neg = (x.double() for x in model(h, t, r, nh, nt))
        exact = {"logistic": (torch.nn.functional.softplus(-pos) + torch.nn.functional.softplus(neg)).sum().item(),
                 "bce": (-torch.clamp(torch.log(torch.sigmoid(pos)), min=-100)
                         - torch.clamp(torch.log(1 - torch.sigmoid(neg)), min=-100)).sum().item()}
        del pos, neg
    for name in ("logistic", "bce"):
        a_, b_ = three_call(name, False).item(), fused(name, False).item()
        agree[name] = {"three_call": a_, "fused": b_, "float64_sum": exact[name],
                       "rel_diff": abs(a_ - b_) / max(abs(a_), 1e-30),
                       "three_call_rel_err_vs_float64": abs(a_ - exact[name]) / abs(exact[name]),
                       "fused_rel_err_vs_float64": abs(b_ - exact[name]) / abs(exact[name]),
                       "within_1e-5": abs(a_ - b_) <= 1e-5 * abs(a_)}
    res["fused_vs_three_call_loss"] = agree
    model.zero_grad(set_to_none=True)
    torch.cuda.empty_cache()

    # ---- 3. 8 emulated shards, logistic loss
    eng = CudaEngine()
    rows = torch.cat([ent[h], ent[t]]).view(2 * b, 1, dim).contiguous()
    hrows, trows = rows[:b], rows[b:]
    idx = torch.cat([h, t])
    per_rank, shard_loss = [], 0.0
    for rank in range(8):
        sh = EntityShard(n_ent, rank, 8)
        local = [ent[sh.lo:sh.hi], None, rel, None]
        step = ShardedStep(_lib.DISTMULT, dim, n_ent, sh.lo, sh.hi - sh.lo, n_neg, 0.0, SEED, OFFSET,
                           _lib.LOSS_LOGISTIC)
        lg = torch.zeros_like(local[0])
        lr_ = torch.zeros_like(rel)
        grows = torch.zeros_like(rows)

        def one():
            eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
            eng.margin_step_bwd(step, local, [lg, None, lr_, None], h, t, r, probs, gl, hrows, trows, grows[:b],
                                grows[b:])
            eng.scatter_rows_add(_lib.DISTMULT, dim, lg, None, sh.lo, idx, grows)

        per_rank.append(timed({"r": one}, args.reps, args.windows)["r"])
        shard_loss += eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows).item()
    res["logistic_8_emulated_shards"] = {
        "rank_ms": per_rank, "max_ms": max(per_rank), "sum_ms": sum(per_rank),
        "loss_sum_over_ranks": shard_loss,
        "rel_diff_vs_unsharded": abs(shard_loss - res["fused_loss"]["logistic"]) / abs(res["fused_loss"]["logistic"]),
        "note": "ranks run one after another on one GPU; collectives not run"}

    # ---- 5. the margin step against the parent commit's library, alternating
    if args.parent_lib:
        parent = ctypes.CDLL(os.path.abspath(args.parent_lib))
        parent.kge_margin_step_fwd.argtypes = [ctypes.POINTER(_lib.MarginStepArgs)]
        parent.kge_margin_step_bwd.argtypes = [ctypes.POINTER(_lib.MarginStepArgs), ctypes.POINTER(_lib.Grads),
                                               ctypes.c_void_p]
        parent.kge_last_error.restype = ctypes.c_char_p
        assert parent.kge_abi_version() == lib.kge_abi_version(), parent.kge_abi_version()
        a, gr = built["margin"]
        cmp_ = timed({"parent_fwd": fwd(parent, a), "this_fwd": fwd(lib, a),
                      "parent_fwd_bwd": fwd_bwd(parent, a, gr), "this_fwd_bwd": fwd_bwd(lib, a, gr)},
                     args.reps, max(args.windows, 7))
        loss_buf.zero_()
        fwd(parent, a)()
        torch.cuda.synchronize()
        cmp_["parent_margin_loss"] = loss_buf.item()
        cmp_["this_margin_loss"] = res["fused_loss"]["margin"]
        cmp_["fwd_bwd_ratio_this_over_parent"] = cmp_["this_fwd_bwd"] / cmp_["parent_fwd_bwd"]
        res["margin_vs_parent"] = cmp_
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
