"""The fused training step and the element-wise losses of this tree against a library built from another
commit (the parent of a refactor of csrc/train.cu): same results, same speed.

    python scripts/train_vs_parent.py --parent-lib build/parent/libkge_b200.so [--out FILE.json]

Both libraries are loaded into one process and called at the C ABI with the same arguments.
1. Results, for TransE-L1, TransE-L2 and DistMult, on a C5-shaped step (d = 200, n_neg = 256: the ring
   kernel, or under KGE_TRAIN_RING=0 the register-resident one), on one n_neg whose ring block passes 96 KB
   (the register-resident kernel), for the three losses, and on an entity-sharded step: pos_out / neg_out
   must be bit-identical; the loss and the gradient tables are sums of float atomics whose order changes
   from run to run, so their difference is reported next to the difference of two runs of the parent.
2. kge_margin_loss_fwd / _bwd on 4M pairs, a quarter of them exact ties margin - pos + neg == 0.
3. Speed on the C5 shape (DistMult, B = 32,768): forward + backward per loss and sharded, windows of the two
   libraries alternating, and the same comparison between two copies of the parent, which shows the spread.
KGE_TRAIN_RING / KGE_TRAIN_BWD_BLOCKS are read once per process by both libraries: run the script again
under them to put the other kernels on the clock.  Records the GPU name and power limit.
"""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchkge_b200 import _lib, synthetic as S  # noqa: E402
from torchkge_b200.engine import _ptr, _stream  # noqa: E402
from torchkge_b200.training import _MarginStep  # noqa: E402

MODELS = {"transe_l1": _lib.TRANSE_L1, "transe_l2": _lib.TRANSE_L2, "distmult": _lib.DISTMULT}
LOSSES = {"margin": _lib.LOSS_MARGIN, "logistic": _lib.LOSS_LOGISTIC, "bce": _lib.LOSS_BCE}


def open_lib(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib.SIGNATURES.items():
        if hasattr(lib, name):
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def ok(lib, rc, what):
    if rc != 0:
        raise RuntimeError("%s: %s" % (what, lib.kge_last_error().decode(errors="replace")))


class Step:
    """One fused step's arguments and buffers; run(lib) gives loss, pos_out, neg_out and the gradients."""

    def __init__(self, dev, model, dim, n_ent, n_rel, b, n_neg, loss, shard=None, outs=True, seed=3):
        g = torch.Generator(device=dev).manual_seed(seed)
        tabs = S.make_tables(model, dim, n_ent, n_rel, 0, n_ent, 1, dev)
        self.ent, self.rel = tabs["ent0"].contiguous(), tabs["rel0"].contiguous()
        self.h = torch.randint(0, n_ent, (b,), generator=g, device=dev)
        self.t = torch.randint(0, n_ent, (b,), generator=g, device=dev)
        self.r = torch.randint(0, n_rel, (b,), generator=g, device=dev)
        self.probs = torch.rand(n_rel, generator=g, device=dev) * 0.8 + 0.1
        self.loss = torch.zeros((), device=dev)
        self.gl = torch.full((), 0.75, device=dev)
        local = self.ent
        if shard:                                   # rows [lo, hi) of the table, positives' rows exchanged
            lo, hi = shard
            local = self.ent[lo:hi].contiguous()
            self.hrows, self.trows = self.ent[self.h].contiguous(), self.ent[self.t].contiguous()
            self.ghrows, self.gtrows = torch.zeros_like(self.hrows), torch.zeros_like(self.trows)
        self.gent, self.grel = torch.zeros_like(local), torch.zeros_like(self.rel)
        a = _MarginStep._args(model, dim, n_ent, 1.0, n_neg, self.h, self.t, self.r, None, None, self.probs, 7, 1,
                              [local, None, self.rel, None], self.loss, dev, LOSSES[loss])
        if shard:
            a.ent_lo, a.n_rows = lo, hi - lo
            a.hrows, a.trows, a.grad_hrows, a.grad_trows = (_ptr(x) for x in (self.hrows, self.trows, self.ghrows,
                                                                              self.gtrows))
        elif outs:
            self.pos, self.neg = torch.zeros(b, device=dev), torch.zeros(b * n_neg, device=dev)
            a.pos_out, a.neg_out = _ptr(self.pos), _ptr(self.neg)
        self.a, self.shard, self.outs = a, shard, outs and not shard
        self.gr = _lib.Grads()
        self.gr.ent0, self.gr.rel0 = _ptr(self.gent), _ptr(self.grel)

    def fwd_bwd(self, lib):
        for x in (self.gent, self.grel) + ((self.ghrows, self.gtrows) if self.shard else ()):
            x.zero_()
        ok(lib, lib.kge_margin_step_fwd(ctypes.byref(self.a)), "kge_margin_step_fwd")
        ok(lib, lib.kge_margin_step_bwd(ctypes.byref(self.a), ctypes.byref(self.gr), _ptr(self.gl)),
           "kge_margin_step_bwd")

    def run(self, lib):
        self.loss.zero_()
        self.fwd_bwd(lib)
        torch.cuda.synchronize()
        out = {"loss": self.loss.double().clone(), "gent": self.gent.clone(), "grel": self.grel.clone()}
        if self.shard:
            out.update(ghrows=self.ghrows.clone(), gtrows=self.gtrows.clone())
        if self.outs:
            out.update(pos=self.pos.clone(), neg=self.neg.clone())
        return out


def rel_diff(x, y):
    return ((x - y).abs().max() / y.abs().max().clamp_min(1e-30)).item()


def compare(step, this, parent):
    p1, p2, n = step.run(parent), step.run(parent), step.run(this)
    res = {"bit_identical": {k: torch.equal(n[k], p1[k]) for k in ("pos", "neg") if k in n}}
    for k in n:
        if k not in ("pos", "neg"):   # max |difference| over the table's largest entry
            res[k] = {"this_vs_parent": rel_diff(n[k], p1[k]), "parent_vs_parent": rel_diff(p2[k], p1[k])}
    return res


def window(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def alternate(fns, reps, windows):
    for fn in fns.values():
        fn()
        fn()
    torch.cuda.synchronize()
    got = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            got[k].append(window(fn, reps))
    return {k: statistics.median(v) for k, v in got.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", required=True)
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--windows", type=int, default=9)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_vs_parent.py compares on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    this = _lib.load()
    parent = open_lib(args.parent_lib)
    with tempfile.TemporaryDirectory() as tmp:      # a second copy of the parent: what two equal libraries show
        parent2 = open_lib(shutil.copy(args.parent_lib, os.path.join(tmp, "libkge_parent2.so")))
    assert parent.kge_abi_version() == this.kge_abi_version()
    q = "name,power.limit,clocks.max.sm"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[:1]
    res = {"gpu": gpu, "env": {k: os.environ.get(k) for k in ("KGE_TRAIN_RING", "KGE_TRAIN_BWD_BLOCKS")}}
    c = S.C5
    dim, n_rel = c["dim"], c["n_rel"]

    # ---- 1. results
    par = {}
    for name, model in MODELS.items():
        par[name + " n_neg=256"] = compare(Step(dev, model, dim, 200000, n_rel, 4096, 256, "margin"), this, parent)
        par[name + " n_neg=4600 (ring block > 96 KB)"] = compare(
            Step(dev, model, dim, 200000, n_rel, 256, 4600, "margin"), this, parent)
        for loss in ("logistic", "bce"):
            par["%s %s" % (name, loss)] = compare(Step(dev, model, dim, 200000, n_rel, 2048, 256, loss), this, parent)
        par[name + " sharded logistic"] = compare(
            Step(dev, model, dim, 200000, n_rel, 2048, 256, "logistic", shard=(50000, 100000)), this, parent)
    res["results"] = par
    res["all_scores_bit_identical"] = all(all(v["bit_identical"].values()) for v in par.values())

    # ---- 2. the element-wise margin loss, with exact ties
    n = 1 << 22
    g = torch.Generator(device=dev).manual_seed(5)
    neg = torch.randint(-64, 64, (n,), generator=g, device=dev).float() / 8
    pos = torch.randint(-64, 64, (n,), generator=g, device=dev).float() / 8
    pos[::4] = neg[::4] + 1.0                      # margin - pos + neg == 0 exactly
    gl = torch.full((), 0.75, device=dev)
    got = {}
    for tag, lib in (("this", this), ("parent", parent), ("parent_again", parent)):
        loss, gp, gn = torch.zeros((), device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev)
        ok(lib, lib.kge_margin_loss_fwd(_ptr(pos), _ptr(neg), n, 1.0, _ptr(loss), _stream(dev)), "kge_margin_loss_fwd")
        ok(lib, lib.kge_margin_loss_bwd(_ptr(pos), _ptr(neg), n, 1.0, _ptr(gl), _ptr(gp), _ptr(gn), _stream(dev)),
           "kge_margin_loss_bwd")
        torch.cuda.synchronize()
        got[tag] = (loss.item(), gp, gn)
    res["margin_loss"] = {
        "ties": int((1.0 - pos + neg == 0).sum().item()),
        "grad_pos_equal": torch.equal(got["this"][1], got["parent"][1]),
        "grad_neg_equal": torch.equal(got["this"][2], got["parent"][2]),
        "loss_this": got["this"][0], "loss_parent": got["parent"][0], "loss_parent_again": got["parent_again"][0]}

    # ---- 3. speed, C5 shape
    speed = {}
    cases = [(k, Step(dev, _lib.DISTMULT, dim, c["n_ent"], n_rel, 32768, c["n_neg"], k, outs=False)) for k in LOSSES]
    cases.append(("sharded logistic, 1 of 8 shards", Step(dev, _lib.DISTMULT, dim, c["n_ent"], n_rel, 32768, c["n_neg"],
                                                          "logistic", shard=(0, c["n_ent"] // 8))))
    for k, st in cases:
        ms = alternate({"parent": lambda: st.fwd_bwd(parent), "this": lambda: st.fwd_bwd(this),
                        "parent_copy": lambda: st.fwd_bwd(parent2)}, args.reps, args.windows)
        ms["this_over_parent"] = ms["this"] / ms["parent"]
        ms["parent_copy_over_parent"] = ms["parent_copy"] / ms["parent"]
        speed[k + " fwd+bwd ms"] = ms
    res["speed"] = speed
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    return 0 if res["all_scores_bit_identical"] and res["margin_loss"]["grad_pos_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
