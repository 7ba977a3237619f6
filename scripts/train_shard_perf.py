"""Single-GPU measurements of the entity-sharded fused margin step (DESIGN.md section 4.4).

    python scripts/train_shard_perf.py [--out FILE.json] [--reps N]

1. C5 shape (DistMult d=200, 1M entities, 1000 relations, B = 32,768, n_neg = 256): the unsharded fused
   forward + backward, then, for W in {2, 4, 8}, every emulated rank's sharded forward + backward kernels
   (engine.margin_step_fwd / _bwd / scatter_rows_add on its row range), timed with CUDA events one rank
   after the other: the maximum over the ranks (what a W-GPU step would wait for in its kernels) and the
   sum.  Collectives are not run here; the bytes they would carry per step are computed from the shapes.
2. One rank of an 8-way C4 shard (RotatE d=1000, 625,000 local rows of 5M, two planes, random positive
   rows, n_neg = 256, B = 8192): time and peak memory of its sharded forward + backward.
Records the GPU name, power limit and SM clock next to the numbers.  No multi-GPU time is measured.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchkge_b200 import _lib, synthetic as S  # noqa: E402
from torchkge_b200.engine import CudaEngine, EntityShard  # noqa: E402
from torchkge_b200.training import ShardedStep, _MarginStep  # noqa: E402


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:      # measurement still valid, the facts are then missing
        return {"error": str(e)}


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def c5(reps, dev, eng):
    c = S.C5
    dim, n_ent, n_rel, n_neg, b = c["dim"], c["n_ent"], c["n_rel"], c["n_neg"], 32768
    tabs = S.make_tables(_lib.DISTMULT, dim, n_ent, n_rel, 0, n_ent, 1, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    probs = torch.rand(n_rel, generator=g, device=dev) * 0.8 + 0.1
    h = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    t = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    r = torch.randint(0, n_rel, (b,), generator=g, device=dev)
    ent = tabs["ent0"].requires_grad_(True)
    rel = tabs["rel0"].requires_grad_(True)

    def unsharded():
        ent.grad = rel.grad = None
        _MarginStep.apply(_lib.DISTMULT, dim, n_ent, 1.0, n_neg, h, t, r, None, None, probs, 7, 1,
                          ent, None, rel, None).backward()

    out = {"shape": "DistMult d=%d, %d entities, %d relations, B=%d, n_neg=%d" % (dim, n_ent, n_rel, b, n_neg),
           "unsharded_fwd_bwd_ms": timed(unsharded, reps)}
    ent.grad = rel.grad = None
    rows = torch.cat([ent.detach()[h], ent.detach()[t]]).view(2 * b, 1, dim).contiguous()
    hrows, trows = rows[:b], rows[b:]
    idx = torch.cat([h, t])
    for world in (2, 4, 8):
        per_rank = []
        for rank in range(world):
            sh = EntityShard(n_ent, rank, world)
            n = sh.hi - sh.lo
            local = [ent.detach()[sh.lo:sh.hi], None, rel.detach(), None]
            step = ShardedStep(_lib.DISTMULT, dim, n_ent, sh.lo, n, n_neg, 1.0, 7, 1)
            gent = torch.zeros_like(local[0])
            grel = torch.zeros_like(rel)
            grows = torch.zeros_like(rows)
            gl = torch.ones((), device=dev)

            def one():
                eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
                eng.margin_step_bwd(step, local, [gent, None, grel, None], h, t, r, probs, gl, hrows, trows,
                                    grows[:b], grows[b:])
                eng.scatter_rows_add(_lib.DISTMULT, dim, gent, None, sh.lo, idx, grows)

            per_rank.append(timed(one, reps))
        planes = 1
        fwd_bytes = 2 * b * planes * dim * 4
        out["W=%d" % world] = {
            "rank_ms": per_rank, "max_ms": max(per_rank), "sum_ms": sum(per_rank),
            "bytes_forward_allreduce": fwd_bytes,
            "bytes_backward_allreduce": fwd_bytes + n_rel * dim * 4,
            "bytes_loss_allreduce": 4}
    del tabs, ent, rel
    torch.cuda.empty_cache()
    return out


def c4_rank(reps, dev, eng, b=8192):
    wl = S.WORKLOADS["c4"]
    dim, n_ent, n_rel, n_neg, world = wl["dim"], wl["n_ent"], wl["n_rel"], 256, 8
    sh = EntityShard(n_ent, 0, world)
    torch.cuda.reset_peak_memory_stats()
    tabs = S.make_tables(_lib.ROTATE, dim, n_ent, n_rel, sh.lo, sh.hi, 1, dev)
    g = torch.Generator(device=dev).manual_seed(2)
    probs = torch.rand(n_rel, generator=g, device=dev) * 0.8 + 0.1
    h = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    t = torch.randint(0, n_ent, (b,), generator=g, device=dev)
    r = torch.randint(0, n_rel, (b,), generator=g, device=dev)
    rows = torch.randn(2 * b, 2, dim, generator=g, device=dev) * 0.05     # random positive rows
    hrows, trows = rows[:b], rows[b:]
    local = [tabs["ent0"], tabs["ent1"], tabs["rel0"], tabs["rel1"]]
    grads = [torch.zeros_like(x) for x in local]
    grows = torch.zeros_like(rows)
    gl = torch.ones((), device=dev)
    step = ShardedStep(_lib.ROTATE, dim, n_ent, sh.lo, sh.hi - sh.lo, n_neg, 1.0, 7, 1)
    idx = torch.cat([h, t])

    def one():
        eng.margin_step_fwd(step, local, h, t, r, probs, hrows, trows)
        eng.margin_step_bwd(step, local, grads, h, t, r, probs, gl, hrows, trows, grows[:b], grows[b:])
        eng.scatter_rows_add(_lib.ROTATE, dim, grads[0], grads[1], sh.lo, idx, grows)

    ms = timed(one, reps, warm=1)
    return {"shape": "RotatE d=%d, rank 0 of 8: %d local rows of %d, two planes, B=%d, n_neg=%d"
                     % (dim, sh.hi - sh.lo, n_ent, b, n_neg),
            "fwd_bwd_scatter_ms": ms, "peak_memory_GB": torch.cuda.max_memory_allocated() / 1e9,
            "table_plus_gradient_GB": 2 * sum(x.numel() for x in local[:2]) * 4 / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    eng = CudaEngine()
    res = {"gpu": gpu_facts(), "c5": c5(args.reps, dev, eng), "c4_rank_of_8": c4_rank(max(1, args.reps // 2), dev, eng),
           "note": "single GPU, emulated ranks run one after another; collectives not run; multi-GPU not measured"}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
