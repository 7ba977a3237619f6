"""Sharded top-k inference probe: EntityInference (k = 10, 20,466 queries, |E| = 1M, d = 200) unsharded,
against the same queries over 8 emulated entity shards run one after another on one GPU (per shard
kge_topk_side with global ids, then one kge_topk_merge per chunk of queries -- the device work of
one rank of topk_entity_inference, times 8, without the collectives).  Scan and merge times come
from CUDA events; the card name and power limit are read in the same run.  The sharded results are
checked against the unsharded ones (ids and score bits).

    python scripts/topk_shard_perf.py [--out DIR] [n_ent] [n_queries] [k] [shards]
"""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchkge_b200 as tk  # noqa: E402
from torchkge_b200 import _lib  # noqa: E402
from torchkge_b200.engine import TOPK_CHUNK, EntityShard, ModelSpec, default_engine  # noqa: E402

REPEATS = 3


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return "%s (%s)" % (name, q)


def sharded_once(eng, spec, packs, ents, rels, k, world):
    """(pred, scores, scan ms, merge ms) of one pass over all queries with `world` emulated shards."""
    dev = spec.ent0.device
    n = ents.shape[0]
    pred = torch.empty((n, k), dtype=torch.int64, device=dev)
    vals = torch.empty((n, k), dtype=torch.float32, device=dev)
    scan_ms = merge_ms = 0.0
    for lo in range(0, n, TOPK_CHUNK):
        hi = min(n, lo + TOPK_CHUNK)
        rows = eng.gather_rows(spec, ents[lo:hi])
        r = rels[lo:hi].contiguous()
        pred_in = torch.full((world, hi - lo, k), -1, dtype=torch.int64, device=dev)
        scores_in = torch.full((world, hi - lo, k), float("-inf"), dtype=torch.float32, device=dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        for rank, (sub, packed) in enumerate(packs):
            k_loc = min(k, sub.n_rows)
            pred_in[rank, :, :k_loc], scores_in[rank, :, :k_loc] = eng.topk_side(
                sub, packed, _lib.SIDE_TAIL, rows, rows, r, k_loc)
        ev[1].record()
        pred[lo:hi], vals[lo:hi] = eng.topk_merge(pred_in, scores_in, k)
        ev[2].record()
        torch.cuda.synchronize()
        scan_ms += ev[0].elapsed_time(ev[1])
        merge_ms += ev[1].elapsed_time(ev[2])
    return pred, vals, scan_ms, merge_ms


def unsharded_scan_ms(eng, spec, packed, ents, rels, k):
    """CUDA-event time of the unsharded kge_topk_side calls over all queries (same chunks)."""
    ms = 0.0
    for lo in range(0, ents.shape[0], TOPK_CHUNK):
        hi = min(ents.shape[0], lo + TOPK_CHUNK)
        rows = eng.gather_rows(spec, ents[lo:hi])
        r = rels[lo:hi].contiguous()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.topk_side(spec, packed, _lib.SIDE_TAIL, rows, rows, r, k)
        b.record()
        torch.cuda.synchronize()
        ms += a.elapsed_time(b)
    return ms


def main():
    args = sys.argv[1:]
    out_dir = None
    if "--out" in args:
        i = args.index("--out")
        out_dir = args[i + 1]
        del args[i:i + 2]
    n_ent = int(args[0]) if len(args) > 0 else 1000000
    n_q = int(args[1]) if len(args) > 1 else 20466
    k = int(args[2]) if len(args) > 2 else 10
    world = int(args[3]) if len(args) > 3 else 8
    dev = torch.device("cuda:0")
    lines = ["card: " + card()]
    print(lines[0], flush=True)
    eng = default_engine()
    for name, cls, d, kw in (("TransE-L2", tk.TransEModel, 200, {"dissimilarity_type": "L2"}),
                             ("DistMult", tk.DistMultModel, 200, {})):
        torch.manual_seed(0)
        model = cls(d, n_ent, 1000, **kw).to(dev)
        g = torch.Generator().manual_seed(1)
        ents = torch.randint(0, n_ent, (n_q,), generator=g)
        rels = torch.randint(0, 1000, (n_q,), generator=g)
        inf = tk.EntityInference(model, ents, rels, top_k=k, missing="tails")
        inf.evaluate(b_size=256, verbose=False)          # warm-up
        spec = ModelSpec.from_model(model)
        e_d, r_d = ents.to(dev), rels.to(dev)
        packed_full = eng.pack(spec)
        unsharded_scan_ms(eng, spec, packed_full, e_d, r_d, k)   # warm-up
        packs = []
        for rank in range(world):
            sh = EntityShard(n_ent, rank, world)
            sub = spec.narrowed(sh.lo, sh.hi)
            packs.append((sub, eng.pack(sub)))
        sharded_once(eng, spec, packs, e_d, r_d, k, world)   # warm-up
        full_ms, full_scan_ms, scan_ms, merge_ms = [], [], [], []
        same = True
        for _ in range(REPEATS):                         # alternate the two forms
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inf.evaluate(b_size=256, verbose=False)
            torch.cuda.synchronize()
            full_ms.append((time.perf_counter() - t0) * 1e3)
            full_scan_ms.append(unsharded_scan_ms(eng, spec, packed_full, e_d, r_d, k))
            pred, vals, s_ms, m_ms = sharded_once(eng, spec, packs, e_d, r_d, k, world)
            scan_ms.append(s_ms)
            merge_ms.append(m_ms)
            same &= bool(torch.equal(pred.cpu(), inf.predictions)
                         and torch.equal(vals.cpu().view(torch.int32), inf.scores.view(torch.int32)))
        med = lambda x: sorted(x)[len(x) // 2]   # noqa: E731
        line = ("%-9s d=%d |E|=%d queries=%d k=%d: unsharded EntityInference.evaluate %.1f ms (host clock, incl. "
                "packing and copies), its kge_topk_side calls %.1f ms (CUDA events) | %d emulated shards, sum of the "
                "shards' kge_topk_side %.1f ms + kge_topk_merge %.3f ms (CUDA events) | medians of %d | "
                "sharded == unsharded (ids, score bits): %s"
                % (name, d, n_ent, n_q, k, med(full_ms), med(full_scan_ms), world, med(scan_ms), med(merge_ms),
                   REPEATS, same))
        print(line, flush=True)
        lines.append(line)
        del model, inf, packs, spec, packed_full
        torch.cuda.empty_cache()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "topk_shard_perf.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
