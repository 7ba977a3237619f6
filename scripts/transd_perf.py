"""TransD evaluation timing: GPU wall time of ``LinkPredictionEvaluator.evaluate`` and
``RelationPredictionEvaluator.evaluate`` on a TransDModel at two synthetic shapes, at the first one the
unmodified reference's CPU evaluation on a sample of the facts when oracle/_ref holds it, and, in a separate
``torch.profiler`` run, the GPU time of link prediction split by kernel.

    python scripts/transd_perf.py [out_dir]   -> one JSON line per shape and one per profile
                                                 (also out_dir/transd_perf.jsonl when given)

Shapes: FB15k-like (14,951 entities, 1,345 relations, 20,466 test facts, widths 100 / 100) and 1M entities with
1,000 relations and 20,000 test facts at widths 200 / 200.  Facts are uniform at random, every relation gets
test facts; the filter sets are the test facts' own.  Each evaluator runs once to warm up, then is timed with
CUDA events around ``REPEATS`` calls (each ends with its ranks on the host); the median is reported.  The
card's name, power limit and maximum SM clock are printed with the numbers.  The profile groups the kernels of
one link-prediction call: the entity scalars, the per-relation projection, the table and query packing, the
rank scans (scalar and tensor-core, with their near-tie recheck) and the filter pass; the largest kernels outside
these groups are listed by name.
"""
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torchkge_b200 as tk  # noqa: E402

SHAPES = {"fb15k_like": (14_951, 1345, 20_466, 100, 100), "1m_entities": (1_000_000, 1000, 20_000, 200, 200)}
REPEATS = 3
REF_SAMPLE = 256       # facts the reference ranks at the first shape (its cost grows linearly with them)
#: kernel-name fragment -> group of the profile (first match wins; the rest is "other")
GROUPS = (("transd_scalars", "scalars"), ("transd_project", "projection"), ("pack", "pack"),
          ("row_norms", "pack"), ("block_max", "pack"), ("recheck", "scan"), ("scan", "scan"), ("filter", "filter"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def graph(n_ent, n_rel, n_test, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, n_ent, (n_test,), generator=g)
    t = torch.randint(0, n_ent, (n_test,), generator=g)
    r = torch.arange(n_test) % n_rel
    return h, t, r


def timed(fn):
    fn()
    times = []
    for _ in range(REPEATS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def kernel_split(fn):
    """({group: GPU ms}, {name: GPU ms} of the five largest kernels outside the groups) of one call of fn,
    from torch.profiler (its own run)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out, other = {}, {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if us <= 0:
            continue
        group = next((g for frag, g in GROUPS if frag in ev.key), "other")
        out[group] = out.get(group, 0.0) + us / 1e3
        if group == "other":
            other[ev.key[:80]] = round(us / 1e3, 3)
    top = dict(sorted(other.items(), key=lambda kv: -kv[1])[:5])
    return {k: round(v, 3) for k, v in sorted(out.items())}, top


def reference_sample(model, h, t, r, n_ent, n_rel):
    """Seconds of the reference's LinkPredictionEvaluator on REF_SAMPLE facts (its projection pass included),
    or None when oracle/_ref does not hold the reference."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchkge")):
        return None
    sys.path.insert(0, ref)
    from torchkge.data_structures import KnowledgeGraph
    from torchkge.evaluation import LinkPredictionEvaluator
    from torchkge.models import TransDModel
    m = TransDModel(model.ent_emb_dim, model.rel_emb_dim, n_ent, n_rel)
    m.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, strict=False)
    n = REF_SAMPLE
    kg = KnowledgeGraph(kg={"heads": h[:n], "tails": t[:n], "relations": r[:n]},
                        ent2ix={i: i for i in range(n_ent)}, rel2ix={i: i for i in range(n_rel)})
    t0 = time.perf_counter()
    LinkPredictionEvaluator(m, kg).evaluate(b_size=32, verbose=False)
    return time.perf_counter() - t0


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    dev = torch.device("cuda:0")
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    lines = []
    for name, (n_ent, n_rel, n_test, d, rd) in SHAPES.items():
        torch.manual_seed(0)
        model = tk.TransDModel(d, rd, n_ent, n_rel).to(dev)
        h, t, r = graph(n_ent, n_rel, n_test)
        kg = tk.KnowledgeGraph(h, t, r, n_ent, n_rel)
        lp = tk.LinkPredictionEvaluator(model, kg)
        rp = tk.RelationPredictionEvaluator(model, kg)
        res = {"shape": name, "n_ent": n_ent, "n_rel": n_rel, "n_test": n_test, "ent_dim": d, "rel_dim": rd,
               "card": info, "lp_ms": timed(lambda: lp.evaluate(b_size=1024)),
               "rp_ms": timed(lambda: rp.evaluate(b_size=1024)), "filt_mrr": lp.mrr()[1]}
        if name == "fb15k_like":
            try:
                s = reference_sample(model, h, t, r, n_ent, n_rel)
            except MemoryError:
                s = None
            res["reference_cpu_s_sample"] = s
            res["reference_sample_facts"] = REF_SAMPLE
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
        groups, other = kernel_split(lambda: lp.evaluate(b_size=1024))
        prof = {"shape": name, "card": info, "profile": "LinkPredictionEvaluator.evaluate, GPU ms by kernel group",
                "kernel_ms": groups, "largest_other_kernels_ms": other}
        lines.append(json.dumps(prof))
        print(lines[-1], flush=True)
        del model, lp, rp
        torch.cuda.empty_cache()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "transd_perf.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
