"""Single-GPU cost of positional negatives in the fused training step (DESIGN.md section 4.4).

    python scripts/pos_step_perf.py [--out FILE.json] [--reps N] [--windows N]

C5 shape: DistMult d=200, 1M entities, 1000 relations, B = 32,768, n_neg = 256, MarginLoss(1.0), on a
synthetic training graph of --facts facts over those tables.  Forward + backward (ms, CUDA events, median of
--windows windows of --reps steps after warm-up, the variants alternated window by window in one process) of
BernoulliNegativeSampler.fused_step, PositionalNegativeSampler.fused_step and
BernoulliRelationNegativeSampler.fused_step at rel_share 0.33.  Positional negatives come from a few
candidates per relation, so the backward's atomics land on fewer rows than with uniform entities.  Prints
the graph's size and the number of CSR entries, and the GPU name, power limit and SM clock of the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torchkge_b200 as tk  # noqa: E402


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:      # measurement still valid, the facts are then missing
        return {"error": str(e)}


class _KG:
    """What the samplers read of a graph: sizes and the facts (for bern_probs)."""

    def __init__(self, n_ent, n_rel, h, t, r):
        self.n_ent, self.n_rel, self.n_facts = n_ent, n_rel, h.shape[0]
        self.head_idx, self.tail_idx, self.relations = h, t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--n-ent", type=int, default=1_000_000)
    ap.add_argument("--n-rel", type=int, default=1000)
    ap.add_argument("--dim", type=int, default=200)
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--n-neg", type=int, default=256)
    ap.add_argument("--facts", type=int, default=1_000_000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pos_step_perf.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    facts = args.facts
    h, t = torch.randint(0, args.n_ent, (facts,), generator=g), torch.randint(0, args.n_ent, (facts,), generator=g)
    r = torch.randint(0, args.n_rel, (facts,), generator=g)
    kg = _KG(args.n_ent, args.n_rel, h, t, r)
    torch.manual_seed(0)
    model = tk.DistMultModel(args.dim, args.n_ent, args.n_rel).to(dev)
    hb, tb, rb = h[:args.batch].to(dev), t[:args.batch].to(dev), r[:args.batch].to(dev)
    positional = tk.PositionalNegativeSampler(kg, seed=1)
    csr_entries = {"heads": int(positional._csr["heads"][1].numel()), "tails": int(positional._csr["tails"][1].numel())}
    samplers = {"entity": tk.BernoulliNegativeSampler(kg, seed=1),
                "positional": positional,
                "relation_share_0.33": tk.BernoulliRelationNegativeSampler(kg, rel_share=0.33, seed=1)}

    def step(s):
        model.zero_grad(set_to_none=True)
        s.fused_step(model, hb, tb, rb, margin=1.0, n_neg=args.n_neg).backward()

    res = {name: [] for name in samplers}
    for s in samplers.values():          # warm-up
        for _ in range(2):
            step(s)
    torch.cuda.synchronize()
    for _ in range(args.windows):        # alternate the variants window by window
        for name, s in samplers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                step(s)
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / args.reps)
    out = {"gpu": gpu_facts(), "shape": vars(args), "graph_facts": facts, "csr_entries": csr_entries,
           "fwd_bwd_ms_median": {k: statistics.median(v) for k, v in res.items()},
           "fwd_bwd_ms_windows": res}
    out["ratio_positional_vs_entity"] = out["fwd_bwd_ms_median"]["positional"] / out["fwd_bwd_ms_median"]["entity"]
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
