"""Data-redundancy timing: GPU wall time of ``duplicates``, ``cartesian_product_relations`` and
``count_triplets`` (torchkge_b200.data_redundancy) at two synthetic shapes, and at the first one the
unmodified reference on the host cores when oracle/_ref holds it.

    python scripts/redundancy_perf.py [out_dir]   -> one JSON line per shape (also out_dir/redundancy_perf.jsonl)

Shapes: FB15k-like (592,213 facts, 14,951 entities, 1,345 relations, every relation non-empty) and
Wikidata5M-like (21M facts, 4.6M entities, 822 relations).  Facts are uniform at random with a planted
share (10%) of copied and reversed relation pairs, split 90/5/5 into train / validation / test; the inputs
are CPU tensors, as in a KnowledgeGraph, so each time includes the copy to the device.  Each function is
run once to warm up (``count_triplets`` on the (r, r + 1) pairs the copies went to), then timed over ``REPEATS`` calls with a device synchronise at the end of each; the
median is reported.  The card's name and power limit are printed with the numbers.
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
from torchkge_b200 import data_redundancy as dr  # noqa: E402

SHAPES = {"fb15k_like": (592_213, 14_951, 1345), "wikidata5m_like": (21_000_000, 4_600_000, 822)}
REPEATS = 5


class Graph:
    """The attributes of a KnowledgeGraph the analysis reads."""

    def __init__(self, h, t, r, n_ent, n_rel):
        self.head_idx, self.tail_idx, self.relations, self.n_ent, self.n_rel = h, t, r, n_ent, n_rel

    def __len__(self):
        return self.head_idx.shape[0]


def make_graphs(n_facts, n_ent, n_rel, seed=0):
    g = torch.Generator().manual_seed(seed)
    n_copy = n_facts // 10
    n_base = n_facts - n_copy
    h = torch.randint(0, n_ent, (n_base,), generator=g)
    t = torch.randint(0, n_ent, (n_base,), generator=g)
    r = torch.arange(n_base) % n_rel       # every relation non-empty
    src = torch.randint(0, n_base, (n_copy,), generator=g)
    flip = torch.rand(n_copy, generator=g) < 0.5
    ch, ct = torch.where(flip, t[src], h[src]), torch.where(flip, h[src], t[src])
    cr = (r[src] + 1) % n_rel                # relation r's copies go to r + 1
    h, t, r = torch.cat([h, ch]), torch.cat([t, ct]), torch.cat([r, cr])
    perm = torch.randperm(n_facts, generator=g)
    h, t, r = h[perm], t[perm], r[perm]
    a, b = int(0.9 * n_facts), int(0.95 * n_facts)
    return [Graph(h[x:y], t[x:y], r[x:y], n_ent, n_rel) for x, y in ((0, a), (a, b), (b, n_facts))]


def timed(fn):
    fn()
    times = []
    for _ in range(REPEATS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return statistics.median(times), out


def reference_run(kgs):
    """{function: (seconds, result)} of the unmodified reference, one call each, or None."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "torchkge")):
        return None
    sys.path.insert(0, ref)
    from torchkge.utils import data_redundancy as ref_dr
    ref_dr.tqdm = lambda it, *a, **k: it       # progress bars off; the loops are unchanged
    out = {}
    for name, fn in (("duplicates", ref_dr.duplicates), ("cartesian_product_relations",
                                                        ref_dr.cartesian_product_relations)):
        t0 = time.perf_counter()
        res = fn(*kgs)
        out[name] = (time.perf_counter() - t0, res)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    if not torch.cuda.is_available():
        raise SystemExit("redundancy_perf: needs a CUDA device")
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    lines = []
    for shape, (n_facts, n_ent, n_rel) in SHAPES.items():
        kgs = make_graphs(n_facts, n_ent, n_rel)
        t_dup, (d, rd) = timed(lambda: dr.duplicates(*kgs))
        t_cart, cart = timed(lambda: dr.cartesian_product_relations(*kgs))
        planted = [(r, r + 1) for r in range(n_rel - 1)]       # where the copies went
        t_cnt, cnt = timed(lambda: dr.count_triplets(kgs[0], kgs[2], planted, planted))
        rec = {"shape": shape, "n_facts": n_facts, "n_ent": n_ent, "n_rel": n_rel, "gpu": card(),
               "duplicates_s": round(t_dup, 4), "cartesian_product_relations_s": round(t_cart, 4),
               "count_triplets_s": round(t_cnt, 4), "n_duplicates": len(d), "n_rev_duplicates": len(rd),
               "n_cartesian": len(cart), "count_train_test_planted": list(cnt), "peak_gpu_bytes": torch.cuda.max_memory_allocated()}
        if shape == "fb15k_like":
            ref = reference_run(kgs)
            rec["host_cores"] = os.cpu_count()
            rec["reference_s"] = None if ref is None else {k: round(v[0], 2) for k, v in ref.items()}
            if ref is not None:
                rec["equal_to_reference"] = (ref["duplicates"][1] == (d, rd)
                                             and ref["cartesian_product_relations"][1] == cart)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
        torch.cuda.reset_peak_memory_stats()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "redundancy_perf.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
