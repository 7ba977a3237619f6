"""Sharded relation prediction probe: RelationPredictionEvaluator's relation scan (20,466 facts, 1k
relations, d = 200, filtered by dict_of_rels) unsharded, against the same facts over W = 8 emulated
ranks run one after another on one GPU -- the device work of rank_relation_prediction's sharded
branches, times W, without the collectives:
  entity-local  EntityShard(local_storage=True): each rank gathers the h / t rows it holds, the sum of
                those (what the all-reduce delivers) is every rank's row block, and each rank ranks its
                QueryShard slice of the facts;
  query         QueryShard (or EntityShard with full storage): each rank ranks its slice of the facts.
The scan time is the sum of the kge_rank_side calls (CUDA events); the bytes exchanged are the
payloads one rank hands the collectives (row all-reduce, rank all-gather), counted from shapes; the
ranks are compared with the unsharded evaluator's.  The card name and power limit are read in the
same run.

    python scripts/relpred_shard_perf.py [--out DIR] [n_ent] [n_facts] [shards]
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchkge_b200 as tk  # noqa: E402
from torchkge_b200 import _lib  # noqa: E402
from torchkge_b200.data import filter_csr  # noqa: E402
from torchkge_b200.engine import (EntityShard, ModelSpec, QueryShard, default_engine,  # noqa: E402
                                  relation_spec)

REPEATS = 5
N_REL, DIM = 1000, 200


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return "%s (%s)" % (name, q)


def scan(eng, spec, rspec, packed, h, t, r, csr, world, mode):
    """(rank, filt_rank, scan ms) of one pass; mode 'unsharded', 'entity-local' or 'query'."""
    dev = h.device
    n = h.shape[0]
    counters = torch.zeros((2, n), dtype=torch.int32, device=dev)
    if mode == "entity-local":
        rows = None
        idx = torch.cat([h, t])
        for rank in range(world):      # what the all-reduce of the gathered rows delivers
            sh = EntityShard(spec.n_ent, rank, world)
            part = eng.gather_rows(spec.narrowed(sh.lo, sh.hi), idx)
            rows = part if rows is None else rows + part
        hrows, trows = rows[:n], rows[n:]
    else:
        hrows, trows = eng.gather_rows(spec, h), eng.gather_rows(spec, t)
    rrows = eng.gather_rows(rspec, r)
    parts = [(0, n)] if mode == "unsharded" else [(q.lo, q.hi) for q in (QueryShard(n, k, world) for k in range(world))]
    offs = csr[0].tolist()
    slices = []
    for a, b in parts:                # the CSR slices (host work, outside the timed window)
        base = offs[a]
        slices.append(((csr[0][a:b + 1] - base).contiguous(), csr[1][base:offs[b]].contiguous()))
    keep = []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for (a, b), f in zip(parts, slices):
        if b > a:
            s_true = torch.empty(b - a, dtype=torch.float32, device=dev)
            keep.append(eng.rank_side(rspec, packed, _lib.SIDE_REL, hrows[a:b], trows[a:b], None, r[a:b], f,
                                      counters[0][a:b], counters[1][a:b], true_score=s_true, true_rows=rrows[a:b]))
            keep.append(s_true)
    ev1.record()
    torch.cuda.synchronize()
    ranks, filt = eng.finalize(counters[0], counters[1])
    return ranks.cpu(), filt.cpu(), ev0.elapsed_time(ev1)


def exchanged_bytes(mode, n, planes, world):
    """Payload one rank hands the collectives: the (2n, planes, dim) fp32 row all-reduce (entity-local)
    and the all-gather of two int64 rank vectors over ceil(n / W) facts."""
    if mode == "unsharded":
        return 0
    per = (n + world - 1) // world
    rows = 2 * n * planes * DIM * 4 if mode == "entity-local" else 0
    return rows + 2 * per * 8


def main():
    args = sys.argv[1:]
    out_dir = None
    if "--out" in args:
        i = args.index("--out")
        out_dir = args[i + 1]
        del args[i:i + 2]
    n_ent = int(args[0]) if len(args) > 0 else 100000
    n_facts = int(args[1]) if len(args) > 1 else 20466
    world = int(args[2]) if len(args) > 2 else 8
    dev = torch.device("cuda:0")
    lines = ["card: " + card()]
    print(lines[0], flush=True)
    eng = default_engine()
    g = torch.Generator().manual_seed(1)
    h = torch.randint(0, n_ent, (n_facts,), generator=g)
    t = torch.randint(0, n_ent, (n_facts,), generator=g)
    r = torch.randint(0, N_REL, (n_facts,), generator=g)
    dict_of_rels = {}
    for a, b, c in zip(h.tolist(), t.tolist(), r.tolist()):
        dict_of_rels.setdefault((a, b), set()).add(c)
    for i in range(0, n_facts, 5):          # filter sets of a few relations on every fifth pair
        dict_of_rels[(int(h[i]), int(t[i]))] |= set(torch.randint(0, N_REL, (4,), generator=g).tolist())
    kg = tk.KnowledgeGraph(h, t, r, n_ent, N_REL, dict_of_heads={}, dict_of_tails={})
    kg.dict_of_rels = dict_of_rels
    csr = tuple(x.to(dev) for x in filter_csr(dict_of_rels, h, t, r))
    h_d, t_d, r_d = h.to(dev), t.to(dev), r.to(dev)
    for name, cls, kw in (("TransE-L2", tk.TransEModel, {"dissimilarity_type": "L2"}),
                          ("DistMult", tk.DistMultModel, {}), ("ComplEx", tk.ComplExModel, {})):
        torch.manual_seed(0)
        model = cls(DIM, n_ent, N_REL, **kw).to(dev)
        ev = tk.RelationPredictionEvaluator(model, kg)
        ev.evaluate(b_size=256, verbose=False)
        spec = ModelSpec.from_model(model)
        rspec = relation_spec(spec)
        packed = eng.pack(rspec)
        modes = ("unsharded", "entity-local", "query")
        for mode in modes:                                  # warm-up
            scan(eng, spec, rspec, packed, h_d, t_d, r_d, csr, world, mode)
        ms = {m: [] for m in modes}
        same = {m: True for m in modes}
        for _ in range(REPEATS):                            # alternate the forms
            for mode in modes:
                ranks, filt, t_ms = scan(eng, spec, rspec, packed, h_d, t_d, r_d, csr, world, mode)
                ms[mode].append(t_ms)
                same[mode] &= bool(torch.equal(ranks, ev.rank_true_rels) and torch.equal(filt, ev.filt_rank_true_rels))
        med = lambda x: sorted(x)[len(x) // 2]   # noqa: E731
        for mode in modes:
            line = ("%-9s d=%d |R|=%d facts=%d %-12s W=%d: relation scan %.3f ms (sum of kge_rank_side, CUDA events, "
                    "median of %d) | bytes into collectives per rank %d | ranks == unsharded evaluator: %s"
                    % (name, DIM, N_REL, n_facts, mode, 1 if mode == "unsharded" else world, med(ms[mode]), REPEATS,
                       exchanged_bytes(mode, n_facts, spec.cand_planes, world), same[mode]))
            print(line, flush=True)
            lines.append(line)
        del model, ev, spec, rspec, packed
        torch.cuda.empty_cache()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "relpred_shard_perf.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
