"""Data-redundancy golden vectors from the UNMODIFIED reference (torchkge v0.17.7,
torchkge/utils/data_redundancy.py).  Run with the reference on the path:

    PYTHONPATH=/root/reference python tests/golden/make_golden_redundancy.py

The reference compares ``combinations(range(1345), 2)`` and divides by every relation's length, so
the graph has exactly 1,345 relations, all non-empty.  Every relation starts with three facts on
entities no other relation uses (no overlap, Cartesian ratio 1/3), except the planted ones:

  duplicates      10/11 share 17 of 21 pairs (17/21 > 0.8), 20/21 share 4 of 5 (exactly 0.8: out),
                  30/31 share 7 of 10 (below), 40/41 one-sided (5 of 5 against 5 of 10),
                  50/51 equal sets but 50's facts all doubled (5/10), 52/53 equal sets, one fact of 52
                  doubled (5/6 > 0.8)
  reverses        61 is 60 reversed; 62 holds 8 of 63's 10 pairs reversed and 2 others (exactly 0.8)
  symmetric       70 holds (a, b) and (b, a), 71 is a copy: duplicate and reverse duplicate
  self-loops      80 and 81 the same six self-loops (both lists); 82 five of them and one of its own
  Cartesian       90: all 2x2 head/tail pairs (1.0); 91: 8 of 2x5 (exactly 0.8: out); 92: 10 of 3x4
                  (0.833); 93: all 2x2 pairs twice (2.0); 94: 3 of 2x2 plus one repeat (4/4)

The facts are shuffled and split 70/15/15 into train / validation / test.  Recorded: ``duplicates``
at the default and at (0.6, 0.5) thresholds, with ``reverses = [(60, 61)]`` and with the list of lists
``[[80, 81]]`` (not excluded: a list is not equal to a tuple), ``count_triplets`` on (train, test) and
(test, test) with the first pair of each list listed twice plus out-of-range pairs,
``cartesian_product_relations`` at 0.8 and 0.5, and the stdout of ``duplicates(..., verbose=True,
counts=True)``.  Output: tests/golden/redundancy.npz.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

sys.path.insert(0, "/root/reference")
from torchkge.data_structures import KnowledgeGraph  # noqa: E402
from torchkge.utils import cartesian_product_relations, count_triplets, duplicates  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "redundancy.npz")
N_REL = 1345
THETAS = [(0.8, 0.8), (0.6, 0.5)]
REVERSES = {"none": None, "tuple": [(60, 61)], "list": [[80, 81]]}
CART_THETAS = [0.8, 0.5]


def planted_facts():
    facts = []
    nxt = [0]

    def fresh(k):
        nxt[0] += k
        return list(range(nxt[0] - k, nxt[0]))

    def pairs(k):
        e = fresh(2 * k)
        return [(e[i], e[k + i]) for i in range(k)]

    planted = {10, 11, 20, 21, 30, 31, 40, 41, 50, 51, 52, 53, 60, 61, 62, 63, 70, 71, 80, 81, 82,
               90, 91, 92, 93, 94}
    for r in range(N_REL):                       # the background: three disjoint facts per relation
        if r not in planted:
            facts += [(h, t, r) for h, t in pairs(3)]
    common = pairs(17)
    facts += [(h, t, 10) for h, t in common + pairs(4)] + [(h, t, 11) for h, t in common + pairs(4)]
    common = pairs(4)
    facts += [(h, t, 20) for h, t in common + pairs(1)] + [(h, t, 21) for h, t in common + pairs(1)]
    common = pairs(7)
    facts += [(h, t, 30) for h, t in common + pairs(3)] + [(h, t, 31) for h, t in common + pairs(3)]
    common = pairs(5)
    facts += [(h, t, 40) for h, t in common] + [(h, t, 41) for h, t in common + pairs(5)]
    common = pairs(5)
    facts += [(h, t, 50) for h, t in common + common] + [(h, t, 51) for h, t in common]
    common = pairs(5)
    facts += [(h, t, 52) for h, t in common + common[:1]] + [(h, t, 53) for h, t in common]
    base = pairs(6)
    facts += [(h, t, 60) for h, t in base] + [(t, h, 61) for h, t in base]
    base = pairs(10)
    facts += [(h, t, 63) for h, t in base] + [(t, h, 62) for h, t in base[:8]] + [(h, t, 62) for h, t in pairs(2)]
    base = pairs(4)
    sym = base + [(t, h) for h, t in base]
    facts += [(h, t, 70) for h, t in sym] + [(h, t, 71) for h, t in sym]
    loops = [(e, e) for e in fresh(6)]
    facts += [(h, t, 80) for h, t in loops] + [(h, t, 81) for h, t in loops]
    facts += [(h, t, 82) for h, t in loops[:5] + [(e, e) for e in fresh(1)]]
    hs, ts = fresh(2), fresh(2)
    facts += [(h, t, 90) for h in hs for t in ts]
    hs, ts = fresh(2), fresh(5)
    facts += [(h, t, 91) for h in hs for t in ts][:8]
    hs, ts = fresh(3), fresh(4)
    facts += [(h, t, 92) for h in hs for t in ts][:10]
    hs, ts = fresh(2), fresh(2)
    facts += [(h, t, 93) for h in hs for t in ts] * 2
    hs, ts = fresh(2), fresh(2)
    f94 = [(h, t, 94) for h in hs for t in ts][:3]
    facts += f94 + f94[:1]
    assert {f[2] for f in facts} == set(range(N_REL))
    return facts, nxt[0]


def graphs():
    facts, n_ent = planted_facts()
    g = torch.Generator().manual_seed(0)
    arr = torch.tensor(facts, dtype=torch.int64)[torch.randperm(len(facts), generator=g)]
    n_tr, n_val = int(0.7 * len(arr)), int(0.15 * len(arr))
    parts = (arr[:n_tr], arr[n_tr:n_tr + n_val], arr[n_tr + n_val:])
    ent2ix = {i: i for i in range(n_ent)}
    rel2ix = {i: i for i in range(N_REL)}
    kgs = [KnowledgeGraph(kg={"heads": p[:, 0].clone(), "tails": p[:, 1].clone(), "relations": p[:, 2].clone()},
                          ent2ix=ent2ix, rel2ix=rel2ix) for p in parts]
    return parts, n_ent, kgs


def main():
    parts, n_ent, (tr, va, te) = graphs()
    out = {"n_ent": n_ent, "n_rel": N_REL}
    for name, p in zip(("tr", "val", "te"), parts):
        out["facts_" + name] = p.numpy()
    for i, (t1, t2) in enumerate(THETAS):
        for tag, rev in REVERSES.items():
            d, rd = duplicates(tr, va, te, theta1=t1, theta2=t2, reverses=rev)
            out["dup_%d_%s" % (i, tag)] = np.array(d, dtype=np.int64).reshape(-1, 2)
            out["rev_%d_%s" % (i, tag)] = np.array(rd, dtype=np.int64).reshape(-1, 2)
    d, rd = (out["dup_0_none"].tolist(), out["rev_0_none"].tolist())
    d_listed = [tuple(x) for x in d] + [tuple(d[0]), (5000, 3), (-1, 10)]
    rd_listed = [tuple(x) for x in rd] + [tuple(rd[0]), (3, 5000)]
    out["count_dup_listed"] = np.array(d_listed, dtype=np.int64)
    out["count_rev_listed"] = np.array(rd_listed, dtype=np.int64)
    out["count_tr_te"] = np.array(count_triplets(tr, te, d_listed, rd_listed), dtype=np.int64)
    out["count_te_te"] = np.array(count_triplets(te, te, d_listed, rd_listed), dtype=np.int64)
    for i, th in enumerate(CART_THETAS):
        out["cart_%d" % i] = np.array(cartesian_product_relations(tr, va, te, theta=th), dtype=np.int64)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        duplicates(tr, va, te, verbose=True, counts=True)
    out["stdout"] = np.array(buf.getvalue())
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")
    for k in sorted(out):
        if k.startswith(("dup_", "rev_", "cart_", "count_")):
            print(k, out[k].tolist())
    print(buf.getvalue())


if __name__ == "__main__":
    main()
