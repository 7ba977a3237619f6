"""TransD golden vectors from the UNMODIFIED reference (torchkge v0.17.7):

    python tests/golden/make_golden_transd.py [torchkge source tree; default: oracle/_ref]

Writes transd_toy.npz and transd_syn.npz, each with the weights of a reference TransDModel (seeded), the
facts, and the reference's outputs on them:
  * LinkPredictionEvaluator (evaluation.py:207-425): the four rank vectors
  * RelationPredictionEvaluator (evaluation.py:16-204): raw and filtered ranks, directed and undirected
  * scoring_function (translation.py:538-568) on the test facts and on fixed negatives
  * the gradients of MarginLoss(margin=1) of model(h, t, r, nh, nt) with respect to ent_emb, rel_emb,
    ent_proj_vect and rel_proj_vect
The toy case has rel_emb_dim < ent_emb_dim, the synthetic one equal widths.  The synthetic case gets two
duplicated entities (both tables) and one ent_emb row of -0.0 (exact ties in every projection); in both the
last relation has no fact.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "oracle", "_ref")
if not os.path.isdir(os.path.join(REF, "torchkge")):
    sys.exit("make_golden_transd: no torchkge package under %s (pass the reference's source tree)" % REF)
sys.path.insert(0, REF)
from torchkge.data_structures import KnowledgeGraph  # noqa: E402
from torchkge.evaluation import LinkPredictionEvaluator, RelationPredictionEvaluator  # noqa: E402
from torchkge.models import TransDModel  # noqa: E402
from torchkge.utils import MarginLoss  # noqa: E402

sys.path.insert(0, HERE)
from make_golden import dicts_to_arrays  # noqa: E402

CASES = {  # name: (n_ent, n_rel, ent_dim, rel_dim, n_facts, n_test, b_size, seed)
    "toy": (40, 5, 10, 7, 120, 30, 7, 13),
    "syn": (400, 24, 40, 40, 3000, 200, 64, 14),
}


def make(name):
    n_ent, n_rel, d, rd, n_facts, n_test, b_size, seed = CASES[name]
    torch.manual_seed(seed)
    model = TransDModel(d, rd, n_ent, n_rel)
    if name == "syn":
        with torch.no_grad():
            for table in (model.ent_emb.weight, model.ent_proj_vect.weight):
                table[7] = table[3]
                table[250] = table[3]
            model.ent_emb.weight[11] = -0.0
    g = torch.Generator().manual_seed(seed)
    heads = torch.randint(0, n_ent, (n_facts,), generator=g)
    tails = torch.randint(0, n_ent, (n_facts,), generator=g)
    rels = torch.randint(0, n_rel - 1, (n_facts,), generator=g)      # relation n_rel - 1 has no fact
    ent2ix = {i: i for i in range(n_ent)}
    rel2ix = {i: i for i in range(n_rel)}
    full = KnowledgeGraph(kg={"heads": heads, "tails": tails, "relations": rels}, ent2ix=ent2ix, rel2ix=rel2ix)
    th, tt, tr = heads[:n_test], tails[:n_test], rels[:n_test]
    test = KnowledgeGraph(kg={"heads": th, "tails": tt, "relations": tr}, ent2ix=ent2ix, rel2ix=rel2ix,
                          dict_of_heads=full.dict_of_heads, dict_of_tails=full.dict_of_tails,
                          dict_of_rels=full.dict_of_rels)
    out = {"n_ent": n_ent, "n_rel": n_rel, "ent_dim": d, "rel_dim": rd, "b_size": b_size,
           "all_heads": heads.numpy(), "all_tails": tails.numpy(), "all_rels": rels.numpy(),
           "heads": th.numpy(), "tails": tt.numpy(), "rels": tr.numpy()}
    for k, v in model.state_dict().items():
        if k != "projected_entities":
            out["w:" + k] = v.numpy().copy()
    weights = {k: v.clone() for k, v in model.state_dict().items()}
    for which, dic in (("dh", full.dict_of_heads), ("dt", full.dict_of_tails), ("dr", full.dict_of_rels)):
        out[which + "_keys"], out[which + "_offs"], out[which + "_vals"] = dicts_to_arrays(dic)

    ev = LinkPredictionEvaluator(model, test)
    ev.evaluate(b_size=b_size, verbose=False)
    out["rank_true_heads"], out["rank_true_tails"] = ev.rank_true_heads.numpy(), ev.rank_true_tails.numpy()
    out["filt_rank_true_heads"] = ev.filt_rank_true_heads.numpy()
    out["filt_rank_true_tails"] = ev.filt_rank_true_tails.numpy()
    for directed in (True, False):
        rev = RelationPredictionEvaluator(model, test, directed=directed)
        rev.evaluate(b_size=b_size, verbose=False)
        tag = "dir" if directed else "undir"
        out["rank_true_rels_" + tag] = rev.rank_true_rels.numpy()
        out["filt_rank_true_rels_" + tag] = rev.filt_rank_true_rels.numpy()

    # the evaluators leave the weights as they were: scoring and gradients on the same tables
    assert all(torch.equal(v, model.state_dict()[k]) for k, v in weights.items() if k != "projected_entities")
    nh = torch.randint(0, n_ent, (n_test,), generator=g)
    nt = torch.randint(0, n_ent, (n_test,), generator=g)
    out["neg_heads"], out["neg_tails"] = nh.numpy(), nt.numpy()
    with torch.no_grad():
        out["scores"] = model.scoring_function(th, tt, tr).numpy()
        out["neg_scores"] = model.scoring_function(nh, nt, tr).numpy()
    model.zero_grad()
    pos, neg = model(th, tt, tr, nh, nt)
    loss = MarginLoss(margin=1.0)(pos, neg)
    loss.backward()
    out["loss"] = np.float32(loss.item())
    for name_ in ("ent_emb", "rel_emb", "ent_proj_vect", "rel_proj_vect"):
        out["grad:" + name_] = getattr(model, name_).weight.grad.numpy().copy()
    return out


def main():
    for name in CASES:
        out = make(name)
        path = os.path.join(HERE, "transd_%s.npz" % name)
        np.savez_compressed(path, **out)
        print(name, "->", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
