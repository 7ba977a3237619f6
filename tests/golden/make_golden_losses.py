"""Generates tests/golden/loss_<case>.npz by running the UNMODIFIED reference (torchkge v0.17.7 at
/root/reference) on the inputs of the ten toy_* / syn_* fixtures of make_golden.py: the same weights,
test facts and fixture negatives, with ``LogisticLoss`` and ``BinaryCrossEntropyLoss`` in place of
``MarginLoss``.  Run in the authoring container only:

    PYTHONPATH=/root/reference python tests/golden/make_golden_losses.py

Each file holds, per loss (``logistic`` / ``bce``): the loss of ``criterion(*model(h, t, r, nh, nt))``
(``loss_<loss>``) and the gradient of every parameter after its backward (``g_<loss>:<name>``).  The
inputs are read back from the toy_* / syn_* fixtures, so they are not repeated here.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, "/root/reference")
from torchkge.models import ComplExModel, DistMultModel, RESCALModel, TransEModel  # noqa: E402
from torchkge.utils import BinaryCrossEntropyLoss, LogisticLoss  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
CASES = ["toy_transe_l1", "toy_transe_l2", "toy_distmult", "toy_rescal", "toy_complex",
         "syn_transe_l1", "syn_transe_l2", "syn_distmult", "syn_rescal", "syn_complex"]


def build(kind, d, n_ent, n_rel):
    if kind == "transe_l1":
        return TransEModel(d, n_ent, n_rel, "L1")
    if kind == "transe_l2":
        return TransEModel(d, n_ent, n_rel, "L2")
    if kind == "distmult":
        return DistMultModel(d, n_ent, n_rel)
    if kind == "rescal":
        return RESCALModel(d, n_ent, n_rel)
    if kind == "complex":
        return ComplExModel(d, n_ent, n_rel)
    raise ValueError(kind)


def run_case(name):
    z = np.load(os.path.join(OUT, name + ".npz"), allow_pickle=False)
    kind, d, n_ent, n_rel = str(z["kind"]), int(z["dim"]), int(z["n_ent"]), int(z["n_rel"])
    model = build(kind, d, n_ent, n_rel)
    model.load_state_dict({k[2:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith("w:")})
    h, t, r, nh, nt = (torch.from_numpy(z[k].copy()).long()
                       for k in ("heads", "tails", "rels", "neg_heads", "neg_tails"))
    out = {"kind": kind, "torch_version": torch.__version__}
    for tag, crit in (("logistic", LogisticLoss()), ("bce", BinaryCrossEntropyLoss())):
        model.zero_grad()
        pos, neg = model(h, t, r, nh, nt)
        loss = crit(pos, neg)
        loss.backward()
        out["loss_" + tag] = np.array(loss.item(), dtype=np.float64)
        for k, p in model.named_parameters():
            out["g_%s:%s" % (tag, k)] = p.grad.numpy().copy()
    path = os.path.join(OUT, "loss_" + name + ".npz")
    np.savez_compressed(path, **out)
    print(name, "->", os.path.getsize(path), "bytes", {k: float(out[k]) for k in out if k.startswith("loss_")})


def main():
    for name in CASES:
        run_case(name)


if __name__ == "__main__":
    main()
