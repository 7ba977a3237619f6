"""The collectives every sharded entry point issues, per rank: tests/golden/shard_collectives.json.

    python tests/golden/make_golden_collectives.py

Every case runs W emulated ranks as threads (tests/shard_threads.py) on the CPU stand-in engines of
the gloo tests and records, per rank, the (op, dtype, shape) of every ``dist.all_reduce`` /
``dist.all_gather`` in call order.  The recording sits at the torch.distributed level, below the
shard objects, so it sees collectives whichever object issues them.  tests/test_shard_collectives.py
runs the same cases and compares; a change of the communication pattern shows there, case by case.
"""
import json
import os
import sys

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import kge_oracle as oracle  # noqa: E402
from tests import helpers, shard_threads  # noqa: E402
from tests.test_relpred_sharding_gloo import OracleRelEngine  # noqa: E402
from tests.test_sharding_gloo import OracleEngine  # noqa: E402
from tests.test_topk_sharding_gloo import OracleTopkEngine, key_order  # noqa: E402
from tests.train_kit import OracleStepEngine  # noqa: E402
from torchkge_b200 import _lib  # noqa: E402
from torchkge_b200.data import filter_csr  # noqa: E402
from torchkge_b200.engine import (EntityShard, ModelSpec, QueryShard, rank_link_prediction,  # noqa: E402
                                  rank_relation_prediction, score_triples_entity_sharded,
                                  topk_entity_inference, topk_relation_inference)
from torchkge_b200.inference import _mask_csr  # noqa: E402
from torchkge_b200.training import sharded_margin_step  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shard_collectives.json")
N_REL, DIM = 4, 8
WORLDS = (1, 2, 3, 8)
#: (n_ent, n_facts): chunks and rank slices of several rows; n_ent and n_facts below most worlds
SIZES = ((23, 11), (2, 2))


class TopkEngine(OracleTopkEngine):
    """OracleTopkEngine plus the dense RESCAL relation path (rescal_rel_scores, topk_dense)."""

    rescal_rel_scores = OracleRelEngine.rescal_rel_scores

    def topk_dense(self, scores, k, mask=None):
        s = scores.clone()
        if mask is not None:
            offs, ids = mask
            for i in range(s.shape[0]):
                s[i, ids[offs[i]:offs[i + 1]]] = float("-inf")
        ids = torch.arange(s.shape[1]).expand(s.shape[0], -1)
        order = key_order(s, ids)[:, :k]
        return ids.gather(1, order), s.gather(1, order)


def _graph(n_ent, n_facts):
    h, t, r = helpers.random_graph(n_ent, N_REL, 4 * n_facts, seed=5, skew=False)
    return h[:n_facts].contiguous(), t[:n_facts].contiguous(), r[:n_facts].contiguous()


def _shard(form, rank, world, group, n_ent, n, spec):
    """(shard, spec) of one rank: form 'query', 'full' (whole table) or 'local' (rows [lo, hi))."""
    if form == "query":
        return QueryShard(n, rank, world, group), spec
    shard = EntityShard(n_ent, rank, world, group, local_storage=form == "local")
    return shard, (spec.narrowed(shard.lo, shard.hi) if form == "local" else spec)


def _lp(kind, form):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=1)
        h, t, r = _graph(n_ent, n)
        dh, dt = oracle.build_filter_dicts(h, t, r)
        shard, spec = _shard(form, rank, world, group, n_ent, n, ModelSpec.from_model(model))
        rank_link_prediction(spec, h, t, r, filter_csr(dt, h, r, t), filter_csr(dh, t, r, h), shard=shard,
                             engine=OracleEngine(), chunk=4)
    return run


def _rp(kind, form, directed):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=2)
        h, t, r = _graph(n_ent, n)
        csr = filter_csr(oracle.build_rel_dict(h, t, r), h, t, r)
        shard, spec = _shard(form, rank, world, group, n_ent, n, ModelSpec.from_model(model))
        rank_relation_prediction(spec, h, t, r, csr, directed=directed, engine=OracleRelEngine(), chunk=4,
                                 shard=shard)
    return run


def _scores(kind):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=3)
        h, t, r = _graph(n_ent, n)
        shard, spec = _shard("local", rank, world, group, n_ent, n, ModelSpec.from_model(model))
        score_triples_entity_sharded(spec, h, t, r, shard, engine=OracleRelEngine(), batch=4)
    return run


def _topk_entity(kind, form, side, masked):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=4)
        h, _, r = _graph(n_ent, n)
        mask = _mask_csr({(int(a), int(b)): {int(a)} for a in h[::2] for b in r[::2]}, h, r) if masked else None
        shard, spec = _shard(form, rank, world, group, n_ent, n, ModelSpec.from_model(model))
        topk_entity_inference(spec, h, r, _lib.SIDE_TAIL if side == "tail" else _lib.SIDE_HEAD, min(3, n_ent),
                              mask, shard=shard, engine=TopkEngine(), chunk=4)
    return run


def _topk_relation(kind, form, masked):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=5)
        h, t, _ = _graph(n_ent, n)
        mask = _mask_csr({(int(a), int(b)): {1} for a in h[::2] for b in t[::2]}, h, t) if masked else None
        shard, spec = _shard(form, rank, world, group, n_ent, n, ModelSpec.from_model(model))
        topk_relation_inference(spec, h, t, 2, mask, shard=shard, engine=TopkEngine(), chunk=4)
    return run


def _train(kind):
    def run(rank, world, group, n_ent, n):
        model = helpers.make_model(kind, DIM, n_ent, N_REL, seed=6)
        h, t, r = _graph(n_ent, n)
        shard = EntityShard(n_ent, rank, world, group, local_storage=True)
        local = helpers.local_model(kind, model, shard.lo, shard.hi, N_REL, DIM)
        with torch.enable_grad():
            loss = sharded_margin_step(local, h, t, r, 0.5, 2, torch.full((N_REL,), 0.5), 7, 1, shard,
                                       engine=OracleStepEngine())
            loss.backward()
    return run


CALLS = {}
for _form in ("full", "local"):
    CALLS["lp-distmult-" + _form] = _lp("distmult", _form)
for _form in ("query", "full", "local"):
    for _kind, _directed in (("distmult", True), ("complex", False), ("rescal", True), ("rescal", False)):
        CALLS["rp-%s-%s-%s" % (_kind, "dir" if _directed else "undir", _form)] = _rp(_kind, _form, _directed)
    for _side in ("tail", "head"):
        for _masked in (False, True):
            CALLS["topk_ent-complex-%s-%s-%s" % (_side, "mask" if _masked else "nomask", _form)] = \
                _topk_entity("complex", _form, _side, _masked)
    for _kind, _masked in (("distmult", True), ("transe_l2", False), ("rescal", True)):
        CALLS["topk_rel-%s-%s-%s" % (_kind, "mask" if _masked else "nomask", _form)] = \
            _topk_relation(_kind, _form, _masked)
CALLS["scores-complex-local"] = _scores("complex")
CALLS["train-distmult-local"] = _train("distmult")


def cases():
    """{case id: (call, world, n_ent, n_facts)}"""
    return {"%s-w%d-e%d-f%d" % (name, w, n_ent, n): (fn, w, n_ent, n)
            for name, fn in CALLS.items() for w in WORLDS for n_ent, n in SIZES}


def record(fn, world, n_ent, n):
    """[[ 'op dtype shape' of every collective, in order ] for every rank]"""
    log = [[] for _ in range(world)]
    with pytest.MonkeyPatch.context() as mp:
        shard_threads.thread_collectives(mp)
        reduce_, gather_ = dist.all_reduce, dist.all_gather

        def all_reduce(t, *a, **k):
            log[shard_threads._me.rank].append("all_reduce %s %s" % (t.dtype, list(t.shape)))
            return reduce_(t, *a, **k)

        def all_gather(out, t, *a, **k):
            log[shard_threads._me.rank].append("all_gather %s %s x%d" % (t.dtype, list(t.shape), len(out)))
            return gather_(out, t, *a, **k)

        mp.setattr(dist, "all_reduce", all_reduce)
        mp.setattr(dist, "all_gather", all_gather)
        shard_threads.run_ranks(world, lambda rank, group: fn(rank, world, group, n_ent, n))
    return log


if __name__ == "__main__":
    torch.set_num_threads(1)
    out = {cid: record(*case) for cid, case in cases().items()}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("%d cases -> %s" % (len(out), OUT))
