"""The communication pattern of every sharded entry point: for each case of
tests/golden/make_golden_collectives.py (link prediction, relation prediction, triple scoring, both
top-k paths and the sharded training step, under every shard form each accepts, W in {1, 2, 3, 8},
with tables and fact lists smaller than W), every rank issues the collectives recorded in
tests/golden/shard_collectives.json: same order, op, dtype and shape.  Arguments that break the table
rule or a QueryShard's length raise before any collective."""
import json

import pytest
import torch

import torchkge_b200 as tk
from tests import helpers
from tests.golden import make_golden_collectives as gen
from tests.test_sharding_gloo import OracleEngine
from tests.train_kit import NoCollectiveShard
from torchkge_b200 import _lib
from torchkge_b200.engine import (ModelSpec, QueryShard, rank_link_prediction, topk_entity_inference,
                                  topk_relation_inference)

with open(gen.OUT) as _f:
    GOLDEN = json.load(_f)
CASES = gen.cases()


def test_fixture_covers_every_case():
    assert sorted(GOLDEN) == sorted(CASES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_collectives_equal_golden(case):
    assert gen.record(*CASES[case]) == GOLDEN[case]


# ------------------------------------------------------------- argument errors before any collective
def _table_case(case, n_ent=20):
    """Rank 1 of 2 (rows [10, 20)) with a table that breaks the table rule: 'local_whole' declares the
    whole table as this rank's rows, 'full_narrowed' declares this rank's rows as the whole table."""
    spec = ModelSpec.from_model(helpers.make_model("distmult", 8, n_ent, gen.N_REL, seed=1))
    if case == "local_whole":
        return spec, NoCollectiveShard(n_ent, 1, 2, local_storage=True), "should hold 10 entity rows .*, the model holds 20 entity rows"
    shard = NoCollectiveShard(n_ent, 1, 2)
    return spec.narrowed(shard.lo, shard.hi), shard, "should hold 20 entity rows .*, the model holds 10 entity rows"


TABLE_CALLS = {
    "link_prediction": lambda spec, shard, h, r: rank_link_prediction(spec, h, h, r, None, None, shard=shard,
                                                                      engine=OracleEngine()),
    "topk_entity": lambda spec, shard, h, r: topk_entity_inference(spec, h, r, _lib.SIDE_TAIL, 3, shard=shard,
                                                                   engine=gen.TopkEngine()),
    "topk_relation": lambda spec, shard, h, r: topk_relation_inference(spec, h, h, 2, shard=shard,
                                                                       engine=gen.TopkEngine()),
}


@pytest.mark.parametrize("case", ["local_whole", "full_narrowed"])
@pytest.mark.parametrize("call", sorted(TABLE_CALLS))
def test_table_rule_is_checked_before_any_collective(call, case):
    spec, shard, message = _table_case(case)
    h = torch.arange(5)
    with pytest.raises(ValueError, match=message):
        TABLE_CALLS[call](spec, shard, h, h % gen.N_REL)


def test_link_prediction_evaluator_checks_the_query_shard_length():
    """Before the model's device: a CPU model reaches it."""
    kg, _, _ = helpers.make_kg(30, 3, 100, 10)
    ev = tk.LinkPredictionEvaluator(tk.DistMultModel(8, 30, 3), kg, shard=QueryShard(kg.n_facts + 1, 0, 2))
    with pytest.raises(ValueError, match="QueryShard covers %d facts or queries, got %d" % (kg.n_facts + 1,
                                                                                          kg.n_facts)):
        ev.evaluate(b_size=4)
