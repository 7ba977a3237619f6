"""The host layer's argument handling, pinned without a GPU: every size query of the grid of
tests/golden/make_golden_abi.py and every malformed call it lists gets the answer recorded in
tests/golden/abi_answers.json -- the same sizes, the same return code and the same kge_last_error()
text.  The calls run in a child process that sees no GPU (CUDA_VISIBLE_DEVICES=""), so a call that
wrongly got past its argument checks fails with KGE_ERR_CUDA instead of launching on dummy pointers."""
import json

import pytest

from tests.golden import make_golden_abi as gen

with open(gen.OUT) as _f:
    GOLDEN = json.load(_f)


@pytest.fixture(scope="module")
def answers():
    return gen.answers()   # raises unless the child exits cleanly


def test_size_queries_equal_golden(answers):
    assert answers["sizes"] == GOLDEN["sizes"]


def test_malformed_calls_equal_golden(answers):
    got = answers["calls"]
    want = {(g, k): v for g, cases in GOLDEN["calls"].items() for k, v in cases.items()}
    missing = [c for c in want if c[1] not in got.get(c[0], {})]
    assert not missing, "cases no longer generated: %s" % missing[:10]
    reached_cuda = [c for c in want if got[c[0]][c[1]][0] == gen.ERR_CUDA]
    assert not reached_cuda, "malformed calls got past their argument checks: %s" % reached_cuda[:10]
    differ = {c: (got[c[0]][c[1]], v) for c, v in want.items() if got[c[0]][c[1]] != v}
    assert not differ, "%d answers differ (got, want): %s" % (len(differ), list(differ.items())[:10])


def test_fixture_covers_every_launching_entry_point():
    assert {g.split("/")[0] for g in GOLDEN["calls"]} >= {
        "kge_rank_side", "kge_filter_side", "kge_score_all", "kge_topk_side", "kge_topk_merge", "kge_topk_dense",
        "kge_pack_table", "kge_tc_pack_table", "kge_tc_pack_table_cached", "kge_gather_rows",
        "kge_margin_step_fwd", "kge_margin_step_bwd", "kge_score_triples_fwd", "kge_score_triples_bwd",
        "kge_scatter_rows_add", "kge_margin_loss_fwd", "kge_margin_loss_bwd", "kge_pair_loss_fwd",
        "kge_pair_loss_bwd"}
    assert all(v[0] != gen.ERR_CUDA for cases in GOLDEN["calls"].values() for v in cases.values())
