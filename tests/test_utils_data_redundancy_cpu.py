"""Data redundancy without a GPU: the CPU oracle (oracle/redundancy_oracle.py) reproduces every output of
the unmodified reference stored in tests/golden/redundancy.npz, printed text included, and every input
check of torchkge_b200.data_redundancy raises ValueError before anything touches CUDA."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from oracle import redundancy_oracle as oracle
from torchkge_b200 import _lib
from torchkge_b200 import data_redundancy as dr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "redundancy.npz")
THETAS = [(0.8, 0.8), (0.6, 0.5)]
REVERSES = {"none": None, "tuple": [(60, 61)], "list": [[80, 81]]}
CART_THETAS = [0.8, 0.5]


class RefStyleKG:
    """The attributes of the reference's KnowledgeGraph that the analysis reads, and nothing else."""

    def __init__(self, h, t, r, n_ent, n_rel):
        self.head_idx, self.tail_idx, self.relations = (torch.as_tensor(x, dtype=torch.int64) for x in (h, t, r))
        self.n_ent, self.n_rel = n_ent, n_rel

    def __len__(self):
        return self.head_idx.shape[0]


def golden_graphs():
    z = np.load(GOLDEN, allow_pickle=False)
    n_ent, n_rel = int(z["n_ent"]), int(z["n_rel"])
    kgs = [RefStyleKG(z[k][:, 0], z[k][:, 1], z[k][:, 2], n_ent, n_rel) for k in ("facts_tr", "facts_val", "facts_te")]
    return z, kgs


def pairs(a):
    return [tuple(p) for p in np.asarray(a).reshape(-1, 2).tolist()]


def test_oracle_reproduces_the_golden_outputs():
    z, (tr, va, te) = golden_graphs()
    assert int(z["n_rel"]) == 1345
    for i, (t1, t2) in enumerate(THETAS):
        for tag, rev in REVERSES.items():
            d, rd = oracle.duplicates(tr, va, te, theta1=t1, theta2=t2, reverses=rev)
            assert d == pairs(z["dup_%d_%s" % (i, tag)]), (i, tag)
            assert rd == pairs(z["rev_%d_%s" % (i, tag)]), (i, tag)
    d_listed, rd_listed = pairs(z["count_dup_listed"]), pairs(z["count_rev_listed"])
    assert oracle.count_triplets(tr, te, d_listed, rd_listed) == tuple(z["count_tr_te"].tolist())
    assert oracle.count_triplets(te, te, d_listed, rd_listed) == tuple(z["count_te_te"].tolist())
    for i, th in enumerate(CART_THETAS):
        assert oracle.cartesian_product_relations(tr, va, te, theta=th) == z["cart_%d" % i].tolist()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        oracle.duplicates(tr, va, te, verbose=True, counts=True)
    assert buf.getvalue() == str(z["stdout"])


def test_golden_fixture_plants_the_edge_cases():
    """What the fixture is for: ratios exactly at the thresholds are excluded, repeated facts change the
    lengths only, a list inside ``reverses`` excludes nothing."""
    z, _ = golden_graphs()
    dup = pairs(z["dup_0_none"])
    assert (10, 11) in dup and (20, 21) not in dup and (30, 31) not in dup and (52, 53) in dup
    assert (50, 51) not in dup and (20, 21) in pairs(z["dup_1_none"])
    assert (60, 61) in pairs(z["rev_0_none"]) and (60, 61) not in pairs(z["rev_0_tuple"])
    assert pairs(z["rev_0_list"]) == pairs(z["rev_0_none"])
    assert z["cart_0"].tolist() == [90, 92, 93, 94] and 91 in z["cart_1"].tolist()


@pytest.fixture
def no_cuda(monkeypatch):
    """Any attempt to reach CUDA or the library fails the test."""
    def boom(*a, **k):
        raise AssertionError("CUDA was reached before the input checks")
    monkeypatch.setattr(torch.cuda, "is_available", boom)
    monkeypatch.setattr(_lib, "load", boom)


def _kg(h=(0, 1), t=(1, 2), r=(0, 1), n_ent=4, n_rel=3):
    return RefStyleKG(list(h), list(t), list(r), n_ent, n_rel)


@pytest.mark.parametrize("where", [0, 1, 2])
@pytest.mark.parametrize("bad", [-1, 3])
def test_relation_ids_outside_the_train_range_raise(no_cuda, where, bad):
    kgs = [_kg(), _kg(), _kg()]
    kgs[where] = _kg(r=(0, bad), n_rel=5 if where else 3)   # the range is kg_tr.n_rel's, not the graph's own
    with pytest.raises(ValueError, match="relation ids"):
        dr.duplicates(*kgs)
    with pytest.raises(ValueError, match="relation ids"):
        dr.cartesian_product_relations(*kgs)


def test_count_triplets_checks_each_graph_against_its_own_n_rel(no_cuda):
    with pytest.raises(ValueError, match="kg2 relation ids"):
        dr.count_triplets(_kg(n_rel=5), _kg(r=(0, 3)), [(0, 1)], [])
    with pytest.raises(ValueError, match="kg1 relation ids"):
        dr.count_triplets(_kg(r=(4, 0)), _kg(n_rel=5), [(0, 1)], [])


def test_entity_ids_outside_n_ent_raise(no_cuda):
    with pytest.raises(ValueError, match="tail ids"):
        dr.duplicates(_kg(t=(1, 4)), _kg(), _kg())
    with pytest.raises(ValueError, match="head ids"):
        dr.count_triplets(_kg(), _kg(h=(-1, 0)), [], [])


@pytest.mark.parametrize("thetas", [(-0.1, 0.8), (0.8, 1.01), (float("nan"), 0.8)])
def test_thresholds_outside_unit_interval_raise(no_cuda, thetas):
    with pytest.raises(ValueError, match="theta"):
        dr.duplicates(_kg(), _kg(), _kg(), theta1=thetas[0], theta2=thetas[1])


def test_key_packing_limit_raises(no_cuda):
    n_ent = 2 ** 30           # n_ent^2 * n_rel = 2^60 * 8 = 2^63
    kg = _kg(n_ent=n_ent, n_rel=8)
    for call in (lambda: dr.duplicates(kg, kg, kg), lambda: dr.cartesian_product_relations(kg, kg, kg),
                 lambda: dr.count_triplets(kg, kg, [], [])):
        with pytest.raises(ValueError, match="int64"):
            call()
    dr._check_sizes(n_ent, 7, counters=False)     # 7 * 2^60 < 2^63


def test_counter_matrix_bound_raises_without_allocating(no_cuda):
    limit = int((dr.MAX_COUNTER_BYTES // 8) ** 0.5)
    assert limit == 8192 and 8 * limit * limit == dr.MAX_COUNTER_BYTES
    dr._check_sizes(10, limit, counters=True)
    big = _kg(n_rel=limit + 1)
    with pytest.raises(ValueError, match="counter matrix"):
        dr.duplicates(big, big, big)
    with pytest.raises(ValueError, match="counter matrix"):
        dr.count_triplets(_kg(), big, [], [])


def test_no_cuda_is_a_library_error(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    for call in (lambda: dr.duplicates(_kg(), _kg(), _kg()), lambda: dr.cartesian_product_relations(_kg(), _kg(), _kg()),
                 lambda: dr.count_triplets(_kg(), _kg(), [(0, 1)], [])):
        with pytest.raises(_lib.KgeLibraryError, match="no CPU fallback"):
            call()


def test_exported_from_utils():
    from torchkge_b200 import utils
    assert utils.duplicates is dr.duplicates
    assert utils.count_triplets is dr.count_triplets
    assert utils.cartesian_product_relations is dr.cartesian_product_relations
