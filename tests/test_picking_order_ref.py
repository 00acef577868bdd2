"""CPU: the picking-order graph rules of ``contrib.picking_order`` (``occlusion_edges``,
``picking_order``) against the picking-order node's own code (select_picking_order.py), run by
oracle/ref_harness/gen_picking_order.py on oracle/picking_order.py's scene counts into
tests/golden/picking_order/cases.npz, and -- where the reference checkout is present -- run
afresh."""

import os

import numpy as np
import pytest

from oracle import picking_order as opo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "picking_order", "cases.npz")
CASES = sorted(opo.CASES)


@pytest.fixture(scope="module")
def models():
    from morefusion_b200 import synthetic
    return synthetic.SyntheticYCBModels()


@pytest.fixture(scope="module")
def counts(models):
    """case -> the oracle's (whole, occluded) of the case's scene."""
    out = {}
    for name in CASES:
        meshes, T, ids, f, H, W = opo.case_scene(name, models)
        _, _, whole, occluded, _ = opo.render_instances(meshes, T, ids, f, H, W)
        out[name] = (whole, occluded)
    return out


def _case(z, name):
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def _rounds(rec):
    ends = np.cumsum(rec["round_len"])
    return [rec["rounds"][e - n:e].tolist() for n, e in zip(rec["round_len"], ends)]


def _ours(name, whole, occluded):
    """(order, edges) by the package's host rules on the counts, as SelectPickingOrder forms them."""
    from morefusion_b200.contrib import picking_order as po
    ids, cls = opo.case_inputs(name)[:2]
    if opo.TARGET not in cls.tolist():
        return None, []
    visible, edges = po.occlusion_edges(ids, whole, occluded)
    targets = [i for i in visible if cls[list(ids).index(i)] == opo.TARGET]
    return (po.picking_order(edges, targets[-1]) if targets else []), edges


def _assert_matches(rec, order, edges):
    kept = [[i, j] for (i, j), r in zip(rec["weighed"].tolist(), rec["weighed_ratio"]) if r >= 0.1]
    assert kept == rec["edges"].tolist()
    assert [[i, j] for i, j, _ in edges] == rec["edges"].tolist()
    want_ratio = {(i, j): r for (i, j), r in zip(rec["weighed"].tolist(), rec["weighed_ratio"])}
    for i, j, r in edges:
        assert np.float64(r).view(np.uint64) == np.float64(want_ratio[(i, j)]).view(np.uint64)
    if not rec["published"]:
        assert order is None
        return
    # the reference emits each round's leaves in set order; ours sorts them
    assert order == [x for leaves in _rounds(rec) for x in sorted(leaves)]
    assert sorted(order) == sorted(rec["order"].tolist())


@pytest.mark.parametrize("name", CASES)
def test_fixture_self_consistent(name):
    """The inputs regenerate, and the reference's flat order is a permutation within its rounds,
    with the target alone in the last round."""
    rec = _case(np.load(GOLDEN), name)
    assert np.array_equal(rec["T_cad2base"], opo.case_inputs(name)[2])
    order = rec["order"].tolist()
    assert int(rec["round_len"].sum()) == len(order)
    pos = 0
    for leaves in _rounds(rec):
        assert sorted(order[pos:pos + len(leaves)]) == leaves
        pos += len(leaves)
    if order:
        assert _rounds(rec)[-1] == [order[-1]]


@pytest.mark.parametrize("name", CASES)
def test_rules_on_oracle_counts_equal_fixture(name, counts):
    rec = _case(np.load(GOLDEN), name)
    order, edges = _ours(name, *counts[name])
    _assert_matches(rec, order, edges)


def test_fixture_covers_the_cases():
    """What each case is there for holds in the fixture."""
    z = np.load(GOLDEN)
    rec = {name: _case(z, name) for name in CASES}
    assert _rounds(rec["chain"]) == [[12], [3], [7]]
    assert _rounds(rec["diamond"]) == [[6], [2, 9], [4]]
    assert rec["clear"]["order"].tolist() == [5]
    assert rec["hidden"]["published"] == 1 and rec["hidden"]["order"].tolist() == []
    assert rec["absent"]["published"] == 0
    assert rec["two_targets"]["order"].tolist() == [5, 8]
    w = dict(zip(map(tuple, rec["threshold"]["weighed"].tolist()), rec["threshold"]["weighed_ratio"]))
    assert 0.09 < w[(3, 10)] < 0.1 <= w[(3, 6)] < 0.11
    assert rec["threshold"]["edges"].tolist() == [[3, 6]]


def test_cycle_raises():
    from morefusion_b200.contrib.picking_order import picking_order
    edges = [(1, 2, 0.3), (2, 3, 0.2), (3, 2, 0.4), (4, 1, 0.5)]
    with pytest.raises(ValueError, match=r"\[2, 3\]"):
        picking_order(edges, 1)
    with pytest.raises(ValueError):
        picking_order([(5, 5, 1.0)], 5)
    # a cycle the target cannot reach is no obstacle
    assert picking_order([(1, 4, 0.2), (2, 3, 0.5), (3, 2, 0.5)], 1) == [4, 1]
    assert picking_order([], 9) == [9]


def test_long_chain():
    """A chain longer than Python's recursion limit orders without recursing."""
    from morefusion_b200.contrib.picking_order import picking_order
    n = 3000
    edges = [(i, i + 1, 0.5) for i in range(n)]
    assert picking_order(edges, 0) == list(range(n, -1, -1))


@pytest.mark.parametrize("name", CASES)
def test_reference_direct(name, models):
    from oracle.ref_harness import shim
    if not shim.reference_available():
        pytest.skip("reference checkout not present")
    from oracle.ref_harness import gen_picking_order as gen
    rec = gen.run_case(name, models)
    z = _case(np.load(GOLDEN), name)
    for k, v in rec.items():
        if k != "order":
            assert np.array_equal(np.asarray(v), z[k]), k
    # the order within a round is the node's set order, which follows the process's hash seed
    assert [x for leaves in _rounds(rec) for x in leaves] == [x for leaves in _rounds(z) for x in leaves]
    pos = 0
    for leaves in _rounds(rec):
        assert sorted(rec["order"][pos:pos + len(leaves)].tolist()) == leaves
        pos += len(leaves)
