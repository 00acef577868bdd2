"""GPU: ``contrib.SelectPickingOrder`` on the picking-order cases against the node's own decisions
(tests/golden/picking_order/cases.npz, tests/test_picking_order_ref.py), end to end behind an
``ObjectMapping`` against the oracle pipeline, and its one host read per call."""

import numpy as np
import pytest

from oracle import picking_order as opo
from test_frame_refine_gpu import _syncs
from test_picking_order_ref import GOLDEN, _case, _rounds

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def models():
    from morefusion_b200 import synthetic
    return synthetic.SyntheticYCBModels()


@pytest.mark.parametrize("name", sorted(opo.CASES))
def test_cases_equal_reference(name, models):
    from morefusion_b200.contrib import SelectPickingOrder
    rec = _case(np.load(GOLDEN), name)
    ids, cls, T, C, K, h, w = opo.case_inputs(name)
    order, edges = SelectPickingOrder(models, opo.TARGET)(ids, cls, T, C, K, h, w)
    if not rec["published"]:
        assert order is None
        return
    assert [[i, j] for i, j, _ in edges] == rec["edges"].tolist()
    ratio = {(i, j): r for (i, j), r in zip(rec["weighed"].tolist(), rec["weighed_ratio"])}
    for i, j, r in edges:
        assert np.float64(r).view(np.uint64) == np.float64(ratio[(i, j)]).view(np.uint64)
    assert order == [x for leaves in _rounds(rec) for x in sorted(leaves)]


def _oracle_pipeline(models, ids, cls, T_cad2base, C, K, h, w):
    """The oracle's scene counts at the same poses, through the package's host graph rules (which
    tests/test_picking_order_ref.py holds to the node's own code)."""
    from morefusion_b200.contrib import picking_order as po
    from oracle import render_cad as orc
    T_cad2cam = np.linalg.inv(C) @ T_cad2base
    f = orc.focal_from_fovy(orc.fovy_from_intrinsics(K[1, 1], h), h)
    meshes = [(models.get_cad(int(c)).vertices, models.get_cad(int(c)).faces) for c in cls]
    _, _, whole, occluded, _ = opo.render_instances(meshes, T_cad2cam, ids, f, h, w)
    visible, edges = po.occlusion_edges(ids, whole, occluded)
    targets = [i for i in visible if cls[list(ids).index(i)] == opo.TARGET]
    return (po.picking_order(edges, targets[-1]) if targets else []), edges


def test_end_to_end_after_object_mapping(models):
    """An ObjectMapping fed four views of the diamond scene and the chain scene together spawns
    its objects; the picking order of their frozen poses at 640x480 equals the oracle's."""
    from morefusion_b200 import geometry
    from morefusion_b200.contrib import ObjectMapping, SelectPickingOrder
    ids_a, cls_a, T_a, C, _, _, _ = opo.case_inputs("diamond")
    ids_b, cls_b, T_b, C_b, _, _, _ = opo.case_inputs("chain")
    # the chain scene moved beside the diamond in the diamond's camera frame
    shift = np.eye(4)
    shift[:3, 3] = (0.25, 0.1, 0.2)
    T_b = C @ shift @ np.linalg.inv(C_b) @ T_b
    ids = np.concatenate([ids_a, ids_b + 100])
    cls = np.concatenate([cls_a, cls_b]).astype(np.int32)
    T_world = np.concatenate([T_a, T_b])
    om = ObjectMapping(models)
    rs = np.random.RandomState(0)
    for _ in range(4):
        dT = np.eye(4)
        dT[:3, 3] = rs.uniform(-0.02, 0.02, 3)
        Ck = C @ dT
        T_cam = np.linalg.inv(Ck) @ T_world
        q = np.array([geometry.quaternion_from_matrix(T) for T in T_cam], np.float32)
        om.add(ids, cls, q, T_cam[:, :3, 3].astype(np.float32), Ck)
    p_ids, p_cls, p_T = om.poses()
    assert sorted(p_ids.tolist()) == sorted(ids.tolist())
    K = np.array([[800.0, 0, 320], [0, 800.0, 240], [0, 0, 1]])
    sel = SelectPickingOrder(models, opo.TARGET)
    order, edges = sel(p_ids, p_cls, p_T, C, K, 480, 640)
    want_order, want_edges = _oracle_pipeline(models, p_ids, p_cls, p_T, C, K, 480, 640)
    assert order == want_order and edges == want_edges
    assert order[-1] == 107 and len(order) == 3          # the chain's target is the last id
    sel(p_ids, p_cls, p_T, C, K, 480, 640)              # warm
    out, syncs = _syncs(lambda: sel(p_ids, p_cls, p_T, C, K, 480, 640))
    assert out == (order, edges)
    assert len(syncs) == 1, syncs


def test_more_than_64_instances_raise(models):
    from morefusion_b200.contrib import SelectPickingOrder
    ids, cls, T, C, K, h, w = opo.case_inputs("clear")
    n = 65
    with pytest.raises(ValueError):
        SelectPickingOrder(models, opo.TARGET)(np.arange(n), np.full(n, opo.TARGET),
                                               np.tile(T[:1], (n, 1, 1)), C, K, h, w)
