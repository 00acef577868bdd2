#!/usr/bin/env python
"""Run the picking-order node's own code (ros/src/morefusion_ros/nodes/select_picking_order.py:
``get_leaves``, ``get_picking_order`` and ``SelectPickingOrder._callback``, taken from the
reference checkout by ``ast``) with the real networkx on the cases of oracle/picking_order.py, and
write what it decides to tests/golden/picking_order/cases.npz.

TEST INFRASTRUCTURE ONLY.  Needs the reference checkout (MOREFUSION_REFERENCE):

    python -m oracle.ref_harness.gen_picking_order

Stand-ins: ``rospy`` (its ``loginfo`` records the caller's ``ins_id_i``, ``ins_id_j`` and ``ratio``
of every occluder the node weighs), ``cv_bridge`` and the message classes; ``nx_graph_to_image``,
which records the graph; ``get_grasp_pose``, which returns a constant; the ``morefusion`` names the
callback touches; and ``self._render_object_pose_array``, which returns oracle/picking_order.py's
``render_instances`` of the whole scene, or of the one instance.  ``set`` in get_picking_order's
namespace records each round's leaves.

cases.npz, per case of CASES: ``<case>/T_cad2base`` (the regenerated inputs, to catch a change of
the generator), ``<case>/weighed`` [K,2] int64 and ``<case>/weighed_ratio`` [K] float64 (every
(i, j) the node logs, in its order), ``<case>/edges`` [E,2] int64 (the graph's edges, in the order
they were added), ``<case>/published`` (0: nothing published, the target class absent; 1:
published), ``<case>/order`` [P] int64 (the published instance ids), ``<case>/rounds`` [P] int64
and ``<case>/round_len`` [R] int64 (the leaf set get_leaves gave in each round of
get_picking_order, each sorted, back to back).
"""

import ast
import copy
import os
import sys
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import picking_order as opo  # noqa: E402
from oracle.ref_harness import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "picking_order")
NODE = os.path.join("ros", "src", "morefusion_ros", "nodes", "select_picking_order.py")


def _namespace():
    """The node's get_leaves, get_picking_order and SelectPickingOrder._callback, exec'd into one
    namespace of stand-ins."""
    import networkx
    text = open(os.path.join(shim.REF_ROOT, NODE)).read()
    g = dict(np=np, copy=copy, networkx=networkx)
    for node in ast.parse(text).body:
        if isinstance(node, ast.FunctionDef) and node.name in ("get_leaves", "get_picking_order"):
            exec(ast.get_source_segment(text, node), g)
        if isinstance(node, ast.ClassDef) and node.name == "SelectPickingOrder":
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name == "_callback":
                    exec(textwrap.dedent(ast.get_source_segment(text, item, padded=True)), g)
    return g


class _Msg:
    def __init__(self):
        self.header = None
        self.poses = []


def run_case(name, models):
    """The node's decision on case ``name``: a dict of the recorded arrays."""
    meshes, T_cad2cam, ids, f, H, W = opo.case_scene(name, models)
    _, cls, T_cad2base, _, K, _, _ = opo.case_inputs(name)
    rec = dict(weighed=[], graph=None, published=None, rounds=[])
    g = _namespace()

    def loginfo(msg):
        loc = sys._getframe(1).f_locals
        rec["weighed"].append((int(loc["ins_id_i"]), int(loc["ins_id_j"]), loc["ratio"]))

    rospy = types.SimpleNamespace(loginfo=loginfo, logwarn_throttle=lambda *a, **k: None)

    def recording_set(it):
        s = set(it)
        rec["rounds"].append(sorted(int(x[0]) for x in s))
        return s

    class _Pub:
        def __init__(self, keep):
            self._keep = keep

        def publish(self, msg):
            if self._keep:
                rec["published"] = [int(p.instance_id) for p in msg.poses]

    def nx_graph_to_image(graph):
        rec["graph"] = graph.copy()
        return np.zeros((1, 1, 3), np.uint8)

    def render(cam_msg, poses_msg, instance_id=None):
        keep = [n for n in range(len(ids)) if instance_id is None or ids[n] == instance_id]
        depth, ins, _, _, _ = opo.render_instances([meshes[n] for n in keep], T_cad2cam[keep],
                                                   ids[keep], f, H, W)
        return np.zeros((H, W, 3), np.uint8), depth, ins

    class_names = [f"class_{c}" for c in range(22)]
    g.update(
        rospy=rospy, set=recording_set, nx_graph_to_image=nx_graph_to_image,
        get_grasp_pose=lambda rgb, pcd, mask: (np.array([1.0, 0, 0, 0]), np.zeros(3)),
        cv_bridge=types.SimpleNamespace(CvBridge=lambda: types.SimpleNamespace(
            cv2_to_imgmsg=lambda img, enc: types.SimpleNamespace(header=None))),
        ObjectPoseArray=_Msg, PoseArray=_Msg,
        morefusion=types.SimpleNamespace(
            datasets=types.SimpleNamespace(ycb_video=types.SimpleNamespace(class_names=class_names)),
            geometry=types.SimpleNamespace(
                pointcloud_from_depth=lambda depth, fx, fy, cx, cy: np.zeros(depth.shape + (3,)))))

    def pose(i, c):
        p = types.SimpleNamespace(position=types.SimpleNamespace(x=0.0, y=0.0, z=0.0),
                                  orientation=types.SimpleNamespace(w=1.0, x=0.0, y=0.0, z=0.0))
        return types.SimpleNamespace(instance_id=int(i), class_id=int(c), pose=p)

    poses_msg = _Msg()
    poses_msg.poses = [pose(i, c) for i, c in zip(ids, cls)]
    self = types.SimpleNamespace(
        _poses_msg=poses_msg, _target=opo.TARGET, _render_object_pose_array=render,
        _pub_rend=_Pub(False), _pub_poses=_Pub(True), _pub_poses_viz=_Pub(False),
        _pub_graph=_Pub(False))
    cam_msg = types.SimpleNamespace(header=None, height=H, width=W, K=K.reshape(-1).tolist())
    g["_callback"](self, cam_msg)

    edges = [(int(i[0]), int(j[0])) for i, j in rec["graph"].edges] if rec["graph"] else []
    # networkx lists edges by node insertion order; the node added them in the order it logged
    logged = [(i, j) for i, j, _ in rec["weighed"]]
    edges.sort(key=logged.index)
    order = rec["published"] or []
    return {"T_cad2base": T_cad2base,
            "weighed": np.array([(i, j) for i, j, _ in rec["weighed"]], np.int64).reshape(-1, 2),
            "weighed_ratio": np.array([r for _, _, r in rec["weighed"]], np.float64),
            "edges": np.array(edges, np.int64).reshape(-1, 2),
            "published": np.int64(rec["published"] is not None),
            "order": np.array(order, np.int64),
            "rounds": np.array([x for leaves in rec["rounds"] for x in leaves], np.int64),
            "round_len": np.array([len(leaves) for leaves in rec["rounds"]], np.int64)}


def main():
    from morefusion_b200 import synthetic
    models = synthetic.SyntheticYCBModels()
    out = {}
    for name in opo.CASES:
        r = run_case(name, models)
        out.update({f"{name}/{k}": v for k, v in r.items()})
    os.makedirs(OUT, exist_ok=True)
    np.savez(os.path.join(OUT, "cases.npz"), **out)


if __name__ == "__main__":
    main()
