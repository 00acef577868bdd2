"""The targeted-pick decision of the picking-order node
(ros/src/morefusion_ros/nodes/select_picking_order.py): which mapped objects must come out before
the target can be reached.

The node renders every mapped object into the camera as one scene, renders each visible object
again alone, and gives object i an edge i -> j ("occluded by j") when the pixels of i's whole
mask where j is visible are at least 10 % of that mask (_callback, :195-296).  Here one
``geometry`` scene render (csrc/render_cad.cu, mf_render_scene) gives every object's whole-mask
pixel count and the per-pair counts in one pass, and the graph is built on the host from them.

Deliberate departures from the node:
  * The order is of instance ids; the node republishes each pose overwritten by a grasp pose
    (get_grasp_pose, :299-331), which is not computed here.
  * Each round's leaves are taken in ascending instance id; the node takes them in ``set`` order,
    which depends on the process's string hash seed.
  * A cycle reachable from the target raises ``ValueError``; the node recurses until
    ``RecursionError``.
  * No RGB render, graph image, ROS stamps or tf: the camera pose comes in as ``sensor_to_world``.
"""

import numpy as np

from .. import geometry

THRESHOLD = 0.1                               # :273, an edge needs ratio >= 0.1


def occlusion_edges(instance_ids, whole, occluded):
    """The node's edges (i, j, ratio) from the counts of one scene render, in its insertion
    order: occluded objects in ascending instance id, then their occluders in ascending id.
    ``whole`` [N] and ``occluded`` [N,N] are in the order of ``instance_ids`` [N].  Returns
    (visible, edges): the instance ids with visible pixels, ascending (the graph's nodes), and
    the edges whose ratio = float64(occluded[i, j]) / float64(whole[i]) is at least 0.1."""
    ids = np.asarray(instance_ids, np.int64).reshape(-1)
    whole = np.asarray(whole, np.int64).reshape(-1)
    occluded = np.asarray(occluded, np.int64).reshape(len(ids), len(ids))
    visible_px = whole - occluded.sum(1)
    order = np.argsort(ids, kind="stable")
    visible = [int(ids[i]) for i in order if visible_px[i] > 0]
    edges = []
    for i in order:
        if visible_px[i] <= 0:
            continue
        for j in order:
            if j == i or occluded[i, j] == 0:
                continue
            ratio = np.float64(occluded[i, j]) / np.float64(whole[i])
            if ratio < THRESHOLD:
                continue
            edges.append((int(ids[i]), int(ids[j]), float(ratio)))
    return visible, edges


def picking_order(edges, target_id):
    """The node's get_picking_order (:27-48) on the graph of ``edges`` [(i, j, ratio)]: round by
    round, the leaves reachable from ``target_id`` (the nodes with no out-edge) are emitted, in
    ascending instance id, and removed, until the target is a leaf itself; the target comes last.
    Raises ``ValueError`` naming the instance ids of a cycle reachable from the target."""
    out = {}
    for i, j, _ in edges:
        out.setdefault(i, set()).add(j)
        out.setdefault(j, set())
    out.setdefault(target_id, set())
    _check_acyclic(out, target_id)
    order = []
    while out[target_id]:
        leaves, seen, stack = set(), {target_id}, [target_id]
        while stack:
            u = stack.pop()
            if not out[u]:
                leaves.add(u)
            for v in out[u]:
                if v not in seen:
                    seen.add(v)
                    stack.append(v)
        for leaf in sorted(leaves):
            order.append(leaf)
            del out[leaf]
            for succ in out.values():
                succ.discard(leaf)
    order.append(target_id)
    return order


def _check_acyclic(out, start):
    state, path = {}, []

    def visit(u):                             # iterative: a long chain must not recurse
        stack = [(u, iter(sorted(out[u])))]
        state[u] = 1
        path.append(u)
        while stack:
            node, it = stack[-1]
            nxt = next(it, None)
            if nxt is None:
                state[node] = 2
                path.pop()
                stack.pop()
            elif state.get(nxt) == 1:
                cycle = path[path.index(nxt):]
                raise ValueError(f"occlusion cycle among instance ids {cycle}: no picking order")
            elif nxt not in state:
                state[nxt] = 1
                path.append(nxt)
                stack.append((nxt, iter(sorted(out[nxt]))))

    visit(start)


class SelectPickingOrder:
    """The picking-order node's decision for one camera frame.  ``models`` has get_cad(class_id)
    (an object with ``.vertices`` and ``.faces``, as ``SyntheticYCBModels.get_cad``); ``target`` is
    the class id of the object to pick (the node's ``~target``)."""

    def __init__(self, models, target):
        self._models = models
        self._target = int(target)
        self._cads = {}

    def _cad(self, class_id):
        if class_id not in self._cads:
            self._cads[class_id] = self._models.get_cad(class_id)
        return self._cads[class_id]

    def __call__(self, instance_ids, class_ids, T_cad2base, sensor_to_world, K, height, width):
        """One frame (_callback, :195-296) on ``ObjectMapping.poses()``'s three outputs as they
        are: instance_ids [N], class_ids [N], T_cad2base [N,4,4]; sensor_to_world the camera's
        4x4 T_cam2base; K the 3x3 intrinsics of a height x width image.  One render and one host
        read.

        Returns (order, edges).  ``order`` is None when no instance has the target class (the node
        publishes nothing), [] when the target is not visible, and otherwise the instance ids in
        picking order, the target last.  ``edges`` are the (i, j, ratio) edges "i is occluded by
        j", in the node's insertion order (``occlusion_edges``)."""
        import torch
        from ..functions.geometry import _util
        ids = geometry._check_instance_ids(instance_ids)
        cls = np.asarray(class_ids, np.int64).reshape(-1)
        N = len(ids)
        if len(cls) != N:
            raise ValueError("instance_ids and class_ids differ in length")
        if N > geometry.MAX_SCENE_OBJECTS:
            raise ValueError(f"at most {geometry.MAX_SCENE_OBJECTS} instances, got {N}")
        if self._target not in cls.tolist():
            return None, []
        T = np.asarray(T_cad2base, np.float64).reshape(N, 4, 4)
        T_cad2cam = np.linalg.inv(np.asarray(sensor_to_world, np.float64).reshape(4, 4)) @ T
        H, W = int(height), int(width)
        fovy = geometry.fovy_from_intrinsics(np.asarray(K, np.float64).reshape(3, 3)[1, 1], H)
        f = geometry.focal_from_fovy(fovy, H)
        v, fc, offsets, mesh = geometry._pack_cads([self._cad(int(c)) for c in cls])
        dev = torch.device("cuda", torch.cuda.current_device())
        _, _, whole, occluded = geometry._render_instances_batch(
            _util.h2d_transient(v, dev, torch.float64), _util.h2d_transient(fc, dev, torch.int32),
            offsets, mesh, T_cad2cam, ids, f=f, height=H, width=W)
        counts = torch.cat([whole, occluded.reshape(-1)]).cpu().numpy()
        visible, edges = occlusion_edges(ids, counts[:N], counts[N:])
        target_nodes = [i for i in visible if cls[list(ids).index(i)] == self._target]
        if not target_nodes:
            return [], edges
        return picking_order(edges, target_nodes[-1]), edges
