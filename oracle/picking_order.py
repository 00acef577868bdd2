"""Float64 NumPy restatement of the picking-order node's scene render
(ros/src/morefusion_ros/nodes/select_picking_order.py:129-190, ``_render_object_pose_array``): the
posed objects rendered together into one camera, and the counts its occlusion graph is built
from.  TEST INFRASTRUCTURE ONLY; csrc/render_cad.cu (mf_render_scene) is checked against it bit
for bit.

The scene is the composite of oracle/render_cad.py's ``render_one`` per object, under the same
rules: each pixel shows the object of smallest float32 depth, the lower input index on an exact
tie (GL_LESS with the objects drawn in input order), and NaN / -1 where nothing covers.  Its
counts: ``whole[i]``, the pixels object i covers rendered alone (the node's ``mask_whole``), and
``occluded[i, j]``, the pixels of i's whole mask where j is visible (the node's per-occluder
``count``).

Also the inputs of the picking-order cases (``CASES``), regenerated from the case name and seed,
which oracle/ref_harness/gen_picking_order.py runs through the node's own code into
tests/golden/picking_order/.
"""

import numpy as np

from oracle import render_cad as orc

H, W = 120, 160                      # small, so that the NumPy oracle stays fast
FY = 200.0
TARGET = 5                           # sphere, 6.5 cm radius


def render_instances(meshes, Ts_cad2cam, instance_ids, f, height, width):
    """meshes: one (vertices, faces) per object; Ts_cad2cam [N,4,4]; instance_ids [N].  Returns
    depth [H,W] float32 (NaN where nothing covers), ins [H,W] int32 (-1 where nothing covers),
    whole [N] int64, occluded [N,N] int64 (zero diagonal) and the per-object masks [N,H,W]."""
    Ts = np.asarray(Ts_cad2cam, np.float64).reshape(-1, 4, 4)
    N = len(Ts)
    masks = np.zeros((N, height, width), bool)
    best = np.full((height, width), np.inf, np.float32)
    idx = np.full((height, width), -1, np.int64)
    for n, ((v, fc), T) in enumerate(zip(meshes, Ts)):
        d, m = orc.render_one(v, fc, T, f, height, width)
        masks[n] = m
        better = m & ((idx < 0) | (d < best))        # strict: a tie keeps the earlier object
        best[better] = d[better]
        idx[better] = n
    depth = np.where(idx >= 0, best, np.float32(np.nan)).astype(np.float32)
    ids = np.asarray(instance_ids, np.int64).reshape(-1)
    ins = np.where(idx >= 0, ids[np.maximum(idx, 0)] if N else -1, -1).astype(np.int32)
    whole = masks.reshape(N, -1).sum(1).astype(np.int64)
    occluded = np.zeros((N, N), np.int64)
    for i in range(N):
        for j in range(N):
            if i != j:
                occluded[i, j] = int((masks[i] & (idx == j)).sum())
    return depth, ins, whole, occluded, masks


# case name -> (seed, [(instance_id, class_id, (x, y, z) of the object's centre in the camera
# frame)]).  Objects lie along the view ray so that the nearer ones cover parts of the farther.
CASES = {
    # the target (7) behind A (3), A behind B (12)
    "chain": (1, [(7, TARGET, (0.0, 0.0, 1.0)), (3, 1, (0.06, 0.0, 0.8)),
                  (12, 3, (0.10, 0.02, 0.6))]),
    # the target (4) behind A (9) and B (2), both behind C (6)
    "diamond": (2, [(9, 1, (-0.05, 0.0, 0.8)), (4, TARGET, (0.0, 0.0, 1.0)),
                    (2, 4, (0.04, 0.0, 0.8)), (6, 6, (0.0, 0.03, 0.6))]),
    # nothing in front of the target (5); another object beside it
    "clear": (3, [(5, TARGET, (0.0, 0.0, 1.0)), (8, 3, (0.25, 0.0, 0.8))]),
    # the target (1) wholly behind a large box (11)
    "hidden": (4, [(11, 12, (0.0, 0.0, 0.4)), (1, TARGET, (0.0, 0.0, 1.2))]),
    # no instance of the target class
    "absent": (5, [(3, 1, (0.0, 0.0, 1.0)), (4, 3, (0.03, 0.0, 0.7))]),
    # two instances of the target class: the last visible one in id order (8) is the target node
    "two_targets": (6, [(8, TARGET, (0.12, 0.0, 1.0)), (2, TARGET, (-0.12, 0.0, 1.0)),
                        (5, 1, (0.16, 0.0, 0.7))]),
    # one occluder (10) just under the 10 % threshold and one (6) just over it
    "threshold": (7, [(3, TARGET, (0.0, 0.0, 1.0)), (10, 1, (-0.0827, 0.0, 0.8)),
                      (6, 4, (0.0715, 0.0, 0.8))]),
}


def _rotation(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def case_inputs(name):
    """(instance_ids [N] int64, class_ids [N] int32, T_cad2base [N,4,4], sensor_to_world [4,4],
    K [3,3], height, width) of a case: the seeded camera pose, and each object at its centre with
    a seeded rotation, moved to the world frame in float64."""
    seed, objs = CASES[name]
    rs = np.random.RandomState(seed)
    C = np.eye(4)
    C[:3, :3], C[:3, 3] = _rotation(rs), rs.uniform(-0.5, 0.5, 3)
    Ts = []
    for _, _, t in objs:
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = _rotation(rs), t
        Ts.append(C @ T)
    K = np.array([[FY, 0, W / 2.0], [0, FY, H / 2.0], [0, 0, 1]])
    return (np.array([o[0] for o in objs], np.int64), np.array([o[1] for o in objs], np.int32),
            np.array(Ts).reshape(-1, 4, 4), C, K, H, W)


def case_scene(name, models):
    """The render inputs of a case as the picking-order node derives them: (meshes, T_cad2cam
    [N,4,4] = inv(sensor_to_world) @ T_cad2base, instance_ids, f, height, width)."""
    ids, cls, T, C, K, height, width = case_inputs(name)
    T_cad2cam = np.linalg.inv(C) @ T
    f = orc.focal_from_fovy(orc.fovy_from_intrinsics(K[1, 1], height), height)
    meshes = []
    for c in cls:
        cad = models.get_cad(int(c))
        meshes.append((cad.vertices, cad.faces))
    return meshes, T_cad2cam, ids, f, height, width
