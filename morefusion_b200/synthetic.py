"""Synthetic YCB-shaped inputs for the volumetric-pose hot path (no datasets offline).

Shapes and conventions follow the reference's data pipeline:
  * 21 YCB classes, voxel pitch = bbox diagonal / 32 (datasets/ycb_video/models.py:113-115;
    table ros/src/morefusion_ros/include/morefusion_ros/utils/data.h:12-32)
  * origin = median(points) - pitch * 15.5 (model.py:197-205, rgbd_pose_estimation/base.py:153-156)
  * 1000 points per object, voxel-frame points = (cam - origin) / pitch (model.py:236)
  * grid_nontarget_empty: free space + other objects as seen from the camera (train.py:50-54)
Objects are boxes / cylinders / spheres whose bbox diagonal is 32 * pitch(class).
"""

import types

import numpy as np

from .contrib.singleview_3d.models.model import YCB_VOXEL_PITCH_32

F32 = np.float32


def init_weights(n_fg_class=21, seed=0, with_occupancy=True):
    """Seeded LeCun-normal weights (chainer's default initialiser) and small random biases for
    the 3-D section of the pose model, keyed by the reference's link names (model.py:62-91):
    {'<link>/W': ndarray, '<link>/b': ndarray}.  No trained weights exist offline."""
    rs = np.random.RandomState(seed)
    w = {}

    def conv(name, cout, cin, *k):
        fan_in = cin * int(np.prod(k)) if k else cin
        shape = (cout, cin) + tuple(k)
        w[name + "/W"] = (rs.normal(0, 1.0 / np.sqrt(fan_in), shape)).astype(np.float32)
        w[name + "/b"] = rs.uniform(-0.05, 0.05, cout).astype(np.float32)

    conv("conv1_rgb", 64, 32, 1)
    conv("conv1_pcd", 8, 3, 1)
    conv("conv2_rgb", 128, 64, 1)
    conv("conv2_pcd", 16, 8, 1)
    if with_occupancy:
        conv("conv1_occ", 8, 1, 3, 3, 3)
        conv("conv2_occ", 16, 8, 3, 3, 3)
    cin3 = 144 + (16 if with_occupancy else 0)
    conv("conv3", 256, cin3, 4, 4, 4)
    conv("conv4", 512, 256, 4, 4, 4)
    for head, cout in (("rot", n_fg_class * 4), ("trans", n_fg_class * 3), ("conf", n_fg_class)):
        conv(f"conv1_{head}", 640, 984, 1)
        conv(f"conv2_{head}", 256, 640, 1)
        conv(f"conv3_{head}", 128, 256, 1)
        conv(f"conv4_{head}", cout, 128, 1)
    return w


def init_weights_pcd(n_fg_class=21, seed=0):
    """Seeded LeCun-normal weights and small random biases for the singleview_pcd model
    (examples/ycb_video/singleview_pcd/contrib/models/model.py:53-67, :299-311), keyed by the
    reference's link paths: {'posenet_extractor/conv3/W': ndarray, 'conv1_rot/b': ndarray, ...}."""
    rs = np.random.RandomState(seed)
    w = {}

    def conv(name, cout, cin):
        w[name + "/W"] = rs.normal(0, 1.0 / np.sqrt(cin), (cout, cin, 1)).astype(np.float32)
        w[name + "/b"] = rs.uniform(-0.05, 0.05, cout).astype(np.float32)

    for name, cout, cin in (("conv1_rgb", 64, 32), ("conv1_pcd", 64, 3), ("conv2_rgb", 128, 64),
                            ("conv2_pcd", 128, 64), ("conv3", 512, 256), ("conv4", 1024, 512)):
        conv("posenet_extractor/" + name, cout, cin)
    for head, cout in (("rot", n_fg_class * 4), ("trans", n_fg_class * 3), ("conf", n_fg_class)):
        conv(f"conv1_{head}", 640, 1408)
        conv(f"conv2_{head}", 256, 640)
        conv(f"conv3_{head}", 128, 256)
        conv(f"conv4_{head}", cout, 128)
    return w


def _rot(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _primitive(class_id, kinds=("box", "cylinder", "sphere")):
    """kind, half-extents (metres) with bbox diagonal = 32 * pitch."""
    diag = 32.0 * YCB_VOXEL_PITCH_32[class_id]
    kind = kinds[class_id % len(kinds)]
    if kind == "box":
        ratio = np.array([1.0, 0.7, 0.45])
    elif kind == "cylinder":
        ratio = np.array([0.6, 0.6, 1.0])
    else:
        ratio = np.array([1.0, 1.0, 1.0])
    half = ratio / np.linalg.norm(2 * ratio) * diag
    return kind, half


def sdf_primitive(kind, half, p):
    """Signed distance, POSITIVE INSIDE (trimesh convention, datasets/ycb_video/models.py:77)."""
    if kind == "sphere":
        return half[0] - np.linalg.norm(p, axis=-1)
    if kind == "box":
        q = np.abs(p) - half
        outside = np.linalg.norm(np.maximum(q, 0), axis=-1)
        inside = np.minimum(q.max(axis=-1), 0)
        return -(outside + inside)
    # cylinder along z
    dr = np.linalg.norm(p[..., :2], axis=-1) - half[0]
    dz = np.abs(p[..., 2]) - half[2]
    outside = np.linalg.norm(np.maximum(np.stack([dr, dz], -1), 0), axis=-1)
    inside = np.minimum(np.maximum(dr, dz), 0)
    return -(outside + inside)


def surface_points(kind, half, n, rs):
    """Uniform-ish points on the primitive's surface (object frame)."""
    if kind == "sphere":
        d = rs.normal(size=(n, 3))
        return d / np.linalg.norm(d, axis=1, keepdims=True) * half[0]
    if kind == "box":
        p = rs.uniform(-1, 1, (n, 3)) * half
        ax = rs.randint(0, 3, n)
        p[np.arange(n), ax] = np.sign(rs.uniform(-1, 1, n)) * half[ax]
        return p
    th = rs.uniform(0, 2 * np.pi, n)
    z = rs.uniform(-1, 1, n) * half[2]
    p = np.stack([np.cos(th) * half[0], np.sin(th) * half[0], z], 1)
    cap = rs.uniform(size=n) < 0.25
    r = np.sqrt(rs.uniform(size=n)) * half[0]
    p[cap] = np.stack([np.cos(th) * r, np.sin(th) * r, np.sign(rs.uniform(-1, 1, n)) * half[2]], 1)[cap]
    return p


class SyntheticYCBModels:
    """Stand-in for morefusion.datasets.YCBVideoModels (a multi-GB download, unavailable
    offline) with the three methods the pose model touches (model.py:199, :353, :416):
    YCB-shaped primitives whose bounding-box diagonal is 32 x the class voxel pitch."""

    # datasets/ycb_video/class_names.py:32-46: bowl, wood_block, large_clamp, extra_large_clamp,
    # foam_brick
    class_ids_symmetric = np.array([13, 16, 19, 20, 21], dtype=np.int32)

    def __init__(self, n_pcd=2000, kinds=("box", "cylinder", "sphere")):
        self._n_pcd = n_pcd
        self._kinds = kinds
        self._pcd = {}

    def get_voxel_pitch(self, dimension, class_id):
        return 32.0 * YCB_VOXEL_PITCH_32[int(class_id)] / dimension

    def get_pcd(self, class_id):
        class_id = int(class_id)
        if class_id not in self._pcd:
            kind, half = _primitive(class_id, self._kinds)
            rs = np.random.RandomState(class_id)
            self._pcd[class_id] = surface_points(kind, half, self._n_pcd, rs).astype(F32)
        return self._pcd[class_id]

    def get_sdf(self, class_id):
        return sdf_lattice(int(class_id), self._kinds)

    def get_cad(self, class_id):
        """Stand-in for YCBVideoModels.get_cad (models.py:88-94, the loaded trimesh of
        textured_simple.obj): an object with ``.vertices`` [V,3] float64 and ``.faces`` [F,3]
        int32, a closed triangulation of the class primitive with every vertex on its surface and
        the faces wound outward.  A box is its 12 triangles; a cylinder has 32 segments around
        (two rings and a centre on each cap: 66 vertices, 128 faces); a sphere has 16 rings of
        latitude and 32 segments of longitude (two poles and 15 rings: 482 vertices, 960 faces)."""
        kind, half = _primitive(int(class_id), self._kinds)
        v, f = cad_mesh(kind, half)
        return types.SimpleNamespace(vertices=v, faces=f)

    def get_solid_voxel_grid(self, class_id):
        """Stand-in for YCBVideoModels.get_solid_voxel_grid (models.py:81-86, a binvox of the CAD
        model): an object whose ``.points`` [n,3] float64 are the lattice points inside the class
        primitive at half the class pitch, centred on the origin, so that the 32^3 grid of the
        class pitch has no holes; ``.pitch`` is that spacing."""
        class_id = int(class_id)
        kind, half = _primitive(class_id, self._kinds)
        pitch = YCB_VOXEL_PITCH_32[class_id] / 2.0
        ax = [np.arange(-np.floor(h / pitch), np.floor(h / pitch) + 1) * pitch for h in half]
        g = np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3)
        return types.SimpleNamespace(points=g[sdf_primitive(kind, half, g) >= 0], pitch=pitch)


def cad_mesh(kind, half, n_around=32, n_rings=16):
    """(vertices [V,3] float64, faces [F,3] int32) of the primitive, as ``get_cad`` states."""
    if kind == "box":
        v = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * half
        quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
        f = [t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))]
        return v, np.array(f, np.int32)
    phi = 2 * np.pi * np.arange(n_around) / n_around
    ring = np.stack([np.cos(phi), np.sin(phi)], 1)
    j = np.arange(n_around)
    k = (j + 1) % n_around
    if kind == "cylinder":
        r, h = half[0], half[2]
        v = np.concatenate([np.c_[r * ring, np.full(n_around, -h)], np.c_[r * ring, np.full(n_around, h)],
                            [[0.0, 0.0, -h], [0.0, 0.0, h]]])
        lo, hi, cb, ct = 0, n_around, 2 * n_around, 2 * n_around + 1
        f = np.concatenate([np.c_[lo + j, lo + k, hi + k], np.c_[lo + j, hi + k, hi + j],
                            np.c_[np.full(n_around, cb), lo + k, lo + j],
                            np.c_[np.full(n_around, ct), hi + j, hi + k]])
        return v, f.astype(np.int32)
    r = half[0]
    theta = np.pi * np.arange(1, n_rings) / n_rings
    body = np.concatenate([np.c_[r * np.sin(t) * ring, np.full(n_around, r * np.cos(t))] for t in theta])
    v = np.concatenate([[[0.0, 0.0, r]], body, [[0.0, 0.0, -r]]])
    south = len(v) - 1
    f = [np.c_[np.zeros(n_around, int), 1 + j, 1 + k]]
    for i in range(n_rings - 2):
        a, b = 1 + i * n_around, 1 + (i + 1) * n_around
        f += [np.c_[a + j, b + j, b + k], np.c_[a + j, b + k, a + k]]
    a = 1 + (n_rings - 2) * n_around
    f.append(np.c_[np.full(n_around, south), a + k, a + j])
    return v, np.concatenate(f).astype(np.int32)


def sdf_lattice(class_id, kinds=("box", "cylinder", "sphere")):
    """Stand-in for YCBVideoModels.get_sdf (models.py:66-79): interior lattice points at the
    class pitch with their signed distance (positive inside)."""
    kind, half = _primitive(class_id, kinds)
    pitch = YCB_VOXEL_PITCH_32[class_id]
    ax = [np.arange(-h, h + 1e-9, pitch) for h in half]
    g = np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3)
    d = sdf_primitive(kind, half, g)
    keep = d >= -0.5 * pitch
    return g[keep].astype(F32), d[keep].astype(F32)


def make_cnn_batch(B=8, P=1000, seed=0, D=32):
    """One batch of objects for the 3D-CNN hot path (BASELINE config 2 shape)."""
    rs = np.random.RandomState(seed)
    class_id = ((np.arange(B) + seed) % 21 + 1).astype(np.int32)
    values = rs.normal(0, 1, (B, 32, P)).astype(F32)      # stands in for PSPNet features
    points = np.zeros((B, 3, P), F32)
    pitch = np.zeros(B, F32)
    origin = np.zeros((B, 3), F32)
    gne = np.zeros((B, D, D, D), bool)
    for i in range(B):
        kind, half = _primitive(int(class_id[i]))
        pitch[i] = YCB_VOXEL_PITCH_32[int(class_id[i])]
        R = _rot(rs)
        t = np.array([rs.uniform(-0.2, 0.2), rs.uniform(-0.15, 0.15), rs.uniform(0.5, 0.8)])
        sp = surface_points(kind, half, 6 * P, rs)
        cam = sp @ R.T + t
        # visible side only: surface normal ~ (p - centre) facing the camera at the origin
        vis = ((cam - t) * (-cam)).sum(1) > 0
        cam = cam[vis]
        cam = cam + rs.normal(0, 0.003, cam.shape) * (cam / np.linalg.norm(cam, axis=1, keepdims=True))
        keep = rs.permutation(cam.shape[0])[:P]
        if keep.shape[0] < P:
            keep = np.r_[keep, rs.randint(0, cam.shape[0], P - keep.shape[0])]
        cam = cam[keep].astype(F32)
        origin[i] = (np.median(cam, axis=0) - pitch[i] * (D / 2.0 - 0.5)).astype(F32)
        points[i] = ((cam - origin[i]) / pitch[i]).T
        # free space in front of the surface along the viewing rays + a random occluder slab
        ijk = np.stack(np.meshgrid(*(np.arange(D),) * 3, indexing="ij"), -1).astype(F32)
        centres = ijk * pitch[i] + origin[i]
        obj = (centres - t) @ R
        inside = sdf_primitive(kind, half, obj) > 0
        front = np.linalg.norm(centres, axis=-1) < np.linalg.norm(t) - 0.3 * half.max()
        slab = np.abs(centres[..., 0] - (t[0] + half.max() * 1.2)) < 2 * pitch[i]
        gne[i] = (front | slab) & ~inside
    return dict(class_id=class_id, values=values, points=points, pitch=pitch, origin=origin,
                grid_nontarget_empty=gne)


CAMERA_K = np.array([[619.44, 0, 326.82], [0, 619.32, 239.52], [0, 0, 1.0]])   # pose_refinement/data/camera_info.yaml


# seeds of the example scripts' synthetic validation batches: batch k is seed VALID_SEED + k, far
# above any training batch's seed ((epoch * iters_per_epoch + it) * n_gpu + rank)
VALID_SEED = 2 ** 31


def make_validation_batch(k, batch_size=48):
    """Validation batch k of the example scripts (make_rgbd_batch with a seed no training batch
    uses)."""
    return make_rgbd_batch(batch_size, seed=VALID_SEED + int(k))


def make_rgbd_batch(B=8, H=256, W=256, seed=0, D=32):
    """Synthetic stand-in for one batch of the RGB-D pose-estimation datasets
    (datasets/rgbd_pose_estimation/base.py:125-156): per object a centred H x W crop with
    ``rgb`` uint8, ``pcd`` float32 camera-frame points (NaN where there is no depth: background,
    5 % dropout), the ground-truth pose, class id, pitch, origin and a non-target/empty grid --
    the keyword arguments of Model.__call__ (model.py:277-288)."""
    rs = np.random.RandomState(seed)
    class_id = ((np.arange(B) * 3 + seed) % 21 + 1).astype(np.int32)
    rgb = rs.randint(0, 255, (B, H, W, 3)).astype(np.uint8)
    pcd = np.full((B, H, W, 3), np.nan, F32)
    q_true = np.zeros((B, 4), F32)
    t_true = np.zeros((B, 3), F32)
    pitch = np.zeros(B, F32)
    origin = np.zeros((B, 3), F32)
    gne = np.zeros((B, D, D, D), bool)
    f = CAMERA_K[0, 0] * 2.2           # crop magnification: the object fills most of the crop
    for i in range(B):
        kind, half = _primitive(int(class_id[i]))
        pitch[i] = YCB_VOXEL_PITCH_32[int(class_id[i])]
        R = _rot(rs)
        t = np.array([rs.uniform(-0.02, 0.02), rs.uniform(-0.02, 0.02), rs.uniform(0.55, 0.75)])
        sp = surface_points(kind, half, 60000, rs)
        cam = sp @ R.T + t
        cam = cam[((cam - t) * (-cam)).sum(1) > 0]                      # camera-facing side
        cam += rs.normal(0, 0.003, cam.shape) * (cam / np.linalg.norm(cam, axis=1, keepdims=True))
        u = np.round(f * cam[:, 0] / cam[:, 2] + W / 2 - f * t[0] / t[2]).astype(int)
        v = np.round(f * cam[:, 1] / cam[:, 2] + H / 2 - f * t[1] / t[2]).astype(int)
        ok = (u >= 0) & (u < W) & (v >= 0) & (v < H)
        order = np.argsort(-cam[ok, 2])                                 # nearest point wins
        uu, vv, cc = u[ok][order], v[ok][order], cam[ok][order]
        pcd[i, vv, uu] = cc.astype(F32)
        drop = rs.rand(H, W) < 0.05
        pcd[i][drop] = np.nan
        rgb[i][~np.isnan(pcd[i, :, :, 2])] //= 2
        # quaternion (w, x, y, z) of R
        tr = np.trace(R)
        w_ = np.sqrt(max(1 + tr, 1e-12)) / 2
        q = np.array([w_, (R[2, 1] - R[1, 2]) / (4 * w_), (R[0, 2] - R[2, 0]) / (4 * w_),
                      (R[1, 0] - R[0, 1]) / (4 * w_)])
        q_true[i] = (q / np.linalg.norm(q)).astype(F32)
        t_true[i] = t.astype(F32)
        valid = pcd[i][~np.isnan(pcd[i]).any(axis=2)]
        origin[i] = (np.median(valid, axis=0) - pitch[i] * (D / 2.0 - 0.5)).astype(F32)
        ijk = np.stack(np.meshgrid(*(np.arange(D),) * 3, indexing="ij"), -1).astype(F32)
        centres = ijk * pitch[i] + origin[i]
        inside = sdf_primitive(kind, half, (centres - t) @ R) > 0
        front = np.linalg.norm(centres, axis=-1) < np.linalg.norm(t) - 0.3 * half.max()
        gne[i] = front & ~inside
    return dict(class_id=class_id, rgb=rgb, pcd=pcd, quaternion_true=q_true, translation_true=t_true,
                pitch=pitch, origin=origin, grid_nontarget_empty=gne)


def make_icc_scene(N=8, seed=0, D=32, t_noise=0.01, rot_noise_deg=10.0,
                   kinds=("box", "cylinder", "sphere"), spacing=0.085):
    """Synthetic stand-in for examples/ycb_video/pose_refinement/data (BASELINE config 4):
    N YCB-shaped primitives resting in contact in a bin, SDF lattice points per object
    (models.get_sdf stand-in), ground-truth poses, perturbed initial poses
    (t ~ N(0, 1 cm), rotation ~ U(0, 10 deg)), per-object 32^3 target / non-target+empty grids."""
    rs = np.random.RandomState(seed)
    class_id = ((np.arange(N) * 5 + seed) % 21 + 1).astype(np.int32)
    prims = [_primitive(int(c), kinds) for c in class_id]
    # place objects on a jittered lattice so that neighbours touch
    T_true = []
    cols = int(np.ceil(np.sqrt(N)))
    for i, (kind, half) in enumerate(prims):
        R = _rot(rs)
        r = float(np.linalg.norm(half))
        cx = (i % cols - (cols - 1) / 2.0) * spacing + rs.uniform(-0.01, 0.01)
        cy = (i // cols - (cols - 1) / 2.0) * spacing + rs.uniform(-0.01, 0.01)
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = [cx, cy, 0.7 + rs.uniform(-0.02, 0.02) + 0.0 * r]
        T_true.append(T)
    T_true = np.stack(T_true)
    points, sdf, pitch, origin = [], [], [], []
    for i, c in enumerate(class_id):
        p, s = sdf_lattice(int(c), kinds)
        points.append(p)
        sdf.append(s)
        pitch.append(YCB_VOXEL_PITCH_32[int(c)])
        origin.append(T_true[i, :3, 3] - pitch[-1] * (D / 2.0 - 0.5))
    pitch = np.array(pitch, F32)
    origin = np.array(origin, F32)
    gt_grid = np.zeros((N, D, D, D), F32)
    gne = np.zeros((N, D, D, D), F32)
    ijk = np.stack(np.meshgrid(*(np.arange(D),) * 3, indexing="ij"), -1).astype(np.float64)
    for i in range(N):
        centres = ijk * pitch[i] + origin[i]
        d_all = []
        for j, (kind, half) in enumerate(prims):
            obj = (centres - T_true[j, :3, 3]) @ T_true[j, :3, :3]
            d_all.append(sdf_primitive(kind, half, obj))
        d_all = np.stack(d_all)
        d_self = d_all[i]
        # visible (camera-facing) surface shell of object i
        normal_out = centres - T_true[i, :3, 3]
        facing = (normal_out * (-centres)).sum(-1) > 0
        gt_grid[i] = ((np.abs(d_self) < 0.75 * pitch[i]) & facing)
        others = np.delete(d_all, i, 0).max(0) > 0 if N > 1 else np.zeros_like(d_self, bool)
        free = (d_all.max(0) < -1.5 * pitch[i]) & (centres[..., 2] < T_true[i, 2, 3])
        gne[i] = (others | free) & ~(d_self > 0)
    # perturbed initial poses
    T_init = []
    for i in range(N):
        ax = rs.normal(size=3)
        ax /= np.linalg.norm(ax)
        ang = np.deg2rad(rs.uniform(0, rot_noise_deg))
        K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        dR = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K
        T = T_true[i].copy()
        T[:3, :3] = T[:3, :3] @ dR
        T[:3, 3] += rs.normal(0, t_noise, 3)
        T_init.append(T)
    return dict(class_id=class_id, points=points, sdf=sdf, pitch=pitch, origin=origin,
                grid_target=gt_grid, grid_nontarget_empty=gne,
                transform_init=np.stack(T_init).astype(F32), transform_true=T_true.astype(F32),
                primitives=prims)


def make_depth_frame(seed=0, H=480, W=640, n_objects=8):
    """A 640x480 synthetic RGB-D frame for the occupancy-map producer (SURVEY.md 8f-3, cfg5
    geometry): `n_objects` YCB-sized boxes at 0.55-0.65 m in front of a tilted table at 0.9-1.1 m,
    camera intrinsics of examples/ycb_video/pose_refinement/data/camera_info.yaml scale (fx ~ 600),
    3 mm depth noise and 5 % dropout (datasets/rgbd_pose_estimation/reindexed.py:70-75).
    Returns (pcd [H,W,3] f32 with NaN rows, instance label [H,W] int32 (0 = background),
    class_ids [n_objects], pitches {instance_id: voxel pitch}); instance ids are 1..n_objects."""
    rs = np.random.RandomState(seed)
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    fx = 600.0
    z = 0.9 + 0.2 * (v / H)
    label = np.zeros((H, W), np.int32)
    class_ids = [1 + (seed + 3 * i) % 21 for i in range(n_objects)]
    pitches = {0: 0.01}
    for ins in range(1, n_objects + 1):
        cu = int(W * (ins - 0.5) / n_objects) + rs.randint(-8, 9)
        cv = H // 2 - 60 + 30 * (ins % 4)
        m = (np.abs(u - cu) < 28) & (np.abs(v - cv) < 36)
        z = np.where(m, 0.55 + 0.03 * (ins % 3) + 0.01 * ((u - cu) / 28.0) ** 2, z)
        label[m] = ins
        pitches[ins] = float(YCB_VOXEL_PITCH_32[class_ids[ins - 1]])
    z = z + 0.003 * rs.randn(H, W)
    pcd = np.stack([(u - W / 2) * z / fx, (v - H / 2) * z / fx, z], -1).astype(F32)
    pcd[rs.rand(H, W) < 0.05] = np.nan
    return pcd, label, class_ids, pitches


# instance ids of make_rgbd_frame's eight fixed objects (not contiguous) and its unlisted label
RGBD_FRAME_IDS = dict(top=3, bottom=7, tall=200, wide=65535, exact=11, large=12, pixel=13,
                      nodepth=14)
RGBD_FRAME_UNLISTED = 99


def _blob(rs, h, w, holes=0.04):
    """Irregular mask filling an h x w box: a wobbly ellipse with scattered holes, touching all
    four sides of the box (so the box is its bounding box)."""
    yy, xx = np.mgrid[0:h, 0:w]
    ang = np.arctan2((yy - (h - 1) / 2) / max(h, 1), (xx - (w - 1) / 2) / max(w, 1))
    r = np.hypot((yy - (h - 1) / 2) / max(h / 2, 0.5), (xx - (w - 1) / 2) / max(w / 2, 0.5))
    k = rs.randint(3, 7)
    m = r < 0.85 + 0.15 * np.sin(k * ang + rs.uniform(0, 2 * np.pi))
    m &= rs.rand(h, w) >= holes
    m[0, w // 2] = m[h - 1, w // 2] = m[h // 2, 0] = m[h // 2, w - 1] = True
    return m


def make_rgbd_frame(seed=0, H=480, W=640, n_objects=8, depth_mm=False):
    """A labelled RGB-D frame for the per-instance front end (FramePoseEstimator): a tilted
    table at 0.9-1.1 m, objects at 0.55-0.7 m, 3 mm depth noise, 5 % dropout, intrinsics
    CAMERA_K.  The first eight objects (RGBD_FRAME_IDS) are the crop's edge cases: irregular
    masks with holes, objects on all four image borders, a 1-pixel instance, an instance with
    no depth at all, a 320 x 6 and a 4 x 300 crop, a crop of exactly 256 x 256 and one of
    300 x 300; further objects are random blobs with ids 20, 21, ... painted underneath.  Label
    99 is an object nobody listed (it belongs to the background), 0 is the table.

    Returns dict(rgb [H,W,3] uint8, depth [H,W] (float32 metres, NaN = none; uint16
    millimetres, 0 = none, with depth_mm), label [H,W] int32, K [3,3], instance_ids [n_objects]
    int64, class_ids [n_objects] int32)."""
    if H < 480 or W < 640:
        raise ValueError("make_rgbd_frame needs at least 480 x 640")
    rs = np.random.RandomState(seed)
    label = np.zeros((H, W), np.int32)
    z = 0.9 + 0.2 * np.arange(H)[:, None] / H * np.ones((1, W))
    ids_fixed = list(RGBD_FRAME_IDS.values())
    extra = list(range(20, 20 + max(0, n_objects - len(ids_fixed))))

    def paint(ins, y, x, m, depth):
        h, w = m.shape
        sl = (slice(y, y + h), slice(x, x + w))
        label[sl][m] = ins
        bulge = 0.02 * ((np.arange(w) - (w - 1) / 2) / max(w / 2, 1))[None, :] ** 2
        z[sl][m] = (depth + bulge + np.zeros((h, 1)))[m]

    for ins in extra:                            # underneath: the fixed objects are painted last
        h, w = rs.randint(8, 90, 2)
        paint(ins, rs.randint(0, H - h), rs.randint(0, W - w), _blob(rs, h, w), rs.uniform(0.55, 0.7))
    fixed = [
        (RGBD_FRAME_IDS["top"], 0, 100, _blob(rs, 61, 161)),
        (RGBD_FRAME_IDS["bottom"], H - 10, 100, _blob(rs, 10, 201)),
        (RGBD_FRAME_IDS["tall"], 100, 0, _blob(rs, 320, 6, holes=0.1)),
        (RGBD_FRAME_IDS["wide"], 100, W - 300, _blob(rs, 4, 300, holes=0.1)),
        (RGBD_FRAME_IDS["exact"], 200, 40, _blob(rs, 256, 256)),
        (RGBD_FRAME_IDS["large"], 170, 330, _blob(rs, 300, 300)),
        (RGBD_FRAME_IDS["pixel"], 130, 20, np.ones((1, 1), bool)),
        (RGBD_FRAME_IDS["nodepth"], 110, 150, _blob(rs, 31, 51)),
        (RGBD_FRAME_UNLISTED, 62, 300, _blob(rs, 29, 31)),
    ]
    for ins, y, x, m in fixed:
        paint(ins, y, x, m, rs.uniform(0.55, 0.7))
    z = z + 0.003 * rs.randn(H, W)
    z[rs.rand(H, W) < 0.05] = np.nan
    z[label == RGBD_FRAME_IDS["pixel"]] = 0.6
    z[label == RGBD_FRAME_IDS["nodepth"]] = np.nan
    z = z.astype(F32)
    rgb = np.empty((H, W, 3), np.uint8)
    rgb[...] = (np.arange(W)[None, :, None] * np.array([1, 2, 3]) // 7 % 256).astype(np.uint8)
    for ins in np.unique(label)[1:]:
        m = label == ins
        rgb[m] = rs.randint(0, 256, 3)
    rgb = np.clip(rgb.astype(np.int64) + rs.randint(-20, 21, (H, W, 3)), 0, 255).astype(np.uint8)
    ids = np.array((ids_fixed + extra)[:n_objects], np.int64)
    class_ids = np.array([1 + (seed + 5 * i) % 21 for i in range(n_objects)], np.int32)
    if depth_mm:
        depth = np.where(np.isnan(z), 0, np.round(z.astype(np.float64) * 1000)).astype(np.uint16)
    else:
        depth = z
    return dict(rgb=rgb, depth=depth, label=label, K=CAMERA_K.copy(), instance_ids=ids,
                class_ids=class_ids)


# make_rgbd_views: the last view stands farther from the scene than this, so that some of its
# rays are clipped by an occupancy server launched with max_range = VIEWS_MAX_RANGE
VIEWS_MAX_RANGE = 1.2


def _look_at(eye, target):
    """sensor_to_world [4,4] of a camera at `eye` looking at `target` (OpenCV axes: z forward,
    x right, y down; world z up)."""
    z = target - eye
    z = z / np.linalg.norm(z)
    x = np.cross(z, [0.0, 0.0, 1.0])
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, eye
    return T


def make_rgbd_views(seed, n_views, H=480, W=640, n_objects=8):
    """One static seeded scene seen by a moving camera, for the occupancy server's multi-view
    map (MultiInstanceOctreeMapping.integrate_scan): `n_objects` YCB-sized oriented boxes
    (bounding-box diagonal 32 x the class pitch) resting on a 1.2 m square table at world z = 0, rendered
    by analytic ray casting from `n_views` camera poses on a ring 0.55-0.8 m from the scene,
    looking down at it.  The last view (of two or more) stands 1.6 m off: its table rays run
    beyond VIEWS_MAX_RANGE.  Intrinsics CAMERA_K scaled to W x H.

    Per view: rgb [H,W,3] uint8, depth [H,W] float32 metres with 3 mm noise and 5 % dropout
    (NaN), label [H,W] int32 -- instance ids 1..n_objects, the same in every view; -1 for the
    table and for pixels that see nothing; -2 on a two-pixel band along object edges --, and
    sensor_to_world [4,4] float64.  Object `peek_id` is labelled on ONE pixel of view 0 (an
    even row and column with depth; the rest of it is -2 there): an object first seen by one
    pixel only.

    Returns dict(views=[dict(rgb, depth, label, sensor_to_world)], K [3,3], instance_ids
    [n_objects] int64, class_ids [n_objects] int32, peek_id)."""
    rs = np.random.RandomState(seed)
    K = CAMERA_K.copy()
    K[0] *= W / 640.0
    K[1] *= H / 480.0
    ids = np.arange(1, n_objects + 1, dtype=np.int64)
    class_ids = rs.randint(1, 22, n_objects).astype(np.int32)
    boxes = []                                           # (centre, R (box -> world), half)
    for n, c in enumerate(class_ids):
        diag = 32.0 * YCB_VOXEL_PITCH_32[int(c)]
        ratio = np.array([1.0, 0.7, 0.45])
        half = ratio / np.linalg.norm(2 * ratio) * diag
        ang = 2 * np.pi * n / n_objects + rs.uniform(-0.3, 0.3)
        r = rs.uniform(0.05, 0.2) if n_objects > 1 else 0.0
        yaw = rs.uniform(0, 2 * np.pi)
        R = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1.0]])
        boxes.append((np.array([r * np.cos(ang), r * np.sin(ang), half[2]]), R, half))
    target = np.array([0.0, 0.0, 0.05])
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    ray_cam = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u, float)], -1)
    colours = rs.randint(0, 256, (n_objects, 3))
    views = []
    for k in range(n_views):
        far = n_views >= 2 and k == n_views - 1
        az = 2 * np.pi * k / max(n_views, 1) + rs.uniform(-0.2, 0.2)
        dist = 1.6 if far else rs.uniform(0.55, 0.8)
        elev = rs.uniform(0.6, 1.0)
        eye = target + dist * np.array([np.cos(az) * np.cos(elev), np.sin(az) * np.cos(elev),
                                        np.sin(elev)])
        T = _look_at(eye, target)
        d = ray_cam @ T[:3, :3].T                        # world direction per pixel, depth units
        depth = np.full((H, W), np.inf)
        label = np.full((H, W), -1, np.int32)
        with np.errstate(divide="ignore", invalid="ignore"):
            t_table = np.where(d[..., 2] < 0, -eye[2] / d[..., 2], np.inf)
            on = (np.abs(eye[:2] + t_table[..., None] * d[..., :2]) < 0.6).all(-1)
        depth = np.where(on, t_table, np.inf)            # a 1.2 m square table
        for n, (c, R, half) in enumerate(boxes):         # slab test in the box frame
            o_b = R.T @ (eye - c)
            d_b = d @ R
            with np.errstate(divide="ignore", invalid="ignore"):
                t1 = (-half - o_b) / d_b
                t2 = (half - o_b) / d_b
            tn = np.nanmax(np.minimum(t1, t2), -1)
            tf = np.nanmin(np.maximum(t1, t2), -1)
            hit = (tn <= tf) & (tn > 0) & (tn < depth)
            depth[hit] = tn[hit]
            label[hit] = ids[n]
        edge = np.zeros((H, W), bool)                    # -2 along object edges, 2 px wide
        for a in (0, 1):
            for s in (1, 2):
                diff = np.roll(label, s, a) != label
                edge |= diff & (label > 0)
                edge |= np.roll(diff & (np.roll(label, s, a) > 0), -s, a)
        label[edge] = -2
        z = depth + 0.003 * rs.randn(H, W)
        z[~np.isfinite(depth) | (rs.rand(H, W) < 0.05)] = np.nan
        label[~np.isfinite(depth)] = -1
        z = z.astype(F32)
        if k == 0:
            peek = int(ids[rs.randint(n_objects)])
            m = label == peek
            even = m & ~np.isnan(z)
            even[1::2] = False
            even[:, 1::2] = False
            label[m] = -2
            if even.any():
                first = np.flatnonzero(even)[0]
                label.reshape(-1)[first] = peek
        rgb = np.empty((H, W, 3), np.int64)
        rgb[...] = 128 + 60 * ((u // 16 + v // 16) % 2)[..., None]
        for n in range(n_objects):
            rgb[label == ids[n]] = colours[n]
        rgb = np.clip(rgb + rs.randint(-20, 21, (H, W, 3)), 0, 255).astype(np.uint8)
        views.append(dict(rgb=rgb, depth=z, label=label, sensor_to_world=T))
    return dict(views=views, K=K, instance_ids=ids, class_ids=class_ids, peek_id=peek)


def _small_rotation(rs, min_deg, max_deg):
    """A rotation about a random axis by an angle uniform in [min_deg, max_deg]."""
    ax = rs.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = np.deg2rad(rs.uniform(min_deg, max_deg))
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def make_icp_scene(M=8, seed=0, n_surface=12000, noise=0.003, n_outliers=5, t_err=0.01,
                   rot_err_deg=5.0, models=None):
    """Posed instances for ICP refinement (contrib.ICPRegistration): per instance the class's CAD
    points (``SyntheticYCBModels.get_pcd``), a true pose in the camera frame (0.6-0.9 m ahead,
    spread over the view), the camera-facing side of a fresh sample of the same surface at that
    pose with `noise` (3 mm) Gaussian noise and `n_outliers` points 3-10 cm off the object, and
    an initial pose off the true one by half to all of `t_err` (1 cm) and `rot_err_deg` (5 deg):
    far enough that a refinement has to move it.

    Returns dict(class_id [M] int32, pcd_depth [M] list of [n_m,3] float32 (camera frame),
    pcd_cad [M] list of [K,3] float32 (object frame), transform_true [M,4,4] and transform_init
    [M,4,4] float64, CAD -> camera)."""
    rs = np.random.RandomState(seed)
    models = models or SyntheticYCBModels()
    class_id = ((np.arange(M) * 7 + seed) % 21 + 1).astype(np.int32)
    cols = int(np.ceil(np.sqrt(M)))
    depth, cad, T_true, T_init = [], [], [], []
    for i, c in enumerate(class_id):
        kind, half = _primitive(int(c))
        T = np.eye(4)
        T[:3, :3] = _rot(rs)
        z = rs.uniform(0.6, 0.9)
        T[:3, 3] = [(i % cols - (cols - 1) / 2.0) * 0.2 * z, (i // cols - (cols - 1) / 2.0) * 0.2 * z, z]
        p = surface_points(kind, half, n_surface, rs) @ T[:3, :3].T + T[:3, 3]
        facing = ((p - T[:3, 3]) * -p).sum(1) > 0
        p = p[facing] + rs.normal(0, noise, (int(facing.sum()), 3))
        d = rs.normal(size=(n_outliers, 3))
        d *= rs.uniform(0.03, 0.1, (n_outliers, 1)) / np.linalg.norm(d, axis=1, keepdims=True)
        p = np.concatenate([p, T[:3, 3] + d * (1 + np.linalg.norm(half) / 0.03)])
        depth.append(p[rs.permutation(len(p))].astype(F32))
        cad.append(models.get_pcd(int(c)))
        T0 = T.copy()
        T0[:3, :3] = T[:3, :3] @ _small_rotation(rs, 0.5 * rot_err_deg, rot_err_deg)
        v = rs.normal(size=3)
        T0[:3, 3] += v / np.linalg.norm(v) * rs.uniform(0.5 * t_err, t_err)
        T_true.append(T)
        T_init.append(T0)
    return dict(class_id=class_id, pcd_depth=depth, pcd_cad=cad, transform_true=np.stack(T_true),
                transform_init=np.stack(T_init))


def make_icp_frame(seed=0, n_objects=8, H=480, W=640, n_surface=40000):
    """``make_icp_scene``'s instances splatted into a labelled RGB-D frame with a z-buffer
    (intrinsics CAMERA_K; every pixel keeps its nearest point; no depth elsewhere), for the frame
    path's ICP.  The 3 mm depth noise is added after the z-buffer, so that it does not pull the
    surface towards the camera.  Returns make_rgbd_frame's dict (float32 metres, NaN = none;
    instance ids 1..n_objects) plus transform_true / transform_init [n_objects,4,4]."""
    s = make_icp_scene(n_objects, seed, n_surface=n_surface, noise=0.0)
    rs = np.random.RandomState(seed + 1)
    K = CAMERA_K
    zbuf = np.full(H * W, np.inf)
    label = np.zeros(H * W, np.int32)
    for i, p in enumerate(s["pcd_depth"]):
        p = p.astype(np.float64)
        u = np.round(p[:, 0] / p[:, 2] * K[0, 0] + K[0, 2]).astype(np.int64)
        v = np.round(p[:, 1] / p[:, 2] * K[1, 1] + K[1, 2]).astype(np.int64)
        ok = (u >= 0) & (u < W) & (v >= 0) & (v < H) & (p[:, 2] > 0)
        pix, z = v[ok] * W + u[ok], p[ok, 2]
        order = np.lexsort((z, pix))                      # per pixel, the nearest point first
        pix, z = pix[order], z[order]
        first = np.r_[True, pix[1:] != pix[:-1]]
        pix, z = pix[first], z[first]
        win = z < zbuf[pix]
        zbuf[pix[win]] = z[win]
        label[pix[win]] = i + 1
    depth = np.where(np.isfinite(zbuf), zbuf + rs.normal(0, 0.003, H * W), np.nan)
    depth = depth.astype(F32).reshape(H, W)
    label = label.reshape(H, W)
    rgb = rs.randint(0, 256, (H, W, 3)).astype(np.uint8)
    return dict(rgb=rgb, depth=depth, label=label, K=K.copy(),
                instance_ids=np.arange(1, n_objects + 1, dtype=np.int64), class_ids=s["class_id"],
                transform_true=s["transform_true"], transform_init=s["transform_init"])


def make_pose_frame(seed, n_objects=8, H=480, W=640, spacing=0.085, n_surface=40000):
    """A labelled RGB-D frame with ground-truth poses for the training-example builder:
    ``make_icc_scene``'s touching primitives (``spacing`` apart on a jittered lattice; less than
    about 0.06 makes neighbours interpenetrate) at about 0.7 m over a table plane 0.12 m behind
    their centres (label 0), splatted with a z-buffer as ``make_icp_frame`` does (intrinsics
    CAMERA_K, every pixel keeps its nearest point), 2 mm depth noise after the z-buffer.  Returns
    get_frame's keys: instance_ids [n] (1..n), class_ids [n] int32, rgb [H,W,3] uint8 (a colour
    per instance, speckled), depth [H,W] float32 metres (NaN = none), instance_label [H,W] int32,
    intrinsic_matrix [3,3], Ts_cad2cam [n,4,4] float64."""
    sc = make_icc_scene(n_objects, seed, spacing=spacing)
    rs = np.random.RandomState(seed + 1)
    K = CAMERA_K
    v, u = np.mgrid[0:H, 0:W]
    zbuf = np.full(H * W, 0.7 + 0.12)                 # the table, facing the camera
    label = np.zeros(H * W, np.int32)
    Ts = sc["transform_true"].astype(np.float64)
    for i, (kind, half) in enumerate(sc["primitives"]):
        p = surface_points(kind, half, n_surface, rs) @ Ts[i, :3, :3].T + Ts[i, :3, 3]
        pu = np.round(p[:, 0] / p[:, 2] * K[0, 0] + K[0, 2]).astype(np.int64)
        pv = np.round(p[:, 1] / p[:, 2] * K[1, 1] + K[1, 2]).astype(np.int64)
        ok = (pu >= 0) & (pu < W) & (pv >= 0) & (pv < H) & (p[:, 2] > 0)
        pix, z = pv[ok] * W + pu[ok], p[ok, 2]
        order = np.lexsort((z, pix))
        pix, z = pix[order], z[order]
        first = np.r_[True, pix[1:] != pix[:-1]]
        pix, z = pix[first], z[first]
        win = z < zbuf[pix]
        zbuf[pix[win]] = z[win]
        label[pix[win]] = i + 1
    depth = (zbuf + rs.normal(0, 0.002, H * W)).astype(F32).reshape(H, W)
    label = label.reshape(H, W)
    colour = rs.randint(0, 256, (n_objects + 1, 3))
    rgb = np.clip(colour[label] + rs.randint(-20, 21, (H, W, 3)), 0, 255).astype(np.uint8)
    return dict(instance_ids=np.arange(1, n_objects + 1, dtype=np.int64),
                class_ids=sc["class_id"].astype(np.int32), rgb=rgb, depth=depth,
                instance_label=label, intrinsic_matrix=K.copy(), Ts_cad2cam=Ts)


def icp_link_clouds(scene, models=None):
    """The clouds of check_iterative_closest_point_link.py for a scene with ``class_id``, ``pitch``,
    ``origin`` and ``grid_target`` (make_icc_scene's, or the committed reference scene's): per
    instance the CAD cloud ``models.get_pcd(class_id)`` (SyntheticYCBModels: 2000 surface points)
    and the target cloud, the voxel centres of grid_target >= 0.5 (argwhere * pitch + origin),
    float32.  Returns (sources, targets), two lists."""
    models = SyntheticYCBModels() if models is None else models
    sources, targets = [], []
    for i, c in enumerate(scene["class_id"]):
        sources.append(models.get_pcd(int(c)))
        ijk = np.argwhere(np.asarray(scene["grid_target"][i]) >= 0.5)
        targets.append((ijk.astype(F32) * F32(scene["pitch"][i]) + np.asarray(scene["origin"][i], F32))
                       .astype(F32))
    return sources, targets
