"""Host-side geometry helpers used at link construction time (NumPy, not on the hot path).

The reference initialises ICC parameters with trimesh.transformations.quaternion_from_matrix /
translation_from_matrix (contrib/iterative_collision_check_link.py:21-25)."""

import numpy as np


def quaternion_from_matrix(matrix):
    """Rotation part of a 4x4 (or 3x3) -> unit quaternion (w, x, y, z) with w >= 0.

    Branch-on-largest-diagonal (Shepperd) extraction: numerically stable and, up to
    round-off, the same quaternion trimesh's eigen-decomposition returns."""
    M = np.asarray(matrix, dtype=np.float64)
    m = M[:3, :3]
    tr = m[0, 0] + m[1, 1] + m[2, 2]
    if tr > 0.0:
        s = np.sqrt(tr + 1.0) * 2.0
        q = np.array([0.25 * s, (m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s,
                      (m[1, 0] - m[0, 1]) / s])
    elif m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
        s = np.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]) * 2.0
        q = np.array([(m[2, 1] - m[1, 2]) / s, 0.25 * s, (m[0, 1] + m[1, 0]) / s,
                      (m[0, 2] + m[2, 0]) / s])
    elif m[1, 1] > m[2, 2]:
        s = np.sqrt(1.0 + m[1, 1] - m[0, 0] - m[2, 2]) * 2.0
        q = np.array([(m[0, 2] - m[2, 0]) / s, (m[0, 1] + m[1, 0]) / s, 0.25 * s,
                      (m[1, 2] + m[2, 1]) / s])
    else:
        s = np.sqrt(1.0 + m[2, 2] - m[0, 0] - m[1, 1]) * 2.0
        q = np.array([(m[1, 0] - m[0, 1]) / s, (m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s,
                      0.25 * s])
    q /= np.linalg.norm(q)
    if q[0] < 0.0:
        q = -q
    return q


def translation_from_matrix(matrix):
    return np.array(matrix, copy=True)[:3, 3]


def quaternion_matrix(quaternion):
    """trimesh.transformations.quaternion_matrix: q (w, x, y, z) -> homogeneous rotation [4,4] in
    float64, q normalised inside; a q with |q|^2 below 4 eps gives the identity."""
    q = np.array(quaternion, dtype=np.float64, copy=True).reshape(4)
    n = np.dot(q, q)
    if n < np.finfo(float).eps * 4.0:
        return np.identity(4)
    q *= np.sqrt(2.0 / n)
    q = np.outer(q, q)
    return np.array([
        [1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0], 0.0],
        [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0], 0.0],
        [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2], 0.0],
        [0.0, 0.0, 0.0, 1.0]])


def compose_transform(R=None, t=None):
    """morefusion.geometry.compose_transform on the host: [4,4] float64 with rotation R [3,3] and
    translation t [3] (identity / zero when None)."""
    T = np.eye(4)
    if R is not None:
        T[:3, :3] = R
    if t is not None:
        T[:3, 3] = t
    return T


def transformation_matrix(quaternion, translation):
    """functions.transformation_matrix on host float32 arrays, in the reference operator's float32
    arithmetic (quaternion_matrix.py:65-78, compose_transform.py): the reference's refinement
    node builds the ICC's initial transforms this way on the host
    (collision_based_pose_refinement.py:152-154).  q [N,4] (w, x, y, z) with t [N,3] gives
    [N,4,4]; q [4] with t [3] gives [4,4]."""
    f32 = np.float32
    q = np.asarray(quaternion, dtype=f32)
    t = np.asarray(translation, dtype=f32)
    single = q.ndim == 1
    q, t = q.reshape(-1, 4), t.reshape(-1, 3)
    assert q.shape[0] == t.shape[0], "one translation [3] per quaternion"
    n = (q * q).sum(axis=1, keepdims=True, dtype=f32)
    qs = q * np.sqrt(f32(2.0) / n)
    Q = qs[:, :, None] * qs[:, None, :]
    T = np.tile(np.eye(4, dtype=f32)[None], (q.shape[0], 1, 1))
    T[:, 0, 0] = 1 - Q[:, 2, 2] - Q[:, 3, 3]
    T[:, 0, 1] = Q[:, 1, 2] - Q[:, 3, 0]
    T[:, 0, 2] = Q[:, 1, 3] + Q[:, 2, 0]
    T[:, 1, 0] = Q[:, 1, 2] + Q[:, 3, 0]
    T[:, 1, 1] = 1 - Q[:, 1, 1] - Q[:, 3, 3]
    T[:, 1, 2] = Q[:, 2, 3] - Q[:, 1, 0]
    T[:, 2, 0] = Q[:, 1, 3] - Q[:, 2, 0]
    T[:, 2, 1] = Q[:, 2, 3] + Q[:, 1, 0]
    T[:, 2, 2] = 1 - Q[:, 1, 1] - Q[:, 2, 2]
    T[:, :3, 3] = t
    return T[0] if single else T


# ------------------------------------------------------------------ per-frame front end (CUDA)
def pointcloud_from_depth(depth, fx, fy, cx, cy, depth_type="z"):
    """depth [H,W] float (metres, NaN = invalid) -> camera-frame points [H,W,3]
    (morefusion/geometry/pointcloud_from_depth.py:4-26) in one kernel.  numpy in -> numpy out,
    CUDA tensor in -> CUDA tensor out (no host round trip on the per-frame path)."""
    import torch
    from .. import _lib
    assert depth_type in ["z", "euclidean"], "Unexpected depth_type"
    is_np = not isinstance(depth, torch.Tensor)
    d = torch.as_tensor(np.asarray(depth), device="cuda") if is_np else depth
    assert d.dtype.is_floating_point, "depth must be float and have meter values"
    _lib.require_cuda(d)
    d = d.to(torch.float32).contiguous()
    H, W = d.shape
    pcd = torch.empty((H, W, 3), dtype=torch.float32, device=d.device)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().mf_pointcloud_from_depth(
            _lib.ptr(d), H, W, float(fx), float(fy), float(cx), float(cy),
            int(depth_type == "euclidean"), _lib.ptr(pcd), _lib.stream()), "pointcloud_from_depth")
    return pcd.cpu().numpy() if is_np else pcd


def masks_to_bboxes(masks):
    """bool masks (N,H,W) or (H,W) -> (y1, x1, y2, x2) boxes, upper bounds exclusive, zeros for
    an empty mask (morefusion/geometry/masks_to_bboxes.py:4-38).  float64 numpy for numpy input
    (as the reference), int32 CUDA tensor for CUDA input."""
    import torch
    from .. import _lib
    is_np = not isinstance(masks, torch.Tensor)
    m = torch.as_tensor(np.asarray(masks), device="cuda") if is_np else masks
    assert m.dtype == torch.bool
    assert m.dim() in [2, 3], "masks must be 2 or 3 dimensional"
    _lib.require_cuda(m)
    squeeze = m.dim() == 2
    m3 = (m[None] if squeeze else m).contiguous().view(torch.uint8)
    N, H, W = m3.shape
    out = torch.empty((N, 4), dtype=torch.int32, device=m.device)
    with torch.cuda.device(m.device):
        _lib.check(_lib.lib().mf_masks_to_bboxes(_lib.ptr(m3), N, H, W, _lib.ptr(out), _lib.stream()),
                   "masks_to_bboxes")
    if is_np:
        out = out.cpu().numpy().astype(np.float64)
    return out[0] if squeeze else out


def _instance_lut(instance_ids):
    """Host look-up table from instance id to slot: (lut int32 [hi - lo + 1], lo)."""
    ids = np.asarray(instance_ids).reshape(-1)
    if ids.size == 0:
        raise ValueError("instance_ids is empty")
    if not np.issubdtype(ids.dtype, np.integer):
        raise ValueError("instance_ids must be integers")
    ids = ids.astype(np.int64)
    if len(np.unique(ids)) != ids.size:
        raise ValueError("instance_ids must be distinct")
    lo, hi = int(ids.min()), int(ids.max())
    if lo < -(1 << 31) or hi >= 1 << 31:
        raise ValueError("instance ids must fit in int32")
    if hi - lo >= 1 << 20:
        raise ValueError("instance ids span too wide a range for a label look-up table")
    lut = np.full(hi - lo + 1, -1, np.int32)
    lut[ids - lo] = np.arange(ids.size, dtype=np.int32)
    return lut, lo, ids.astype(np.int32)


def _frame_crops(rgb, pcd, label, instance_ids, size=256):
    """CUDA tensors rgb [H,W,3] u8, pcd [H,W,3] f32, label [H,W] int32 and host instance ids ->
    rgb_ins [N,S,S,3] u8, pcd_ins [N,S,S,3] f32, stats [N,6] int32 (y1, x1, y2, x2, n_mask,
    n_valid); three launches (csrc/frontend.cu), nothing read back."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    _lib.require_cuda(rgb, pcd, label)
    if rgb.dtype != torch.uint8 or pcd.dtype != torch.float32 or label.dtype != torch.int32:
        raise ValueError("rgb must be uint8, pcd float32 and label int32")
    if rgb.dim() != 3 or rgb.shape[2] != 3 or tuple(pcd.shape) != tuple(rgb.shape) \
            or tuple(label.shape) != tuple(rgb.shape[:2]):
        raise ValueError("rgb and pcd must be [H,W,3] and label [H,W]")
    if size <= 0:
        raise ValueError("size must be positive")
    lut, lo, ids = _instance_lut(instance_ids)
    dev = rgb.device
    N = ids.size
    H, W = label.shape
    rgb, pcd, label = rgb.contiguous(), pcd.contiguous(), label.contiguous()
    d_lut = _util.h2d(lut, dev, torch.int32, "crops/lut")
    d_ids = _util.h2d(ids, dev, torch.int32, "crops/ids")
    L = _lib.lib()
    ws_bytes = L.mf_label_bboxes_workspace_bytes(N)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    stats = torch.empty((N, 6), dtype=torch.int32, device=dev)
    rgb_ins = torch.empty((N, size, size, 3), dtype=torch.uint8, device=dev)
    pcd_ins = torch.empty((N, size, size, 3), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.mf_label_bboxes(
            _lib.ptr(label), _lib.ptr(pcd), H, W, _lib.ptr(d_lut), lo, lut.size, N,
            _lib.ptr(stats), _lib.ptr(ws), ws_bytes, _lib.stream()), "label_bboxes")
        _lib.check(L.mf_instance_crops(
            _lib.ptr(rgb), _lib.ptr(pcd), _lib.ptr(label), H, W, _lib.ptr(d_ids), _lib.ptr(stats),
            N, size, _lib.ptr(rgb_ins), _lib.ptr(pcd_ins), _lib.stream()), "instance_crops")
    return rgb_ins, pcd_ins, stats


def instance_crops(rgb, pcd, label, instance_ids, *, size=256):
    """Per-instance crops of a labelled frame, as datasets/rgbd_pose_estimation/base.py:113-161
    and the ROS pose node build them: for each id, the mask ``label == id``, its bounding box, the
    RGB zeroed and the points NaN'd outside the mask, cropped and centred into ``size`` x
    ``size`` by imgviz.centerize with OpenCV's resize (RGB bilinear with 0 padding, points
    nearest with NaN padding).

    rgb [H,W,3] uint8, pcd [H,W,3] float32, label [H,W] integer, instance_ids [N] distinct
    integers (an id absent from ``label`` gives an empty box, zero RGB and NaN points).
    Returns (rgb_ins [N,S,S,3] uint8, pcd_ins [N,S,S,3] float32, bboxes [N,4] int32 (y1, x1,
    y2, x2), upper bounds exclusive, zeros when empty, n_valid [N] int32: mask pixels whose
    point has no NaN).  numpy in -> numpy out, CUDA tensors in -> CUDA tensors out.

    Crops of up to 1024 instances are made by one pass over the label image and one launch of
    one thread per output pixel; no per-instance host work and no host read."""
    import torch
    from .. import _lib
    is_np = not isinstance(rgb, torch.Tensor)
    if is_np:
        rgb, pcd, label = (torch.as_tensor(np.ascontiguousarray(a), device="cuda")
                           for a in (rgb, pcd, label))
    _lib.require_cuda(rgb, pcd, label)
    if label.dtype.is_floating_point or label.dtype == torch.bool:
        raise ValueError("label must be an integer image")
    if isinstance(instance_ids, torch.Tensor):
        instance_ids = instance_ids.cpu().numpy()
    rgb_ins, pcd_ins, stats = _frame_crops(rgb, pcd.to(torch.float32), label.to(torch.int32),
                                           instance_ids, size=size)
    out = (rgb_ins, pcd_ins, stats[:, :4], stats[:, 5])
    if is_np:
        out = tuple(o.cpu().numpy() for o in out)
    return out


def _check_faces(faces, n_vertices):
    """Host check of a mesh's faces before upload: [F,3] integer indices in [0, n_vertices),
    returned as int32."""
    f = np.asarray(faces)
    if f.size and not np.issubdtype(f.dtype, np.integer):
        raise ValueError("faces must be integer vertex indices")
    f = f.reshape(-1, 3).astype(np.int64)
    if f.size and (f.min() < 0 or f.max() >= n_vertices):
        raise ValueError("face index outside [0, len(vertices))")
    return np.ascontiguousarray(f.astype(np.int32))


def _check_mesh(vertices, faces):
    """Host checks of a mesh before upload: vertices [V,3] float64, faces [F,3] int32 in [0, V)."""
    v = np.ascontiguousarray(np.asarray(vertices, dtype=np.float64).reshape(-1, 3))
    return v, _check_faces(faces, len(v))


def focal_from_fovy(fovy, height):
    """The focal length in pixels of computeProjectionMatrixFOV's frustum of vertical field of
    view ``fovy`` degrees over ``height`` rows (float64)."""
    import math
    return (height / 2.0) / math.tan(math.radians(float(fovy)) / 2.0)


def fovy_from_intrinsics(fy, height):
    """The vertical field of view in degrees that trimesh.scene.Camera(resolution=(W, H),
    focal=(fx, fy)).fov[1] gives, as get_example passes it to render_cad."""
    return float(2.0 * np.degrees(np.arctan(height / (2.0 * float(fy)))))


def _render_cad_batch(vertices, faces, offsets, mesh, Ts_cad2cam, *, f, height, width):
    """N poses of S meshes packed back to back, each pose rendered alone (csrc/render_cad.cu).

    vertices [V,3] float64 and faces [F,3] int32 CUDA tensors, already checked on the host
    (``_check_mesh``; face indices of mesh s index the packed vertices); offsets [S+1] host
    int64, mesh s is faces[offsets[s]:offsets[s+1]]; mesh [N] (the mesh of each pose) and
    Ts_cad2cam [N,4,4] float64 CUDA tensors or host arrays (uploaded without a host sync); f
    the focal length in pixels.  Returns CUDA tensors depth [N,H,W] float32 (NaN where nothing
    covers), mask [N,H,W] bool and count [N] int32.  Three launches, no host read."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    _lib.require_cuda(vertices, faces)
    dev = vertices.device
    offsets = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
    d_mesh = _util.h2d(mesh, dev, torch.int32, "render_cad/mesh").contiguous()
    d_T = _util.h2d(Ts_cad2cam, dev, torch.float64, "render_cad/T").contiguous()
    N = d_mesh.numel()
    if tuple(d_T.shape) != (N, 4, 4):
        raise ValueError("Ts_cad2cam must be [N,4,4] with one mesh index per pose")
    H, W = int(height), int(width)
    depth = torch.empty((N, H, W), dtype=torch.float32, device=dev)
    mask = torch.empty((N, H, W), dtype=torch.bool, device=dev)
    count = torch.empty(N, dtype=torch.int32, device=dev)
    L = _lib.lib()
    F = faces.shape[0]
    ws_bytes = L.mf_render_cad_workspace_bytes(N, F, H, W)
    ws = _util.workspace(ws_bytes, dev) if ws_bytes else None
    with torch.cuda.device(dev):
        _lib.check(L.mf_render_cad(
            _lib.ptr(vertices), vertices.shape[0], _lib.ptr(faces), F,
            offsets.ctypes.data_as(_lib.ctypes.c_void_p), offsets.size - 1, _lib.ptr(d_mesh),
            _lib.ptr(d_T), N, float(f), H, W, _lib.ptr(depth), _lib.ptr(mask.view(torch.uint8)),
            _lib.ptr(count), _lib.ptr(ws), ws_bytes, _lib.stream()), "render_cad")
    return depth, mask, count


def render_cad(vertices, faces, Ts_cad2cam, *, fovy, height, width):
    """Depth and mask of a CAD mesh at one pose [4,4] or N poses [N,4,4], each pose rendered
    alone, as morefusion/extra/_pybullet.py:215-288 ``render_cad`` renders them with pybullet.

    The reference takes a mesh file; here the caller passes the mesh: vertices [V,3] and faces
    [F,3] integer indices (a loaded ``trimesh.Trimesh`` passes ``.vertices`` and ``.faces``).
    Ts_cad2cam maps CAD points into the camera frame (OpenCV axes).  The camera is pybullet's
    computeProjectionMatrixFOV(fovy, W / H, 0.01, 1000): square pixels of focal length
    (H / 2) / tan(fovy / 2) and the principal point at the image centre.  RGB is not produced:
    textures are out of scope.

    Returns (depth, mask): depth float32 camera-frame Z of the nearest surface, NaN where the
    mesh does not cover; mask bool, the covered pixels; [H,W] for one pose, [N,H,W] for N
    poses.  NumPy in gives NumPy out; CUDA tensors in give CUDA tensors out.  The rasterisation
    rules (snapping, fill rule, triangles crossing the near plane) are DESIGN's render_cad
    section.  Faces are checked on the host, so CUDA faces are read back once."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    is_np = not isinstance(vertices, torch.Tensor)
    if is_np:
        v, fc = _check_mesh(vertices, faces)
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        _lib.require_cuda(vertices)
        dev = vertices.device
        v = None
        fc = _check_faces(faces.cpu().numpy() if isinstance(faces, torch.Tensor) else faces,
                          vertices.shape[0])
    Ts = Ts_cad2cam
    if isinstance(Ts, torch.Tensor):
        _lib.require_cuda(Ts)
        squeeze = Ts.dim() == 2
        Ts = Ts.to(torch.float64).reshape(-1, 4, 4).contiguous()
    else:
        Ts = np.asarray(Ts, np.float64)
        squeeze = Ts.ndim == 2
        Ts = Ts.reshape(-1, 4, 4)
    height, width = int(height), int(width)
    f = focal_from_fovy(fovy, height)
    if not (np.isfinite(f) and f > 0):
        raise ValueError("fovy must be in (0, 180) degrees")
    d_v = (_util.h2d_transient(v, dev, torch.float64) if is_np
           else vertices.to(torch.float64).contiguous())
    d_f = _util.h2d_transient(fc, dev, torch.int32)
    N = Ts.shape[0]
    depth, mask, _ = _render_cad_batch(d_v, d_f, [0, len(fc)], np.zeros(N, np.int32), Ts,
                                       f=f, height=height, width=width)
    if squeeze:
        depth, mask = depth[0], mask[0]
    if is_np:
        return depth.cpu().numpy(), mask.cpu().numpy()
    return depth, mask


MAX_SCENE_OBJECTS = 64                    # MF_RENDER_SCENE_MAX_OBJECTS


def _check_instance_ids(instance_ids, n=None):
    """Host checks of a scene's instance ids: distinct integers in [0, 2^31), n of them when n is
    given."""
    ids = np.asarray(instance_ids).reshape(-1)
    if ids.size and not np.issubdtype(ids.dtype, np.integer):
        raise ValueError("instance_ids must be integers")
    ids = ids.astype(np.int64)
    if n is not None and len(ids) != n:
        raise ValueError(f"{len(ids)} instance ids for {n} objects")
    if ids.size and (ids.min() < 0 or ids.max() > np.iinfo(np.int32).max):
        raise ValueError("instance ids must be in [0, 2^31)")
    if len(np.unique(ids)) != len(ids):
        raise ValueError("instance ids must be distinct")
    return ids.astype(np.int32)


def _pack_cads(cads):
    """One mesh per object, packed back to back with identical meshes stored once: (vertices
    [V,3] float64, faces [F,3] int32 indexing the packed vertices, offsets [S+1] int64, mesh [N]
    int32), host arrays, each mesh checked by ``_check_mesh``."""
    keys, vs, fs, offsets, mesh, base = {}, [], [], [0], [], 0
    for cad in cads:
        v, fc = _check_mesh(cad.vertices, cad.faces)
        key = (v.tobytes(), fc.tobytes())
        if key not in keys:
            keys[key] = len(vs)
            vs.append(v)
            fs.append(fc + base)
            base += len(v)
            offsets.append(offsets[-1] + len(fc))
        mesh.append(keys[key])
    if not vs:                                # no object: one empty mesh keeps S >= 1
        vs, fs, offsets = [np.zeros((0, 3))], [np.zeros((0, 3), np.int32)], [0, 0]
    return (np.concatenate(vs), np.concatenate(fs).astype(np.int32), np.asarray(offsets, np.int64),
            np.asarray(mesh, np.int32))


def _render_instances_batch(vertices, faces, offsets, mesh, Ts_cad2cam, instance_ids, *, f, height,
                            width):
    """N <= 64 posed objects of S packed meshes rendered together into one camera
    (csrc/render_cad.cu, mf_render_scene).  Arguments as ``_render_cad_batch``, and instance_ids
    [N] int32, already checked on the host (``_check_instance_ids``).  Returns CUDA tensors depth
    [H,W] float32 (NaN where nothing covers), ins [H,W] int32 (-1 where nothing covers), whole
    [N] int32 (the pixels each object covers alone) and occluded [N,N] int32 (occluded[i, j]: the
    pixels of object i's whole mask where object j is visible).  Four launches, no host read."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    _lib.require_cuda(vertices, faces)
    dev = vertices.device
    offsets = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
    d_mesh = _util.h2d_transient(np.asarray(mesh, np.int32).reshape(-1), dev, torch.int32)
    d_ids = _util.h2d_transient(np.asarray(instance_ids, np.int32).reshape(-1), dev, torch.int32)
    d_T = _util.h2d(Ts_cad2cam, dev, torch.float64, "render_instances/T").contiguous()
    N = d_mesh.numel()
    if N > MAX_SCENE_OBJECTS:
        raise ValueError(f"at most {MAX_SCENE_OBJECTS} objects per scene, got {N}")
    if tuple(d_T.shape) != (N, 4, 4) or d_ids.numel() != N:
        raise ValueError("Ts_cad2cam must be [N,4,4] with one mesh index and instance id per pose")
    H, W = int(height), int(width)
    depth = torch.empty((H, W), dtype=torch.float32, device=dev)
    ins = torch.empty((H, W), dtype=torch.int32, device=dev)
    whole = torch.empty(N, dtype=torch.int32, device=dev)
    occluded = torch.empty((N, N), dtype=torch.int32, device=dev)
    L = _lib.lib()
    F = faces.shape[0]
    ws_bytes = L.mf_render_cad_workspace_bytes(N, F, H, W)
    ws = _util.workspace(ws_bytes, dev) if ws_bytes else None
    with torch.cuda.device(dev):
        _lib.check(L.mf_render_scene(
            _lib.ptr(vertices), vertices.shape[0], _lib.ptr(faces), F,
            offsets.ctypes.data_as(_lib.ctypes.c_void_p), offsets.size - 1, _lib.ptr(d_mesh),
            _lib.ptr(d_T), _lib.ptr(d_ids), N, float(f), H, W, _lib.ptr(depth), _lib.ptr(ins),
            _lib.ptr(whole), _lib.ptr(occluded), _lib.ptr(ws), ws_bytes, _lib.stream()),
            "render_scene")
    return depth, ins, whole, occluded


def render_instances(cads, Ts_cad2cam, instance_ids, *, fovy, height, width):
    """Depth and instance image of posed objects rendered together into one camera, as the
    picking-order node's ``_render_object_pose_array`` renders them with pybullet
    (ros/src/morefusion_ros/nodes/select_picking_order.py:129-190).

    ``cads`` holds one mesh per object, each with ``.vertices`` [V,3] and ``.faces`` [F,3] host
    arrays (as ``get_cad`` returns them); identical meshes are uploaded once.  Ts_cad2cam [N,4,4]
    maps each object's CAD points into the camera frame (OpenCV axes); instance_ids [N] are
    distinct integers in [0, 2^31), at most 64 objects.  The camera and the rasterisation rules
    are ``render_cad``'s; each pixel shows the object of smallest float32 depth, the earlier
    object on an exact tie.

    Returns (depth, ins): depth [H,W] float32, NaN where nothing covers; ins [H,W] int32, the
    instance id of the visible object, -1 where nothing covers.  NumPy Ts_cad2cam gives NumPy
    out; a CUDA tensor gives CUDA tensors out, with no host read."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    cads = list(cads)
    if len(cads) > MAX_SCENE_OBJECTS:
        raise ValueError(f"at most {MAX_SCENE_OBJECTS} objects per scene, got {len(cads)}")
    ids = _check_instance_ids(instance_ids, len(cads))
    is_np = not isinstance(Ts_cad2cam, torch.Tensor)
    if is_np:
        Ts = np.asarray(Ts_cad2cam, np.float64).reshape(-1, 4, 4)
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        _lib.require_cuda(Ts_cad2cam)
        Ts = Ts_cad2cam.to(torch.float64).reshape(-1, 4, 4).contiguous()
        dev = Ts.device
    f = focal_from_fovy(fovy, int(height))
    if not (np.isfinite(f) and f > 0):
        raise ValueError("fovy must be in (0, 180) degrees")
    v, fc, offsets, mesh = _pack_cads(cads)
    depth, ins, _, _ = _render_instances_batch(
        _util.h2d_transient(v, dev, torch.float64), _util.h2d_transient(fc, dev, torch.int32),
        offsets, mesh, Ts, ids, f=f, height=height, width=width)
    if is_np:
        return depth.cpu().numpy(), ins.cpu().numpy()
    return depth, ins


MAX_MODEL_MESHES = 64                     # MF_MESH_MODELS_MAX_MESHES
MAX_GRID_DIMENSION = 128                  # MF_MESH_MODELS_MAX_DIM


def _check_model_mesh(vertices, faces):
    """``_check_mesh`` plus what the model data needs: at least one face, finite vertices and a
    non-zero extent of the referenced vertices."""
    v, fc = _check_mesh(vertices, faces)
    if len(fc) == 0:
        raise ValueError("the mesh has no faces")
    used = v[fc.reshape(-1)]
    if not np.isfinite(v).all():
        raise ValueError("vertices must be finite")
    if not (used.max(0) - used.min(0)).max() > 0:
        raise ValueError("the mesh's referenced vertices span no extent")
    return v, fc


def _pack_meshes(meshes):
    """(vertices, faces) pairs checked by ``_check_model_mesh`` and packed back to back: (vertices
    [V,3] float64, faces [F,3] int32 indexing the packed vertices, offsets [S+1] int64)."""
    vs, fs, offsets, base = [], [], [0], 0
    for v, fc in meshes:
        v, fc = _check_model_mesh(v, fc)
        vs.append(v)
        fs.append(fc + base)
        base += len(v)
        offsets.append(offsets[-1] + len(fc))
    if not 1 <= len(vs) <= MAX_MODEL_MESHES:
        raise ValueError(f"1 to {MAX_MODEL_MESHES} meshes per call, got {len(vs)}")
    return np.concatenate(vs), np.concatenate(fs).astype(np.int32), np.asarray(offsets, np.int64)


def _voxelize_solid_batch(vertices, faces, offsets, dimension):
    """The solid grids of S packed meshes (csrc/mesh_models.cu, mf_mesh_voxelize_solid): vertices
    [V,3] float64 and faces [F,3] int32 CUDA tensors checked on the host, offsets [S+1] host
    int64.  Returns CUDA tensors matrix [S,D,D,D] bool, counts [S] int32, points [S,D^3,3]
    float64 (mesh s's filled centres in its first counts[s] rows, NaN after), translate [S,3],
    scale [S] and pitch [S] float64.  Seven launches, no host read."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    _lib.require_cuda(vertices, faces)
    D = int(dimension)
    if not 1 <= D <= MAX_GRID_DIMENSION:
        raise ValueError(f"dimension must be in [1, {MAX_GRID_DIMENSION}], got {dimension}")
    dev = vertices.device
    offsets = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
    S = offsets.size - 1
    matrix = torch.empty((S, D, D, D), dtype=torch.bool, device=dev)
    counts = torch.empty(S, dtype=torch.int32, device=dev)
    points = torch.empty((S, D ** 3, 3), dtype=torch.float64, device=dev)
    translate = torch.empty((S, 3), dtype=torch.float64, device=dev)
    scale = torch.empty(S, dtype=torch.float64, device=dev)
    pitch = torch.empty(S, dtype=torch.float64, device=dev)
    L = _lib.lib()
    ws_bytes = L.mf_mesh_voxelize_workspace_bytes(S, D)
    ws = _util.workspace(ws_bytes, dev)
    with torch.cuda.device(dev):
        _lib.check(L.mf_mesh_voxelize_solid(
            _lib.ptr(vertices), vertices.shape[0], _lib.ptr(faces), faces.shape[0],
            offsets.ctypes.data_as(_lib.ctypes.c_void_p), S, D, _lib.ptr(matrix.view(torch.uint8)),
            _lib.ptr(counts), _lib.ptr(points), _lib.ptr(translate), _lib.ptr(scale),
            _lib.ptr(pitch), _lib.ptr(ws), ws_bytes, _lib.stream()), "voxelize_solid")
    return matrix, counts, points, translate, scale, pitch


def _signed_distance_batch(vertices, faces, offsets, points, mesh):
    """Signed distances of points [P,3] float64 (CUDA) to S packed meshes (csrc/mesh_models.cu,
    mf_mesh_signed_distance); mesh [P] int32 CUDA, the mesh of each point (a point outside [0, S)
    gets NaN and -1).  Returns CUDA tensors sdf [P] float64 (positive inside) and face [P] int32
    (the nearest face, an index into the packed faces).  Two launches, no host read."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    _lib.require_cuda(vertices, faces, points, mesh)
    dev = vertices.device
    offsets = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1))
    points = points.to(torch.float64).reshape(-1, 3).contiguous()
    mesh = mesh.to(torch.int32).reshape(-1).contiguous()
    P = points.shape[0]
    if mesh.numel() != P:
        raise ValueError("one mesh index per point")
    sdf = torch.empty(P, dtype=torch.float64, device=dev)
    face = torch.empty(P, dtype=torch.int32, device=dev)
    if P == 0:
        return sdf, face
    L = _lib.lib()
    f_max = int(np.diff(offsets).max())
    with torch.cuda.device(dev):
        ws_bytes = L.mf_mesh_signed_distance_workspace_bytes(P, f_max)
        ws = _util.workspace(ws_bytes, dev)
        _lib.check(L.mf_mesh_signed_distance(
            _lib.ptr(vertices), vertices.shape[0], _lib.ptr(faces), faces.shape[0],
            offsets.ctypes.data_as(_lib.ctypes.c_void_p), offsets.size - 1, _lib.ptr(points),
            _lib.ptr(mesh), P, _lib.ptr(sdf), _lib.ptr(face), _lib.ptr(ws), ws_bytes,
            _lib.stream()), "signed_distance")
    return sdf, face


def _host_mesh(vertices, faces):
    """Host copies of a mesh given as NumPy or CUDA tensors, and the device to run on."""
    import torch
    from .. import _lib
    if isinstance(vertices, torch.Tensor):
        _lib.require_cuda(vertices)
        dev = vertices.device
        v = vertices.detach().cpu().numpy()
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
        v = vertices
    fc = faces.detach().cpu().numpy() if isinstance(faces, torch.Tensor) else faces
    return v, fc, dev


def voxelize_solid(vertices, faces, dimension=64):
    """The solid D^3 voxel grid of a mesh, as YCBVideoModels.get_solid_voxel_grid gets it from
    ``binvox -d 64`` (datasets/ycb_video/models.py:81-86), by the rules of DESIGN section 4.22:
    the grid spans the referenced vertices' bounding box from its minimum corner, with cubic
    voxels of side scale / D (scale: the largest extent); a voxel is filled when a face overlaps
    its closed box or its centre is inside by +z ray parity.  The winding need not be consistent.

    Returns an object with ``.matrix`` [D,D,D] bool (i along x), ``.points`` [n,3] float64 (the
    filled voxel centres in ascending (i, j, k)), ``.translate`` [3] (the grid's minimum corner),
    ``.pitch`` (the voxel side) and ``.scale`` (floats).  NumPy in gives NumPy out; CUDA tensors
    in give CUDA tensors out, after one host read (the number of points).  ValueError, before any
    launch, for a mesh without faces, face indices outside [0, V), non-finite vertices, a zero
    extent or a dimension outside [1, 128]."""
    import types
    import torch
    from ..functions.geometry import _util
    is_np = not isinstance(vertices, torch.Tensor)
    v, fc, dev = _host_mesh(vertices, faces)
    v, fc = _check_model_mesh(v, fc)
    matrix, counts, points, translate, scale, pitch = _voxelize_solid_batch(
        _util.h2d_transient(v, dev, torch.float64), _util.h2d_transient(fc, dev, torch.int32),
        [0, len(fc)], dimension)
    head = torch.cat([counts.to(torch.float64), scale, pitch]).cpu().numpy()
    n = int(head[0])
    out = types.SimpleNamespace(matrix=matrix[0], points=points[0, :n], translate=translate[0],
                                scale=float(head[1]), pitch=float(head[2]))
    if is_np:
        out.matrix = out.matrix.cpu().numpy()
        out.points = out.points.cpu().numpy()
        out.translate = out.translate.cpu().numpy()
    return out


def signed_distance(vertices, faces, points):
    """Signed distance of points [P,3] to a mesh, as trimesh's ``nearest.signed_distance``
    gives it to YCBVideoModels._get_sdf (datasets/ycb_video/models.py:77): the distance to the
    closest point of the nearest face, positive inside.  Inside is the +z ray parity rule of
    ``voxelize_solid``, so the grid and the sign agree.  Returns sdf [P] float64.  NumPy in gives
    NumPy out; CUDA tensors in give CUDA tensors out, with no host read besides the face check.
    ValueError, before any launch, as ``voxelize_solid``."""
    import torch
    from .. import _lib
    from ..functions.geometry import _util
    is_np = not isinstance(points, torch.Tensor)
    v, fc, dev = _host_mesh(vertices, faces)
    v, fc = _check_model_mesh(v, fc)
    if is_np:
        p = np.asarray(points, np.float64).reshape(-1, 3)
        d_p = _util.h2d_transient(p, dev, torch.float64)
    else:
        _lib.require_cuda(points)
        d_p = points.to(torch.float64).reshape(-1, 3).contiguous()
    mesh = torch.zeros(d_p.shape[0], dtype=torch.int32, device=dev)
    sdf, _ = _signed_distance_batch(_util.h2d_transient(v, dev, torch.float64),
                                    _util.h2d_transient(fc, dev, torch.int32), [0, len(fc)], d_p,
                                    mesh)
    return sdf.cpu().numpy() if is_np else sdf
