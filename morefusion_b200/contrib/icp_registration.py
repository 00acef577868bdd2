"""Point-to-point ICP refinement: ``ICPRegistration`` (morefusion/contrib/icp_registration.py), the
reference's wrapper over Open3D, on the sm_90a kernels of csrc/icp.cu.

``register_batch`` is the one entry: M source clouds on the device (the frame path's crops, NaN
rows skipped), each registered to its down-sampled CAD cloud (``ICPTarget``, built once and kept
on the device), in two launches with no host read between them -- the down-sampling of every
source cloud, then every iteration of every instance.  Everything is float64, as Open3D computes.
"""

import ctypes

import numpy as np
import torch

from .. import _lib
from ..functions.geometry import _util

ITERATION = 100          # icp_registration.py:28
VOXEL_SIZE = 0.01        # icp_registration.py:29
RELATIVE_FITNESS = 1e-6  # Open3D's ICPConvergenceCriteria defaults
RELATIVE_RMSE = 1e-6


class _TargetC(ctypes.Structure):
    _fields_ = [("points", ctypes.c_void_p), ("cells", ctypes.c_void_p), ("index", ctypes.c_void_p),
                ("count", ctypes.c_void_p), ("origin", ctypes.c_void_p), ("cell_size", ctypes.c_double)]


def _points(x, device=None):
    """A CUDA [M,N,3] float32 / float64 tensor of M clouds; host input is uploaded to `device`
    when one is given."""
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)
    if t.dim() < 2 or t.shape[-1] != 3:
        raise ValueError("point clouds must be [..., 3]")
    if not t.is_cuda:
        if device is None:
            _lib.require_cuda(t)
        t = _util.h2d_transient(t.numpy(), device, t.dtype)
    return t.reshape(t.shape[0] if t.dim() > 2 else 1, -1, 3).contiguous()


def voxel_down_sample(points, voxel_size):
    """Open3D's ``voxel_down_sample`` of M clouds at once.  points: CUDA [M,N,3] (or [M,H,W,3])
    float32 / float64; rows with a non-finite coordinate are skipped.  Returns CUDA tensors
    (means [M,N,3] float64, keys [M,N,3] int32, counts [M,N] int32, n [M] int32): cloud m's n[m]
    voxels are its first rows, in ascending (i, j, k).  n[m] = -1 refuses a cloud that spans
    2^31 - 1 voxels or more on an axis, whose keys would not fit in int32."""
    pts = _points(points)
    _lib.require_cuda(pts)
    M, N = pts.shape[0], pts.shape[1]
    dev = pts.device
    means = torch.empty((M, N, 3), dtype=torch.float64, device=dev)
    keys = torch.empty((M, N, 3), dtype=torch.int32, device=dev)
    counts = torch.empty((M, N), dtype=torch.int32, device=dev)
    n = torch.empty(M, dtype=torch.int32, device=dev)
    L = _lib.lib()
    nb = L.mf_icp_sort_workspace_bytes(M, N)
    ws = _util.workspace(nb, dev)
    _lib.check(L.mf_icp_voxel_down_sample(
        _lib.ptr(pts), int(pts.dtype == torch.float64), M, N, float(voxel_size), _lib.ptr(means),
        _lib.ptr(keys), _lib.ptr(counts), _lib.ptr(n), _lib.ptr(ws), nb, _lib.stream()),
        "voxel_down_sample")
    return means, keys, counts, n


class ICPTarget:
    """A CAD cloud down-sampled at voxel_size with a uniform cell list of side max_distance over
    it, on the device: what each ICP iteration searches (csrc/icp.cu)."""

    def __init__(self, points, voxel_size, max_distance, device=None):
        device = torch.device(device if device is not None else "cuda")
        pts = _points(points, device)
        if pts.shape[0] != 1:
            raise ValueError("one target cloud")
        means, _, _, n = voxel_down_sample(pts, voxel_size)
        N = means.shape[1]
        self.points = torch.empty((N, 3), dtype=torch.float64, device=means.device)
        self.cells = torch.empty((N, 3), dtype=torch.int32, device=means.device)
        self.index = torch.empty(N, dtype=torch.int32, device=means.device)
        self.origin = torch.empty(3, dtype=torch.float64, device=means.device)
        self.count = n
        self.voxel_size = float(voxel_size)
        self.max_distance = float(max_distance)
        if not self.max_distance > 0:
            raise ValueError("max_distance must be positive")
        L = _lib.lib()
        nb = L.mf_icp_sort_workspace_bytes(1, N)
        ws = _util.workspace(nb, means.device)
        _lib.check(L.mf_icp_cell_list(
            _lib.ptr(means), _lib.ptr(n), N, self.max_distance, _lib.ptr(self.points),
            _lib.ptr(self.cells), _lib.ptr(self.index), _lib.ptr(self.origin), _lib.ptr(ws), nb,
            _lib.stream()), "icp cell list")
        self._keep = means                     # the cell list's input stays alive with it

    def _c(self):
        return _TargetC(self.points.data_ptr(), self.cells.data_ptr(), self.index.data_ptr(),
                        self.count.data_ptr(), self.origin.data_ptr(), self.max_distance)


def register_batch(source, targets, transform_init, *, voxel_size=VOXEL_SIZE, max_distance=None,
                   max_iteration=ITERATION, relative_fitness=RELATIVE_FITNESS,
                   relative_rmse=RELATIVE_RMSE):
    """Open3D's ``registration_icp`` (point to point, no scaling) of M instances in two launches.

    source: CUDA [M,N,3] or [M,H,W,3] float32 / float64 clouds (non-finite rows skipped),
    down-sampled here at voxel_size; targets: M ``ICPTarget`` (one object may serve several
    instances); transform_init: host [M,4,4], source -> target.  max_distance defaults to
    2 * voxel_size and must equal each target's.

    Returns CUDA tensors (transform [M,4,4] float64, fitness [M], inlier_rmse [M] float64,
    iterations [M] int32).  No host read.  An instance whose source or target spans 2^31 - 1
    voxels (or target cells) or more on an axis is refused: NaN transform, fitness and rmse, 0
    iterations."""
    src = _points(source)
    _lib.require_cuda(src)
    M, N = src.shape[0], src.shape[1]
    max_distance = 2.0 * voxel_size if max_distance is None else float(max_distance)
    targets = list(targets)
    if len(targets) != M:
        raise ValueError(f"one target per source cloud: {len(targets)} targets, {M} clouds")
    for t in targets:
        if t.max_distance != max_distance:
            raise ValueError("a target's cell list was built for another max_distance")
    init = np.ascontiguousarray(np.asarray(transform_init, dtype=np.float64).reshape(M, 4, 4))
    dev = src.device
    means, _, _, n = voxel_down_sample(src, voxel_size)
    T = torch.empty((M, 4, 4), dtype=torch.float64, device=dev)
    fit = torch.empty(M, dtype=torch.float64, device=dev)
    rmse = torch.empty(M, dtype=torch.float64, device=dev)
    iters = torch.empty(M, dtype=torch.int32, device=dev)
    if M == 0:
        return T, fit, rmse, iters
    table = (_TargetC * M)(*[t._c() for t in targets])
    d_table = _util.h2d(np.frombuffer(bytes(table), np.uint8).copy(), dev, torch.uint8, "icp/targets")
    d_init = _util.h2d(init, dev, torch.float64, "icp/init")
    L = _lib.lib()
    nb = L.mf_icp_run_workspace_bytes(M, N)
    ws = _util.workspace(nb, dev)
    _lib.check(L.mf_icp_run(
        M, _lib.ptr(means), N, _lib.ptr(n), _lib.ptr(d_table), _lib.ptr(d_init),
        init.ctypes.data_as(ctypes.c_void_p), max_distance, int(max_iteration),
        float(relative_fitness), float(relative_rmse), _lib.ptr(T), _lib.ptr(fit), _lib.ptr(rmse),
        _lib.ptr(iters), _lib.ptr(ws), nb, _lib.stream()), "icp")
    return T, fit, rmse, iters


class ICPRegistration:
    """morefusion.contrib.ICPRegistration (icp_registration.py:6-71): pcd_depth [N,3] and pcd_cad
    [K,3] host arrays, transform_init [4,4] (CAD -> camera, default identity).  ``register``
    returns the refined float64 [4,4]; ``register_iterative`` yields the initial transform, then
    one per single-iteration step.  Source = depth, target = CAD, max_distance = 2 voxel_size,
    init = inv(transform) and result = inv(T), both by np.linalg.inv, as the wrapper does."""

    def __init__(self, pcd_depth, pcd_cad, transform_init=None, device=None):
        self._pcd_depth = pcd_depth
        self._pcd_cad = pcd_cad
        if transform_init is None:
            transform_init = np.eye(4)
        self._transform = transform_init
        self._device = torch.device(device if device is not None else "cuda")

    def _run(self, iteration, voxel_size):
        src = _points(np.asarray(self._pcd_depth).reshape(1, -1, 3), self._device)
        tgt = ICPTarget(self._pcd_cad, voxel_size, 2 * voxel_size, self._device)
        init = np.linalg.inv(self._transform)
        T, fit, rmse, _ = register_batch(src, [tgt], init[None], voxel_size=voxel_size,
                                         max_iteration=iteration)
        out = torch.cat([T.reshape(-1), fit, rmse]).cpu().numpy()
        if not np.isfinite(out).all():
            raise ValueError("a cloud spans 2^31 - 1 voxels or more on an axis")
        return np.linalg.inv(out[:16].reshape(4, 4)), float(out[16]), float(out[17])

    def register(self, iteration=None, voxel_size=None):
        iteration = ITERATION if iteration is None else iteration
        voxel_size = VOXEL_SIZE if voxel_size is None else voxel_size
        return self._run(iteration, voxel_size)[0]

    def register_iterative(self, iteration=None, voxel_size=None):
        iteration = ITERATION if iteration is None else iteration
        voxel_size = VOXEL_SIZE if voxel_size is None else voxel_size
        yield self._transform
        for i in range(iteration):
            T, fit, rmse = self._run(1, voxel_size)
            print(f"[{i:08d}] fitness={fit:.2g} inlier_rmse={rmse:.2g}")
            self._transform = T
            yield self._transform
