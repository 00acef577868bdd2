"""Occupancy-grid producer on the GPU (SURVEY.md 8f-3).

API of morefusion/contrib/multi_instance_octree_mapping.py:7-133 -- ``MultiInstanceOctreeMapping``
with ``instance_ids``, ``initialize(instance_id, *, pitch)``, ``integrate(instance_id, mask, pcd,
origin=(0, 0, 0))``, ``update(instance_id, occupied)``, ``get_target_grids(target_id, *,
dimensions, pitch, origin)`` and ``get_target_pcds(target_id, aabb_min=None, aabb_max=None)`` --
which is what builds ``grid_target / grid_nontarget / grid_empty`` for the pose network and the ICC
(datasets/rgbd_pose_estimation/base.py:30-50,157-162).

The reference keeps one OctoMap ``OcTree`` per instance on the host and queries it voxel by voxel
from Python (32 768 ``search`` calls per instance and target).  Here every instance lives in one
device-resident hash table of log-odds cells (csrc/mapping.cu): a depth scan is two launches, the
grids of any number of targets are one launch (``get_target_grids_batch`` returns CUDA tensors for
the per-frame path; ``get_target_grids`` returns numpy arrays like the reference).  OctoMap's
sensor model and key arithmetic are kept (hit 0.7, miss 0.4, clamping [0.1192, 0.971], 16-bit keys);
the library itself is absent from the reference tree, see oracle/octomap.py for the statement of
what is reproduced.  No CPU path: tensors live on a CUDA device.
"""

import ctypes
import math

import numpy as np
import torch

from .. import _lib

_TREE_MAX_VAL = 32768
# an instance box as stored on the device ([6] of box_enc, csrc/mapping.cu): OctoMap's default box
# (0,0,0)-(0,0,0), the sign bit set on +0's bits
_BOX_DEFAULT = -(1 << 31)


def _logodds(p):
    return np.float32(math.log(p / (1.0 - p)))


def _matrix4f(sensor_to_world):
    """A finite 4x4 host transform as the server's Eigen::Matrix4f (float32)."""
    T = np.asarray(sensor_to_world, dtype=np.float64).reshape(4, 4)
    if not np.isfinite(T).all():
        raise ValueError("sensor_to_world must be finite")
    return T.astype(np.float32)


def _host_xform(m):
    """Rows 0-2 of a float32 4x4 as the C ABI's host float[12]."""
    return (ctypes.c_float * 12)(*np.ascontiguousarray(m[:3], np.float32).reshape(-1).tolist())


def rigid_inverse_f32(m):
    """World -> sensor for a float32 rigid sensor -> world transform m: [R^T | -R^T t] computed
    in float64 from the float32 entries, rounded to float32.  publishGrids uses Eigen's general
    ``Matrix4f::inverse()`` (OctomapServer.cpp:536); its float rounding is not reproduced."""
    m = np.asarray(m, np.float32).astype(np.float64)
    R, t = m[:3, :3], m[:3, 3]
    inv = np.eye(4)
    inv[:3, :3] = R.T
    inv[:3, 3] = -((R[0] * t[0] + R[1] * t[1]) + R[2] * t[2])
    return inv.astype(np.float32)


class MultiInstanceOctreeMapping:
    PROB_HIT, PROB_MISS, CLAMP_MIN, CLAMP_MAX = 0.7, 0.4, 0.1192, 0.971     # OctoMap defaults
    # the occupancy server's sensor_model/max (OctomapServer.cpp:24): another instance's cell at or
    # above it is no-entry for get_noentry_grids_batch
    PROBABILITY_MAX = 0.97

    def __init__(self, device=None, capacity=1 << 22):
        """capacity: initial number of hash slots (power of two, 20 bytes each; the table grows x4
        when a quarter full)."""
        if capacity < 64 or capacity & (capacity - 1):
            raise ValueError("capacity must be a power of two >= 64")
        self.device = torch.device("cuda" if device is None else device)
        self._ids = {}                           # instance_id -> dense index (insertion order)
        self._pitch = []                         # per dense index
        self._scan = 0
        self._cap = int(capacity)
        self._hit, self._miss = _logodds(self.PROB_HIT), _logodds(self.PROB_MISS)
        self._lo_min, self._lo_max = _logodds(self.CLAMP_MIN), _logodds(self.CLAMP_MAX)
        self._alloc_table(self._cap)
        self._counters = torch.zeros(8, dtype=torch.int32, device=self.device)
        self._host_counters = None
        self._pending = None                     # event of the last asynchronous counter read-back
        self._res_factor = None                  # cached device array of 1 / pitch
        self._lut = None                         # cached (lut, lut_lo, resolutions) device arrays
        self._res = None                         # cached device array of every instance's resolution
        self._query_cache = None                 # cached (key, targets, pitches, origins) device arrays
        self._walk = None                        # cached (background id, walk order, its dense index)
        self._render_walk = None                 # cached (background id, walk [2, n] device array)
        # integrate_scan's per-instance world centres (by dense index), their "set" flags, the
        # scan's centre accumulators, and a host mirror of the flags (True = known to be set);
        # the instance boxes that render reads, and whether the server would have created the
        # instance's tree yet (1) or not (0: listed to integrate_scan, never in its labels)
        self._centres = self._centre_set = self._centre_sums = self._centre_first = None
        self._centre_known = None
        self._boxes = self._tree_state = None

    # ------------------------------------------------------------------ table management
    def _alloc_table(self, cap):
        dev = self.device
        # 16-byte cells {u64 key | f32 log-odds, u32 stamp}: column 0 = key (-1 = free slot),
        # column 1 = the value / stamp pair
        self._cells = torch.zeros((cap, 2), dtype=torch.int64, device=dev)
        self._cells[:, 0] = -1
        self._cnt = torch.zeros(cap, dtype=torch.int32, device=dev)
        self._cap = cap

    @property
    def _keys(self):
        return self._cells[:, 0]

    @property
    def _lo(self):
        return self._cells.view(torch.float32)[:, 2]

    def _table_args(self):
        p = _lib.ptr
        return (p(self._cells), p(self._cnt), self._cap, p(self._counters))

    def _read_back(self):
        """Asynchronous copy of the counters into pinned host memory; looked at by the next call."""
        if self._host_counters is None:
            self._host_counters = torch.zeros(8, dtype=torch.int32).pin_memory()
        self._host_counters.copy_(self._counters, non_blocking=True)
        self._pending = torch.cuda.Event()
        self._pending.record(torch.cuda.current_stream(self.device))

    def _check(self, wait=True):
        """Act on the counters of the previous operation: errors for dropped work, growth.
        `wait=False` (the per-frame calls integrate_labels / get_target_grids_batch) never blocks
        the host: if the read-back of the previous operation has not landed yet it is looked at by
        a later call (the table grows at a quarter full, so a decision that lags a scan is still
        early; overflow is sticky and cannot be missed).  The reference-style calls wait, which
        keeps growth decisions exact for small tables."""
        if self._pending is None:
            return
        if not wait and not self._pending.query():
            return
        self._pending.synchronize()
        self._pending = None
        c = self._host_counters.tolist()
        if c[1]:
            raise RuntimeError(
                f"occupancy map: hash table of {self._cap} slots overflowed during the previous "
                "operation and updates were dropped; construct the mapping with a larger capacity")
        if c[0] * 4 > self._cap:
            self._grow(self._cap * 4)

    def _grow(self, new_cap):
        L = _lib.lib()
        old = (self._cells, self._cap)
        self._alloc_table(new_cap)
        with self._dev_ctx():
            _lib.check(L.mf_map_rehash(_lib.ptr(old[0]), old[1], *self._table_args(), _lib.stream()),
                       "map_rehash")

    def _dev_ctx(self):
        return torch.cuda.device(self.device)

    # ------------------------------------------------------------------ reference API
    @property
    def instance_ids(self):
        return list(self._ids.keys())

    def initialize(self, instance_id, *, pitch):
        if instance_id in self._ids:
            raise ValueError("instance {instance_id} already exists")
        if not pitch > 0:
            raise ValueError("pitch must be positive")
        if len(self._ids) >= 0xFFFF:
            raise ValueError("too many instances")
        self._ids[instance_id] = len(self._ids)
        self._pitch.append(float(pitch))
        self._res_factor = None
        self._lut = None
        self._res = None
        self._walk = None
        self._render_walk = None

    def integrate(self, instance_id, mask, pcd, origin=(0, 0, 0)):
        """octree.insertPointCloud(pcd[mask & nonnan], origin) (:21-27).  mask [H,W] bool, pcd
        [H,W,3]; numpy arrays or tensors (CUDA tensors are used in place)."""
        idx = self._ids[instance_id]                       # KeyError for an unknown instance, as the dict
        dev = self.device
        pts = torch.as_tensor(pcd).to(device=dev, dtype=torch.float32).contiguous()
        msk = torch.as_tensor(mask).to(device=dev)
        if pts.dim() < 2 or pts.shape[-1] != 3 or tuple(msk.shape) != tuple(pts.shape[:-1]):
            raise ValueError("pcd must be [..., 3] and mask its leading shape")
        if msk.dtype != torch.bool:
            raise ValueError("mask must be bool")
        _lib.require_cuda(pts, msk)
        msk = msk.contiguous().view(torch.uint8)
        n = pts.numel() // 3
        org = np.asarray(origin, dtype=np.float64).astype(np.float32)      # point3d: floats
        self._check()
        if n == 0:
            return
        self._scan += 1
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_integrate(
                _lib.ptr(pts), _lib.ptr(msk), n, float(org[0]), float(org[1]), float(org[2]),
                self._pitch[idx], idx, self._scan, float(self._hit), float(self._miss),
                float(self._lo_min), float(self._lo_max), *self._table_args(), _lib.stream()),
                "map_integrate")
            self._read_back()

    def integrate_labels(self, label, pcd, origin=(0, 0, 0)):
        """Every initialised instance of a labelled frame in one scan: equal to
        ``for i in instance_ids: integrate(i, label == i, pcd, origin)`` (what build_octomap,
        datasets/rgbd_pose_estimation/base.py:30-50, does instance by instance), as two launches.
        label [H,W] integer image; pixels whose label is not an initialised instance are skipped."""
        dev = self.device
        pts = torch.as_tensor(pcd).to(device=dev, dtype=torch.float32).contiguous()
        lab = torch.as_tensor(label).to(device=dev)
        if pts.dim() < 2 or pts.shape[-1] != 3 or tuple(lab.shape) != tuple(pts.shape[:-1]):
            raise ValueError("pcd must be [..., 3] and label its leading shape")
        if lab.dtype.is_floating_point or lab.dtype == torch.bool:
            raise ValueError("label must be an integer image")
        _lib.require_cuda(pts, lab)
        lab = lab.to(torch.int32).contiguous()
        n = pts.numel() // 3
        org = np.asarray(origin, dtype=np.float64).astype(np.float32)
        self._check(wait=False)
        if n == 0 or not self._ids:
            return
        lut, lo, res = self._label_lut()
        self._scan += 1
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_integrate_labelled(
                _lib.ptr(pts), _lib.ptr(lab), n, float(org[0]), float(org[1]), float(org[2]),
                _lib.ptr(lut), lo, lut.numel(), _lib.ptr(res), self._scan, float(self._hit),
                float(self._miss), float(self._lo_min), float(self._lo_max), *self._table_args(),
                _lib.stream()), "map_integrate_labelled")
            self._read_back()

    def update(self, instance_id, occupied):
        """octree.updateNodes(occupied, True) (:29-34): one hit update per row of occupied [M,3]."""
        idx = self._ids[instance_id]
        pts = torch.as_tensor(occupied).to(device=self.device, dtype=torch.float64).reshape(-1, 3).contiguous()
        _lib.require_cuda(pts)
        self._check()
        if pts.shape[0] == 0:
            return
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_update_points(
                _lib.ptr(pts), pts.shape[0], self._pitch[idx], idx, float(self._hit),
                float(self._lo_min), float(self._lo_max), *self._table_args(), _lib.stream()),
                "map_update_points")
            self._read_back()

    def get_target_grids_batch(self, target_ids, *, dimensions, pitches, origins):
        """The three grids of several targets from one launch.  Returns CUDA tensors
        (grid_target, grid_nontarget, grid_empty), each [T, X, Y, Z] float32.

        pitches [T] / origins [T,3] are host arrays, or CUDA tensors that stay on the device (no
        host read: their positivity / NaN checks are then the caller's)."""
        T, X, Y, Z, d_tix, d_pit, d_org = self._query_args(target_ids, dimensions, pitches, origins)
        out = torch.empty((3, T, X, Y, Z), dtype=torch.float32, device=self.device)
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_query_grids(
                _lib.ptr(d_tix), _lib.ptr(d_pit), _lib.ptr(d_org), T, X, Y, Z,
                _lib.ptr(self._res_factor), len(self._pitch), *self._table_args(),
                _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(out[2]), _lib.stream()), "map_query_grids")
        return out[0], out[1], out[2]

    def get_noentry_grids_batch(self, target_ids, *, dimensions, pitches, origins, background_id=0,
                                sensor_to_world=None, ground_as_noentry=False):
        """The grid / grid_noentry pair the ROS occupancy server publishes for the refinement node
        (OctomapServer::publishGrids, ros/src/morefusion_ros/src/OctomapServer.cpp:510-618), for
        several targets from one launch.  Returns CUDA tensors (grid, grid_noentry), each
        [T, X, Y, Z] float32.

        grid is the target's occupancy where it is > 0.5.  Elsewhere grid_noentry is the occupancy
        of another instance where it is >= PROBABILITY_MAX, or 1 - occupancy where the
        background instance ``background_id`` is free (< 0.5); where several instances qualify the
        one the server pushes last wins (the background first, then ascending instance id).  The
        voxel centre is rounded to float before the look-up, as the server's PCL point is.
        pitches / origins as in ``get_target_grids_batch``; targets must not be the background.
        A ``background_id`` that is not initialised means no free-space no-entry.

        sensor_to_world [4,4] (host): the origins are in the camera's frame and the map in the
        world's, as for a map fed by ``integrate_scan``; each float voxel centre is moved to the
        world in float32 before the look-up (:573-576).  ground_as_noentry (with
        sensor_to_world): a voxel whose world z < 0 is no-entry at PROBABILITY_MAX and is not
        looked up (:579-583; the reference launches the server with it off)."""
        if background_id in target_ids:
            raise ValueError("the background instance cannot be a refinement target")
        T, X, Y, Z, d_tix, d_pit, d_org = self._query_args(target_ids, dimensions, pitches, origins)
        if self._walk is None or self._walk[0] != background_id:
            # the server's std::map order, with its background (-1) first, reversed
            others = sorted((i for i in self._ids if i != background_id), reverse=True)
            walk = [self._ids[i] for i in others]
            if background_id in self._ids:
                walk.append(self._ids[background_id])
            self._walk = (background_id, torch.as_tensor(np.asarray(walk, np.int32)).to(self.device),
                          self._ids.get(background_id, -1))
        _, d_walk, bg = self._walk
        out = torch.empty((2, T, X, Y, Z), dtype=torch.float32, device=self.device)
        with self._dev_ctx():
            if sensor_to_world is None:
                if ground_as_noentry:
                    raise ValueError("ground_as_noentry needs sensor_to_world")
                _lib.check(_lib.lib().mf_map_query_node_grids(
                    _lib.ptr(d_tix), _lib.ptr(d_pit), _lib.ptr(d_org), T, X, Y, Z,
                    _lib.ptr(self._res_factor), _lib.ptr(d_walk), len(self._pitch), bg,
                    float(self.PROBABILITY_MAX), *self._table_args(), _lib.ptr(out[0]),
                    _lib.ptr(out[1]), _lib.stream()), "map_query_node_grids")
            else:
                _lib.check(_lib.lib().mf_map_query_node_grids_world(
                    _lib.ptr(d_tix), _lib.ptr(d_pit), _lib.ptr(d_org), T, X, Y, Z,
                    _lib.ptr(self._res_factor), _lib.ptr(d_walk), len(self._pitch), bg,
                    float(self.PROBABILITY_MAX), _host_xform(_matrix4f(sensor_to_world)),
                    int(bool(ground_as_noentry)), *self._table_args(), _lib.ptr(out[0]),
                    _lib.ptr(out[1]), _lib.stream()), "map_query_node_grids_world")
        return out[0], out[1]

    # ------------------------------------------------------------------ the occupancy server
    def integrate_scan(self, label, pcd, sensor_to_world, class_ids, *, max_range=-1.0,
                       background_id=-1, uncertain_id=-2, background_pitch=0.01):
        """One frame of a moving camera into the map in the world frame, as the ROS occupancy
        server's ``insertScan`` does it (OctomapServer.cpp:283-448); five launches, no host sync.

        label [H,W] integer image, pcd [H,W,3] organised camera-frame cloud (NaN = no depth),
        sensor_to_world [4,4] host array, class_ids {instance_id: class_id}.

        Listed instances that are new are initialised at their class pitch
        (``YCB_VOXEL_PITCH_32``, the server's class_id_to_voxel_pitch), the background at
        ``background_pitch`` (the reference launches the server at 0.01, setup_static.xml:41).
        Only pixels of even row and column are used.  Points are moved to the world in float32
        as pcl::transformPointCloud does with a Matrix4f; the sensor origin is float32(T[:3, 3]).
        Inside ``max_range`` (< 0: no limit) every pixel casts a free ray through the
        background's cells only, a pixel labelled with an instance (the background included) is
        a hit in that instance, and a pixel not labelled background, ``uncertain_id`` included,
        frees its end cell in the background.  Beyond ``max_range`` the free ray stops at
        max_range and nothing is hit.  Each cell is updated at most once per scan and a
        background cell hit in the scan is not freed; instances other than the background are
        never freed.

        Labels that are neither initialised, listed, the background nor ``uncertain_id`` are
        skipped.  (The server aborts the whole scan there.)  Instance ids must be consistent
        across frames: the server's instance tracking is not part of this map.

        The first scan in which an instance pushes a point sets its world centre for good
        (``server_grid_params``): the mean of its listed points of that scan, beyond max_range
        too, except the one of lowest pixel index (the server does not push an instance's first
        point, :345-349).  The sum is exact in a fixed point of 2^-32 m, so it does not depend
        on thread order.  An instance with no pushed point has no centre yet (the server would
        read an uninitialised centroid).

        Each instance other than the background keeps a box (``boxes``, read by ``render``),
        widened by the points it pushed (insertScan's setBBXMin/Max, :404-437); in the first scan
        whose labels hold its id on any pixel (where the server creates its tree) the box is set
        to those points alone."""
        from .singleview_3d.models.model import YCB_VOXEL_PITCH_32
        dev = self.device
        T = _matrix4f(sensor_to_world)
        pts = torch.as_tensor(pcd).to(device=dev, dtype=torch.float32).contiguous()
        lab = torch.as_tensor(label).to(device=dev)
        if pts.dim() != 3 or pts.shape[2] != 3 or tuple(lab.shape) != tuple(pts.shape[:2]):
            raise ValueError("pcd must be [H,W,3] and label [H,W]")
        if lab.dtype.is_floating_point or lab.dtype == torch.bool:
            raise ValueError("label must be an integer image")
        _lib.require_cuda(pts, lab)
        classes = {int(i): int(c) for i, c in dict(class_ids).items()}
        if uncertain_id == background_id:
            raise ValueError("uncertain_id and background_id must differ")
        if background_id in classes:
            raise ValueError("the background must not be listed in class_ids")
        if uncertain_id in classes or uncertain_id in self._ids:
            raise ValueError("uncertain_id must not be an instance id")
        for c in classes.values():
            if not 1 <= c < len(YCB_VOXEL_PITCH_32):
                raise IndexError(f"class_id {c} out of range")
        if not background_pitch > 0:
            raise ValueError("background_pitch must be positive")
        first_new = len(self._pitch)       # created below: no tree until the labels hold them
        for i, c in classes.items():
            if i not in self._ids:
                self.initialize(i, pitch=YCB_VOXEL_PITCH_32[c])
        if background_id not in self._ids:
            self.initialize(background_id, pitch=background_pitch)
        self._ensure_centres()
        self._tree_state[first_new:len(self._pitch)] = 0
        H, W = int(pts.shape[0]), int(pts.shape[1])
        lab = lab.to(torch.int32).contiguous()
        self._check(wait=False)
        if H * W == 0:
            return
        lut, lo, res = self._label_lut()
        bg = self._ids[background_id]
        self._scan += 1
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_integrate_server(
                _lib.ptr(pts), _lib.ptr(lab), H, W, _host_xform(T), float(max_range),
                _lib.ptr(lut), lo, lut.numel(), _lib.ptr(res), len(self._pitch), bg,
                self._pitch[bg], int(uncertain_id), self._scan, float(self._hit), float(self._miss),
                float(self._lo_min), float(self._lo_max), _lib.ptr(self._centre_sums),
                _lib.ptr(self._centre_first), _lib.ptr(self._centres), _lib.ptr(self._centre_set),
                *self._table_args(), _lib.ptr(self._tree_state), _lib.ptr(self._boxes),
                _lib.stream()),
                "map_integrate_server")
            self._read_back()

    def server_grid_params(self, target_ids, sensor_to_world, dimensions=(32, 32, 32)):
        """The pitch and origin of each target's grids as the ROS occupancy server publishes them
        in the current camera's frame (publishGrids, OctomapServer.cpp:534-551): CUDA float64
        tensors pitches [T] (the instance's pitch) and origins [T,3] = centre_sensor - (D / 2 -
        0.5) * pitch, centre_sensor the world centre of ``integrate_scan`` moved to the camera by
        the rigid inverse of sensor_to_world in float.  No host read, except once when the host
        has not yet seen a target's centre being set.  A target without a centre raises
        ValueError."""
        dims = np.asarray(dimensions, np.float64).reshape(3)
        tix = np.asarray([self._ids[t] for t in target_ids], dtype=np.int32)
        T = len(tix)
        if T == 0:
            return (torch.empty(0, dtype=torch.float64, device=self.device),
                    torch.empty((0, 3), dtype=torch.float64, device=self.device))
        self._ensure_centres()
        if not self._centre_known[tix].all():
            self._centre_known[:len(self._pitch)] = self._centre_set[:len(self._pitch)].cpu().numpy() != 0
            missing = [t for t, q in zip(target_ids, tix) if not self._centre_known[q]]
            if missing:
                raise ValueError(f"instances {missing} have no centre yet: no scan has pushed a "
                                 "point of them")
        inv = rigid_inverse_f32(_matrix4f(sensor_to_world))
        from ..functions.geometry import _util
        d_tix = _util.h2d(tix, self.device, torch.int32, "map/grid_params_targets")
        pitch = torch.empty(T, dtype=torch.float64, device=self.device)
        origin = torch.empty((T, 3), dtype=torch.float64, device=self.device)
        off = dims / 2.0 - 0.5
        res = self._label_lut()[2]
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_server_grid_params(
                _lib.ptr(d_tix), T, _lib.ptr(res), _lib.ptr(self._centres), _host_xform(inv),
                float(off[0]), float(off[1]), float(off[2]), _lib.ptr(pitch), _lib.ptr(origin),
                _lib.stream()), "map_server_grid_params")
        return pitch, origin

    def _centre_flags(self, instance_ids):
        """Device int32 [N]: 1 where the instance has a centre (0 for ids not in the map), for a
        caller that folds it into a read it does anyway and then calls ``_note_centres``."""
        self._ensure_centres()
        idx = np.asarray([self._ids.get(int(i), -1) for i in instance_ids], np.int64)
        from ..functions.geometry import _util
        d_idx = _util.h2d(np.maximum(idx, 0), self.device, torch.int64, "map/centre_flags")
        flags = self._centre_set.index_select(0, d_idx)
        return flags * _util.h2d((idx >= 0).astype(np.int32), self.device, torch.int32,
                                 "map/centre_flags_known")

    def _note_centres(self, instance_ids, flags):
        """Record host-read flags of ``_centre_flags`` in the host mirror."""
        for i, f in zip(instance_ids, np.asarray(flags).reshape(-1)):
            if f and int(i) in self._ids:
                self._centre_known[self._ids[int(i)]] = True

    def _ensure_centres(self):
        """Per-instance centre arrays for every initialised instance (grown x2 on demand)."""
        n = len(self._pitch)
        cap = 0 if self._centres is None else self._centres.shape[0]
        if n <= cap:
            return
        new = max(16, 1 << (n - 1).bit_length())
        dev = self.device
        sums = torch.zeros((new, 4), dtype=torch.int64, device=dev)
        first = torch.zeros(new, dtype=torch.int32, device=dev)
        centres = torch.zeros((new, 3), dtype=torch.float32, device=dev)
        cset = torch.zeros(new, dtype=torch.int32, device=dev)
        known = np.zeros(new, bool)
        boxes = torch.full((new, 6), _BOX_DEFAULT, dtype=torch.int32, device=dev)
        trees = torch.ones(new, dtype=torch.int32, device=dev)
        if cap:
            sums[:cap] = self._centre_sums
            first[:cap] = self._centre_first
            centres[:cap] = self._centres
            cset[:cap] = self._centre_set
            known[:cap] = self._centre_known
            boxes[:cap] = self._boxes
            trees[:cap] = self._tree_state
        self._centre_sums, self._centre_first = sums, first
        self._centres, self._centre_set, self._centre_known = centres, cset, known
        self._boxes, self._tree_state = boxes, trees

    def centres(self):
        """{instance_id: world centre float32 [3]} of the instances that have one (host read;
        for tests and tools)."""
        self._ensure_centres()
        c = self._centres.cpu().numpy()
        s = self._centre_set.cpu().numpy()
        return {i: c[q].copy() for i, q in self._ids.items() if s[q]}

    def boxes(self, background_id=-1):
        """{instance_id: float32 [2, 3] (min, max)} of every instance but the background: the box
        ``integrate_scan`` keeps and ``render`` tests points against.  An instance that no scan
        has boxed has OctoMap's default box, all zeros.  (Host read; for tests and tools.)"""
        self._ensure_centres()
        if not self._ids:
            return {}
        e = self._boxes[:len(self._pitch)].cpu().numpy().view(np.uint32)
        bits = np.where(e & 0x80000000, e & 0x7FFFFFFF, ~e).astype(np.uint32)
        b = bits.view(np.float32).reshape(-1, 2, 3)
        return {i: b[q].copy() for i, q in self._ids.items() if i != background_id}

    def render(self, pcd, sensor_to_world, K, *, background_id=-1, uncertain_id=-2):
        """The map's own label image of the current view, as the ROS occupancy server's
        ``render`` draws it (OctomapServer.cpp:193-281).  Returns CUDA tensors label [H, W]
        int32 and depth [H, W] float32; two launches, no host sync.

        pcd [H, W, 3] organised camera-frame cloud (NaN = no depth) and sensor_to_world [4, 4]
        (host) as ``integrate_scan`` takes them, K [3, 3] host intrinsics.  For every pixel of
        even row and column and every instance but ``background_id``: a pixel with depth is moved
        to the world as in ``integrate_scan`` and is skipped unless it lies in the instance's box
        (``boxes``); a pixel without depth targets the z = 1 point of its ray, (u - cx) / fx,
        (v - cy) / fy in float, with no box test.  OctoMap's castRay from the sensor origin
        towards the target, unknown cells ignored, up to 1.1 times the target's distance, finds
        the first occupied cell of the instance (log-odds >= 0) in its own key space.  Of the
        instances hit, the nearest cell centre wins the pixel -- on an exact tie the lower
        instance id, as the server run on one thread --: its float distance is depth[v, u] and its
        id fills label[v-1:v+1, u-1:u+1] (clipped at the image edge).  Every other label pixel is
        ``uncertain_id``, every other depth pixel NaN."""
        dev = self.device
        T = _matrix4f(sensor_to_world)
        K = np.asarray(K, np.float64).reshape(3, 3)
        if not np.isfinite(K).all():
            raise ValueError("K must be finite")
        fx, fy, cx, cy = (float(np.float32(k)) for k in (K[0, 0], K[1, 1], K[0, 2], K[1, 2]))
        pts = torch.as_tensor(pcd).to(device=dev, dtype=torch.float32).contiguous()
        if pts.dim() != 3 or pts.shape[2] != 3:
            raise ValueError("pcd must be [H,W,3]")
        _lib.require_cuda(pts)
        H, W = int(pts.shape[0]), int(pts.shape[1])
        label = torch.empty((H, W), dtype=torch.int32, device=dev)
        depth = torch.empty((H, W), dtype=torch.float32, device=dev)
        self._check(wait=False)
        if H * W == 0:
            return label, depth
        if self._render_walk is None or self._render_walk[0] != background_id:
            ids = sorted(i for i in self._ids if i != background_id)       # the server's std::map order
            walk = np.asarray([[self._ids[i] for i in ids], ids], np.int64).reshape(2, -1)
            if walk.size and not (np.abs(walk[1]) < 1 << 31).all():
                raise ValueError("instance ids must fit in int32 to be rendered")
            self._render_walk = (background_id, torch.as_tensor(walk.astype(np.int32)).to(dev))
        walk = self._render_walk[1]
        n_walk = walk.shape[1]
        self._ensure_centres()
        res = self._resolutions() if n_walk else None
        zbuf = torch.empty(((H + 1) // 2) * ((W + 1) // 2), dtype=torch.int64, device=dev)
        with self._dev_ctx():
            _lib.check(_lib.lib().mf_map_render(
                _lib.ptr(pts), H, W, _host_xform(T), fx, fy, cx, cy, _lib.ptr(walk[0]),
                _lib.ptr(walk[1]), n_walk, _lib.ptr(res), _lib.ptr(self._boxes), int(uncertain_id),
                _lib.ptr(zbuf), _lib.ptr(label), _lib.ptr(depth), *self._table_args(),
                _lib.stream()), "map_render")
        return label, depth

    def _resolutions(self):
        """Cached float64 device array of every instance's resolution, by dense index."""
        if self._res is None:
            self._res = torch.as_tensor(np.asarray(self._pitch, dtype=np.float64)).to(self.device)
        return self._res

    def _label_lut(self):
        """Cached (lut, lut_lo, resolutions) device arrays: label - lut_lo -> dense index."""
        if self._lut is None:
            ids = [int(i) for i in self._ids]            # instance ids must be integers here
            lo, hi = min(ids), max(ids)
            if hi - lo >= 1 << 20:
                raise ValueError("instance ids span too wide a range for a label look-up table")
            lut = np.full(hi - lo + 1, -1, np.int32)
            for i, idx in self._ids.items():
                lut[int(i) - lo] = idx
            dev = self.device
            self._lut = (torch.as_tensor(lut).to(dev), lo, self._resolutions())
        return self._lut

    def _query_args(self, target_ids, dimensions, pitches, origins):
        """Checks and device arrays shared by the grid queries: T, X, Y, Z and the targets' dense
        indices, pitches and origins on the device."""
        assert len(dimensions) == 3
        assert (np.asarray(dimensions) > 0).all()
        T = len(target_ids)
        on_device = isinstance(pitches, torch.Tensor) and isinstance(origins, torch.Tensor)
        if on_device:
            _lib.require_cuda(pitches, origins)
        else:
            pit = np.asarray(pitches, dtype=np.float64).reshape(T)
            org = np.asarray(origins, dtype=np.float64).reshape(T, 3)
            assert not np.isnan(org).any()
            assert (pit > 0).all()
        tix = np.asarray([self._ids[t] for t in target_ids], dtype=np.int32)
        dev = self.device
        self._check(wait=False)
        if self._res_factor is None:
            self._res_factor = torch.as_tensor(1.0 / np.asarray(self._pitch, dtype=np.float64)).to(dev)
        X, Y, Z = (int(d) for d in dimensions)
        if on_device:
            from ..functions.geometry import _util
            d_tix = _util.h2d(tix, dev, torch.int32, "map/query_targets")
            d_pit = pitches.to(device=dev, dtype=torch.float64).reshape(T).contiguous()
            d_org = origins.to(device=dev, dtype=torch.float64).reshape(T, 3).contiguous()
        else:
            # the per-frame path asks for the same targets frame after frame: their small device
            # arrays are uploaded once per distinct (targets, pitches, origins)
            key = (tix.tobytes(), pit.tobytes(), org.tobytes())
            if self._query_cache is None or self._query_cache[0] != key:
                self._query_cache = (key, torch.as_tensor(tix).to(dev), torch.as_tensor(pit).to(dev),
                                     torch.as_tensor(org).to(dev))
            _, d_tix, d_pit, d_org = self._query_cache
        return T, X, Y, Z, d_tix, d_pit, d_org

    def get_target_grids(self, target_id, *, dimensions, pitch, origin):
        """(grid_target, grid_nontarget, grid_empty) as float32 numpy arrays of shape `dimensions`
        (:35-94)."""
        assert not np.isnan(origin).any()
        assert pitch > 0
        self._check()
        gt, gn, ge = self.get_target_grids_batch(
            [target_id], dimensions=dimensions, pitches=[pitch], origins=[origin])
        return gt[0].cpu().numpy(), gn[0].cpu().numpy(), ge[0].cpu().numpy()

    def get_target_pcds(self, target_id, aabb_min=None, aabb_max=None):
        """Centres of the occupied / free cells of one instance, float64 [N,3] / [M,3] (:96-133).
        Rows are in key order (the reference returns them in OctoMap's tree-iteration order)."""
        idx = self._ids[target_id]
        self._check()
        keys = self._keys
        sel = (keys != -1) & (((keys >> 48) & 0xFFFF) == idx)
        k = keys[sel]
        lo = self._lo[sel]
        order = torch.argsort(k)
        k, lo = k[order], lo[order]
        kxyz = torch.stack([(k >> 32) & 0xFFFF, (k >> 16) & 0xFFFF, k & 0xFFFF], 1)
        coords = ((kxyz - _TREE_MAX_VAL).to(torch.float64) + 0.5) * self._pitch[idx]
        coords = coords.to(torch.float32).to(torch.float64).cpu().numpy()   # point3d floats -> float64
        occ = (lo >= 0).cpu().numpy()
        # axis-aligned box [aabb_min, aabb_max): lower bound inclusive, upper exclusive (:124-131)
        inside = np.ones(len(coords), dtype=bool)
        if aabb_min is not None:
            inside &= (coords >= np.asarray(aabb_min)).all(axis=1)
        if aabb_max is not None:
            inside &= (coords < np.asarray(aabb_max)).all(axis=1)
        return coords[occ & inside], coords[~occ & inside]

    # ------------------------------------------------------------------ introspection (tests, bench)
    def n_cells(self):
        return int(self._counters[0].item())

    def cells(self, instance_id):
        """{(kx, ky, kz): log-odds} of one instance (host dict; for tests)."""
        idx = self._ids[instance_id]
        cells = self._cells.cpu()
        keys = cells[:, 0].numpy()
        lo = cells.view(torch.float32)[:, 2].numpy()
        sel = (keys != -1) & (((keys >> 48) & 0xFFFF) == idx)
        out = {}
        for k, v in zip(keys[sel].tolist(), lo[sel].tolist()):
            out[((k >> 32) & 0xFFFF, (k >> 16) & 0xFFFF, k & 0xFFFF)] = np.float32(v)
        return out
