"""get_example of morefusion/datasets/rgbd_pose_estimation/base.py:78-197 on the device: the map,
the crops, the origins and the target grids of ``contrib.singleview_3d.frame.build_examples``,
and the ground-truth full grids of every kept instance (csrc/training_examples.cu)."""

import numpy as np
import torch

from .. import _lib
from .. import geometry
from .. import synthetic
from ..contrib.singleview_3d.frame import build_examples, empty_examples
from ..functions.geometry import _util

MAX_INSTANCES = 64          # the Transform's non-target id mask is 64 bits wide
VOXEL_DIM = 32


def full_grids(points, offsets, seg, R, t, origin, pitch, d_offsets=None):
    """``_get_grid_full`` (base.py:52-76) for every kept instance of a frame, as get_example
    calls it (:179-195): grid_target_full [M,32,32,32] int32 (1 where instance i's own solid
    points land) and grid_nontarget_full [M,32,32,32] int32 (where instance j != i lands, j's
    position in examples_nontarget + 1; where several land, the largest, which is the
    reference loop's last writer).

    points [Ntot,3] CUDA float64, the solid points of every class back to back; offsets [S+1]
    host int64 (d_offsets: the same on the device, uploaded here when None); seg [M] host, the
    segment of each instance; R [M,3,3], t [M,3] host float64, the ground-truth cad->camera
    transforms; origin [M,3] float32 and pitch [M] float64, the instances' grids (CUDA tensors,
    or host arrays uploaded here).  p' = ((r0 x + r1 y) + r2 z) + t in float64 and index =
    round_half_even((p' - origin) / pitch), kept inside the grid.  Two launches, no host read.
    More than 64 instances raise ValueError before any launch."""
    seg = np.asarray(seg, np.int64).reshape(-1)
    M = seg.size
    if M > MAX_INSTANCES:
        raise ValueError(f"at most {MAX_INSTANCES} kept instances per frame, got {M}")
    _lib.require_cuda(points)
    dev = points.device
    offsets = np.asarray(offsets, np.int64).reshape(-1)
    if ((seg < 0) | (seg >= offsets.size - 1)).any():
        raise IndexError("full_grids: segment index out of range")
    out = torch.empty((2, M, VOXEL_DIM, VOXEL_DIM, VOXEL_DIM), dtype=torch.int32, device=dev)
    if M == 0:
        return out[0], out[1]
    Rt = np.concatenate([np.asarray(R, np.float64).reshape(M, 3, 3),
                         np.asarray(t, np.float64).reshape(M, 3, 1)], 2)
    d_rt = _util.h2d(Rt, dev, torch.float64, "full_grids/Rt")
    d_seg = _util.h2d(seg.astype(np.int32), dev, torch.int32, "full_grids/seg")
    d_org = _util.h2d(origin, dev, torch.float32, "full_grids/origin").contiguous()
    d_pit = _util.h2d(pitch, dev, torch.float64, "full_grids/pitch").contiguous()
    if d_offsets is None:
        d_offsets = _util.h2d_transient(offsets, dev, torch.int64)
    max_points = int(np.diff(offsets)[seg].max())
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().mf_training_full_grids(
            M, _lib.ptr(points), _lib.ptr(d_offsets), _lib.ptr(d_seg), max_points, _lib.ptr(d_rt),
            _lib.ptr(d_org), _lib.ptr(d_pit), _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.stream()),
            "training full_grids")
    return out[0], out[1]


class RGBDPoseEstimationDatasetBase:
    """RGBDPoseEstimationDatasetBase(models, class_ids=None, with_visibility=False): subclasses implement ``get_frame``
    (a dict with instance_ids [N], class_ids [N], rgb [H,W,3] uint8, depth [H,W] float metres,
    instance_label [H,W], intrinsic_matrix [3,3] and Ts_cad2cam [N,4,4]) and ``__len__``.

    models: ``get_voxel_pitch(dimension, class_id)`` and ``get_solid_voxel_grid(class_id)``
    (an object with ``.points`` [n,3], the solid voxel centres in the CAD frame).  class_ids:
    the classes an example may have (the others still go into the map).  device: where the
    examples are built (the current CUDA device when None).  with_visibility: examples also hold
    ``visibility`` (``get_example``), which needs ``models.get_cad(class_id)`` (an object with
    ``.vertices`` [V,3] and ``.faces`` [F,3]); off by default, as in the reindexed datasets that
    training uses (reindexed.py:159-160 drop it)."""

    _n_points_minimal = 1
    _image_size = 256
    _voxel_dim = VOXEL_DIM
    _n_fg_class = 21

    def __init__(self, models, class_ids=None, device=None, with_visibility=False):
        self._models = models
        self._with_visibility = bool(with_visibility)
        self._cad_cache = {}
        self._class_ids = tuple(class_ids) if class_ids is not None else None
        self._device = torch.device(device) if device is not None else None
        self._pitch_table = np.array(
            [np.nan] + [models.get_voxel_pitch(self._voxel_dim, c)
                        for c in range(1, self._n_fg_class + 1)], dtype=np.float64)
        self._solid_cache = {}

    def get_frame(self, index):
        raise NotImplementedError

    def _dev(self):
        if self._device is not None:
            return self._device
        return torch.device("cuda", torch.cuda.current_device())

    def _solid_table(self, dev):
        """Every class's solid points back to back on the device in float64 (uploaded once), the
        host int64 offsets [n_fg_class + 1] (class c is segment c - 1) and the same offsets on
        the device."""
        key = str(dev)
        if key not in self._solid_cache:
            pts = [np.asarray(self._models.get_solid_voxel_grid(c).points, np.float64).reshape(-1, 3)
                   for c in range(1, self._n_fg_class + 1)]
            offsets = np.r_[0, np.cumsum([len(p) for p in pts])].astype(np.int64)
            self._solid_cache[key] = (
                _util.h2d_transient(np.concatenate(pts), dev, torch.float64), offsets,
                _util.h2d_transient(offsets, dev, torch.int64))
        return self._solid_cache[key]

    def _cad_table(self, dev):
        """Every class's CAD mesh back to back on the device (checked on the host and uploaded
        once): vertices [V,3] float64, faces [F,3] int32 indexing the packed vertices, and the
        host int64 face offsets [n_fg_class + 1] (class c is mesh c - 1)."""
        key = str(dev)
        if key not in self._cad_cache:
            vs, fs, offsets, base = [], [], [0], 0
            for c in range(1, self._n_fg_class + 1):
                cad = self._models.get_cad(c)
                v, f = geometry._check_mesh(cad.vertices, cad.faces)
                vs.append(v)
                fs.append(f + base)
                base += len(v)
                offsets.append(offsets[-1] + len(f))
            self._cad_cache[key] = (
                _util.h2d_transient(np.concatenate(vs), dev, torch.float64),
                _util.h2d_transient(np.concatenate(fs), dev, torch.int32),
                np.asarray(offsets, np.int64))
        return self._cad_cache[key]

    def _visibility(self, ex, cls_kept, Ts, K, height, width, dev):
        """visibility [M] float64: each kept instance's label-mask pixel count over the pixel
        count of its CAD model rendered alone at Ts_cad2cam (base.py:139-148), every instance in
        one render call; 0/0 gives NaN and x/0 inf, as NumPy does under the reference's
        errstate."""
        n_mask = ex.pop("n_mask")
        if len(cls_kept) == 0:
            return torch.empty(0, dtype=torch.float64, device=dev)
        vertices, faces, offsets = self._cad_table(dev)
        fovy = geometry.fovy_from_intrinsics(K[1, 1], height)
        _, _, count = geometry._render_cad_batch(
            vertices, faces, offsets, cls_kept.astype(np.int32) - 1, Ts,
            f=geometry.focal_from_fovy(fovy, height), height=height, width=width)
        return n_mask.to(torch.float64) / count.to(torch.float64)

    def get_example(self, index):
        """The kept instances of frame ``index`` as one batched dict of CUDA tensors, with
        get_example's keys except visibility: class_id [M] int32, rgb [M,256,256,3] uint8, pcd
        [M,256,256,3] float32, quaternion_true [M,4] and translation_true [M,3] float64
        (quaternion_from_matrix / translation_from_matrix of Ts_cad2cam), origin [M,3] float32,
        pitch [M] float64, grid_target / grid_nontarget / grid_empty [M,32,32,32] float32 as the
        map query returns them, grid_target_full / grid_nontarget_full [M,32,32,32] int32
        (``full_grids``); and instance_ids [M] (numpy).  With ``with_visibility``, also
        visibility [M] float64 (``_visibility``).  The keep rules are the reference's
        (``build_examples``).  Host reads: those of ``build_examples`` with the map built from the
        frame; the full grids and the visibility add none."""
        frame = self.get_frame(index)
        dev = self._dev()
        D = self._voxel_dim
        ids = np.asarray(frame["instance_ids"]).reshape(-1)
        cls = np.asarray(frame["class_ids"]).reshape(-1)
        Ts = np.asarray(frame["Ts_cad2cam"], np.float64).reshape(-1, 4, 4)
        if ids.size == 0:                       # the reference returns before building the map
            ex, cls_kept = empty_examples(dev, D, self._image_size), np.empty(0, np.int32)
        else:
            ex, cls_kept, _ = build_examples(
                frame["rgb"], frame["depth"], frame["intrinsic_matrix"], frame["instance_label"],
                ids, cls, self._pitch_table, dev=dev, n_points_minimal=self._n_points_minimal,
                dimensions=D, image_size=self._image_size, class_filter=self._class_ids or None,
                with_n_mask=self._with_visibility)
        if self._with_visibility and "n_mask" not in ex:
            ex["n_mask"] = torch.empty(0, dtype=torch.int32, device=dev)
        Ts = Ts[ex.pop("index")]
        q = np.zeros((len(Ts), 4))
        R = np.zeros((len(Ts), 3, 3))
        for m, T in enumerate(Ts):
            q[m] = geometry.quaternion_from_matrix(T)
            R[m] = geometry.quaternion_matrix(q[m])[:3, :3]
        t = Ts[:, :3, 3].copy()
        points, offsets, d_offsets = self._solid_table(dev)
        gtf, gnf = full_grids(points, offsets, cls_kept.astype(np.int64) - 1, R, t, ex["origin"],
                              ex["pitch"], d_offsets=d_offsets)
        ex["quaternion_true"] = _util.h2d(q, dev, torch.float64, "example/q")
        ex["translation_true"] = _util.h2d(t, dev, torch.float64, "example/t")
        ex["grid_target_full"] = gtf
        ex["grid_nontarget_full"] = gnf
        if self._with_visibility:
            H, W = np.shape(frame["instance_label"])[:2]
            ex["visibility"] = self._visibility(
                ex, cls_kept, Ts, np.asarray(frame["intrinsic_matrix"], np.float64).reshape(3, 3),
                H, W, dev)
        return ex


class SyntheticRGBDPoseEstimationDataset(RGBDPoseEstimationDatasetBase):
    """Frames of ``synthetic.make_pose_frame``: frame i is seed ``seed + i``."""

    def __init__(self, size, seed=0, n_objects=8, class_ids=None, models=None, device=None,
                 with_visibility=False):
        super().__init__(synthetic.SyntheticYCBModels() if models is None else models,
                         class_ids=class_ids, device=device, with_visibility=with_visibility)
        self._size = int(size)
        self._seed = int(seed)
        self._n_objects = int(n_objects)

    def __len__(self):
        return self._size

    def get_frame(self, index):
        if not 0 <= index < self._size:
            raise IndexError(index)
        return synthetic.make_pose_frame(self._seed + index, n_objects=self._n_objects)
