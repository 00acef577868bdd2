"""From a labelled RGB-D frame to object poses: the per-frame front end of the singleview_3d
model, as the dataset code (datasets/rgbd_pose_estimation/base.py:27-161) and the ROS pose node
(ros/src/morefusion_ros/nodes/singleview_3d_pose_estimation.py:113-282) build it around
``Model.predict``, on the device: depth -> points, per-instance crops (csrc/frontend.cu), the
median origin, the labelled occupancy map and the non-target / empty grid of every instance."""

import numpy as np
import torch

from ... import geometry
from ...functions.geometry import _util
from .. import icp_registration
from .. import occupancy_registration
from ..iterative_collision_check_link import IterativeCollisionCheckLink
from ..multi_instance_octree_mapping import MultiInstanceOctreeMapping
from .models.model import masked_median

_EXAMPLE_KEYS = ("class_id", "rgb", "pcd", "pitch", "origin", "grid_nontarget_empty")
BACKGROUND_PITCH = 0.01             # build_octomap's instance 0 (base.py:44)
SERVER_BACKGROUND_ID = -1           # the occupancy server's background (OctomapServer.cpp:295)


def frame_inputs(rgb, depth, label, dev):
    """rgb [H,W,3] uint8, depth [H,W] float metres (NaN = none) or integer millimetres (0 = none)
    and label [H,W] integer, as contiguous CUDA tensors (uint8, float32 metres, int32)."""
    rgb = torch.as_tensor(rgb, device=dev)
    depth = torch.as_tensor(depth, device=dev)
    label = torch.as_tensor(label, device=dev)
    if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3:
        raise ValueError("rgb must be uint8 [H,W,3]")
    if label.dtype.is_floating_point or label.dtype == torch.bool:
        raise ValueError("label must be an integer image")
    if tuple(depth.shape) != tuple(rgb.shape[:2]) or tuple(label.shape) != tuple(rgb.shape[:2]):
        raise ValueError("depth and label must be [H,W] like rgb")
    if depth.dtype == torch.uint16 or not depth.dtype.is_floating_point:
        # millimetres, 0 = no depth (singleview_3d_pose_estimation.py:119-121); dividing by a
        # device scalar keeps the division correctly rounded, as NumPy's
        depth = depth.to(torch.int32).to(torch.float32) / torch.full((), 1000.0, device=dev)
        depth = torch.where(depth == 0, torch.full_like(depth, float("nan")), depth)
    return rgb.contiguous(), depth.to(torch.float32).contiguous(), label.to(torch.int32).contiguous()


def build_map(pcd, label, instance_ids, class_ids, pitch_table):
    """The occupancy map of build_octomap (base.py:30-50): every instance with class_id > 0 at
    its class pitch (pitch_table[class_id]), then instance 0 at 0.01 m holding every label that
    is not listed.  The foreground is one labelled scan (its instances' cells are disjoint); the
    background is one scan per distinct unlisted label, because a cell seen by two of them gets
    two updates there.  Host reads: the distinct labels of the frame and the map's own table
    checks."""
    ids = np.asarray(instance_ids).reshape(-1)
    cls = np.asarray(class_ids).reshape(-1)
    mapping = MultiInstanceOctreeMapping(device=pcd.device)
    fg = cls > 0
    for i, p in zip(ids[fg].tolist(), pitch_table[cls[fg]].tolist()):
        mapping.initialize(i, pitch=p)
    if fg.any():
        mapping.integrate_labels(label, pcd)
    mapping.initialize(0, pitch=BACKGROUND_PITCH)
    labels = torch.unique(label).cpu().numpy()
    for lab in labels[~np.isin(labels, ids)].tolist():
        mapping.integrate(0, label == lab, pcd)
    return mapping


def empty_examples(dev, D, S):
    """The result of ``build_examples`` for a frame without a kept instance."""
    return dict(class_id=torch.empty(0, dtype=torch.int32, device=dev),
                rgb=torch.empty((0, S, S, 3), dtype=torch.uint8, device=dev),
                pcd=torch.empty((0, S, S, 3), dtype=torch.float32, device=dev),
                pitch=torch.empty(0, dtype=torch.float64, device=dev),
                origin=torch.empty((0, 3), dtype=torch.float32, device=dev),
                grid_target=torch.empty((0, D, D, D), dtype=torch.float32, device=dev),
                grid_nontarget=torch.empty((0, D, D, D), dtype=torch.float32, device=dev),
                grid_empty=torch.empty((0, D, D, D), dtype=torch.float32, device=dev),
                instance_ids=np.empty(0, dtype=np.int64), index=np.empty(0, dtype=np.int64))


def build_examples(rgb, depth, K, label, instance_ids, class_ids, pitch_table, mapping=None, *,
                   dev, n_points_minimal=1, dimensions=32, image_size=256, class_filter=None,
                   sensor_to_world=None, with_n_mask=False):
    """The model-free part of an example of every instance of one labelled frame, as get_example
    builds it (datasets/rgbd_pose_estimation/base.py:78-197) and the pose node (ros/src/
    morefusion_ros/nodes/singleview_3d_pose_estimation.py:113-185) around it: the map, the
    crops, the medians, the origins, the keep rule and the target grids, on the device.

    rgb / depth / label as ``frame_inputs`` takes them, K [3,3] intrinsics, instance_ids /
    class_ids [N] host arrays, pitch_table [n_fg_class + 1] float64 (the class pitch at
    ``dimensions``, entry 0 unused).  mapping: a ``MultiInstanceOctreeMapping`` that already holds
    the scene, or None to build it from this frame (``build_map``, every instance with
    class_id > 0).  class_filter: class ids an example may have (get_example's ``class_ids``);
    the others stay in the map.

    Instances are skipped when class_id <= 0, their class is filtered out, their mask is empty,
    fewer than n_points_minimal mask pixels have depth (base.py:118-129), or no valid point
    survives the nearest resize of the crop (its median, hence its origin, would be undefined).

    Returns (examples, kept class ids (host int32), mapping).  examples: a dict of CUDA tensors
    -- class_id [M] int32, rgb [M,S,S,3] uint8, pcd [M,S,S,3] float32, pitch [M] float64,
    origin [M,3] float32 (median of the crop's valid points - (D/2 - 0.5) pitch) and the map's
    grid_target / grid_nontarget / grid_empty [M,D,D,D] float32 -- plus instance_ids [M] and
    index [M] (positions in instance_ids), numpy.  Host reads: with a mapping passed in and CUDA
    inputs, one (the counts that decide which instances are kept); with mapping=None also those
    of ``build_map``.

    sensor_to_world [4,4] (host), with a mapping fed by ``integrate_scan``: the occupancy
    server's grids in this camera's frame instead (:129-148, :162-164, :181-185).  An instance
    without a server centre yet is skipped; origin is the server's grid origin rounded to
    float32, pitch the server's, and the three map grids are replaced by grid_nontarget_empty
    [M,D,D,D] bool, the server's grid_noentry > 0.  The "set" flags of the centres travel in the
    one host read.

    with_n_mask: the examples of kept instances also hold n_mask [M] int32, each one's
    label-mask pixel count (a gather of the crop pass's counts, no host read)."""
    ids =np.asarray(instance_ids).reshape(-1)
    cls = np.asarray(class_ids).reshape(-1).astype(np.int64)
    if ids.shape != cls.shape:
        raise ValueError("instance_ids and class_ids must have the same length")
    if ((cls < 0) | (cls >= len(pitch_table))).any():
        raise IndexError("class_id out of range for n_fg_class")
    rgb, depth, label = frame_inputs(rgb, depth, label, dev)
    K = np.asarray(K, dtype=np.float64).reshape(3, 3)
    pcd = geometry.pointcloud_from_depth(depth, K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    server = sensor_to_world is not None
    if mapping is None:
        if server:
            raise ValueError("sensor_to_world needs the mapping fed by integrate_scan")
        mapping = build_map(pcd, label, ids, cls, pitch_table)
    fg = cls > 0
    if class_filter is not None:
        fg &= np.isin(cls, np.asarray(tuple(class_filter), dtype=np.int64))
    D, S = int(dimensions), int(image_size)
    if not fg.any():
        return empty_examples(dev, D, S), np.empty(0, np.int32), mapping
    ids_fg, cls_fg = ids[fg], cls[fg]
    rgb_ins, pcd_ins, stats = geometry._frame_crops(rgb, pcd, label, ids_fg, size=S)
    N = ids_fg.size
    flat = pcd_ins.reshape(N, S * S, 3).permute(0, 2, 1)
    valid = ~torch.isnan(flat).any(1)
    n_crop = valid.sum(1)
    center = masked_median(flat, valid, n_crop)
    pitch64 = pitch_table[cls_fg]
    # base.py:153-156 origin = center - (dim / 2 - 0.5) * pitch: float32 centre minus the
    # float64 offset rounded to float32 (NumPy's rule for a float32 array and a Python float)
    off = _util.h2d((pitch64 * (D / 2.0 - 0.5)).astype(np.float32), dev, torch.float32,
                    "frame/offset")
    origin = center - off[:, None]
    cols = [stats[:, 4], stats[:, 5], n_crop.to(torch.int32)]
    if server:
        cols.append(mapping._centre_flags(ids_fg).to(torch.int32))
    counts = torch.stack(cols, 1).cpu().numpy()
    keep = (counts[:, 0] > 0) & (counts[:, 1] >= n_points_minimal) & (counts[:, 2] > 0)
    if server:                        # no server grid for an instance without a centre (:162-164)
        mapping._note_centres(ids_fg, counts[:, 3])
        keep &= counts[:, 3] > 0
    if not keep.any():
        return empty_examples(dev, D, S), np.empty(0, np.int32), mapping
    k = np.flatnonzero(keep)
    kd = _util.h2d(k.astype(np.int64), dev, torch.int64, "frame/keep")
    kept_ids = ids_fg[k]
    cls_kept = cls_fg[k].astype(np.int32)
    ex = dict(class_id=_util.h2d(cls_kept, dev, torch.int32, "frame/class"),
              rgb=rgb_ins.index_select(0, kd), pcd=pcd_ins.index_select(0, kd),
              instance_ids=kept_ids, index=np.flatnonzero(fg)[k])
    if with_n_mask:
        ex["n_mask"] = stats[:, 4].index_select(0, kd)
    if server:
        # the node's decoding of grids_noentry (:131-148): every listed index is True, the
        # origin a float32 array of the message's float64 origin
        d_pitch, d_origin = mapping.server_grid_params(kept_ids.tolist(), sensor_to_world,
                                                       (D, D, D))
        _, noentry = mapping.get_noentry_grids_batch(
            kept_ids.tolist(), dimensions=(D, D, D), pitches=d_pitch, origins=d_origin,
            background_id=SERVER_BACKGROUND_ID, sensor_to_world=sensor_to_world)
        ex.update(pitch=d_pitch, origin=d_origin.to(torch.float32),
                  grid_nontarget_empty=noentry > 0)
    else:
        origin = origin.index_select(0, kd)
        d_pitch = _util.h2d(pitch64[k], dev, torch.float64, "frame/pitch")
        gt, gn, ge = mapping.get_target_grids_batch(
            kept_ids.tolist(), dimensions=(D, D, D), pitches=d_pitch,
            origins=origin.to(torch.float64))
        ex.update(pitch=d_pitch, origin=origin, grid_target=gt, grid_nontarget=gn, grid_empty=ge)
    return ex, cls_kept, mapping


class FramePoseEstimator:
    """Poses of every listed instance of one frame from a ``Model``.

    model: a ``Model`` on a CUDA device.  n_points_minimal: instances with fewer mask pixels of
    valid depth are skipped (the dataset's rule is 1, the ROS node uses 50).  dimensions: side of
    the voxel grid the model was built for (the class pitch is the model's ``get_voxel_pitch``
    at that side)."""

    image_size = 256
    background_pitch = BACKGROUND_PITCH
    server_background_id = SERVER_BACKGROUND_ID

    def __init__(self, model, *, n_points_minimal=1, dimensions=32):
        self.model = model
        self.n_points_minimal = int(n_points_minimal)
        self.dimensions = int(dimensions)
        n = model._n_fg_class
        self._pitch_table = np.array(
            [np.nan] + [model._models.get_voxel_pitch(self.dimensions, c) for c in range(1, n + 1)],
            dtype=np.float64)
        self._sdf_cache = {}                 # (class_id, device) -> SDF points and values
        self._icp_cache = {}                 # (class_id, voxel_size, device) -> ICPTarget
        # (class_id, dimensions, device) -> occupancy registration's pitch and CAD cloud
        self._occupancy_cache = {}

    def build_map(self, pcd, label, instance_ids, class_ids):
        """``build_map`` at the model's class pitches."""
        return build_map(pcd, label, instance_ids, class_ids, self._pitch_table)

    def examples(self, rgb, depth, K, label, instance_ids, class_ids, mapping=None, *,
                 sensor_to_world=None):
        """The keyword arguments of ``Model.predict`` for the instances of one frame.

        rgb [H,W,3] uint8, depth [H,W] float metres (NaN = none) or uint16 millimetres (0 =
        none), K [3,3] intrinsics, label [H,W] integer instance image; instance_ids / class_ids
        [N] host arrays.  mapping: a ``MultiInstanceOctreeMapping`` that already holds the scene
        (every kept instance initialised), or None to build it from this frame (``build_map``).

        Instances are skipped when class_id <= 0, their mask is empty, fewer than
        n_points_minimal mask pixels have depth (base.py:118-129), or no valid point survives the
        nearest resize of the crop (its median, hence its origin, would be undefined).

        Returns a dict of CUDA tensors -- class_id [M] int32, rgb [M,256,256,3] uint8, pcd
        [M,256,256,3] float32, pitch [M] float32, origin [M,3] float32 (median of the crop's valid
        points - 15.5 pitch), grid_nontarget_empty [M,D,D,D] bool -- and instance_ids [M] (numpy)
        of the kept instances.

        Host reads: with a mapping passed in and CUDA inputs, one -- the mask / valid-point counts
        that decide which instances are kept.  With mapping=None, also those of ``build_map``.

        sensor_to_world [4,4] (host), with a mapping fed by ``integrate_scan``: the pose node's
        occupancy branch (singleview_3d_pose_estimation.py:129-148, :162-164, :181-185) on the
        occupancy server's grids in this camera's frame.  An instance without a server centre
        yet is skipped; origin is the server's grid origin rounded to float32, pitch the class
        pitch, and grid_nontarget_empty is the server's grid_noentry > 0
        (``get_noentry_grids_batch`` with the server's background).  The "set" flags of the
        centres travel in the one host read."""
        return self._examples(rgb, depth, K, label, instance_ids, class_ids, mapping,
                              sensor_to_world)[0]

    def _examples(self, rgb, depth, K, label, instance_ids, class_ids, mapping,
                  sensor_to_world=None):
        """examples(), the kept class ids on the host and the map."""
        dev = self.model.conv4_conf.weight.device
        if dev.type != "cuda":
            raise RuntimeError("FramePoseEstimator runs on CUDA only (no CPU fallback)")
        ex, cls_kept, mapping = build_examples(
            rgb, depth, K, label, instance_ids, class_ids, self._pitch_table, mapping, dev=dev,
            n_points_minimal=self.n_points_minimal, dimensions=self.dimensions,
            image_size=self.image_size, sensor_to_world=sensor_to_world)
        if "grid_nontarget_empty" not in ex:                      # train.py:50-54, :92-93
            t = ex["grid_target"] > 0.5
            ex["grid_nontarget_empty"] = (((ex["grid_nontarget"] > 0.5) ^ t)
                                          | ((ex["grid_empty"] > 0.5) ^ t))
        out = {k: ex[k] for k in _EXAMPLE_KEYS}
        out["pitch"] = ex["pitch"].to(torch.float32)
        out["instance_ids"] = ex["instance_ids"]
        return out, cls_kept, mapping

    def __call__(self, rgb, depth, K, label, instance_ids, class_ids, mapping=None, *,
                 confidence_threshold=0.0, refine=False, icp=False, occupancy=False,
                 sensor_to_world=None):
        """Poses of the instances of one frame (the ROS node's callback, :113-282): ``examples``,
        ``Model.predict``, and per instance the point of highest confidence.  Instances whose
        confidence is below confidence_threshold are dropped (:266-268).  icp=True refines each
        kept pose by point-to-point ICP of its crop's points against the class's CAD points
        (``icp``; the node's ~icp option, :246-264).  occupancy=True refines each kept pose by
        occupancy registration against the frame's map (``occupancy``; the DenseFusion occupancy
        evaluation), an alternative to icp=True (both raise ValueError) that has no world-frame
        variant (with sensor_to_world it raises ValueError).  refine=True refines the poses that
        are kept (after ICP or occupancy registration, when set) as one scene with ``refine`` (the
        refinement node that follows the pose node), on grids placed at the origins the model
        used.

        Returns numpy arrays (instance_ids [M], quaternion [M,4] (w, x, y, z), translation [M,3],
        confidence [M]); the confidence is the model's also after refinement.  Host reads besides
        ``Model.predict``'s own: those of ``examples``, one of the picked poses, with icp=True one
        of the ICP poses, with occupancy=True one of the registered poses and with refine=True one
        of the refined poses.  sensor_to_world: the occupancy server's grids,
        as in ``examples`` and ``refine``; poses are in the camera's frame."""
        if occupancy and icp:
            raise ValueError("occupancy and icp are alternative refinements: choose one")
        if occupancy and sensor_to_world is not None:
            raise ValueError("occupancy registration has no world-frame (sensor_to_world) grids")
        ex, cls_kept, mapping = self._examples(rgb, depth, K, label, instance_ids, class_ids,
                                               mapping, sensor_to_world)
        M = len(ex["instance_ids"])
        if M == 0:
            return (ex["instance_ids"], np.zeros((0, 4), np.float32), np.zeros((0, 3), np.float32),
                    np.zeros(0, np.float32))
        # the point-cloud model (singleview_pcd) takes no voxel grid: its predict reads the
        # example's rgb and pcd only
        keys = _EXAMPLE_KEYS if getattr(self.model, "takes_voxel_grid", True) else ("class_id", "rgb", "pcd")
        kw = {k: ex[k] for k in keys}
        kw["class_id"] = cls_kept
        with torch.no_grad():
            rot, trans, conf = self.model.predict(**kw)
        best = conf.argmax(1)
        q = rot.gather(1, best[:, None, None].expand(M, 1, 4))[:, 0]
        t = trans.gather(1, best[:, None, None].expand(M, 1, 3))[:, 0]
        c = conf.gather(1, best[:, None])[:, 0]
        out = torch.cat([q, t, c[:, None]], 1).cpu().numpy()
        keep = out[:, 7] >= confidence_threshold
        ids, q, t, c = ex["instance_ids"][keep], out[keep, :4], out[keep, 4:7], out[keep, 7]
        if (icp or refine) and keep.any():
            kd = _util.h2d(np.flatnonzero(keep), ex["origin"].device, torch.int64, "frame/refine_keep")
        if icp and keep.any():
            q, t, _ = self.icp(ex["pcd"].index_select(0, kd), cls_kept[keep], q, t)
        if occupancy and keep.any():
            q, t = self.occupancy(mapping, ids, cls_kept[keep], q, t)
        if refine and keep.any():
            q, t, _ = self.refine(mapping, ids, cls_kept[keep], q, t,
                                  ex["origin"].index_select(0, kd), sensor_to_world=sensor_to_world)
        return ids, q, t, c

    def refine(self, mapping, instance_ids, class_ids, quaternion, translation, origin=None, *,
               n_iter=30, early_stop=True, sensor_to_world=None):
        """Refine the poses of the instances of one scene together against the occupancy map:
        the ROS refinement node's callback (collision_based_pose_refinement.py:108-211) with the
        occupancy server's grids (``get_noentry_grids_batch``, background instance 0 as
        ``build_map`` makes it) and one ``IterativeCollisionCheckLink.refine`` call (Adam,
        ``n_iter`` iterations at most, the node's early stop when ``early_stop`` is True).

        mapping: a ``MultiInstanceOctreeMapping`` that holds every instance.  instance_ids /
        class_ids [M] host arrays; quaternion [M,4] (w, x, y, z) and translation [M,3] host
        arrays, the initial poses; origin [M,3] float32 (host or CUDA), the grid origins.

        Returns numpy (quaternion [M,4], translation [M,3], iterations run).  An instance whose
        refined pose is not finite -- its scene's target grids are empty, and the ICC loss
        divides by their sum -- keeps its initial pose.  One host read, of the result.  M = 0
        launches nothing; M > 32 (the ICC's limit per scene) raises ValueError.

        sensor_to_world [4,4] (host), with a mapping fed by ``integrate_scan``: the refinement
        node on the occupancy server's grid / grid_noentry in this camera's frame
        (collision_based_pose_refinement.py:86-98, :123-133): both grids at the server's pitches
        and origins (``server_grid_params``; ``origin`` is not used), the ICC at those origins
        rounded to float32."""
        ids = np.asarray(instance_ids).reshape(-1)
        cls = np.asarray(class_ids).reshape(-1).astype(np.int64)
        q0 = np.asarray(quaternion, np.float32).reshape(-1, 4)
        t0 = np.asarray(translation, np.float32).reshape(-1, 3)
        M = ids.size
        if not (cls.shape == (M,) and q0.shape[0] == M and t0.shape[0] == M):
            raise ValueError("instance_ids, class_ids, quaternion and translation must have one row "
                             "per instance")
        if M > 32:
            raise ValueError(f"at most 32 instances per scene can be refined together, got {M}")
        if ((cls < 1) | (cls > self.model._n_fg_class)).any():
            raise IndexError("class_id out of range for n_fg_class")
        if M == 0:
            return q0, t0, 0
        dev = self.model.conv4_conf.weight.device
        D = self.dimensions
        pitch64 = self._pitch_table[cls]
        # the node: the class pitch in float64 for the query, float32 for the ICC (:159-160)
        if sensor_to_world is None:
            if origin is None:
                raise ValueError("origin is needed without sensor_to_world")
            d_pitch = _util.h2d(pitch64, dev, torch.float64, "refine/pitch")
            d_origin = _util.h2d(origin, dev, torch.float32, "refine/origin").reshape(M, 3).contiguous()
            grid, grid_noentry = mapping.get_noentry_grids_batch(
                ids.tolist(), dimensions=(D, D, D), pitches=d_pitch,
                origins=d_origin.to(torch.float64), background_id=0)
        else:
            d_pitch, o64 = mapping.server_grid_params(ids.tolist(), sensor_to_world, (D, D, D))
            grid, grid_noentry = mapping.get_noentry_grids_batch(
                ids.tolist(), dimensions=(D, D, D), pitches=d_pitch, origins=o64,
                background_id=self.server_background_id, sensor_to_world=sensor_to_world)
            d_origin = o64.to(torch.float32)
        # initial parameters by the reference's route: host transform -> quaternion_from_matrix
        link = IterativeCollisionCheckLink(geometry.transformation_matrix(q0, t0), voxel_dim=D)
        for name in ("quaternion", "translation"):
            p = getattr(link, name)
            p.data = _util.h2d(p.data, dev, torch.float32, "refine/" + name)
        sdf = [self._sdf(int(c), dev) for c in cls]
        link.refine([s[0] for s in sdf], [s[1] for s in sdf], d_pitch.to(torch.float32), d_origin,
                    grid, grid_noentry, n_iter=n_iter, early_stop=early_stop)
        n_run = link.n_iter_run
        if n_run is None:
            n_run = torch.full((), n_iter, dtype=torch.int32, device=dev)
        out = torch.cat([link.quaternion.data.reshape(-1), link.translation.data.reshape(-1),
                         n_run.reshape(1).view(torch.float32)]).cpu().numpy()
        q = out[:4 * M].reshape(M, 4)
        t = out[4 * M:7 * M].reshape(M, 3)
        ok = np.isfinite(q).all(1) & np.isfinite(t).all(1)
        q = np.where(ok[:, None], q, q0)
        t = np.where(ok[:, None], t, t0)
        return q, t, int(out[7 * M:].view(np.int32)[0])

    def icp(self, pcd, class_ids, quaternion, translation, *, iteration=None, voxel_size=None):
        """Refine each instance's pose by point-to-point ICP, as the pose node does with ~icp
        (singleview_3d_pose_estimation.py:246-264, ``ICPRegistration.register``): the crop's valid
        points (depth, source) against the class's CAD points (``get_pcd``, target), both
        down-sampled at voxel_size (0.01), matches within 2 voxel_size, at most ``iteration``
        (100) iterations; init = inv(transformation_matrix(q, t)) in float32 and the result
        inverted, as the node and the wrapper do.  All instances in one ``register_batch``.

        pcd [M,S,S,3] float32 CUDA (the crops of ``examples``, NaN = no point); class_ids [M],
        quaternion [M,4] (w, x, y, z) and translation [M,3] host arrays.  Returns numpy
        (quaternion [M,4] float32 (w >= 0), translation [M,3] float32, iterations run [M]).  One
        host read, of the result; M = 0 launches nothing."""
        iteration = icp_registration.ITERATION if iteration is None else int(iteration)
        voxel_size = icp_registration.VOXEL_SIZE if voxel_size is None else float(voxel_size)
        cls = np.asarray(class_ids).reshape(-1).astype(np.int64)
        q0 = np.asarray(quaternion, np.float32).reshape(-1, 4)
        t0 = np.asarray(translation, np.float32).reshape(-1, 3)
        M = cls.size
        if not (q0.shape[0] == M and t0.shape[0] == M and pcd.shape[0] == M):
            raise ValueError("pcd, class_ids, quaternion and translation must have one row per "
                             "instance")
        if ((cls < 1) | (cls > self.model._n_fg_class)).any():
            raise IndexError("class_id out of range for n_fg_class")
        if M == 0:
            return q0, t0, np.zeros(0, np.int32)
        dev = pcd.device
        init = np.linalg.inv(geometry.transformation_matrix(q0, t0))     # float32, as the node
        targets = [self._icp_target(int(c), voxel_size, dev) for c in cls]
        T, _, _, n_it = icp_registration.register_batch(
            pcd, targets, init, voxel_size=voxel_size, max_iteration=iteration)
        out = torch.cat([T.reshape(-1), n_it.to(torch.float64)]).cpu().numpy()
        Ts = np.linalg.inv(out[:16 * M].reshape(M, 4, 4))
        q = np.stack([geometry.quaternion_from_matrix(T) for T in Ts]).astype(np.float32)
        t = Ts[:, :3, 3].astype(np.float32)
        return q, t, out[16 * M:].astype(np.int32)

    def occupancy(self, mapping, instance_ids, class_ids, quaternion, translation, *,
                  iteration=100, dimensions=16, threshold=2, alpha=0.01):
        """Refine each instance's pose by occupancy registration, as the DenseFusion occupancy
        evaluation does per instance (examples/ycb_video/dense_fusion/
        eval_densefusion_occupancy.py:68-120), all instances in one ``register_batch``:
        pitch = |max - min| of the class's CAD points (``get_pcd``) / dimensions in float64, a
        dimensions^3 grid centred on the initial translation (origin = t - (dimensions / 2 - 0.5)
        pitch), the map's three target grids of the instance, the CAD points down-sampled at that
        pitch (float32), init = compose_transform(quaternion_matrix(q), t) in float32, then
        ``iteration`` Adam steps (alpha, translation alpha * 0.1) at ``threshold``.  The result is
        rebuilt on the host in float64 as OccupancyRegistration._transform does; a non-finite one
        (an empty target grid makes the loss 0/0) keeps the initial pose.

        mapping: a ``MultiInstanceOctreeMapping`` holding every instance (the script labels its
        map by class id, YCB-Video labels being class ids; here the instance id is the target).
        instance_ids / class_ids [M], quaternion [M,4] (w, x, y, z) and translation [M,3] host
        arrays.  Returns numpy (quaternion [M,4], translation [M,3]) float32.  One host read, of
        the result; M = 0 launches nothing."""
        ids = np.asarray(instance_ids).reshape(-1)
        cls = np.asarray(class_ids).reshape(-1).astype(np.int64)
        q0 = np.asarray(quaternion).reshape(-1, 4)
        t0 = np.asarray(translation).reshape(-1, 3)
        M = ids.size
        if not (cls.shape == (M,) and q0.shape[0] == M and t0.shape[0] == M):
            raise ValueError("instance_ids, class_ids, quaternion and translation must have one row "
                             "per instance")
        if ((cls < 1) | (cls > self.model._n_fg_class)).any():
            raise IndexError("class_id out of range for n_fg_class")
        if M == 0:
            return q0.astype(np.float32), t0.astype(np.float32)
        dev = self.model.conv4_conf.weight.device
        D = int(dimensions)
        clouds = [self._occupancy_cloud(int(c), D, dev) for c in cls]
        pitch = np.array([c[0] for c in clouds])
        origin, init = self.occupancy_frame(pitch, q0, t0, D)
        N = max(c[1].shape[0] for c in clouds)
        points = torch.zeros((M, N, 3), dtype=torch.float32, device=dev)
        for m, c in enumerate(clouds):
            points[m, :c[1].shape[0]] = c[1]
        n_points = torch.cat([c[2] for c in clouds])
        gt, gn, ge = mapping.get_target_grids_batch(
            ids.tolist(), dimensions=(D, D, D),
            pitches=_util.h2d(pitch, dev, torch.float64, "occupancy/pitch"),
            origins=_util.h2d(origin, dev, torch.float64, "occupancy/origin"))
        grids = torch.stack([gt, gn, ge], 1)
        q, t, _, _ = occupancy_registration.register_batch(
            points, n_points, grids, pitch=pitch.astype(np.float32),
            origin=origin.astype(np.float32), threshold=threshold,
            transform_init=init.astype(np.float32), iteration=iteration, alpha=alpha)
        out = torch.cat([q, t], 1).cpu().numpy()
        qs, ts = [], []
        for m in range(M):
            T = geometry.compose_transform(geometry.quaternion_matrix(out[m, :4])[:3, :3],
                                           out[m, 4:])
            if np.isnan(T).sum():
                T = init[m]
            qs.append(geometry.quaternion_from_matrix(T))
            ts.append(geometry.translation_from_matrix(T))
        return np.stack(qs).astype(np.float32), np.stack(ts).astype(np.float32)

    @staticmethod
    def occupancy_pitch(pcd_cad, dimensions):
        """The registration pitch of a class: its CAD bounding-box diagonal / dimensions
        (eval_densefusion_occupancy.py:86-90), a Python float."""
        pcd = np.asarray(pcd_cad)
        return float(np.linalg.norm(np.nanmax(pcd, axis=0) - np.nanmin(pcd, axis=0))) / dimensions

    @staticmethod
    def occupancy_frame(pitch, quaternion, translation, dimensions):
        """The grid origins [M,3] (centred on the initial translations, :91-92) and the initial
        transforms [M,4,4] (compose_transform(quaternion_matrix(q), t), :74-76), float64."""
        t = np.asarray(translation).reshape(-1, 3)
        origin = t - (dimensions / 2.0 - 0.5) * np.asarray(pitch, np.float64).reshape(-1, 1)
        init = np.stack([geometry.compose_transform(geometry.quaternion_matrix(q)[:3, :3], tt)
                         for q, tt in zip(np.asarray(quaternion).reshape(-1, 4), t)])
        return origin, init

    def _occupancy_cloud(self, class_id, dimensions, dev):
        """The class's registration pitch (float64) and its CAD points down-sampled at that pitch
        (CUDA float32 [N,3], the first n rows, n a CUDA int32 [1]), built once."""
        key = (class_id, dimensions, str(dev))
        if key not in self._occupancy_cache:
            pcd = np.asarray(self.model._models.get_pcd(class_id))
            pitch = self.occupancy_pitch(pcd, dimensions)
            means, _, _, n = icp_registration.voxel_down_sample(
                _util.h2d_transient(pcd.reshape(1, -1, 3), dev, torch.float64), pitch)
            self._occupancy_cache[key] = (pitch, means[0].to(torch.float32), n)
        return self._occupancy_cache[key]

    def _icp_target(self, class_id, voxel_size, dev):
        """The class's CAD points down-sampled with their cell list on the device, built once."""
        key = (class_id, voxel_size, str(dev))
        if key not in self._icp_cache:
            self._icp_cache[key] = icp_registration.ICPTarget(
                self.model._models.get_pcd(class_id), voxel_size, 2 * voxel_size, dev)
        return self._icp_cache[key]

    def _sdf(self, class_id, dev):
        """The class's SDF points and values on the device, uploaded once (the node's _get_sdf)."""
        key = (class_id, str(dev))
        if key not in self._sdf_cache:
            pcd, sdf = self.model._models.get_sdf(class_id)
            self._sdf_cache[key] = (_util.h2d_transient(pcd, dev, torch.float32),
                                    _util.h2d_transient(sdf, dev, torch.float32))
        return self._sdf_cache[key]
