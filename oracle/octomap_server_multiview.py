"""CPU restatement of the ROS occupancy server's scan of a moving camera's frame and of the
grids it publishes in the current camera's frame, for the pose node's occupancy branch
(singleview_3d_pose_estimation.py:129-148, :162-164, :181-185) and the refinement node
(collision_based_pose_refinement.py:86-98, :123-133).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): imported by tests/, never by the product.

It extends oracle/octomap_server.py (``publishGrids`` in the map's own frame), which stays as it
is, with the rules of ros/src/morefusion_ros/src/OctomapServer.cpp that need a sensor-to-world
transform, over the restated ``OcTree`` of oracle/octomap.py:

insert_scan (``insertScan``, :283-448):
  :111-119  the cloud moved sensor -> world by ``pcl::transformPointCloud`` with a Matrix4f
            (``transform_f32``: ((m0 x + m1 y) + m2 z) + m3 in float, PCL's generic path; its SSE
            path may associate differently, so the order is unpinned); the sensor origin is the
            transform's float translation
  :290-321  instances initialised at their class pitch, the background (-1 there) at the
            server's resolution; -2 (uncertain) is not an instance
  :329-338  pixels of even row and column only, NaN points skipped
  :340-349  every listed point is pushed for the centre, except the first of each instance
  :352-374  inside max_range: the free ray in the background's key space (computeRayKeys, here
            ``ray_keys``: every ray stepped in lockstep with its arithmetic), the end point a hit
            in its instance unless uncertain, and free in the background unless labelled
            background
  :375-383  beyond max_range: the free ray to o + normalized(p - o) * max_range in float
  :386-402  background cells freed once unless hit by the background; hits once per instance
  :404-447  centres_.insert(compute3DCentroid): set by the first scan that pushed a point, never
            overwritten
grid_params (publishGrids, :534-551): the world centre moved to the camera by the inverse
            transform in float, origin = centre - (dims / 2 - 0.5) * pitch in double
publish_grids (publishGrids, :510-618) with sensor_to_world:
  :566-576  voxel centre ``origin + pitch * i`` in double, stored in a float ``PCLPoint``, moved
            to the world in float; ``search`` takes it back as double
  :579-583  ground_as_noentry: a voxel whose world z < 0 is no-entry at probability_max and is
            not looked at otherwise
  the other rules as oracle/octomap_server.py states them.

Not restated: ``render`` (:193-281), instance tracking (utils/geometry.h:79-281; callers pass
instance ids that are consistent across frames), the bounding boxes (:410-437, read by render
only), markers, ``publishAll`` and pruning.

**PARITY UNPINNED**, as for oracle/octomap_server.py (ROS and PCL cannot be built here).
Departures from the server that are deliberate and shared with the product, besides those of
oracle/octomap_server.py: a label that is neither listed, the background nor uncertain is
skipped (the server aborts the scan, :302-304); an instance whose first scan pushes no point has
no centre yet (the server reads an uninitialised centroid); the centroid is summed exactly in a
fixed point of 2^-32 m (``centre``), not in float in OpenMP order; the inverse transform is the
rigid inverse computed in float64 from the float matrix and rounded to float
(``rigid_inverse_f32``), not Eigen's general ``Matrix4f::inverse()``; the background's centre is
never read (publishGrids skips the background) and is not computed.
"""

import numpy as np

from .octomap import TREE_MAX_VAL, probability
from .octomap_server import map_order
from .octomap_server import publish_grids as _publish_grids


def publish_grids(octrees, target_ids, *, dimensions, pitches, origins, background_id=0,
                  probability_max=0.97, sensor_to_world=None, ground_as_noentry=False):
    """``oracle.octomap_server.publish_grids`` with the voxel centres in the camera's frame.

    (grid, grid_noentry) float32 [T, X, Y, Z] of every target.  octrees: {instance_id:
    oracle.octomap.OcTree}; pitches [T] and origins [T, 3] in float64.  sensor_to_world [4, 4]:
    the origins are in the camera's frame and the map in the world's; each float voxel centre is
    moved to the world in float before the look-up (:573-576).  ground_as_noentry (with
    sensor_to_world): :579-583.  With sensor_to_world=None this is
    ``oracle.octomap_server.publish_grids`` itself."""
    if sensor_to_world is None:
        if ground_as_noentry:
            raise ValueError("ground_as_noentry needs sensor_to_world")
        return _publish_grids(octrees, target_ids, dimensions=dimensions, pitches=pitches,
                              origins=origins, background_id=background_id,
                              probability_max=probability_max)
    X, Y, Z = (int(d) for d in dimensions)
    T = len(target_ids)
    pitches = np.asarray(pitches, np.float64).reshape(T)
    origins = np.asarray(origins, np.float64).reshape(T, 3)
    grid = np.zeros((T, X, Y, Z), np.float32)
    noentry = np.zeros((T, X, Y, Z), np.float32)
    order = map_order(list(octrees), background_id)
    tables = {}
    for t, target in enumerate(target_ids):
        p, o = pitches[t], origins[t]
        # :566-575 double centre -> float PCLPoint -> double search coordinate
        c = [np.float32(o[a] + p * np.arange(n, dtype=np.float64)) for a, n in enumerate((X, Y, Z))]
        w = transform_f32(matrix4f(sensor_to_world),
                          np.stack(np.meshgrid(*c, indexing="ij"), -1))          # :573-576
        ground = (w[..., 2] < 0) if ground_as_noentry else np.zeros((X, Y, Z), bool)   # :579
        wd = w.astype(np.float64)

        def look(tree):
            if id(tree) not in tables:
                tables[id(tree)] = _table(tree)
            return _lookup_points(tree, wd, tables[id(tree)])
        occ_t = look(octrees[target])
        occupied = (occ_t > 0.5) & ~ground                                       # :586
        grid[t][occupied] = occ_t[occupied].astype(np.float32)                   # :587-588
        noentry[t][ground] = np.float32(probability_max)                         # :580-582
        for other in order:                                                      # :591-593
            if other == target:                                                  # :594-596
                continue
            occ = look(octrees[other])
            known = ~np.isnan(occ) & ~occupied & ~ground                         # :598
            free = known & (other == background_id) & (occ < 0.5)                # :599-600
            full = known & ~free & (occ >= probability_max)                      # :603
            # later instances overwrite earlier ones: the node's fancy assignment keeps the last
            noentry[t][free] = (1.0 - occ[free]).astype(np.float32)              # :601-602
            noentry[t][full] = occ[full].astype(np.float32)                      # :604-605
    return grid, noentry


def _table(octree):
    """The tree's packed keys, sorted, and the occupancy of each."""
    keys = np.array([(a << 32) | (b << 16) | c for a, b, c in octree.cells], np.int64)
    lo = np.array(list(octree.cells.values()), np.float32)
    order = np.argsort(keys)
    keys, lo = keys[order], lo[order]
    uniq, inv = np.unique(lo, return_inverse=True)
    return keys, np.array([probability(v) for v in uniq], np.float64)[inv.reshape(-1)]


def _lookup_points(octree, pts, table):
    """oracle.octomap_server._lookup at arbitrary double coordinates pts [..., 3]; table =
    _table(octree)."""
    rf = octree.resolution_factor
    f = np.floor(rf * pts) + TREE_MAX_VAL
    ok = ((f >= 0) & (f < 2 * TREE_MAX_VAL)).all(-1)
    k = np.where(ok[..., None], f, 0).astype(np.int64)
    packed = (k[..., 0] << 32) | (k[..., 1] << 16) | k[..., 2]
    occ = np.full(packed.shape, np.nan)
    if not octree.cells:
        return occ
    keys, p = table
    pos = np.clip(np.searchsorted(keys, packed), 0, len(keys) - 1)
    hit = ok & (keys[pos] == packed)
    occ[hit] = p[pos[hit]]
    return occ


# --------------------------------------------------------------------------------------------
# transforms (:111-119, :536)
# --------------------------------------------------------------------------------------------
def matrix4f(sensor_to_world):
    """The transform as the server's Eigen::Matrix4f."""
    return np.asarray(sensor_to_world, np.float64).reshape(4, 4).astype(np.float32)


def transform_f32(m, pts):
    """pcl::transformPointCloud with a Matrix4f, PCL's generic path: each row
    ((m0 x + m1 y) + m2 z) + m3, every operation rounded to float32 (no FMA).  pts [..., 3]."""
    m = np.asarray(m, np.float32)
    p = np.asarray(pts, np.float32)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return np.stack([((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3] for r in range(3)],
                    -1).astype(np.float32)


def rigid_inverse_f32(m):
    """[R^T | -R^T t] in float64 from the float32 matrix, rounded to float32 (stands in for
    Eigen's Matrix4f::inverse(), whose rounding is not reproduced: unpinned)."""
    m = np.asarray(m, np.float32).astype(np.float64)
    R, t = m[:3, :3], m[:3, 3]
    inv = np.eye(4)
    inv[:3, :3] = R.T
    inv[:3, 3] = -((R[0] * t[0] + R[1] * t[1]) + R[2] * t[2])
    return inv.astype(np.float32)


# --------------------------------------------------------------------------------------------
# insertScan (:283-448)
# --------------------------------------------------------------------------------------------
def _keys(tree, pts):
    """coordToKeyChecked of float32 points [N, 3]: packed int64 keys and the ok mask."""
    f = np.floor(tree.resolution_factor * np.asarray(pts, np.float32).astype(np.float64)) + TREE_MAX_VAL
    ok = ((f >= 0) & (f < 2 * TREE_MAX_VAL)).all(-1)
    k = np.where(ok[:, None], f, 0).astype(np.int64)
    return (k[:, 0] << 32) | (k[:, 1] << 16) | k[:, 2], ok


def ray_keys(tree, origin, ends, counts=False):
    """The union of ``OcTree.computeRayKeys(origin, end)`` (oracle/octomap.py, first cell
    included, end cell excluded, nothing for a ray with an end outside the key range) over the
    rows of ends [N, 3] float32, as packed int64 keys: the same arithmetic, every ray stepped in
    lockstep.  counts: also the number of rays whose key list holds each key (a ray never
    crosses a cell twice), as (keys, counts)."""
    origin = np.asarray(origin, np.float32)
    ends = np.asarray(ends, np.float32).reshape(-1, 3)
    none = (np.empty(0, np.int64), np.empty(0, np.int64)) if counts else np.empty(0, np.int64)
    ko, ok_o = _keys(tree, origin[None])
    if not ok_o[0] or not len(ends):
        return none
    ke, ok_e = _keys(tree, ends)
    act = ok_e & (ke != ko[0])
    ends, ke = ends[act], ke[act]
    if not len(ends):
        return none
    out = [np.full(len(ends) if counts else 1, ko[0])]
    res = tree.resolution
    d = (ends - origin).astype(np.float32)
    nsq = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float32)
    length = np.sqrt(nsq.astype(np.float64)).astype(np.float32)
    d = (d / length[:, None]).astype(np.float32).astype(np.float64)
    step = np.where(d > 0, 1, np.where(d < 0, -1, 0))
    cur = np.stack([(ko[0] >> 32) & 0xFFFF, (ko[0] >> 16) & 0xFFFF, ko[0] & 0xFFFF])
    cur = np.repeat(cur[None], len(d), 0).astype(np.int64)
    dmax = float(np.finfo(np.float64).max)
    border = ((cur - TREE_MAX_VAL).astype(np.float64) + 0.5) * res
    border = border + (step * res * 0.5).astype(np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        tmax = np.where(step != 0, (border - origin.astype(np.float64)) / d, dmax)
        tdelta = np.where(step != 0, res / np.abs(d), dmax)
    flen = length.astype(np.float64)
    kend = np.stack([(ke >> 32) & 0xFFFF, (ke >> 16) & 0xFFFF, ke & 0xFFFF], 1)
    rows = np.arange(len(d))
    while len(rows):
        t0, t1, t2 = tmax[:, 0], tmax[:, 1], tmax[:, 2]
        dim = np.where(t0 < t1, np.where(t0 < t2, 0, 2), np.where(t1 < t2, 1, 2))
        r = np.arange(len(rows))
        cur[r, dim] += step[r, dim]
        with np.errstate(over="ignore"):
            tmax[r, dim] += tdelta[r, dim]
        done = (cur == kend).all(1)
        done |= tmax.min(1) > flen
        cd = cur[r, dim]
        done |= (cd < 0) | (cd >= 2 * TREE_MAX_VAL)
        go = ~done
        c = cur[go]
        out.append((c[:, 0] << 32) | (c[:, 1] << 16) | c[:, 2])
        cur, tmax, tdelta, step, kend, flen = cur[go], tmax[go], tdelta[go], step[go], kend[go], flen[go]
        rows = rows[go]
    return np.unique(np.concatenate(out), return_counts=counts)


def centre(points):
    """compute3DCentroid of the pushed points [N, 3] float32, N >= 1, summed exactly in a fixed
    point of 2^-32 m (each coordinate rounded to nearest, ties to even), then divided in
    double and rounded to float."""
    q = np.rint(np.asarray(points, np.float32).astype(np.float64) * 4294967296.0).astype(np.int64)
    s = q.sum(0)
    return (s.astype(np.float64) * (1.0 / 4294967296.0) / np.float64(len(q))).astype(np.float32)


def insert_scan(octrees, centres, label, pcd, sensor_to_world, class_ids, *, pitch_of,
                max_range=-1.0, background_id=-1, uncertain_id=-2, background_pitch=0.01):
    """One scan of an organised camera-frame cloud pcd [H, W, 3] with label [H, W] into
    octrees {instance_id: OcTree} and centres {instance_id: float32 [3]} (both updated in
    place).  class_ids {instance_id: class_id}; pitch_of(class_id) the class pitch."""
    from .octomap import OcTree
    for i, c in class_ids.items():                                               # :290-321
        if i not in octrees:
            octrees[i] = OcTree(pitch_of(c))
    if background_id not in octrees:
        octrees[background_id] = OcTree(background_pitch)
    bg = octrees[background_id]
    m = matrix4f(sensor_to_world)
    o = m[:3, 3]
    H, W = label.shape
    pix = np.arange(H * W).reshape(H, W)[0::2, 0::2].reshape(-1)                 # :329-333
    p = transform_f32(m, np.asarray(pcd, np.float32).reshape(-1, 3)[pix])        # :111-119
    lab = np.asarray(label).reshape(-1)[pix]
    listed = np.isin(lab, list(octrees))
    keep = ~np.isnan(p).any(1) & (listed | (lab == uncertain_id))                # :334-338
    p, lab, pix = p[keep], lab[keep], pix[keep]
    d = (p - o).astype(np.float32)
    nsq = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float32)
    length = np.sqrt(nsq.astype(np.float64))                                     # point3d::norm
    inside = (max_range < 0) | (length <= max_range)                             # :352
    with np.errstate(divide="ignore", invalid="ignore"):
        clipped = (o + (d / length.astype(np.float32)[:, None]) * np.float32(max_range)).astype(np.float32)
    ends = np.where(inside[:, None], p, clipped)                                 # :376
    free = [ray_keys(bg, o, ends)]                                               # :355-359, :377-381
    k, ok = _keys(bg, p[inside & (lab != background_id)])                        # :367-372
    free.append(k[ok])
    free = set(np.concatenate(free).tolist())
    hits = {}
    for i in np.unique(lab[inside & (lab != uncertain_id)]).tolist():            # :361-366
        k, ok = _keys(octrees[i], p[inside & (lab == i)])
        hits[i] = set(k[ok].tolist())

    def unpack(key):
        return ((key >> 32) & 0xFFFF, (key >> 16) & 0xFFFF, key & 0xFFFF)
    for key in sorted(free - hits.get(background_id, set())):                    # :386-392
        bg._update(unpack(key), False)
    for i, keys in hits.items():                                                 # :394-402
        for key in sorted(keys):
            octrees[i]._update(unpack(key), True)
    for i in np.unique(lab[lab != uncertain_id]).tolist():                        # :404-447
        if i == background_id or i in centres:
            continue
        pts = p[lab == i]                    # pixel order; the first is not pushed (:345-349)
        if len(pts) >= 2:
            centres[i] = centre(pts[1:])


def grid_params(centres, pitches, target_ids, sensor_to_world, dimensions=(32, 32, 32)):
    """publishGrids' pitch [T] and origin [T, 3] (float64) of each target (:534-551)."""
    inv = rigid_inverse_f32(matrix4f(sensor_to_world))
    off = np.asarray(dimensions, np.float64) / 2.0 - 0.5
    pitch = np.array([pitches[t] for t in target_ids], np.float64)
    c = transform_f32(inv, np.array([centres[t] for t in target_ids], np.float32).reshape(-1, 3))
    return pitch, c.astype(np.float64) - off * pitch[:, None]
