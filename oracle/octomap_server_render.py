"""CPU restatement of the ROS occupancy server's ``render`` (OctomapServer.cpp:193-281) and of the
instance boxes it reads, which ``insertScan`` keeps (:404-437), over the restated ``OcTree`` of
oracle/octomap.py.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): imported by tests/ and scripts/, never by the
product.  It extends oracle/octomap_server_multiview.py, which stays as it is.

OctoMap 1.9 (OccupancyOcTreeBase), restated rule by rule in its float / double mix:

castRay(origin, direction, end, ignoreUnknownCells=true, maxRange)  ``cast_ray`` (one ray, line
    by line) and ``cast_rays`` (many rays stepped in lockstep, the same arithmetic):
  - the origin's key by coordToKeyChecked; outside the key range: false
  - the origin's own cell occupied: true, end = its centre; unknown: go on (ignoreUnknownCells)
  - direction.normalized(): the float norm_sq, its double sqrt, each float component divided by
    the float of it (no division for a zero vector); a zero direction: false
  - voxelBorder = keyToCoord(key) + double(step * resolution * 0.5): castRay keeps the half step
    in double, where computeRayKeys rounds it to float
  - tMax = (voxelBorder - origin) / direction, tDelta = resolution / |direction| in double; the
    axis of the smallest tMax with strict <, as computeRayKeys
  - before a step: key 0 stepping down or 65535 stepping up: false
  - after a step: end = keyToCoord(key) as floats; maxRange > 0 and the double sum of the float
    (end - origin)^2 > maxRange^2: false
  - the cell occupied (isNodeOccupied: log-odds >= the threshold's log-odds, 0): true; free and
    unknown cells are passed
inBBX(p)  ``in_bbx``: bbx_min <= p <= bbx_max on every axis, in float.  The box of a tree that
    no scan has boxed is the default-constructed point3d pair, (0,0,0)-(0,0,0) (``DEFAULT_BBX``):
    inBBX holds at (0,0,0) only.
insertScan's boxes  ``insert_scan``: the points an instance pushes (every listed point but its
    first of the scan, range or not, the background's included; here the background is not
    boxed: render skips it); pcl::getMinMax3D of them, (+FLT_MAX, -FLT_MAX) for none; a tree
    created by this scan takes that box, an older one the union with its box.  An instance with
    no listed point is not boxed.  The server creates a tree for every id of ``unique(label_ins)``
    (:290-319): the first scan whose label image holds the id on any pixel, odd rows and columns
    and NaN points included.  oracle/octomap_server_multiview.py (and the map) create an
    instance as soon as it is listed, so which instances have a tree in the server's sense is
    kept apart, in ``trees``.
render  ``render``: see its docstring.

**PARITY UNPINNED**, as for computeRayKeys (oracle/octomap.py) and the rest of the server
(oracle/octomap_server.py): neither OctoMap nor ROS / PCL can be built here, so what is pinned
is this statement of the published source, and the tests check its castRay against a float64
slab test that does not share its DDA.  Departures shared with the product: ties between
instances go to the lower instance id (the server's OpenMP loop leaves them to thread order);
a zero box bound is +0 (the server's sign of a zero bound depends on its OpenMP order; inBBX
does not see it).
"""

import math

import numpy as np

from .octomap import TREE_MAX_VAL
from .octomap_server_multiview import insert_scan as _insert_scan
from .octomap_server_multiview import matrix4f, transform_f32

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)
DBL_MAX = float(np.finfo(np.float64).max)
DEFAULT_BBX = (np.zeros(3, F32), np.zeros(3, F32))


def _centre(tree, k):
    """keyToCoord(key) as a point3d: double arithmetic, float result."""
    return F32((float(int(k) - TREE_MAX_VAL) + 0.5) * tree.resolution)


def _occupied(tree, key):
    lo = tree.cells.get(tuple(int(k) for k in key))
    return lo is not None and lo >= F32(0.0)


def cast_ray(tree, origin, direction, max_range):
    """castRay(origin, direction, end, ignoreUnknownCells=true, max_range) of one ray.
    origin, direction float32 [3]; max_range double.  Returns (hit, end float32 [3] or None)."""
    origin = np.asarray(origin, F32)
    direction = np.asarray(direction, F32)
    cur = tree.coords_to_key(origin.astype(np.float64))
    if cur is None:
        return False, None
    cur = list(cur)
    if _occupied(tree, cur):
        return True, np.array([_centre(tree, k) for k in cur], F32)
    nsq = F32(F32(direction[0] * direction[0] + direction[1] * direction[1])
              + direction[2] * direction[2])
    length = math.sqrt(float(nsq))
    d = (direction / F32(length)).astype(F32) if length > 0 else direction
    step, tmax, tdelta = [0] * 3, [0.0] * 3, [0.0] * 3
    for i in range(3):
        step[i] = 1 if d[i] > 0 else (-1 if d[i] < 0 else 0)
        if step[i] != 0:
            border = tree.key_to_coord(cur[i])
            border += float(step[i] * tree.resolution * 0.5)
            tmax[i] = (border - float(origin[i])) / float(d[i])
            tdelta[i] = tree.resolution / abs(float(d[i]))
        else:
            tmax[i] = tdelta[i] = DBL_MAX
    if step == [0, 0, 0]:
        return False, None
    range_set = max_range > 0.0
    range_sq = max_range * max_range
    while True:
        if tmax[0] < tmax[1]:
            dim = 0 if tmax[0] < tmax[2] else 2
        else:
            dim = 1 if tmax[1] < tmax[2] else 2
        if (step[dim] < 0 and cur[dim] == 0) or (step[dim] > 0 and cur[dim] == 2 * TREE_MAX_VAL - 1):
            return False, None
        cur[dim] += step[dim]
        tmax[dim] += tdelta[dim]
        end = np.array([_centre(tree, k) for k in cur], F32)
        if range_set:
            dsq = 0.0
            for j in range(3):
                e = F32(end[j] - origin[j])
                dsq += float(F32(e * e))
            if dsq > range_sq:
                return False, None
        if _occupied(tree, cur):
            return True, end


def _occupied_table(tree):
    keys = [(a << 32) | (b << 16) | c for (a, b, c), lo in tree.cells.items() if lo >= F32(0.0)]
    return np.sort(np.asarray(keys, np.int64))


def _lookup(table, cur):
    packed = (cur[:, 0] << 32) | (cur[:, 1] << 16) | cur[:, 2]
    if not len(table):
        return np.zeros(len(cur), bool)
    pos = np.clip(np.searchsorted(table, packed), 0, len(table) - 1)
    return table[pos] == packed


def cast_rays(tree, origin, directions, max_ranges):
    """``cast_ray`` of every row of directions [N, 3] float32 (max_ranges [N] double) from one
    origin, all rays stepped in lockstep with the same arithmetic.  Returns hit [N] bool and end
    [N, 3] float32 (NaN where there is no hit)."""
    origin = np.asarray(origin, F32)
    d = np.asarray(directions, F32).reshape(-1, 3)
    max_ranges = np.asarray(max_ranges, np.float64).reshape(-1)
    N = len(d)
    hit = np.zeros(N, bool)
    end = np.full((N, 3), np.nan, F32)
    ko = tree.coords_to_key(origin.astype(np.float64))
    if ko is None or not N:
        return hit, end
    res = tree.resolution
    table = _occupied_table(tree)
    cur = np.repeat(np.asarray(ko, np.int64)[None], N, 0)

    def centres(c):
        return (((c - TREE_MAX_VAL).astype(np.float64) + 0.5) * res).astype(F32)
    if _lookup(table, cur[:1])[0]:
        return np.ones(N, bool), np.repeat(centres(cur[:1]), N, 0)
    nsq = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)
    length = np.sqrt(nsq.astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.where((length > 0)[:, None], d / length.astype(F32)[:, None], d).astype(F32)
    d64 = d.astype(np.float64)
    step = np.where(d > 0, 1, np.where(d < 0, -1, 0))
    border = ((cur - TREE_MAX_VAL).astype(np.float64) + 0.5) * res + step * res * 0.5
    with np.errstate(divide="ignore", invalid="ignore"):
        tmax = np.where(step != 0, (border - origin.astype(np.float64)) / d64, DBL_MAX)
        tdelta = np.where(step != 0, res / np.abs(d64), DBL_MAX)
    rows = np.flatnonzero((step != 0).any(1))
    cur, step, tmax, tdelta = cur[rows], step[rows], tmax[rows], tdelta[rows]
    range_set = max_ranges[rows] > 0.0
    range_sq = max_ranges[rows] ** 2
    while len(rows):
        t0, t1, t2 = tmax[:, 0], tmax[:, 1], tmax[:, 2]
        dim = np.where(t0 < t1, np.where(t0 < t2, 0, 2), np.where(t1 < t2, 1, 2))
        r = np.arange(len(rows))
        s, c = step[r, dim], cur[r, dim]
        out = ((s < 0) & (c == 0)) | ((s > 0) & (c == 2 * TREE_MAX_VAL - 1))
        cur[r, dim] += s
        with np.errstate(over="ignore"):
            tmax[r, dim] += tdelta[r, dim]
        e = centres(cur)
        f = ((e - origin) * (e - origin)).astype(F32).astype(np.float64)
        out |= range_set & (((f[:, 0] + f[:, 1]) + f[:, 2]) > range_sq)
        occ = ~out & _lookup(table, np.where(out[:, None], 0, cur))
        hit[rows[occ]] = True
        end[rows[occ]] = e[occ]
        go = ~out & ~occ
        rows, cur, step, tmax, tdelta = rows[go], cur[go], step[go], tmax[go], tdelta[go]
        range_set, range_sq = range_set[go], range_sq[go]
    return hit, end


def in_bbx(bbx, points):
    """inBBX of points [N, 3] float32 against bbx = (min, max) float32 [3]."""
    lo, hi = bbx
    p = np.asarray(points, F32)
    return ((p >= lo) & (p <= hi)).all(-1)


def _plus_zero(v):
    return np.where(v == 0, F32(0.0), v).astype(F32)


def insert_scan(octrees, centres, boxes, trees, label, pcd, sensor_to_world, class_ids, *,
                pitch_of, max_range=-1.0, background_id=-1, uncertain_id=-2, background_pitch=0.01):
    """oracle.octomap_server_multiview.insert_scan, and the boxes {instance_id: (min, max)
    float32 [3]} that insertScan sets (:404-437), updated in place.  trees: the set of instance
    ids whose tree the server has created (:290-319), updated in place; an instance a caller adds
    to the map outside the server's scan (integrate_labels, update) belongs in it."""
    _insert_scan(octrees, centres, label, pcd, sensor_to_world, class_ids, pitch_of=pitch_of,
                 max_range=max_range, background_id=background_id, uncertain_id=uncertain_id,
                 background_pitch=background_pitch)
    seen = set(np.unique(np.asarray(label)).tolist()) & set(octrees)             # :290-319
    new = seen - trees - {background_id}
    trees |= seen
    m = matrix4f(sensor_to_world)
    H, W = np.asarray(label).shape
    pix = np.arange(H * W).reshape(H, W)[0::2, 0::2].reshape(-1)                 # :329-333
    p = transform_f32(m, np.asarray(pcd, F32).reshape(-1, 3)[pix])
    lab = np.asarray(label).reshape(-1)[pix]
    keep = ~np.isnan(p).any(1) & np.isin(lab, list(octrees))                      # :334-344
    p, lab = p[keep], lab[keep]
    for i in np.unique(lab).tolist():
        if i == background_id:
            continue
        pts = p[lab == i][1:]                 # pixel order; the first is not pushed (:345-349)
        lo = pts.min(0) if len(pts) else np.full(3, FLT_MAX, F32)                 # getMinMax3D
        hi = pts.max(0) if len(pts) else np.full(3, -FLT_MAX, F32)
        if i not in new:                                                          # :415-424
            old = boxes.get(i, DEFAULT_BBX)
            lo, hi = np.minimum(old[0], lo), np.maximum(old[1], hi)
        boxes[i] = (_plus_zero(lo), _plus_zero(hi))                               # :434-437


def render(octrees, boxes, pcd, sensor_to_world, K, *, background_id=-1, uncertain_id=-2):
    """OctomapServer::render (:193-281).  octrees {instance_id: OcTree}, boxes as kept by
    ``insert_scan`` (an instance without one has ``DEFAULT_BBX``), pcd [H, W, 3] camera frame,
    K [3, 3].  Returns label [H, W] int32 and depth [H, W] float32.

    Instances in ascending id (std::map), the background skipped (:205-209); pixels of even row
    and column (:212-217); a pixel with depth targets its world point if it is inBBX (:238-247),
    one without depth the z = 1 point of its ray, fx, fy, cx, cy rounded to float, moved to the
    world the same way (:219-237); castRay with maxRange = 1.1 |target - origin| (:250); the hit
    is the cell centre (:255-260); d = |end - origin| in float, strictly nearer wins, so of exact
    ties the lower id (:262-278); the winner writes depth at the pixel and its id on rows v-1..v,
    columns u-1..u (:268-276)."""
    m = matrix4f(sensor_to_world)
    o = m[:3, 3]
    pcd = np.asarray(pcd, F32)
    H, W = pcd.shape[:2]
    label = np.full((H, W), uncertain_id, np.int32)
    depth = np.full((H, W), np.nan, F32)
    vv, uu = np.meshgrid(np.arange(0, H, 2), np.arange(0, W, 2), indexing="ij")
    vv, uu = vv.reshape(-1), uu.reshape(-1)
    p = transform_f32(m, pcd[vv, uu])
    nodepth = np.isnan(p).any(1)
    K = np.asarray(K, np.float64)
    fx, fy, cx, cy = F32(K[0, 0]), F32(K[1, 1]), F32(K[0, 2]), F32(K[1, 2])
    ray = np.stack([(uu.astype(F32) - cx) / fx, (vv.astype(F32) - cy) / fy,
                    np.ones(len(uu), F32)], 1).astype(F32)
    p[nodepth] = transform_f32(m, ray[nodepth])
    d = (p - o).astype(F32)
    nsq = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)
    max_range = np.sqrt(nsq.astype(np.float64)) * 1.1
    best = np.full(len(p), np.nan, F32)
    best_id = np.zeros(len(p), np.int64)
    for i in sorted(octrees):
        if i == background_id:
            continue
        sel = np.flatnonzero(nodepth | in_bbx(boxes.get(i, DEFAULT_BBX), p))
        hit, end = cast_rays(octrees[i], o, d[sel], max_range[sel])
        sel, end = sel[hit], end[hit]
        e = (end - o).astype(F32)
        dist = np.sqrt((((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
                        .astype(F32)).astype(np.float64)).astype(F32)
        new = np.isnan(best[sel]) | (dist < best[sel])
        best[sel[new]] = dist[new]
        best_id[sel[new]] = i
    won = ~np.isnan(best)
    depth[vv[won], uu[won]] = best[won]
    for dj in (-1, 0):
        for di in (-1, 0):
            j, i = vv[won] + dj, uu[won] + di
            ok = (j >= 0) & (i >= 0) & (j < H) & (i < W)
            label[j[ok], i[ok]] = best_id[won][ok]
    return label, depth
