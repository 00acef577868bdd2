"""The dataset rules of oracle/octomap.py in bulk, for scans of whole 640x480 frames.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): imported by tests/, never by the product.

``OcTree.insertPointCloud`` of oracle/octomap.py walks one ray at a time in Python, hours for the
~290k rays of a frame.  ``Tree`` here computes the same cells with the same arithmetic over
whole arrays:

  insertPointCloud(points, origin)
      free = the union of ``octomap_server_multiview.ray_keys`` (every ray stepped in lockstep
             with computeRayKeys' arithmetic), chunk by chunk; occ = ``_keys`` of the end points
             (float32 points, double key arithmetic); one miss for each key of free - occ and one
             hit for each key of occ, as float32 adds clamped as ``OcTree._update`` clamps them.
  updateNodes(values)
      float64 rows keyed in double, one hit per row, no de-duplication: a key with n rows gets n
      sequential clamped adds.

``MultiInstanceOctreeMapping`` restates oracle/octomap.py's class of the same name over these
trees; ``get_target_grids_batch`` is its ``get_target_grids`` for T targets at once (voxel
centres ``idx * pitch + origin`` in float64, keyed in double, octomap::probability in double).

A tree is a sorted int64 array of packed keys (kx << 32 | ky << 16 | kz) and the float32
log-odds of each.  tests/test_octomap_batch.py pins this module to oracle/octomap.py cell for
cell and grid for grid, bit for bit.
"""

import numpy as np

from .octomap import TREE_MAX_VAL, OcTree, probability
from .octomap_server_multiview import _keys, ray_keys

CHUNK = 1 << 14                     # rays walked together: bounds the arrays of one ray_keys call


def unpack(keys):
    """Packed int64 keys [N] -> the (kx, ky, kz) tuples of OcTree.cells."""
    k = np.asarray(keys, np.int64)
    return list(zip(((k >> 32) & 0xFFFF).tolist(), ((k >> 16) & 0xFFFF).tolist(),
                    (k & 0xFFFF).tolist()))


def pack(cells_keys):
    """(kx, ky, kz) tuples -> packed int64 keys."""
    k = np.asarray(list(cells_keys), np.int64).reshape(-1, 3)
    return (k[:, 0] << 32) | (k[:, 1] << 16) | k[:, 2]


def double_keys(tree, pts):
    """coordToKeyChecked of float64 points [..., 3] (OcTree.coords_to_key): packed keys, ok mask."""
    f = np.floor(tree.resolution_factor * np.asarray(pts, np.float64)) + TREE_MAX_VAL
    ok = ((f >= 0) & (f < 2 * TREE_MAX_VAL)).all(-1)
    k = np.where(ok[..., None], f, 0).astype(np.int64)
    return (k[..., 0] << 32) | (k[..., 1] << 16) | k[..., 2], ok


def _walk(resolution, origin, ends):
    """ray_keys with counts for one chunk of rays (a pool worker's job)."""
    return ray_keys(OcTree(resolution), origin, ends, counts=True)


class Tree:
    """One OcTree of oracle/octomap.py as sorted key / log-odds arrays."""

    def __init__(self, resolution):
        self.octree = OcTree(resolution)        # constants and key arithmetic; holds no cells
        self.keys = np.empty(0, np.int64)
        self.lo = np.empty(0, np.float32)

    @property
    def resolution(self):
        return self.octree.resolution

    def copy(self):
        t = Tree(self.resolution)
        t.keys, t.lo = self.keys.copy(), self.lo.copy()
        return t

    @property
    def cells(self):
        """{(kx, ky, kz): np.float32 log-odds}, as OcTree.cells."""
        return dict(zip(unpack(self.keys), (np.float32(v) for v in self.lo)))

    def scan_keys(self, pointcloud, origin, chunk=CHUNK, pool=None):
        """The keys of one insertPointCloud: (free, rays, occ).  free: sorted keys of every ray's
        computeRayKeys; rays [len(free)]: how many rays cross each; occ: sorted end-point keys.
        pool: a multiprocessing pool that walks the chunks of rays in parallel."""
        pts = np.asarray(pointcloud, np.float64).astype(np.float32).reshape(-1, 3)
        org = np.asarray(origin, np.float64).astype(np.float32)
        jobs = [(self.resolution, org, pts[s:s + chunk]) for s in range(0, len(pts), chunk)]
        walked = pool.starmap(_walk, jobs) if pool is not None and len(jobs) > 1 else \
            [_walk(*j) for j in jobs]
        keys = [np.empty(0, np.int64)] + [k for k, _ in walked]
        counts = [np.empty(0, np.int64)] + [c for _, c in walked]
        free, inv = np.unique(np.concatenate(keys), return_inverse=True)
        rays = np.bincount(inv.reshape(-1), weights=np.concatenate(counts),
                           minlength=len(free)).astype(np.int64)
        k, ok = _keys(self.octree, pts)
        return free, rays, np.unique(k[ok])

    def apply(self, keys, update, times=1):
        """``times`` clamped float32 adds of ``update`` to each of the distinct keys (a cell not
        in the tree starts at 0).  times: int or [len(keys)]."""
        keys = np.asarray(keys, np.int64)
        if not len(keys):
            return
        upd = np.float32(update)
        lo_min, lo_max = self.octree.clamping_thres_min, self.octree.clamping_thres_max
        times = np.broadcast_to(np.asarray(times, np.int64), keys.shape)
        pos = np.searchsorted(self.keys, keys)
        found = pos < len(self.keys)
        found[found] = self.keys[pos[found]] == keys[found]
        v = np.zeros(len(keys), np.float32)
        v[found] = self.lo[pos[found]]
        # the clamp a run of equal updates ends at: once there, further adds stay there
        bound = lo_max if upd > 0 else lo_min
        n = 0
        while True:
            n += 1
            sel = (times >= n) & (v != bound)
            if not sel.any():
                break
            w = (v[sel] + upd).astype(np.float32)                  # float add
            v[sel] = np.minimum(np.maximum(w, lo_min), lo_max)
        self.lo[pos[found]] = v[found]
        keys = np.concatenate([self.keys, keys[~found]])
        lo = np.concatenate([self.lo, v[~found]])
        order = np.argsort(keys, kind="stable")
        self.keys, self.lo = keys[order], lo[order]

    def apply_scan(self, free, occ):
        """insertPointCloud's updates: a miss for every key of free - occ, a hit for every key of
        occ."""
        self.apply(np.setdiff1d(free, occ, assume_unique=True), self.octree.prob_miss_log)
        self.apply(occ, self.octree.prob_hit_log)

    def insertPointCloud(self, pointcloud, origin, pool=None):
        """OcTree.insertPointCloud(pointcloud, origin).  Returns (rays, distinct free cells, largest
        number of rays through one cell) of the scan."""
        free, rays, occ = self.scan_keys(pointcloud, origin, pool=pool)
        self.apply_scan(free, occ)
        return len(np.asarray(pointcloud).reshape(-1, 3)), len(free), int(rays.max(initial=0))

    def updateNodes(self, values):
        """OcTree.updateNodes(values, True): one hit per row of float64 values [M, 3]."""
        k, ok = double_keys(self.octree, np.asarray(values, np.float64).reshape(-1, 3))
        keys, n = np.unique(k[ok], return_counts=True)
        self.apply(keys, self.octree.prob_hit_log, n)

    def lookup(self, pts):
        """Log-odds at float64 points [..., 3] (search(depth=0)), NaN for unknown space."""
        k, ok = double_keys(self.octree, pts)
        out = np.full(k.shape, np.nan, np.float32)
        if not len(self.keys):
            return out
        pos = np.clip(np.searchsorted(self.keys, k), 0, len(self.keys) - 1)
        hit = ok & (self.keys[pos] == k)
        out[hit] = self.lo[pos[hit]]
        return out


def occupancy(lo):
    """octomap::probability (oracle.octomap.probability, math.exp in double) of float32 log-odds,
    NaN -> -1 (unknown, as get_target_grids marks it)."""
    lo = np.asarray(lo, np.float32)
    out = np.full(lo.shape, -1.0)
    known = ~np.isnan(lo)
    uniq, inv = np.unique(lo[known], return_inverse=True)
    out[known] = np.array([probability(v) for v in uniq], np.float64)[inv.reshape(-1)]
    return out


class MultiInstanceOctreeMapping:
    """oracle.octomap.MultiInstanceOctreeMapping over ``Tree``s.  pool: a multiprocessing pool
    for the ray walks of ``integrate`` (see Tree.scan_keys)."""

    def __init__(self, pool=None):
        self._trees = {}
        self.pool = pool

    @property
    def instance_ids(self):
        return list(self._trees.keys())

    def initialize(self, instance_id, *, pitch):
        if instance_id in self._trees:
            raise ValueError("instance {instance_id} already exists")
        self._trees[instance_id] = Tree(pitch)

    def copy(self):
        m = MultiInstanceOctreeMapping(self.pool)
        m._trees = {i: t.copy() for i, t in self._trees.items()}
        return m

    def integrate(self, instance_id, mask, pcd, origin=(0, 0, 0)):
        """Returns insertPointCloud's (rays, distinct free cells, largest rays through one cell)."""
        origin = np.asarray(origin, dtype=float)
        nonnan = ~np.isnan(pcd).any(axis=2)
        return self._trees[instance_id].insertPointCloud(pcd[mask & nonnan], origin=origin,
                                                         pool=self.pool)

    def update(self, instance_id, occupied):
        self._trees[instance_id].updateNodes(occupied)

    def cells(self, instance_id):
        return self._trees[instance_id].cells

    def n_cells(self):
        return sum(len(t.keys) for t in self._trees.values())

    def get_target_grids(self, target_id, *, dimensions, pitch, origin):
        g = self.get_target_grids_batch([target_id], dimensions=dimensions, pitches=[pitch],
                                        origins=[origin])
        return tuple(a[0] for a in g)

    def get_target_grids_batch(self, target_ids, *, dimensions, pitches, origins):
        """(grid_target, grid_nontarget, grid_empty), each float32 [T, X, Y, Z]: oracle.octomap's
        get_target_grids of every target."""
        X, Y, Z = (int(d) for d in dimensions)
        T = len(target_ids)
        pitches = np.asarray(pitches, np.float64).reshape(T)
        origins = np.asarray(origins, np.float64).reshape(T, 3)
        ii, jj, kk = np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij")
        idx = np.stack([ii.ravel(), jj.ravel(), kk.ravel()], 1)
        centers = idx[None] * pitches[:, None, None] + origins[:, None, :]   # [T, V, 3]
        gt, gn, ge = (np.zeros((T, X * Y * Z), np.float32) for _ in range(3))
        for ins_id, tree in self._trees.items():
            occ = occupancy(tree.lookup(centers))
            q = occ >= 0.5
            is_t = np.array([t == ins_id for t in target_ids], bool)[:, None]
            gt[q & is_t] = occ[q & is_t]
            gn[q & ~is_t] = occ[q & ~is_t]
            e = (0 <= occ) & (occ < 0.5)
            ge[e] = 1 - occ[e]
        shape = (T, X, Y, Z)
        return gt.reshape(shape), gn.reshape(shape), ge.reshape(shape)
