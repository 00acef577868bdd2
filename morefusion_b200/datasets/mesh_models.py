"""Per-class model data from CAD meshes, as YCBVideoModels derives it
(morefusion/datasets/ycb_video/models.py:56-115), built on the GPU (csrc/mesh_models.cu).

``MeshModels`` answers the ``models`` interface every component here reads (``get_pcd``,
``get_sdf``, ``get_solid_voxel_grid``, ``get_cad``, ``get_voxel_pitch``, ``get_bbox_diagonal``
and ``class_ids_symmetric``) for meshes the caller gives, or that ``from_directory`` reads in the
YCB layout.  Differences from the reference (DESIGN.md section 4.22):
  * the solid grid is the rule of ``geometry.voxelize_solid``, not binvox's carving;
  * the signed distance takes its sign from +z ray parity, not trimesh's ``contains``;
  * an existing ``sdf.npz`` is read as the reference reads it, but one is written only when
    ``write_sdf_cache`` is set (the reference writes into the dataset directory unasked);
  * nothing is downloaded: a missing directory raises FileNotFoundError.
"""

import os
import types

import numpy as np

SDF_DIMENSION = 32            # _get_sdf down-samples at get_voxel_pitch(32) (models.py:74)
GRID_DIMENSION = 64           # binvox -d 64 (utils/get_binvox_file.py)


def read_obj(path):
    """(vertices [V,3] float64, faces [F,3] int32) of a Wavefront OBJ file: ``v`` lines (x y z;
    any further numbers ignored) and ``f`` lines whose entries are ``a``, ``a/b``, ``a//c`` or
    ``a/b/c`` (1-based, negative counts back from the last vertex read); polygons are
    fan-triangulated from their first vertex.  Every other line is ignored."""
    vs, fs = [], []
    with open(path) as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                vs.append([float(t) for t in tok[1:4]])
            elif tok[0] == "f":
                idx = []
                for t in tok[1:]:
                    i = int(t.split("/")[0])
                    idx.append(i - 1 if i > 0 else len(vs) + i)
                if any(i < 0 or i >= len(vs) for i in idx):
                    raise ValueError(f"{path}: face index outside the vertices read so far")
                fs += [(idx[0], idx[k], idx[k + 1]) for k in range(1, len(idx) - 1)]
    return np.asarray(vs, np.float64).reshape(-1, 3), np.asarray(fs, np.int32).reshape(-1, 3)


class MeshModels:
    """Model data of the classes in ``meshes`` ({class_id: (vertices [V,3], faces [F,3])}), with
    the points of ``pcds`` ({class_id: [N,3]}) as each class's point cloud and
    ``class_ids_symmetric`` as the reference lists them.  ``sdf_files`` ({class_id: path}) names
    each class's ``sdf.npz``: an existing file is read instead of computing the SDF, and with
    ``write_sdf_cache`` a computed SDF is written there.

    The grids and SDFs are built on ``device`` (default: the current CUDA device) when first
    asked for; ``prepare(class_ids)`` builds many classes in one launch sequence."""

    def __init__(self, meshes, pcds, class_ids_symmetric=(), *, sdf_files=None,
                 write_sdf_cache=False, device=None):
        from .. import geometry
        self._meshes = {}
        for c, (v, f) in meshes.items():
            self._meshes[int(c)] = geometry._check_model_mesh(v, f)
        self._pcds = {int(c): np.asarray(p, np.float64).reshape(-1, 3) for c, p in pcds.items()}
        self.class_ids_symmetric = np.asarray(class_ids_symmetric, np.int32).reshape(-1)
        self._sdf_files = {int(c): str(p) for c, p in (sdf_files or {}).items()}
        self._write_sdf_cache = bool(write_sdf_cache)
        self._device = device
        self._grid = {}
        self._sdf = {}

    @classmethod
    def from_directory(cls, root, class_names, class_ids_symmetric=(), **kw):
        """Models in the YCB layout: class c's mesh is ``<root>/<class_names[c]>/
        textured_simple.obj``, its points ``points.xyz`` and its SDF cache ``sdf.npz`` beside
        them.  ``class_names[c]`` names class c; class 0 is the background and has no model.  A
        missing root or class directory raises FileNotFoundError (nothing is downloaded)."""
        root = str(root)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"models directory not found: {root}")
        meshes, pcds, sdf_files = {}, {}, {}
        for c, name in enumerate(class_names):
            if c == 0:
                continue
            d = os.path.join(root, name)
            if not os.path.isdir(d):
                raise FileNotFoundError(f"class {c} ({name}): directory not found: {d}")
            meshes[c] = read_obj(os.path.join(d, "textured_simple.obj"))
            pcds[c] = np.loadtxt(os.path.join(d, "points.xyz")).reshape(-1, 3)
            sdf_files[c] = os.path.join(d, "sdf.npz")
        return cls(meshes, pcds, class_ids_symmetric, sdf_files=sdf_files, **kw)

    # --------------------------------------------------------------------------------------------
    def _dev(self):
        import torch
        if self._device is not None:
            return torch.device(self._device)
        return torch.device("cuda", torch.cuda.current_device())

    def _mesh(self, class_id):
        c = int(class_id)
        if c not in self._meshes:
            raise KeyError(f"no mesh for class {c}")
        return self._meshes[c]

    def get_cad(self, class_id):
        v, f = self._mesh(class_id)
        return types.SimpleNamespace(vertices=v, faces=f)

    def get_pcd(self, class_id):
        return self._pcds[int(class_id)]

    def get_bbox_diagonal(self, class_id):
        v, f = self._mesh(class_id)
        used = v[f.reshape(-1)]
        extents = used.max(0) - used.min(0)
        return np.sqrt((extents ** 2).sum())

    def get_voxel_pitch(self, dimension, class_id):
        return 1.0 * self.get_bbox_diagonal(class_id) / dimension

    def get_solid_voxel_grid(self, class_id):
        """The class's 64^3 solid grid (``geometry.voxelize_solid``): ``.matrix``, ``.points``,
        ``.translate``, ``.pitch`` and ``.scale``, host arrays."""
        c = int(class_id)
        if c not in self._grid:
            self.prepare([c], sdf=False)
        return self._grid[c]

    def get_sdf(self, class_id):
        """(points [n,3], sdf [n]) float64, as _get_sdf composes them: the solid grid's points
        down-sampled at get_voxel_pitch(32) by Open3D's voxel_down_sample rule, and their signed
        distance (positive inside)."""
        c = int(class_id)
        if c not in self._sdf:
            self.prepare([c])
        return self._sdf[c]

    # --------------------------------------------------------------------------------------------
    def prepare(self, class_ids, sdf=True):
        """Build the grids (and, with ``sdf``, the SDFs) of the given classes that are not built
        yet: one voxelize launch sequence for every class, one down-sampling per class, one host
        read of the down-sampled counts, one signed-distance launch sequence for every class and
        one read of the results."""
        import torch
        from .. import geometry
        from ..contrib import icp_registration
        from ..functions.geometry import _util
        todo_sdf = []
        if sdf:
            for c in dict.fromkeys(int(c) for c in class_ids):
                if c in self._sdf:
                    continue
                f = self._sdf_files.get(c)
                if f is not None and os.path.exists(f):
                    data = np.load(f)
                    self._sdf[c] = (data["points"], data["sdf"])
                else:
                    todo_sdf.append(c)
        if sdf:                                   # grids only where an SDF is computed
            todo_grid = todo_sdf
        else:
            todo_grid = [c for c in dict.fromkeys(int(c) for c in class_ids) if c not in self._grid]
        if not todo_grid:
            return
        for c in todo_grid:
            self._mesh(c)
        dev = self._dev()
        classes = [todo_grid[i:i + geometry.MAX_MODEL_MESHES]
                   for i in range(0, len(todo_grid), geometry.MAX_MODEL_MESHES)]
        for group in classes:
            v, fc, offsets = geometry._pack_meshes([self._meshes[c] for c in group])
            d_v = _util.h2d_transient(v, dev, torch.float64)
            d_f = _util.h2d_transient(fc, dev, torch.int32)
            matrix, counts, points, translate, scale, pitch = geometry._voxelize_solid_batch(
                d_v, d_f, offsets, GRID_DIMENSION)
            want_sdf = [i for i, c in enumerate(group) if c in todo_sdf]
            n_ds = []
            for i in want_sdf:
                means, _, _, n = icp_registration.voxel_down_sample(
                    points[i:i + 1], self.get_voxel_pitch(SDF_DIMENSION, group[i]))
                n_ds.append((means[0], n))
            head = torch.cat([counts.to(torch.float64), scale, pitch, translate.reshape(-1)]
                             + [n.to(torch.float64) for _, n in n_ds]).cpu().numpy()
            S = len(group)
            cnt, sc, pt = head[:S].astype(np.int64), head[S:2 * S], head[2 * S:3 * S]
            tr = head[3 * S:6 * S].reshape(S, 3)
            nds = head[6 * S:].astype(np.int64)
            if want_sdf:
                pts = torch.cat([m[:k] for (m, _), k in zip(n_ds, nds)])
                tags = torch.cat([torch.full((int(k),), i, dtype=torch.int32, device=dev)
                                  for i, k in zip(want_sdf, nds)])
                d, _ = geometry._signed_distance_batch(d_v, d_f, offsets, pts, tags)
                pts_h, d_h = pts.cpu().numpy(), d.cpu().numpy()
            grids_h = [(matrix[i].cpu().numpy(), points[i, :cnt[i]].cpu().numpy())
                       for i in range(S)]
            for i, c in enumerate(group):
                m_h, p_h = grids_h[i]
                self._grid[c] = types.SimpleNamespace(matrix=m_h, points=p_h, translate=tr[i],
                                                      pitch=float(pt[i]), scale=float(sc[i]))
            off = 0
            for i, k in zip(want_sdf, nds):
                c = group[i]
                self._sdf[c] = (pts_h[off:off + k], d_h[off:off + k])
                off += k
                f = self._sdf_files.get(c)
                if self._write_sdf_cache and f is not None:
                    np.savez_compressed(f, points=self._sdf[c][0], sdf=self._sdf[c][1])
