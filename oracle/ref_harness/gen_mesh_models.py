#!/usr/bin/env python
"""Run the reference's own ``YCBVideoModels`` methods (morefusion/datasets/ycb_video/models.py:
``get_sdf``, ``_get_sdf_file``, ``_get_sdf``, ``get_solid_voxel_grid``, ``get_cad``,
``get_cad_file``, ``get_bbox_diagonal`` and ``get_voxel_pitch``, taken from the reference
checkout by ``ast``) on seeded meshes, and write what they compose to
tests/golden/mesh_models/cases.npz with a digest in tests/golden/mesh_models/digest.json.

TEST INFRASTRUCTURE ONLY.  Needs the reference checkout (MOREFUSION_REFERENCE):

    python -m oracle.ref_harness.gen_mesh_models

Stand-ins, in the style of open3d_stub.py (binvox, trimesh and Open3D are not installed):
  * ``trimesh.load(path, process=False)`` returns the case's mesh, whose ``bounding_box.extents``
    are the extents of its referenced vertices and whose ``nearest.signed_distance`` is
    oracle/mesh_models.py's;
  * ``utils_module.get_binvox_file`` writes an empty placeholder beside the OBJ (the methods open
    it) and ``trimesh.exchange.binvox.load_binvox`` returns the oracle's 64^3 grid of the mesh;
  * ``extra_module.open3d.voxel_down_sample`` is oracle/icp.py's.
So this pins the composition -- which points, which pitch, in what order, and what an existing
sdf.npz gives -- not binvox's carving or trimesh's sign (DESIGN.md section 4.22).

cases.npz, per case of CASES: ``<case>/vertices``, ``<case>/faces`` (the inputs),
``<case>/points`` and ``<case>/sdf`` (what get_sdf returns), ``<case>/bbox_diagonal`` and
``<case>/pitch32`` (get_bbox_diagonal, get_voxel_pitch(32)), ``<case>/written_points`` and
``<case>/written_sdf`` (what _get_sdf wrote to sdf.npz); and ``cache/points``, ``cache/sdf``: what
get_sdf returns for a class whose sdf.npz already exists (the file's arrays, not a recomputation).
"""

import ast
import hashlib
import json
import os
import pathlib
import sys
import tempfile
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import icp as oicp  # noqa: E402
from oracle import mesh_models as omm  # noqa: E402
from oracle.ref_harness import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mesh_models")
MODELS = os.path.join("morefusion", "datasets", "ycb_video", "models.py")
METHODS = ("get_sdf", "_get_sdf_file", "_get_sdf", "get_solid_voxel_grid", "get_cad", "get_cad_file",
           "get_bbox_diagonal", "get_voxel_pitch")


def cases():
    """name -> (vertices, faces): small seeded meshes of every kind the kernels handle."""
    import _mesh_cases as mc
    from morefusion_b200 import synthetic
    sm = synthetic.SyntheticYCBModels()
    out = {f"class{c}": (sm.get_cad(c).vertices, sm.get_cad(c).faces) for c in (1, 2, 3)}
    out["torus"] = mc.torus(n_major=16, n_minor=8)
    out["extruded_l"] = mc.extruded_l()
    out["mixed_winding"] = mc.mixed_winding(*mc.icosphere(1, radius=0.04), seed=3)
    return out


def _reference_class(meshes):
    """A class whose methods are the reference's own, over the stand-ins."""
    text = open(os.path.join(shim.REF_ROOT, MODELS)).read()
    mesh_of = {}

    class _Cad:
        def __init__(self, v, f):
            self.vertices, self.faces = v, f
            used = v[f.reshape(-1)]
            self.bounding_box = types.SimpleNamespace(extents=used.max(0) - used.min(0))
            self.nearest = types.SimpleNamespace(
                signed_distance=lambda p: omm.signed_distance(v, f, p)[0])

    def load(path, process=True):
        assert process is False
        return _Cad(*meshes[mesh_of[str(path)]])

    def get_binvox_file(cad_file, solid=True):
        out = pathlib.Path(str(cad_file)).with_suffix(".solid.binvox")
        out.write_bytes(b"")
        mesh_of[str(out)] = mesh_of[str(cad_file)]
        return out

    def load_binvox(f):
        v, fc = meshes[mesh_of[f.name]]
        return types.SimpleNamespace(points=omm.voxelize_solid(v, fc, 64)["points"])

    trimesh = types.SimpleNamespace(load=load, Trimesh=object, exchange=types.SimpleNamespace(
        binvox=types.SimpleNamespace(load_binvox=load_binvox)))
    g = dict(np=np, trimesh=trimesh, typing=__import__("typing"),
             utils_module=types.SimpleNamespace(get_binvox_file=get_binvox_file),
             extra_module=types.SimpleNamespace(open3d=types.SimpleNamespace(
                 voxel_down_sample=lambda p, s: oicp.voxel_down_sample(p, s))))
    body = {}
    for node in ast.parse(text).body:
        if isinstance(node, ast.ClassDef) and node.name == "YCBVideoModels":
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in METHODS:
                    ns = dict(g)
                    exec(textwrap.dedent(ast.get_source_segment(text, item, padded=True)), ns)
                    body[item.name] = ns[item.name]
    assert set(body) == set(METHODS), set(METHODS) - set(body)
    return body, mesh_of


def run(meshes, root):
    """The reference's get_sdf / get_bbox_diagonal / get_voxel_pitch(32) of every mesh, with its
    models directory at root."""
    body, mesh_of = _reference_class(meshes)
    names = sorted(meshes)
    root = pathlib.Path(root)
    attrs = dict(body, class_names=names, _root_dir=root, root_dir=root, _bbox_diagonal_cache={},
                 _cad_cache={}, _pcd_cache={}, _sdf_cache={})
    Models = type("ReferenceYCBVideoModels", (), attrs)
    models = Models()
    out = {}
    for c, name in enumerate(names):
        (root / name).mkdir(parents=True, exist_ok=True)
        mesh_of[str(root / name / "textured_simple.obj")] = name
        points, sdf = models.get_sdf(c)
        written = np.load(root / name / "sdf.npz")
        out[name] = dict(points=np.asarray(points), sdf=np.asarray(sdf),
                         bbox_diagonal=np.float64(models.get_bbox_diagonal(c)),
                         pitch32=np.float64(models.get_voxel_pitch(32, class_id=c)),
                         written_points=written["points"], written_sdf=written["sdf"])
    return out


def run_cache(root):
    """What get_sdf returns for a class whose sdf.npz exists: seeded arrays written first."""
    rs = np.random.RandomState(5)
    pts, sdf = rs.uniform(-1, 1, (17, 3)), rs.uniform(-1, 1, 17)
    name = "cached"
    d = pathlib.Path(root) / name
    d.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(d / "sdf.npz", points=pts, sdf=sdf)
    body, mesh_of = _reference_class({name: cases()["torus"]})
    Models = type("ReferenceYCBVideoModels", (), dict(
        body, class_names=[name], _root_dir=pathlib.Path(root), root_dir=pathlib.Path(root),
        _bbox_diagonal_cache={}, _cad_cache={}, _pcd_cache={}, _sdf_cache={}))
    p, s = Models().get_sdf(0)
    return pts, sdf, np.asarray(p), np.asarray(s)


def digest(arrays):
    return {k: hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest()
            for k, v in sorted(arrays.items())}


def main():
    meshes = cases()
    with tempfile.TemporaryDirectory() as tmp:
        got = run(meshes, os.path.join(tmp, "models"))
        cpts, csdf, gpts, gsdf = run_cache(os.path.join(tmp, "cache"))
    assert np.array_equal(cpts, gpts) and np.array_equal(csdf, gsdf)
    arrays = {"cache/points": gpts, "cache/sdf": gsdf}
    for name, (v, f) in meshes.items():
        arrays[f"{name}/vertices"] = np.asarray(v, np.float64)
        arrays[f"{name}/faces"] = np.asarray(f, np.int32)
        for k, a in got[name].items():
            arrays[f"{name}/{k}"] = a
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "cases.npz"), **arrays)
    with open(os.path.join(OUT, "digest.json"), "w") as fh:
        json.dump(digest(arrays), fh, indent=1, sort_keys=True)
        fh.write("\n")
    print("wrote", OUT, {k: got[k]["points"].shape[0] for k in got})


if __name__ == "__main__":
    main()
