"""CPU-only: the solid grid and the signed distance of morefusion_b200/csrc/mesh_models.cu, its
per-face and per-pair code executed serially on the host (tests/emu/mesh_models_emu.cpp,
g++ -DMF_HOST_EMU), bit for bit against oracle/mesh_models.py.  The GPU run is
tests/test_mesh_models_gpu.py."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import _mesh_cases as mc
from oracle import mesh_models as omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "mesh_models_emu.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17",
                    "-I" + os.path.join(ROOT, "tests", "emu"),
                    os.path.join(ROOT, "tests", "emu", "mesh_models_emu.cpp"), "-o", so], check=True)
    return ctypes.CDLL(so)


def pack(meshes):
    vs, fs, offsets, base = [], [], [0], 0
    for v, f in meshes:
        vs.append(np.asarray(v, np.float64).reshape(-1, 3))
        fs.append(np.asarray(f, np.int32).reshape(-1, 3) + base)
        base += len(vs[-1])
        offsets.append(offsets[-1] + len(fs[-1]))
    return (np.ascontiguousarray(np.concatenate(vs)), np.ascontiguousarray(np.concatenate(fs)),
            np.asarray(offsets, np.int64))


def voxelize(emu, meshes, D):
    v, f, off = pack(meshes)
    S = len(meshes)
    matrix = np.empty((S, D, D, D), np.uint8)
    counts = np.empty(S, np.int32)
    points = np.empty((S, D ** 3, 3))
    t, sc, pitch = np.empty((S, 3)), np.empty(S), np.empty(S)
    p = ctypes.c_void_p
    fn = emu.emu_voxelize_solid
    fn.argtypes = [p, ctypes.c_int, p, ctypes.c_int, p, ctypes.c_int, ctypes.c_int] + [p] * 6
    assert fn(v.ctypes.data, len(v), f.ctypes.data, len(f), off.ctypes.data, S, D,
              matrix.ctypes.data, counts.ctypes.data, points.ctypes.data, t.ctypes.data,
              sc.ctypes.data, pitch.ctypes.data) == 0
    return matrix.astype(bool), counts, points, t, sc, pitch


def signed_distance(emu, meshes, pts, mesh):
    v, f, off = pack(meshes)
    pts = np.ascontiguousarray(pts, np.float64)
    mesh = np.ascontiguousarray(mesh, np.int32)
    sdf = np.empty(len(pts))
    face = np.empty(len(pts), np.int32)
    p = ctypes.c_void_p
    fn = emu.emu_signed_distance
    fn.argtypes = [p, ctypes.c_int, p, ctypes.c_int, p, ctypes.c_int, p, p, ctypes.c_int, p, p]
    assert fn(v.ctypes.data, len(v), f.ctypes.data, len(f), off.ctypes.data, len(meshes),
              pts.ctypes.data, mesh.ctypes.data, len(pts), sdf.ctypes.data, face.ctypes.data) == 0
    return sdf, face


def crossings(emu, mesh, px, py):
    v, f, off = pack([mesh])
    p = ctypes.c_void_p
    fn = emu.emu_column_crossings
    fn.argtypes = [p, ctypes.c_int, p, ctypes.c_int, p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                   ctypes.c_double]
    return fn(v.ctypes.data, len(v), f.ctypes.data, len(f), off.ctypes.data, 1, 0, px, py)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def synthetic_cads(class_ids):
    from morefusion_b200 import synthetic
    m = synthetic.SyntheticYCBModels()
    return [(m.get_cad(c).vertices, m.get_cad(c).faces) for c in class_ids]


def check_grid(emu, meshes, D):
    matrix, counts, points, t, sc, pitch = voxelize(emu, meshes, D)
    for s, (v, f) in enumerate(meshes):
        want = omm.voxelize_solid(v, f, D)
        assert np.array_equal(matrix[s], want["matrix"]), s
        assert counts[s] == len(want["points"])
        assert np.array_equal(bits(points[s, :counts[s]]), bits(want["points"]))
        assert np.isnan(points[s, counts[s]:]).all()
        assert np.array_equal(bits(t[s]), bits(want["translate"]))
        assert bits(sc[s]) == bits(want["scale"]) and bits(pitch[s]) == bits(want["pitch"])
    return matrix, counts


@pytest.mark.parametrize("D", [16, 40])
def test_grid_synthetic_classes(emu, D):
    matrix, counts = check_grid(emu, synthetic_cads([1, 2, 3]), D)
    assert (counts > 0).all()


@pytest.mark.parametrize("name", sorted(mc.all_cases()))
def test_grid_cases(emu, name):
    matrix, counts = check_grid(emu, [mc.all_cases()[name]], 24)
    assert counts[0] > 0


def test_grid_is_solid_and_not_convex(emu):
    # the L's notch stays empty, its arms are filled through
    v, f = mc.extruded_l()
    matrix, _, _, t, _, pitch = voxelize(emu, [(v, f)], 32)
    c = t[0][:, None] + (np.arange(32) + 0.5) * pitch[0]
    ix = np.searchsorted(c[0], 0.04)
    iy = np.searchsorted(c[1], 0.05)
    assert not matrix[0, ix, iy].any()
    col = matrix[0, np.searchsorted(c[0], 0.01), np.searchsorted(c[1], 0.01)]
    assert col[c[2] < 0.04].all() and not col[c[2] > 0.04 + pitch[0]].any()
    # the torus's hole stays empty
    matrix, _, _, t, _, pitch = voxelize(emu, [mc.torus()], 32)
    assert not matrix[0, 15:17, 15:17].any() and matrix[0].sum() > 0


def test_columns_through_shared_edges_and_vertices(emu):
    # every column centre of the edge-aligned box's grid, and lines exactly through its vertices
    # and along its cap diagonal: a closed mesh is crossed an even number of times
    D = 16
    v, f = mc.edge_aligned_box(D)
    s = 1.0 / D
    c = (np.arange(D) + 0.5) * s
    xs, ys = np.meshgrid(c, c, indexing="ij")
    pts = np.c_[xs.reshape(-1), ys.reshape(-1)]
    pts = np.concatenate([pts, v[:, :2], [[7.5 * s, 3.5 * s], [0.0, 3.5 * s]]])
    for px, py in pts:
        n = crossings(emu, (v, f), px, py)
        assert n % 2 == 0, (px, py, n)
        assert n == omm.column_parity_counts(v, f, [px], [py])[0]
    # inside the cross-section the column meets the two caps exactly once each
    diag = [crossings(emu, (v, f), x, x) for x in c[:7]]
    assert diag == [2] * 7
    # closed meshes with shared vertices on column lines: the torus and the sphere at their grids
    for mesh in (mc.torus(), synthetic_cads([3])[0], mc.extruded_l()):
        g = omm.voxelize_solid(*mesh, 20)
        cc = omm.centres(g["translate"], g["pitch"], 20)
        cols = np.concatenate([np.stack(np.meshgrid(cc[0], cc[1], indexing="ij"), -1).reshape(-1, 2),
                               mesh[0][:, :2]])
        n = omm.column_parity_counts(*mesh, cols[:, 0], cols[:, 1])
        assert (n % 2 == 0).all()


def test_signed_distance_cases(emu):
    meshes = synthetic_cads([1, 2, 3]) + [mc.all_cases()[k] for k in sorted(mc.all_cases())]
    pts, tags = [], []
    for s, (v, f) in enumerate(meshes):
        p = mc.sample_points(v, f, 200, seed=s)
        pts.append(p)
        tags.append(np.full(len(p), s, np.int32))
    pts, tags = np.concatenate(pts), np.concatenate(tags)
    sdf, face = signed_distance(emu, meshes, pts, tags)
    v_all, f_all, off = pack(meshes)
    for s, (v, f) in enumerate(meshes):
        sel = tags == s
        want, arg = omm.signed_distance(v, f, pts[sel])
        assert np.array_equal(bits(sdf[sel]), bits(want)), s
        assert np.array_equal(face[sel], arg + off[s])
    # a point outside every mesh's range of tags
    sdf2, face2 = signed_distance(emu, meshes[:1], pts[:3], np.array([0, -1, 5], np.int32))
    assert np.isfinite(sdf2[0]) and np.isnan(sdf2[1:]).all() and (face2[1:] == -1).all()


def test_signed_distance_signs(emu):
    from morefusion_b200 import synthetic
    kind, half = synthetic._primitive(3)
    assert kind == "box"
    v, f = synthetic.cad_mesh(kind, half)
    pts = np.array([[0.0, 0.0, 0.0], [2 * half[0], 0, 0], [half[0], 0.3 * half[1], 0.1 * half[2]]])
    sdf, _ = signed_distance(emu, [(v, f)], pts, np.zeros(3, np.int32))
    assert sdf[0] > 0 and sdf[1] < 0 and abs(sdf[2]) < 1e-15
