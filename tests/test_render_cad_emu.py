"""CPU-only: the CAD render of morefusion_b200/csrc/render_cad.cu, its set-up kernel and per-pixel
code executed serially on the host (tests/emu/render_cad_emu.cpp, g++ -DMF_HOST_EMU), bit for bit
against oracle/render_cad.py; that oracle against a float64 Moller-Trumbore control and the
fill rule on constructed edges; and ``SyntheticYCBModels.get_cad``.  The GPU run is
tests/test_render_cad_gpu.py."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import render_cad as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 500.0                                     # focal length in pixels of the constructed cases


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "render_cad_emu.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17",
                    "-I" + os.path.join(ROOT, "tests", "emu"),
                    os.path.join(ROOT, "tests", "emu", "render_cad_emu.cpp"), "-o", so], check=True)
    fn = ctypes.CDLL(so).emu_render_cad
    fn.restype = ctypes.c_int
    p, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    fn.argtypes = [p, i, p, i, p, i, p, p, i, d, i, i, p, p, p]

    def render(meshes, mesh_of_pose, Ts, f, H, W):
        vs, fs, offsets, base = [], [], [0], 0
        for v, fc in meshes:
            vs.append(np.asarray(v, np.float64).reshape(-1, 3))
            fs.append(np.asarray(fc, np.int32).reshape(-1, 3) + base)
            base += len(vs[-1])
            offsets.append(offsets[-1] + len(fs[-1]))
        v = np.ascontiguousarray(np.concatenate(vs))
        fc = np.ascontiguousarray(np.concatenate(fs))
        off = np.asarray(offsets, np.int64)
        mesh = np.ascontiguousarray(mesh_of_pose, np.int32)
        Ts = np.ascontiguousarray(np.asarray(Ts, np.float64).reshape(-1, 4, 4))
        N = len(Ts)
        depth = np.empty((N, H, W), np.float32)
        mask = np.empty((N, H, W), np.uint8)
        count = np.empty(N, np.int32)
        assert fn(v.ctypes.data, len(v), fc.ctypes.data, len(fc), off.ctypes.data, len(meshes),
                  mesh.ctypes.data, Ts.ctypes.data, N, f, H, W, depth.ctypes.data,
                  mask.ctypes.data, count.ctypes.data) == 0
        return depth, mask.astype(bool), count
    return render


def assert_same(got, want):
    d, m, c = got
    wd, wm, wc = want
    assert np.array_equal(m, wm)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(c, wc)


def check(emu, v, fc, Ts, f, H, W):
    want = orc.render_cad(v, fc, Ts, f, H, W)
    got = emu([(v, fc)], np.zeros(len(np.reshape(Ts, (-1, 4, 4))), np.int32), Ts, f, H, W)
    assert_same(got, want)
    return want


def pose(R=np.eye(3), t=(0, 0, 1)):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def random_rotation(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def primitive_poses(rs, n, H, W, f):
    """n random poses at 0.3-1.2 m, centred somewhere on (or just off) the image."""
    Ts = []
    for _ in range(n):
        z = rs.uniform(0.3, 1.2)
        u, v = rs.uniform(-0.2, 1.2) * W, rs.uniform(-0.2, 1.2) * H
        Ts.append(pose(random_rotation(rs), ((u - W / 2) / f * z, (v - H / 2) / f * z, z)))
    return np.array(Ts)


def cads():
    from morefusion_b200 import synthetic
    m = synthetic.SyntheticYCBModels()
    return [m.get_cad(c) for c in (1, 2, 3)]


@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (480, 640)])
def test_primitives_random_poses(emu, H, W):
    """The three synthetic primitives at random poses, some partly or wholly off the image."""
    rs = np.random.RandomState(H * 1000 + W)
    f = orc.focal_from_fovy(orc.fovy_from_intrinsics(1066.778 * H / 480, H), H)
    for cad in cads():
        Ts = primitive_poses(rs, 3, H, W, f)
        d, m, c = check(emu, cad.vertices, cad.faces, Ts, f, H, W)
        if H > 1:
            assert c.max() > 0


def test_several_meshes_one_call(emu):
    """Poses of several packed meshes in one call, as the dataset renders them."""
    rs = np.random.RandomState(1)
    H, W = 48, 64
    cs = cads()
    mesh = np.array([2, 0, 1, 1, 0, 2], np.int32)
    Ts = primitive_poses(rs, len(mesh), H, W, 60.0)
    got = emu([(c.vertices, c.faces) for c in cs], mesh, Ts, 60.0, H, W)
    for n, s in enumerate(mesh):
        want = orc.render_cad(cs[s].vertices, cs[s].faces, Ts[n], 60.0, H, W)
        assert_same(tuple(a[n:n + 1] for a in got), want)


def test_behind_near_and_straddling(emu):
    """A pose behind the camera covers nothing; a mesh straddling the near plane loses exactly
    the triangles with a vertex in front of it."""
    cad = cads()[0]
    H, W = 60, 80
    T_behind = pose(t=(0, 0, -0.5))
    T_straddle = pose(t=(0, 0, 0.012))
    T_far_off = pose(t=(50, 0, 1))
    d, m, c = check(emu, cad.vertices, cad.faces, [T_behind, T_straddle, T_far_off], 70.0, H, W)
    assert c[0] == 0 and c[2] == 0
    s = orc.setup(cad.vertices, cad.faces, T_straddle, 70.0, H, W)
    assert (~s["valid"]).any() and s["valid"].any()


def test_full_image_degenerate_nan_empty(emu):
    H, W = 7, 5
    big = np.array([[-10, -10, 1], [10, -10, 1], [0, 10, 1]], np.float64)
    degenerate = np.array([[0, 0, 1], [0.1, 0, 1], [0.2, 0, 1], [0, 0, 1], [0, 0, 1], [0.1, 0.1, 1]])
    v = np.concatenate([big, degenerate])
    fc = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8]], np.int32)
    d, m, c = check(emu, v, fc, [pose(t=(0, 0, 0)), pose(t=(0, 0, 1))], 3.0, H, W)
    assert m[0].all() and np.all(d[0] == np.float32(1.0))
    # degenerate faces alone cover nothing
    d, m, c = check(emu, v, fc[1:], [pose(t=(0, 0, 0))], 3.0, H, W)
    assert c[0] == 0 and np.isnan(d).all()
    # F = 0, N = 0, NaN in a pose
    T_nan = pose()
    T_nan[0, 1] = np.nan
    check(emu, v, np.zeros((0, 3), np.int32), [pose()], 3.0, H, W)
    check(emu, v, fc, np.zeros((0, 4, 4)), 3.0, H, W)
    d, m, c = check(emu, v, fc[:1], [T_nan, pose()], 3.0, H, W)
    assert c[0] == 0 and c[1] == H * W


def _pixel_faces(v2, f=1.0):
    """Camera-frame vertices at Z = 1 whose projection with focal f and a 0x0 offset is v2."""
    v2 = np.asarray(v2, np.float64)
    return np.c_[v2[:, 0] / f, v2[:, 1] / f, np.ones(len(v2))]


def test_shared_edge_covered_once():
    """A square split into two triangles along a diagonal through pixel centres: every centre on
    the shared edge (and on the square's edges) is covered by exactly one triangle."""
    H = W = 16
    # pixel coordinates relative to the image centre (W / 2, H / 2) = (8, 8)
    sq = np.array([[2.5, 2.5], [12.5, 2.5], [12.5, 12.5], [2.5, 12.5]]) - 8
    v = _pixel_faces(sq)
    for tris in ([[0, 1, 2], [0, 2, 3]], [[0, 2, 1], [0, 3, 2]]):     # both windings
        masks = [orc.render_one(v, np.array([t]), pose(t=(0, 0, 0)), 1.0, H, W)[1] for t in tris]
        assert not (masks[0] & masks[1]).any()
        union = masks[0] | masks[1]
        # centres 2.5..12.5 on the square's boundary: left/top edges in, right/bottom out
        want = np.zeros((H, W), bool)
        want[2:12, 2:12] = True
        assert np.array_equal(union, want)
        diag = np.arange(2, 12)
        assert (masks[0] | masks[1])[diag, diag].all()


def test_fill_rule_each_edge_kind():
    """A triangle with pixel centres exactly on a top edge, a left edge, a right edge and a bottom
    edge: only the top and left ones count."""
    H = W = 16
    tri = np.array([[2.5, 2.5], [10.5, 2.5], [2.5, 10.5]]) - 8    # top, left, hypotenuse
    for fc in ([0, 1, 2], [0, 2, 1]):
        m = orc.render_one(_pixel_faces(tri), np.array([fc]), pose(t=(0, 0, 0)), 1.0, H, W)[1]
        assert m[2, 2:10].all() and m[2:10, 2].all()      # top row and left column in
        assert not m[2, 10] and not m[10, 2]               # the far ends lie on the hypotenuse
        assert not m[3, 9] and m[3, 8]                     # centre on the hypotenuse: out
    # bottom and right edges: the mirrored triangle
    tri = np.array([[10.5, 10.5], [2.5, 10.5], [10.5, 2.5]]) - 8
    m = orc.render_one(_pixel_faces(tri), np.array([[0, 1, 2]]), pose(t=(0, 0, 0)), 1.0, H, W)[1]
    assert not m[10, 3:11].any() and not m[3:11, 10].any()
    assert m[9, 9] and m[8, 4]          # its hypotenuse, running up and right, is a left edge


@pytest.mark.parametrize("case", range(6))
def test_oracle_matches_moller_trumbore(case):
    rs = np.random.RandomState(case)
    H, W = 48, 64
    f = 60.0
    if case < 3:
        cad = cads()[case]
        v, fc = cad.vertices, cad.faces
        Ts = primitive_poses(rs, 2, H, W, f)
    else:                                                  # a random soup in front of the camera
        v = rs.uniform(-0.3, 0.3, (90, 3)) + [0, 0, 1.0]
        fc = rs.randint(0, 90, (30, 3)).astype(np.int32)
        Ts = [pose(random_rotation(rs) if case > 3 else np.eye(3), t=(0, 0, rs.uniform(0, 0.5)))]
    for T in Ts:
        _, m = orc.render_one(v, fc, T, f, H, W)
        covered, decided = orc.moller_trumbore_mask(v, fc, T, f, H, W)
        assert decided.mean() > 0.9
        assert np.array_equal(m[decided], covered[decided])


def test_camera_chain_gl():
    """The oracle's projection equals gluPerspective's matrix applied to the view matrix
    render_camera builds, through the viewport."""
    rs = np.random.RandomState(0)
    for H, W, fovy in [(480, 640, 48.0), (5, 7, 30.0), (100, 50, 90.0)]:
        f = orc.focal_from_fovy(fovy, H)
        T = pose(random_rotation(rs), (0.1, -0.05, 1.0))
        P = orc.projection_matrix(fovy, W / H)
        for x in rs.uniform(-0.1, 0.1, (5, 3)):
            u, v = orc.gl_pixel(orc.view_matrix(T), P, H, W, x)
            c = T[:3, :3] @ x + T[:3, 3]
            np.testing.assert_allclose([u, v], [f * c[0] / c[2] + W / 2, f * c[1] / c[2] + H / 2],
                                       rtol=0, atol=1e-9)


def test_get_cad_surface_and_closed():
    from morefusion_b200 import synthetic
    m = synthetic.SyntheticYCBModels()
    for c in range(1, 22):
        kind, half = synthetic._primitive(c)
        cad = m.get_cad(c)
        assert cad.vertices.dtype == np.float64 and cad.faces.dtype == np.int32
        assert np.abs(synthetic.sdf_primitive(kind, half, cad.vertices)).max() <= 1e-12
        fc = cad.faces
        directed = np.concatenate([fc[:, [0, 1]], fc[:, [1, 2]], fc[:, [2, 0]]])
        # closed and consistently wound: every directed edge once, and its reverse once
        assert len(np.unique(directed, axis=0)) == len(directed)
        rev = {tuple(e) for e in directed[:, ::-1]}
        assert rev == {tuple(e) for e in directed}
        a, b, cc = (cad.vertices[fc[:, k]] for k in range(3))
        assert np.einsum("ij,ij->i", a, np.cross(b, cc)).sum() > 0      # wound outward
