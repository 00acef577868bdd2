"""GPU: the CAD render (csrc/render_cad.cu, ``geometry.render_cad`` / ``_render_cad_batch``) bit
for bit against oracle/render_cad.py, its argument checks and output bounds, and the
``visibility`` of ``get_example``.  The host emulation of the same code is
tests/test_render_cad_emu.py."""

import ctypes

import numpy as np
import pytest
import torch

from oracle import render_cad as orc
from test_frame_refine_gpu import _syncs
from test_render_cad_emu import cads, pose, primitive_poses, random_rotation

pytestmark = pytest.mark.gpu


def _pack(meshes):
    vs, fs, offsets, base = [], [], [0], 0
    for v, f in meshes:
        vs.append(np.asarray(v, np.float64).reshape(-1, 3))
        fs.append(np.asarray(f, np.int32).reshape(-1, 3) + base)
        base += len(vs[-1])
        offsets.append(offsets[-1] + len(fs[-1]))
    return (torch.tensor(np.concatenate(vs), device="cuda"),
            torch.tensor(np.concatenate(fs), device="cuda"), np.asarray(offsets, np.int64))


def _render(meshes, mesh, Ts, f, H, W):
    from morefusion_b200 import geometry
    v, fc, off = _pack(meshes)
    d, m, c = geometry._render_cad_batch(v, fc, off, np.asarray(mesh, np.int32),
                                         np.asarray(Ts, np.float64).reshape(-1, 4, 4),
                                         f=f, height=H, width=W)
    return d.cpu().numpy(), m.cpu().numpy(), c.cpu().numpy()


def _assert_oracle(got, meshes, mesh, Ts, f, H, W):
    d, m, c = got
    Ts = np.asarray(Ts, np.float64).reshape(-1, 4, 4)
    for n, s in enumerate(mesh):
        wd, wm, wc = orc.render_cad(meshes[s][0], meshes[s][1], Ts[n], f, H, W)
        assert np.array_equal(m[n], wm[0]), n
        assert np.array_equal(d[n].view(np.uint32), wd[0].view(np.uint32)), n
        assert c[n] == wc[0], n


@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (480, 640)])
def test_primitives_random_poses(H, W):
    rs = np.random.RandomState(H + W)
    f = orc.focal_from_fovy(orc.fovy_from_intrinsics(1066.778 * H / 480, H), H)
    meshes = [(c.vertices, c.faces) for c in cads()]
    mesh = np.repeat(np.arange(3), 3)
    Ts = primitive_poses(rs, len(mesh), H, W, f)
    _assert_oracle(_render(meshes, mesh, Ts, f, H, W), meshes, mesh, Ts, f, H, W)


def test_edge_cases():
    cad = cads()[0]
    H, W = 60, 80
    big = np.array([[-10, -10, 1], [10, -10, 1], [0, 10, 1]], np.float64)
    degenerate = np.array([[0, 0, 1], [0.1, 0, 1], [0.2, 0, 1], [0, 0, 1], [0, 0, 1], [0.1, 0.1, 1]])
    soup = (np.concatenate([big, degenerate]), np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8]]))
    meshes = [(cad.vertices, cad.faces), soup, (soup[0], soup[1][1:])]
    T_nan = pose()
    T_nan[1, 2] = np.nan
    Ts = [pose(t=(0, 0, -0.5)), pose(t=(0, 0, 0.012)), pose(t=(50, 0, 1)), pose(t=(0.05, 0, 0.3)),
          pose(t=(0, 0, 0)), pose(t=(0, 0, 0)), T_nan]
    mesh = [0, 0, 0, 0, 1, 2, 1]
    got = _render(meshes, mesh, Ts, 70.0, H, W)
    _assert_oracle(got, meshes, mesh, Ts, 70.0, H, W)
    assert got[2][4] == H * W and got[2][5] == 0 and got[2][6] == 0 and got[2][0] == 0
    # F = 0 and N = 0
    empty = [(cad.vertices, np.zeros((0, 3), np.int32))]
    d, m, c = _render(empty, [0, 0], [pose(), pose()], 70.0, H, W)
    assert not m.any() and np.isnan(d).all() and (c == 0).all()
    d, m, c = _render(meshes, np.zeros(0, np.int32), np.zeros((0, 4, 4)), 70.0, H, W)
    assert d.shape == (0, H, W) and c.shape == (0,)


def test_64_poses_and_repeat_bitwise():
    rs = np.random.RandomState(64)
    H, W = 480, 640
    f = orc.focal_from_fovy(orc.fovy_from_intrinsics(1066.778, H), H)
    meshes = [(c.vertices, c.faces) for c in cads()]
    mesh = rs.randint(0, 3, 64)
    Ts = primitive_poses(rs, 64, H, W, f)
    a = _render(meshes, mesh, Ts, f, H, W)
    _assert_oracle(a, meshes, mesh, Ts, f, H, W)
    b = _render(meshes, mesh, Ts, f, H, W)
    assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))


def test_large_soup():
    """10^5 random triangles: the pose's face records cross hundreds of shared-memory chunks."""
    rs = np.random.RandomState(5)
    H, W = 480, 640
    f = 600.0
    V = 60000
    v = rs.uniform(-0.25, 0.25, (V, 3))
    centre = rs.randint(0, V, 100000)
    fc = np.stack([centre, (centre + rs.randint(1, 40, centre.size)) % V,
                   (centre + rs.randint(1, 40, centre.size)) % V], 1)
    v = v[np.argsort(v[:, 0])]             # neighbouring indices are nearby: small triangles
    Ts = [pose(t=(0, 0, 0.8)), pose(random_rotation(rs), (0.05, 0.02, 0.6))]
    got = _render([(v, fc)], [0, 0], Ts, f, H, W)
    _assert_oracle(got, [(v, fc)], [0, 0], Ts, f, H, W)
    assert got[2].min() > 1000


def _raw_call(L, args):
    return L.mf_render_cad(*args)


def test_bounds_and_bad_arguments():
    from morefusion_b200 import _lib
    L = _lib.lib()
    cad = cads()[2]
    v = torch.tensor(cad.vertices, device="cuda")
    fc = torch.tensor(cad.faces, device="cuda")
    N, H, W, G = 3, 33, 47, 4096
    off = np.array([0, len(cad.faces)], np.int64)
    rs = np.random.RandomState(3)
    Ts = torch.tensor(primitive_poses(rs, N, H, W, 40.0), device="cuda")
    mesh = torch.zeros(N, dtype=torch.int32, device="cuda")
    ws_bytes = L.mf_render_cad_workspace_bytes(N, len(cad.faces), H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    depth = torch.full((N * H * W + 2 * G,), 7.5, dtype=torch.float32, device="cuda")
    mask = torch.full((N * H * W + 2 * G,), 0xA5, dtype=torch.uint8, device="cuda")
    count = torch.full((N + 2 * G,), -7, dtype=torch.int32, device="cuda")
    p = lambda t, k=0: ctypes.c_void_p(t.data_ptr() + k * t.element_size())  # noqa: E731
    offp = off.ctypes.data_as(ctypes.c_void_p)

    def args(**kw):
        a = dict(vertices=p(v), V=len(cad.vertices), faces=p(fc), F=len(cad.faces), offsets=offp,
                 S=1, mesh=p(mesh), Ts=p(Ts), N=N, f=40.0, H=H, W=W, depth=p(depth, G),
                 mask=p(mask, G), count=p(count, G), ws=p(ws), ws_bytes=ws_bytes,
                 stream=_lib.stream())
        a.update(kw)
        return list(a.values())

    def untouched():
        torch.cuda.synchronize()
        return bool((depth == 7.5).all() and (mask == 0xA5).all() and (count == -7).all())

    bad_off = np.array([0, len(cad.faces) - 1], np.int64)
    dec_off = np.array([0, 5, 3, len(cad.faces)], np.int64)
    for kw, rc in [(dict(H=0), -1), (dict(W=-1), -1), (dict(H=1 << 15, W=1 << 15), -1),
                   (dict(N=-1), -1), (dict(F=-1), -1), (dict(V=-1), -1), (dict(S=0), -1),
                   (dict(offsets=None), -1),
                   (dict(offsets=bad_off.ctypes.data_as(ctypes.c_void_p)), -1),
                   (dict(offsets=dec_off.ctypes.data_as(ctypes.c_void_p), S=3), -1),
                   (dict(f=0.0), -1), (dict(f=float("nan")), -1), (dict(vertices=None), -1),
                   (dict(faces=None), -1), (dict(mesh=None), -1), (dict(Ts=None), -1),
                   (dict(depth=None), -1), (dict(mask=None), -1), (dict(count=None), -1),
                   (dict(ws=None), -1), (dict(ws_bytes=ws_bytes - 1), -3)]:
        assert _raw_call(L, args(**kw)) == rc, kw
        assert untouched(), kw
    assert _raw_call(L, args(N=0)) == 0 and untouched()
    # a face index outside [0, V) is rejected on the host before upload
    from morefusion_b200 import geometry
    with pytest.raises(ValueError):
        geometry.render_cad(cad.vertices, cad.faces + len(cad.vertices), np.eye(4), fovy=45,
                            height=H, width=W)
    assert _raw_call(L, args()) == 0
    torch.cuda.synchronize()
    for t, fill in ((depth, 7.5), (mask, 0xA5)):
        assert (t[:G] == fill).all() and (t[G + N * H * W:] == fill).all()
    assert (count[:G] == -7).all() and (count[G + N:] == -7).all()
    got = (depth[G:G + N * H * W].view(N, H, W).cpu().numpy(),
           mask[G:G + N * H * W].view(N, H, W).cpu().numpy().astype(bool), count[G:G + N].cpu().numpy())
    _assert_oracle(got, [(cad.vertices, cad.faces)], [0] * N, Ts.cpu().numpy(), 40.0, H, W)


def test_public_render_cad_numpy_and_cuda():
    from morefusion_b200 import geometry
    cad = cads()[1]
    rs = np.random.RandomState(9)
    H, W, fovy = 120, 160, 50.0
    f = orc.focal_from_fovy(fovy, H)
    Ts = primitive_poses(rs, 2, H, W, f)
    d, m = geometry.render_cad(cad.vertices, cad.faces, Ts[0], fovy=fovy, height=H, width=W)
    wd, wm, _ = orc.render_cad(cad.vertices, cad.faces, Ts[0], f, H, W)
    assert d.shape == (H, W) and m.dtype == bool
    assert np.array_equal(d.view(np.uint32), wd[0].view(np.uint32)) and np.array_equal(m, wm[0])
    d, m = geometry.render_cad(torch.tensor(cad.vertices, device="cuda"),
                               torch.tensor(cad.faces, device="cuda"),
                               torch.tensor(Ts, device="cuda"), fovy=fovy, height=H, width=W)
    wd, wm, _ = orc.render_cad(cad.vertices, cad.faces, Ts, f, H, W)
    assert d.is_cuda and d.shape == (2, H, W)
    assert np.array_equal(d.cpu().numpy().view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(m.cpu().numpy(), wm)


def _bits(t):
    return t.contiguous().view(torch.uint8)


@pytest.mark.parametrize("seed", [0, 3])
def test_get_example_visibility(seed):
    from morefusion_b200 import datasets, synthetic
    models = synthetic.SyntheticYCBModels()
    on = datasets.SyntheticRGBDPoseEstimationDataset(4, seed=seed, models=models, device="cuda",
                                                     with_visibility=True)
    off = datasets.SyntheticRGBDPoseEstimationDataset(4, seed=seed, models=models, device="cuda")
    for i in range(2):
        on.get_example(i), off.get_example(i)             # warm caches
        a, s_on = _syncs(lambda: on.get_example(i))
        b, s_off = _syncs(lambda: off.get_example(i))
        assert len(s_on) == len(s_off), (s_on, s_off)
        assert set(a) == set(b) | {"visibility"}
        for k in b:
            if k == "instance_ids":
                assert np.array_equal(a[k], b[k])
            else:
                assert torch.equal(_bits(a[k]), _bits(b[k])), k
        frame = on.get_frame(i)
        H, W = frame["instance_label"].shape
        f = orc.focal_from_fovy(orc.fovy_from_intrinsics(frame["intrinsic_matrix"][1, 1], H), H)
        want = []
        for iid, c in zip(a["instance_ids"], a["class_id"].cpu().numpy()):
            T = frame["Ts_cad2cam"][list(frame["instance_ids"]).index(iid)]
            cad = models.get_cad(c)
            count = orc.render_cad(cad.vertices, cad.faces, T, f, H, W)[2][0]
            n_mask = (frame["instance_label"] == iid).sum()
            with np.errstate(all="ignore"):
                want.append(np.float64(n_mask) / np.float64(count))
        got = a["visibility"].cpu().numpy()
        assert got.dtype == np.float64 and len(got) > 0
        assert np.array_equal(got.view(np.uint64), np.array(want).view(np.uint64))
        assert np.all(got > 0)
