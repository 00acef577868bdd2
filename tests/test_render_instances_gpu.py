"""GPU: the scene render (csrc/render_cad.cu, mf_render_scene; ``geometry.render_instances`` /
``_render_instances_batch``) against mf_render_cad's per-object renders, bit for bit, and against
oracle/picking_order.py's composite; its edge cases and argument checks."""

import ctypes

import numpy as np
import pytest
import torch

from oracle import picking_order as opo
from oracle import render_cad as orc
from test_render_cad_emu import cads, pose, primitive_poses
from test_render_cad_gpu import _pack

pytestmark = pytest.mark.gpu
H, W = 480, 640
F_VGA = orc.focal_from_fovy(orc.fovy_from_intrinsics(1066.778, H), H)


def _scene(meshes, mesh, Ts, ids, f, height, width):
    from morefusion_b200 import geometry
    v, fc, off = _pack(meshes)
    out = geometry._render_instances_batch(v, fc, off, np.asarray(mesh, np.int32),
                                           np.asarray(Ts, np.float64).reshape(-1, 4, 4),
                                           np.asarray(ids, np.int32), f=f, height=height,
                                           width=width)
    return tuple(t.cpu().numpy() for t in out)


def _alone(meshes, mesh, Ts, f, height, width):
    from morefusion_b200 import geometry
    v, fc, off = _pack(meshes)
    d, m, c = geometry._render_cad_batch(v, fc, off, np.asarray(mesh, np.int32),
                                         np.asarray(Ts, np.float64).reshape(-1, 4, 4), f=f,
                                         height=height, width=width)
    return d.cpu().numpy(), m.cpu().numpy(), c.cpu().numpy()


def _assert_composite(got, alone, ids):
    """depth, ins, whole and occluded of the scene from the per-object renders of mf_render_cad."""
    depth, ins, whole, occluded = got
    d, m, c = alone
    N = len(ids)
    assert np.array_equal(whole, c)
    best = np.full(depth.shape, np.inf, np.float32)
    idx = np.full(depth.shape, -1, np.int64)
    for n in range(N):
        better = m[n] & ((idx < 0) | (d[n] < best))
        best[better] = d[n][better]
        idx[better] = n
    want_depth = np.where(idx >= 0, best, np.float32(np.nan)).astype(np.float32)
    assert np.array_equal(depth.view(np.uint32), want_depth.view(np.uint32))
    want_ins = np.where(idx >= 0, np.asarray(ids)[np.maximum(idx, 0)] if N else -1, -1)
    assert np.array_equal(ins, want_ins)
    want_occ = np.zeros((N, N), np.int64)
    for i in range(N):
        for j in range(N):
            if i != j:
                want_occ[i, j] = (m[i] & (ins == ids[j])).sum()
    assert np.array_equal(occluded, want_occ)
    assert not np.diag(occluded).any()
    return idx


@pytest.mark.parametrize("N", [1, 8, 32, 64])
def test_scene_equals_per_object_renders(N):
    rs = np.random.RandomState(N)
    meshes = [(c.vertices, c.faces) for c in cads()]
    mesh = rs.randint(0, 3, N)
    Ts = primitive_poses(rs, N, H, W, F_VGA)
    Ts[:, 0, 3] *= 0.4                                   # crowd the centre: real overlaps
    Ts[:, 1, 3] *= 0.4
    ids = rs.permutation(1000)[:N] + 3
    got = _scene(meshes, mesh, Ts, ids, F_VGA, H, W)
    _assert_composite(got, _alone(meshes, mesh, Ts, F_VGA, H, W), ids)
    if N >= 8:
        assert got[3].sum() > 0
    again = _scene(meshes, mesh, Ts, ids, F_VGA, H, W)
    assert all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
               for a, b in zip(got, again))


@pytest.mark.parametrize("name", sorted(opo.CASES))
def test_scene_equals_oracle(name):
    from morefusion_b200 import synthetic
    meshes, T, ids, f, h, w = opo.case_scene(name, synthetic.SyntheticYCBModels())
    got = _scene(meshes, np.arange(len(meshes)), T, ids, f, h, w)
    wd, wi, ww, wo, _ = opo.render_instances(meshes, T, ids, f, h, w)
    assert np.array_equal(got[0].view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(got[1], wi)
    assert np.array_equal(got[2], ww) and np.array_equal(got[3], wo)


def test_edge_cases():
    cad = cads()[0]
    meshes = [(cad.vertices, cad.faces)]
    h, w, f = 60, 80, 70.0
    # the same mesh twice at the same pose: the later object is never visible
    got = _scene(meshes, [0, 0], [pose(), pose()], [4, 2], f, h, w)
    _assert_composite(got, _alone(meshes, [0, 0], [pose(), pose()], f, h, w), [4, 2])
    depth, ins, whole, occ = got
    assert whole[1] > 0 and not (ins == 2).any() and occ[1, 0] == whole[1] and occ[0, 1] == 0
    # wholly in front of the near plane (every Z < 0.01: the cylinder's half height is 0.077), behind
    # the camera, wholly outside the image, straddling the near plane, and a visible one
    Ts = [pose(t=(0, 0, -0.07)), pose(t=(0, 0, -0.5)), pose(t=(50, 0, 1)), pose(t=(0.05, 0, 0.3)),
          pose(t=(-0.05, 0, 0.02))]
    got = _scene(meshes, [0] * 5, Ts, [1, 2, 3, 4, 5], f, h, w)
    _assert_composite(got, _alone(meshes, [0] * 5, Ts, f, h, w), [1, 2, 3, 4, 5])
    assert got[2][:3].tolist() == [0, 0, 0] and got[2][3] > 0
    assert not (np.isin(got[1], [1, 2, 3])).any() and (got[1] == 4).any()
    # N = 0 still writes one image
    depth, ins, whole, occ = _scene(meshes, np.zeros(0, np.int32), np.zeros((0, 4, 4)),
                                    np.zeros(0, np.int32), f, h, w)
    assert np.isnan(depth).all() and (ins == -1).all() and whole.shape == (0,)
    assert occ.shape == (0, 0)


def test_bad_arguments():
    from morefusion_b200 import _lib
    L = _lib.lib()
    cad = cads()[2]
    v = torch.tensor(cad.vertices, device="cuda")
    fc = torch.tensor(cad.faces, device="cuda")
    N, h, w = 65, 33, 47
    off = np.array([0, len(cad.faces)], np.int64)
    rs = np.random.RandomState(3)
    Ts = torch.tensor(primitive_poses(rs, N, h, w, 40.0), device="cuda")
    mesh = torch.zeros(N, dtype=torch.int32, device="cuda")
    ids = torch.arange(N, dtype=torch.int32, device="cuda")
    ws_bytes = L.mf_render_cad_workspace_bytes(N, len(cad.faces), h, w)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    depth = torch.full((h * w,), 7.5, dtype=torch.float32, device="cuda")
    ins = torch.full((h * w,), -7, dtype=torch.int32, device="cuda")
    whole = torch.full((N,), -7, dtype=torch.int32, device="cuda")
    occ = torch.full((N * N,), -7, dtype=torch.int32, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    offp = off.ctypes.data_as(ctypes.c_void_p)

    def call(**kw):
        a = dict(vertices=p(v), V=len(cad.vertices), faces=p(fc), F=len(cad.faces), offsets=offp,
                 S=1, mesh=p(mesh), Ts=p(Ts), ids=p(ids), N=8, f=40.0, H=h, W=w, depth=p(depth),
                 ins=p(ins), whole=p(whole), occ=p(occ), ws=p(ws), ws_bytes=ws_bytes,
                 stream=_lib.stream())
        a.update(kw)
        return L.mf_render_scene(*a.values())

    def untouched():
        torch.cuda.synchronize()
        return bool((depth == 7.5).all() and (ins == -7).all() and (whole == -7).all()
                    and (occ == -7).all())

    bad_off = np.array([0, len(cad.faces) - 1], np.int64)
    for kw, rc in [(dict(N=65), -4), (dict(N=1000), -4), (dict(H=0), -1), (dict(W=-1), -1),
                   (dict(H=1 << 15, W=1 << 15), -1), (dict(N=-1), -1), (dict(F=-1), -1),
                   (dict(V=-1), -1), (dict(S=0), -1), (dict(offsets=None), -1),
                   (dict(offsets=bad_off.ctypes.data_as(ctypes.c_void_p)), -1),
                   (dict(f=0.0), -1), (dict(f=float("nan")), -1), (dict(vertices=None), -1),
                   (dict(faces=None), -1), (dict(mesh=None), -1), (dict(Ts=None), -1),
                   (dict(ids=None), -1), (dict(depth=None), -1), (dict(ins=None), -1),
                   (dict(whole=None), -1), (dict(occ=None), -1), (dict(ws=None), -1),
                   (dict(ws_bytes=L.mf_render_cad_workspace_bytes(8, len(cad.faces), h, w) - 1),
                    -3)]:
        assert call(**kw) == rc, kw
        assert untouched(), kw
    assert call(N=64) == 0
    torch.cuda.synchronize()
    got = (depth.view(h, w).cpu().numpy(), ins.view(h, w).cpu().numpy(),
           whole[:64].cpu().numpy(), occ[:64 * 64].view(64, 64).cpu().numpy())
    assert (whole[64:] == -7).all() and (occ[64 * 64:] == -7).all()
    _assert_composite(got, _alone([(cad.vertices, cad.faces)], [0] * 64, Ts[:64].cpu().numpy(),
                                  40.0, h, w), list(range(64)))
    # the public op rejects what the kernel cannot take, on the host
    from morefusion_b200 import geometry
    with pytest.raises(ValueError):
        geometry.render_instances([cad] * 65, Ts.cpu().numpy(), range(65), fovy=45, height=h,
                                  width=w)
    for bad in ([1, 1], [-1, 2], [0, 1 << 31], [0.5, 1]):
        with pytest.raises(ValueError):
            geometry.render_instances([cad] * 2, Ts[:2].cpu().numpy(), np.asarray(bad), fovy=45,
                                      height=h, width=w)


def test_public_render_instances_numpy_and_cuda():
    from morefusion_b200 import geometry
    from morefusion_b200 import synthetic
    models = synthetic.SyntheticYCBModels()
    rs = np.random.RandomState(11)
    cls = [1, 5, 1, 3, 5, 3]
    cs = [models.get_cad(c) for c in cls]                 # identical meshes are packed once
    h, w, fovy = 120, 160, 50.0
    f = orc.focal_from_fovy(fovy, h)
    Ts = primitive_poses(rs, len(cls), h, w, f)
    ids = np.array([9, 4, 17, 2, 30, 5])
    v, fc, off, mesh = geometry._pack_cads(cs)
    assert len(off) == 4 and mesh.tolist() == [0, 1, 0, 2, 1, 2]
    wd, wi, _, _, _ = opo.render_instances([(c.vertices, c.faces) for c in cs], Ts, ids, f, h, w)
    d, ins = geometry.render_instances(cs, Ts, ids, fovy=fovy, height=h, width=w)
    assert isinstance(d, np.ndarray) and d.shape == (h, w) and ins.dtype == np.int32
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)) and np.array_equal(ins, wi)
    T_cuda = torch.tensor(Ts, device="cuda")
    geometry.render_instances(cs, T_cuda, ids, fovy=fovy, height=h, width=w)    # warm up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        d, ins = geometry.render_instances(cs, T_cuda, ids, fovy=fovy, height=h, width=w)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert d.is_cuda and ins.is_cuda
    assert np.array_equal(d.cpu().numpy().view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ins.cpu().numpy(), wi)
