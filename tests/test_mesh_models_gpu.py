"""GPU: csrc/mesh_models.cu (``geometry.voxelize_solid``, ``geometry.signed_distance`` and
``datasets.MeshModels``) bit for bit against oracle/mesh_models.py, batched against per-mesh
calls and run against run, and MeshModels driving the ICC refinement end to end."""

import warnings

import numpy as np
import pytest
import torch

import _mesh_cases as mc
from oracle import icp as oicp
from oracle import mesh_models as omm

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def synthetic_meshes():
    from morefusion_b200 import synthetic
    m = synthetic.SyntheticYCBModels()
    return {c: (m.get_cad(c).vertices, m.get_cad(c).faces) for c in range(1, 22)}


def assert_grid(got, want):
    assert np.array_equal(got.matrix, want["matrix"])
    assert np.array_equal(bits(got.points), bits(want["points"]))
    assert np.array_equal(bits(got.translate), bits(want["translate"]))
    assert bits(got.pitch) == bits(want["pitch"]) and bits(got.scale) == bits(want["scale"])


def test_synthetic_classes_match_oracle():
    from morefusion_b200 import geometry
    for c, (v, f) in synthetic_meshes().items():
        assert_grid(geometry.voxelize_solid(v, f), omm.voxelize_solid(v, f, 64))
        p = mc.sample_points(v, f, 300, seed=c)
        assert np.array_equal(bits(geometry.signed_distance(v, f, p)),
                              bits(omm.signed_distance(v, f, p)[0]))


@pytest.mark.parametrize("name", sorted(mc.all_cases()))
def test_cases_match_oracle(name):
    from morefusion_b200 import geometry
    v, f = mc.all_cases()[name]
    for D in (16, 64, 128) if name == "torus" else (64,):
        assert_grid(geometry.voxelize_solid(v, f, D), omm.voxelize_solid(v, f, D))
    p = mc.sample_points(v, f, 1000, seed=1)
    assert np.array_equal(bits(geometry.signed_distance(v, f, p)),
                          bits(omm.signed_distance(v, f, p)[0]))


def test_large_mesh_sampled():
    # 81,920 faces: the grid in full, the SDF on a sample of points (both against the oracle)
    from morefusion_b200 import geometry
    v, f = mc.icosphere(6)
    assert len(f) >= 50000
    assert_grid(geometry.voxelize_solid(v, f, 32), omm.voxelize_solid(v, f, 32))
    p = mc.sample_points(v, f, 2000, seed=2)
    sdf = geometry.signed_distance(v, f, p)
    rs = np.random.RandomState(0)
    sel = rs.choice(len(p), 96, replace=False)
    assert np.array_equal(bits(sdf[sel]), bits(omm.signed_distance(v, f, p[sel])[0]))
    # a sphere of radius r: |sdf| is close to | r - |p| | and the sign agrees away from the surface
    r = np.linalg.norm(p, axis=1)
    far = np.abs(r - 0.05) > 1e-3
    assert (np.sign(sdf[far]) == np.sign(0.05 - r[far])).all()


def test_batched_equals_per_mesh_and_repeatable():
    from morefusion_b200 import geometry
    meshes = list(synthetic_meshes().values())[:5] + list(mc.all_cases().values())
    v, fc, off = geometry._pack_meshes(meshes)
    dv = torch.as_tensor(v, device="cuda")
    df = torch.as_tensor(fc, device="cuda")
    runs = [geometry._voxelize_solid_batch(dv, df, off, 48) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a, b) if a.dtype != torch.float64 else \
            np.array_equal(bits(a.cpu().numpy()), bits(b.cpu().numpy()))
    matrix, counts, points = runs[0][0].cpu().numpy(), runs[0][1].cpu().numpy(), runs[0][2].cpu().numpy()
    pts, tags = [], []
    for s, (vs, fs) in enumerate(meshes):
        one = geometry.voxelize_solid(vs, fs, 48)
        assert np.array_equal(matrix[s], one.matrix)
        assert np.array_equal(bits(points[s, :counts[s]]), bits(one.points))
        assert np.isnan(points[s, counts[s]:]).all()
        p = mc.sample_points(vs, fs, 400, seed=s)
        pts.append(p)
        tags.append(np.full(len(p), s, np.int32))
    P = np.concatenate(pts)
    T = np.concatenate(tags)
    rs = np.random.RandomState(0)
    perm = rs.permutation(len(P))                     # interleaved meshes within a CTA
    dP, dT = torch.as_tensor(P[perm], device="cuda"), torch.as_tensor(T[perm], device="cuda")
    out = [geometry._signed_distance_batch(dv, df, off, dP, dT) for _ in range(2)]
    assert np.array_equal(bits(out[0][0].cpu().numpy()), bits(out[1][0].cpu().numpy()))
    assert torch.equal(out[0][1], out[1][1])
    sdf = np.empty(len(P))
    sdf[perm] = out[0][0].cpu().numpy()
    face = np.empty(len(P), np.int64)
    face[perm] = out[0][1].cpu().numpy()
    for s, (vs, fs) in enumerate(meshes):
        sel = T == s
        assert np.array_equal(bits(sdf[sel]), bits(geometry.signed_distance(vs, fs, P[sel])))
        want, arg = omm.signed_distance(vs, fs, P[sel])
        assert np.array_equal(bits(sdf[sel]), bits(want)) and np.array_equal(face[sel], arg + off[s])


def test_cuda_in_cuda_out():
    from morefusion_b200 import geometry
    v, f = mc.torus()
    g = geometry.voxelize_solid(torch.as_tensor(v, device="cuda"), torch.as_tensor(f, device="cuda"))
    assert g.matrix.is_cuda and g.points.is_cuda and g.translate.is_cuda
    assert_grid(type("G", (), dict(matrix=g.matrix.cpu().numpy(), points=g.points.cpu().numpy(),
                                   translate=g.translate.cpu().numpy(), pitch=g.pitch,
                                   scale=g.scale)), omm.voxelize_solid(v, f, 64))
    p = torch.as_tensor(mc.sample_points(v, f, 100), device="cuda")
    d = geometry.signed_distance(torch.as_tensor(v, device="cuda"), f, p)
    assert d.is_cuda
    assert np.array_equal(bits(d.cpu().numpy()), bits(omm.signed_distance(v, f, p.cpu().numpy())[0]))


def test_value_errors():
    from morefusion_b200 import geometry
    v, f = mc.torus()
    bad = [(v, np.zeros((0, 3), np.int32)), (v, f + len(v)), (v, -f - 1),
           (np.where(np.arange(len(v))[:, None] == 3, np.nan, v), f),
           (np.zeros_like(v), f), (v, f.astype(np.float64))]
    for vv, ff in bad:
        with pytest.raises(ValueError):
            geometry.voxelize_solid(vv, ff)
        with pytest.raises(ValueError):
            geometry.signed_distance(vv, ff, np.zeros((2, 3)))
    for D in (0, 129):
        with pytest.raises(ValueError):
            geometry.voxelize_solid(v, f, D)


def test_mesh_models_composition():
    # get_sdf: the grid's points down-sampled at get_voxel_pitch(32), then signed_distance
    from morefusion_b200.datasets import MeshModels
    from morefusion_b200 import synthetic
    meshes = synthetic_meshes()
    sm = synthetic.SyntheticYCBModels()
    models = MeshModels(meshes, {c: sm.get_pcd(c) for c in meshes}, sm.class_ids_symmetric)
    models.prepare(list(meshes))
    for c in (1, 2, 3, 13):
        v, f = meshes[c]
        want_pts, want_sdf = omm.get_sdf(v, f)
        pts, sdf = models.get_sdf(c)
        assert pts.dtype == np.float64 and sdf.dtype == np.float64
        assert np.array_equal(bits(pts), bits(want_pts)) and np.array_equal(bits(sdf), bits(want_sdf))
        grid = models.get_solid_voxel_grid(c)
        assert_grid(grid, omm.voxelize_solid(v, f, 64))
        assert np.array_equal(bits(pts), bits(oicp.voxel_down_sample(grid.points,
                                                                     models.get_voxel_pitch(32, c))))
        # the class pitch agrees with the synthetic stand-in's (its diagonal is 32 pitches)
        assert np.isclose(models.get_voxel_pitch(32, c), sm.get_voxel_pitch(32, c), rtol=1e-12)
        assert (sdf > 0).mean() > 0.5


def test_refine_with_mesh_models():
    """MeshModels from the synthetic meshes in place of the synthetic stand-in: the frame-level
    ICC refinement runs with finite poses, the loss falls, and refine() reads the host once."""
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib import IterativeCollisionCheckLink
    from morefusion_b200.contrib.singleview_3d import FramePoseEstimator
    from morefusion_b200.contrib.singleview_3d.models import Model
    from morefusion_b200.datasets import MeshModels
    torch.manual_seed(0)
    model = Model(n_fg_class=21, with_occupancy=True).cuda()
    model.load_reference_weights(synthetic.init_weights(21, seed=1))
    model.eval()
    sm = model._models
    meshes = synthetic_meshes()
    model._models = MeshModels(meshes, {c: sm.get_pcd(c) for c in meshes}, sm.class_ids_symmetric)
    est = FramePoseEstimator(model)
    f = synthetic.make_rgbd_frame(0)
    from morefusion_b200 import geometry
    pcd = geometry.pointcloud_from_depth(torch.as_tensor(f["depth"], device="cuda"), f["K"][0, 0],
                                         f["K"][1, 1], f["K"][0, 2], f["K"][1, 2])
    label = torch.as_tensor(f["label"], device="cuda")
    mapping = est.build_map(pcd, label, f["instance_ids"], f["class_ids"])
    fc = dict(rgb=torch.as_tensor(f["rgb"], device="cuda"), depth=torch.as_tensor(f["depth"], device="cuda"),
              K=f["K"], label=label, instance_ids=f["instance_ids"], class_ids=f["class_ids"])
    ex = est.examples(**fc, mapping=mapping)
    ids = ex["instance_ids"]
    cls = ex["class_id"].cpu().numpy()
    rs = np.random.RandomState(0)
    M = len(ids)
    q = rs.randn(M, 4)
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    pitch = ex["pitch"].cpu().numpy()
    t = (ex["origin"].cpu().numpy() + (32 / 2 - 0.5) * pitch[:, None]
         + rs.uniform(-0.01, 0.01, (M, 3))).astype(np.float32)
    est.refine(mapping, ids, cls, q, t, ex["origin"])                   # builds the SDFs once
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            qr, tr, n_run = est.refine(mapping, ids, cls, q, t, ex["origin"])
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "called a synchronizing CUDA operation" in str(x.message)]
    assert len(syncs) <= 1, [str(x.message) for x in syncs]
    assert np.isfinite(qr).all() and np.isfinite(tr).all() and n_run >= 1
    assert not np.array_equal(tr, t)
    # the loss of the same problem falls over the iterations
    pitch64 = est._pitch_table[cls]
    grid, gne = mapping.get_noentry_grids_batch(
        ids.tolist(), dimensions=(32, 32, 32), pitches=torch.as_tensor(pitch64, device="cuda"),
        origins=ex["origin"].to(torch.float64), background_id=0)
    link = IterativeCollisionCheckLink(geometry.transformation_matrix(q, t)).cuda()
    sdf = [model._models.get_sdf(int(c)) for c in cls]
    loss = link.refine([s[0] for s in sdf], [s[1] for s in sdf],
                       torch.as_tensor(pitch64.astype(np.float32), device="cuda"),
                       ex["origin"].to(torch.float32), grid, gne, n_iter=30).cpu().numpy()
    loss = loss[np.isfinite(loss)]
    assert len(loss) > 1 and loss[-1] < loss[0], loss
