"""GPU: the occupancy map's dataset-rule path (csrc/mapping.cu: k_map_scan_hits,
k_map_scan_free<ScanParams>, k_map_update_*, k_map_query_grids, k_map_rehash) cell for cell
against the OctoMap restatement, at the sizes its callers run: 640x480 frames of 8 instances and
a background, integrated frame after frame into one map, as bench.py's bench_mapping and the
frame path (FramePoseEstimator: integrate_labels, get_target_grids_batch) do.

The restatement is oracle/octomap_batch.py, pinned bit for bit to oracle/octomap.py by
tests/test_octomap_batch.py.  Every comparison is exact: the same key set per instance and the
same float32 log-odds bits, the same grid bits.  At full frame every scan's rays start in the
same few cells at the camera, so the once-per-scan stamp of map_scan_update is contended hardest
there; the report printed by the fixture says how hard (run with -s to see it)."""

import multiprocessing
import os
import time
import types

import numpy as np
import pytest
import torch

from oracle import frame as of
from oracle import octomap_batch as ob

pytestmark = pytest.mark.gpu
D = 32
N_FRAMES = 6                              # bench_mapping's frames (seeds 0-5)
CHECKED = (1, 2, 6)                       # frames after which the map is compared


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.time()
    yield
    print(f"\n[test_mapping_frames_gpu] wall time {time.time() - t0:.1f} s")


@pytest.fixture(scope="module")
def pool(cuda_device):
    """Worker processes for the restatement's ray walks (spawned: they never touch CUDA)."""
    n = max(1, min(16, len(os.sched_getaffinity(0))))
    with multiprocessing.get_context("spawn").Pool(n) as p:
        yield p


@pytest.fixture(scope="module")
def bench(pool):
    """bench_mapping's workload restated: frames of make_depth_frame(0..5), every instance at
    the pitches bench_mapping initialises them with (those make_depth_frame returns for its last
    frame), one insertPointCloud per instance and frame.  Snapshots after the CHECKED frames, the
    keys of frame 1's scans (for the controls) and per-scan statistics."""
    from morefusion_b200 import synthetic
    t0 = time.time()
    made = [synthetic.make_depth_frame(seed=s) for s in range(N_FRAMES)]
    frames = [(pcd, label) for pcd, label, _, _ in made]
    pitches = made[-1][3]
    ids = sorted(i for i in pitches if i != 0) + [0]      # foreground instances, then background
    R = ob.MultiInstanceOctreeMapping(pool)
    for ins in ids:
        R.initialize(ins, pitch=pitches[ins])
    snaps, scan1, stats = {}, {}, []
    for f, (pcd, label) in enumerate(frames, 1):
        nonnan = ~np.isnan(pcd).any(axis=2)
        for ins in ids:
            tree = R._trees[ins]
            pts = pcd[(label == ins) & nonnan]
            free, rays, occ = tree.scan_keys(pts, np.zeros(3), pool=pool)
            tree.apply_scan(free, occ)
            if f == 1:
                scan1[ins] = (free, rays, occ)
            stats.append(dict(frame=f, ins=ins, rays=len(pts), free=len(free), hits=len(occ),
                              max_rays=int(rays.max(initial=0)),
                              max_rays_not_origin=int(np.sort(rays)[-2]) if len(rays) > 1 else 0))
        if f in CHECKED:
            snaps[f] = R.copy()
    R6 = snaps[N_FRAMES]
    lo = np.concatenate([t.lo for t in R6._trees.values()])
    t = R6._trees[0].octree
    n_max, n_min = int((lo == t.clamping_thres_max).sum()), int((lo == t.clamping_thres_min).sum())
    bg = [s for s in stats if s["ins"] == 0]
    print(f"\n[bench workload] {N_FRAMES} frames x {len(ids)} scans, "
          f"{sum(s['rays'] for s in stats) // N_FRAMES} rays per frame "
          f"({bg[0]['rays']} in the background scan); cells after frames "
          + ", ".join(f"{f}: {snaps[f].n_cells()}" for f in CHECKED)
          + f"; frame {N_FRAMES}: {n_max} cells at clamping_thres_max, {n_min} at "
          f"clamping_thres_min; largest number of rays through one cell in a scan "
          f"{max(s['max_rays'] for s in stats)} (the origin's cell; next largest "
          f"{max(s['max_rays_not_origin'] for s in stats)}); distinct cells freed by one "
          f"background scan {bg[0]['free']}; restated in {time.time() - t0:.1f} s")
    return types.SimpleNamespace(frames=frames, pitches=pitches, ids=ids, snaps=snaps,
                                 scan1=scan1, n_clamped=(n_max, n_min))


# ------------------------------------------------------------------------------------ helpers
def mapping(ids, pitches, **kw):
    from morefusion_b200.contrib import MultiInstanceOctreeMapping
    m = MultiInstanceOctreeMapping(**kw)
    for ins in ids:
        m.initialize(ins, pitch=pitches[ins])
    return m


def device_frames(frames):
    return [(torch.as_tensor(pcd, device="cuda"), torch.as_tensor(label, device="cuda"))
            for pcd, label in frames]


def device_cells(m):
    """{instance_id: (sorted packed keys, float32 log-odds)} of the device map, one table read."""
    c = m._cells.cpu()
    keys = c[:, 0].numpy()
    lo = c.view(torch.float32)[:, 2].numpy()
    sel = keys != -1
    keys, lo = keys[sel], lo[sel]
    inst = (keys >> 48) & 0xFFFF
    out = {}
    for ins, q in m._ids.items():
        s = inst == q
        k, v = keys[s] & 0xFFFFFFFFFFFF, lo[s]
        o = np.argsort(k)
        out[ins] = (k[o], v[o])
    return out


def differences(m, R):
    """{instance_id: (keys only on the device, keys only restated, keys whose bits differ)}."""
    got = device_cells(m)
    out = {}
    for ins in R.instance_ids:
        k, v = got[ins]
        t = R._trees[ins]
        only_dev = np.setdiff1d(k, t.keys, assume_unique=True)
        only_ref = np.setdiff1d(t.keys, k, assume_unique=True)
        both, i, j = np.intersect1d(k, t.keys, assume_unique=True, return_indices=True)
        bad = both[v[i].view(np.uint32) != t.lo[j].view(np.uint32)]
        if len(only_dev) or len(only_ref) or len(bad):
            out[ins] = (only_dev, only_ref, bad, got[ins], t)
    return out


def assert_map_equal(m, R, what):
    diff = differences(m, R)
    lines = []
    for ins, (only_dev, only_ref, bad, (k, v), t) in diff.items():
        lines.append(f"instance {ins}: {len(only_dev)} cells only on the device, {len(only_ref)} "
                     f"only restated, {len(bad)} with other log-odds")
        for key in bad[:5]:
            a, b = v[np.searchsorted(k, key)], t.lo[np.searchsorted(t.keys, key)]
            lines.append(f"  key {ob.unpack([key])[0]}: device {a!r}, restated {b!r}")
        for key in only_dev[:3]:
            lines.append(f"  key {ob.unpack([key])[0]} only on the device: "
                         f"{v[np.searchsorted(k, key)]!r}")
        for key in only_ref[:3]:
            lines.append(f"  key {ob.unpack([key])[0]} only restated: "
                         f"{t.lo[np.searchsorted(t.keys, key)]!r}")
    assert not lines, what + ":\n" + "\n".join(lines)
    assert m.n_cells() == R.n_cells(), (what, m.n_cells(), R.n_cells())


def assert_bitwise(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype == np.float32 and a.shape == b.shape
    n = int((a.view(np.uint32) != b.view(np.uint32)).sum())
    assert n == 0, f"{n} voxels differ"


# ------------------------------------------------------------------------------------- tests
def test_bench_frames_nine_integrate_calls(bench):
    """bench_mapping's calls: 9 integrate() calls per frame, device inputs, one map."""
    m = mapping(bench.ids, bench.pitches)
    cap0 = m._cap
    for f, (pcd, lab) in enumerate(device_frames(bench.frames), 1):
        for ins in bench.ids:
            m.integrate(ins, lab == ins, pcd)
        if f in CHECKED:
            assert_map_equal(m, bench.snaps[f], f"after frame {f}")
        if f == 1:                                  # the public accessor, every instance
            for ins in bench.ids:
                want = bench.snaps[1].cells(ins)
                got = m.cells(ins)
                assert set(got) == set(want), ins
                assert all(got[k].view(np.uint32) == want[k].view(np.uint32) for k in want), ins
    n_max, n_min = bench.n_clamped
    # six seeds do put five hits into one cell, and five misses
    assert n_max > 0 and n_min > 0
    print(f"\n[integrate x9] {m.n_cells()} cells, table {cap0} -> {m._cap} slots")


def test_bench_frames_labelled(bench):
    """The frame path's call: one integrate_labels per frame."""
    m = mapping(bench.ids, bench.pitches)
    for f, (pcd, lab) in enumerate(device_frames(bench.frames), 1):
        m.integrate_labels(lab, pcd)
        if f in CHECKED:
            assert_map_equal(m, bench.snaps[f], f"after frame {f}")


def test_growth_mid_frame(bench):
    """A table a quarter full or more after frame 1: k_map_rehash runs inside the next
    integrate_labels, before its scan."""
    n1 = bench.snaps[1].n_cells()
    cap = 1 << int(np.ceil(np.log2(2 * n1)))          # frame 1 fills it to between 1/4 and 1/2
    m = mapping(bench.ids, bench.pitches, capacity=cap)
    caps = [cap]
    for f, (pcd, lab) in enumerate(device_frames(bench.frames), 1):
        torch.cuda.synchronize()                      # the growth decision sees frame f - 1
        m.integrate_labels(lab, pcd)
        caps.append(m._cap)
        if f in CHECKED:
            assert_map_equal(m, bench.snaps[f], f"after frame {f}")
    assert caps[2] > caps[1] == cap
    print(f"\n[growth] table slots per frame {caps}: {int(np.log(caps[-1] / cap) / np.log(4))} "
          f"growths")


@pytest.mark.parametrize("origin", [(0.25, -0.5, 0.75), (-0.6131, -0.4729, -1.7343)],
                         ids=["on_cell_borders", "negative"])
def test_sensor_origin_off_zero(bench, pool, origin):
    """integrate(..., origin=o) with the cloud shifted by o.  (0.25, -0.5, 0.75) lies exactly on
    cell borders of the background's 0.01 m key space; the other puts every coordinate below 0."""
    o = np.asarray(origin)
    pcd, label = bench.frames[0]
    cloud = pcd + o.astype(np.float32)
    R = ob.MultiInstanceOctreeMapping(pool)
    for ins in bench.ids:
        R.initialize(ins, pitch=bench.pitches[ins])
        R.integrate(ins, label == ins, cloud, o)
    m = mapping(bench.ids, bench.pitches)
    cd, ld = torch.as_tensor(cloud, device="cuda"), torch.as_tensor(label, device="cuda")
    for ins in bench.ids:
        m.integrate(ins, ld == ins, cd, origin=o)
    assert_map_equal(m, R, f"origin {origin}")


def test_update_at_scale(bench):
    """update() of ~200k float64 rows after six frames: existing cells hit back (free ones
    included), new cells, one row 60 times (clamps), a NaN row and rows outside the key range."""
    ins = 5
    R = bench.snaps[N_FRAMES].copy()
    tree = R._trees[ins]
    res = tree.resolution
    xyz = np.stack([(tree.keys >> 32) & 0xFFFF, (tree.keys >> 16) & 0xFFFF, tree.keys & 0xFFFF], 1)
    centres = ((xyz - 32768).astype(np.float64) + 0.5) * res
    rs = np.random.RandomState(0)
    lo, hi = centres.min(0) - 2 * res, centres.max(0) + 2 * res
    rows = np.concatenate([
        rs.uniform(lo, hi, (150000, 3)),
        centres[rs.randint(0, len(centres), 50000)],                      # duplicates as they come
        np.repeat(centres[np.argmin(tree.lo)][None], 60, 0),             # a free cell, to the clamp
        [[np.nan, 0.0, 0.5], [1e9, 0.0, 0.5], [0.0, 0.0, -1e12]]])
    rows = rows[rs.permutation(len(rows))]
    m = mapping(bench.ids, bench.pitches)
    for pcd, lab in device_frames(bench.frames):
        m.integrate_labels(lab, pcd)
    before = R.n_cells()
    m.update(ins, rows)
    R.update(ins, rows)
    assert_map_equal(m, R, "after update")
    assert R.n_cells() > before and len(rows) > 200000
    assert (R._trees[ins].lo == tree.octree.clamping_thres_max).sum() > 100


def test_target_grids_batch(bench):
    """8 targets at 32^3 on the six-frame map: origins as FramePoseEstimator sets them, the
    same moved so that voxel centres land on the targets' key borders, and one target whose grid
    reaches past the mapped region."""
    m = mapping(bench.ids, bench.pitches)
    for pcd, lab in device_frames(bench.frames):
        m.integrate_labels(lab, pcd)
    R = bench.snaps[N_FRAMES]
    pcd, label = bench.frames[-1]
    tids = bench.ids[:-1]
    p = np.array([bench.pitches[t] for t in tids], np.float64)
    med = np.stack([np.nanmedian(pcd[label == t], axis=0) for t in tids]).astype(np.float64)
    plain = med - 15.5 * p[:, None]
    border = np.round(plain / p[:, None]) * p[:, None]
    far = plain.copy()
    far[-1] += [0.05, 0.0, 0.40]                         # its back half lies behind the table
    idx = np.arange(D, dtype=np.float64)
    f = (idx[None, :, None] * p[:, None, None] + border[:, None, :]) / p[:, None, None]
    on = np.abs(f - np.round(f)) < 1e-9
    assert on.mean() > 0.5                               # most voxel coordinates sit on a border
    for name, origins in (("plain", plain), ("on key borders", border), ("past the map", far)):
        got = m.get_target_grids_batch(tids, dimensions=(D, D, D), pitches=p, origins=origins)
        want = R.get_target_grids_batch(tids, dimensions=(D, D, D), pitches=p, origins=origins)
        for g, w in zip(got, want):
            assert_bitwise(g.cpu().numpy(), w)
        assert (want[0] > 0).sum() > 1000 and (want[2] > 0).sum() > 10000, name
    unknown = (want[0][-1] == 0) & (want[1][-1] == 0) & (want[2][-1] == 0)
    assert unknown.sum() > 1000 and (~unknown).sum() > 1000


def test_frame_estimator_examples(pool):
    """FramePoseEstimator.examples on make_rgbd_frame(0): its map, cell for cell, and its
    grid_nontarget_empty against the grids of the restatement's map of the same point image."""
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib.singleview_3d import FramePoseEstimator
    from morefusion_b200.contrib.singleview_3d.models import Model
    from test_frame_gpu import _frame_cuda, _pcd
    f = synthetic.make_rgbd_frame(0)
    torch.manual_seed(0)
    est = FramePoseEstimator(Model(n_fg_class=21, with_occupancy=True).cuda().eval())
    fc = _frame_cuda(f)
    ex = est.examples(**fc)
    pcd = _pcd(f["depth"], f["K"])
    R = of.build_octomap(ob.MultiInstanceOctreeMapping(pool), pcd.cpu().numpy(), f["label"],
                         list(f["instance_ids"]), f["class_ids"],
                         lambda c: est.model._models.get_voxel_pitch(D, c))
    assert_map_equal(est.build_map(pcd, fc["label"], f["instance_ids"], f["class_ids"]), R,
                     "FramePoseEstimator.build_map")
    grids = R.get_target_grids_batch(list(ex["instance_ids"]), dimensions=(D, D, D),
                                     pitches=ex["pitch"].cpu().numpy(),
                                     origins=ex["origin"].cpu().numpy().astype(np.float64))
    want = of.combine_grids(*grids)
    got = ex["grid_nontarget_empty"].cpu().numpy()
    assert got.shape == want.shape and len(ex["instance_ids"]) == 7
    assert np.array_equal(got, want) and want.any()


def test_controls_break_the_comparison(bench):
    """The frames exercise both per-scan rules: a restatement that frees a cell once per ray
    instead of once per scan, and one that also frees the scan's hit cells, each differ from the
    device's frame-1 map."""
    m = mapping(bench.ids, bench.pitches)
    pcd, lab = device_frames(bench.frames[:1])[0]
    for ins in bench.ids:
        m.integrate(ins, lab == ins, pcd)
    assert_map_equal(m, bench.snaps[1], "after frame 1")
    per_ray, hits_freed = ob.MultiInstanceOctreeMapping(), ob.MultiInstanceOctreeMapping()
    for ins in bench.ids:
        per_ray.initialize(ins, pitch=bench.pitches[ins])
        hits_freed.initialize(ins, pitch=bench.pitches[ins])
        free, rays, occ = bench.scan1[ins]
        t = per_ray._trees[ins]
        miss = ~np.isin(free, occ)
        t.apply(free[miss], t.octree.prob_miss_log, rays[miss])
        t.apply(occ, t.octree.prob_hit_log)
        t = hits_freed._trees[ins]
        t.apply(free, t.octree.prob_miss_log)
        t.apply(occ, t.octree.prob_hit_log)
    report = []
    for name, R in (("once per ray", per_ray), ("hits not removed from free", hits_freed)):
        diff = differences(m, R)
        n = sum(len(d[2]) + len(d[0]) + len(d[1]) for d in diff.values())
        report.append(f"{name}: {n} cells differ")
        assert n > 0, name
    print("\n[controls] " + "; ".join(report))
