"""CPU-only: oracle/octomap_batch.py (the dataset rules of oracle/octomap.py in bulk, the
restatement tests/test_mapping_frames_gpu.py compares full frames with) against
oracle/octomap.py's OcTree and MultiInstanceOctreeMapping, cell for cell and grid for grid, bit
for bit.  oracle/octomap.py is itself pinned to the reference's code
(test_oracle_golden.py::test_octree_mapping_oracle_equals_reference_code_over_it)."""

import collections

import numpy as np
import pytest

from oracle import octomap as oc
from oracle import octomap_batch as ob
from oracle import octomap_server_multiview as osv
from test_mapping_emu import make_scene, scans_for


def assert_same_cells(got, want):
    """Two {(kx, ky, kz): float32 log-odds} dicts: the same keys, the same bits."""
    assert set(got) == set(want), (len(got), len(want), len(set(got) ^ set(want)))
    a = np.array([got[k] for k in want], np.float32)
    b = np.array(list(want.values()), np.float32)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def assert_same_maps(fast, ref):
    assert fast.instance_ids == ref.instance_ids
    for ins in ref.instance_ids:
        assert_same_cells(fast.cells(ins), ref._octrees[ins].cells)
    assert fast.n_cells() == sum(len(t.cells) for t in ref._octrees.values())


def assert_same_grids(fast, ref, targets, dimensions, pitches, origins):
    got = fast.get_target_grids_batch(targets, dimensions=dimensions, pitches=pitches,
                                      origins=origins)
    for t, (tid, p, o) in enumerate(zip(targets, pitches, origins)):
        want = ref.get_target_grids(tid, dimensions=dimensions, pitch=p, origin=o)
        for g, w in zip(got, want):
            assert g[t].dtype == w.dtype == np.float32
            assert np.array_equal(g[t].view(np.uint32), w.view(np.uint32))
    return got


def pair(pitches):
    fast, ref = ob.MultiInstanceOctreeMapping(), oc.MultiInstanceOctreeMapping()
    for ins, p in pitches.items():
        fast.initialize(ins, pitch=p)
        ref.initialize(ins, pitch=p)
    return fast, ref


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_small_scans_equal_octree(seed):
    """The scans of test_mapping_emu.py (two frames, a shifted sensor origin, three pitches)."""
    fast, ref = pair({3: 0.008, 7: 0.011, 0: 0.02})
    for ins, mask, pcd, origin in scans_for(seed):
        fast.integrate(ins, mask, pcd, origin)
        ref.integrate(ins, mask, pcd, origin)
    assert_same_maps(fast, ref)
    assert fast.n_cells() > 1500
    pcd, fg = make_scene(seed)
    c = np.nanmedian(pcd[fg], axis=0)
    g = assert_same_grids(fast, ref, [3, 7, 0, 3], (16, 16, 16), [0.008, 0.011, 0.02, 0.005],
                          [c - 7.5 * 0.008, c - 7.5 * 0.011, c - 7.5 * 0.02, c - 7.5 * 0.005])
    assert (g[0] > 0).sum() > 20 and (g[1] > 0).sum() > 20 and (g[2] > 0).sum() > 100
    # a non-cubic grid, voxel centres on the key borders of instance 3 and past the mapped region
    o = np.round(c / 0.008) * 0.008 - 3 * 0.008
    assert_same_grids(fast, ref, [3, 7], (6, 9, 40), [0.008, 0.011], [o, o + [0, 0, 0.1]])


def test_strided_sample_of_a_full_frame():
    """A few thousand rays of a 640x480 make_depth_frame frame, at the class pitches and the
    background's, in two scans per instance (the second one from a shifted origin)."""
    from morefusion_b200 import synthetic
    pcd, label, _, pitches = synthetic.make_depth_frame(0)
    ids = [2, 5, 0]
    fast, ref = pair({i: pitches[i] for i in ids})
    sample = np.zeros(label.shape, bool)
    sample.reshape(-1)[::97] = True
    org = np.float32([0.02, -0.013, 0.031])
    for o, shift in ((np.zeros(3), 0), (org, 1)):
        cloud = np.roll(pcd, shift, axis=1) + o.astype(np.float32)
        for ins in ids:
            m = sample & (np.roll(label, shift, axis=1) == ins)
            fast.integrate(ins, m, cloud, o)
            ref.integrate(ins, m, cloud, o)
    assert sample.sum() > 3000
    assert_same_maps(fast, ref)
    tids = [2, 5]
    origins = [np.nanmedian(pcd[label == t], axis=0) - 15.5 * pitches[t] for t in tids]
    assert_same_grids(fast, ref, tids, (32, 32, 32), [pitches[t] for t in tids], origins)


def test_hand_built_rays():
    """An end in the origin's cell, ends and an origin outside the key range, NaN, an origin
    exactly on cell borders (of both pitches), negative coordinates; and the ray counts of
    ``ray_keys`` against computeRayKeys ray by ray."""
    rs = np.random.RandomState(7)
    on_border = np.float32([0.25, -0.5, 0.75])              # x / 0.01 and x / 0.0125 are integers
    ends = (on_border + rs.uniform(-0.3, 0.3, (300, 3))).astype(np.float32)
    ends[:8] = on_border + np.float32([0.001, 0.002, 0.003])         # in the origin's cell
    ends[8:16, 1:] = on_border[1:]                                   # along x only
    ends[16] = [700.0, 0.0, 0.0]                                     # outside the key range
    ends[17] = [np.nan, 0.1, 0.2]
    ends[18] = on_border                                             # zero-length ray
    ends[19:30] = -rs.uniform(0.01, 0.4, (11, 3))                    # every coordinate negative
    fast, ref = pair({1: 0.01, 2: 0.0125})
    scans = [(on_border, ends), (np.float32([-0.137, -0.291, -0.05]), ends[::-1]),
             (np.float32([-1000.0, 0.0, 0.0]), ends[:40]),          # origin outside the key range
             (np.zeros(3, np.float32), ends[19:40])]
    for origin, e in scans:
        for ins in (1, 2):
            fast._trees[ins].insertPointCloud(e, origin)
            ref._octrees[ins].insertPointCloud(e, origin)
    assert_same_maps(fast, ref)
    for res in (0.01, 0.0125):
        tree = oc.OcTree(res)
        want = collections.Counter()
        for e in ends:
            want.update(tree.computeRayKeys(on_border, e) or [])
        keys, counts = osv.ray_keys(tree, on_border, ends, counts=True)
        got = dict(zip(ob.unpack(keys), counts.tolist()))
        assert got == dict(want) and max(got.values()) > 50
        assert np.array_equal(keys, osv.ray_keys(tree, on_border, ends))


def test_update_nodes_with_duplicates_reaching_the_clamp():
    fast, ref = pair({3: 0.008, 7: 0.011, 0: 0.02})
    for ins, mask, pcd, origin in scans_for(1)[:2]:
        fast.integrate(ins, mask, pcd, origin)
        ref.integrate(ins, mask, pcd, origin)
    rs = np.random.RandomState(5)
    free = [k for k, v in ref._octrees[3].cells.items() if v < 0][:50]
    centres = np.array([[ref._octrees[3].key_to_coord(a) for a in k] for k in free])
    occupied = np.concatenate([
        rs.uniform(-0.05, 0.05, (2000, 3)) + [0, 0, 0.4],
        np.repeat([[0.001, 0.002, 0.4]], 9, 0),                      # 9 hits on one cell: clamps
        np.repeat(centres[:5], 3, 0),                                # free cells hit back
        centres[5:],
        [[np.nan, 0, 0], [1e9, 0, 0], [0.0, -1e12, 0.0]]])
    occupied = occupied[rs.permutation(len(occupied))]
    fast.update(3, occupied)
    ref.update(3, occupied)
    assert_same_maps(fast, ref)
    lo = np.array(list(ref._octrees[3].cells.values()), np.float32)
    assert (lo == ref._octrees[3].clamping_thres_max).any()
