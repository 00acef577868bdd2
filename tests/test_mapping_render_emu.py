"""CPU-only: the occupancy server's render and the instance boxes its scan keeps -- the kernels
k_map_server_boxes* and k_map_render_* of morefusion_b200/csrc/mapping.cu, executed serially on
the host (tests/emu/mapping_render_emu.cpp, g++ -DMF_HOST_EMU) through
``MultiInstanceOctreeMapping.integrate_scan`` / ``boxes`` / ``render`` -- bit for bit against
oracle/octomap_server_render.py, and that oracle's castRay against a float64 slab test.  The GPU
run is tests/test_mapping_render_gpu.py."""

import contextlib
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import octomap as oc
from oracle import octomap_server_render as osr
from test_mapping_node_grids_emu import assert_bitwise
from test_mapping_server_emu import pcd_of, pitch_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("integrate", "integrate_labelled", "update_points", "rehash", "integrate_server", "render")
F32 = np.float32
EMPTY = (np.full(3, osr.FLT_MAX, F32), np.full(3, -osr.FLT_MAX, F32))


def _build(tmp_path_factory, src, names, without_boxes=()):
    """ctypes adapters of the emulated entry points; those in `without_boxes` are the scan of
    tests/emu/mapping_server_emu.cpp, which takes neither tree_state nor boxes: their prototype
    and calls drop those two trailing arguments along with the stream."""
    so = str(tmp_path_factory.mktemp("emu") / (src + ".so"))
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17",
                    "-I" + os.path.join(ROOT, "tests", "emu"),
                    os.path.join(ROOT, "tests", "emu", src + ".cpp"), "-o", so], check=True)
    L = ctypes.CDLL(so)
    from morefusion_b200 import _lib

    class Adapter:
        pass
    a = Adapter()
    for name in names:
        res, args = _lib.SIGNATURES["mf_map_" + name]
        fn = getattr(L, "emu_map_" + name)
        fn.restype = res
        k = 3 if name in without_boxes else 1                    # no stream (nor boxes)
        fn.argtypes = args[:-k]
        setattr(a, "mf_map_" + name, (lambda f, k: (lambda *args: f(*args[:-k])))(fn, k))
    return a


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _build(tmp_path_factory, "mapping_render_emu", NAMES)


def _mapping_class(monkeypatch, lib):
    from morefusion_b200 import _lib
    from morefusion_b200.contrib.multi_instance_octree_mapping import MultiInstanceOctreeMapping
    from morefusion_b200.functions.geometry import _util
    monkeypatch.setattr(_lib, "lib", lambda: lib)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    monkeypatch.setattr(_lib, "require_cuda", lambda *a: None)
    monkeypatch.setattr(_util, "h2d", lambda x, device, dtype=None, tag="":
                        torch.as_tensor(np.asarray(x)).to(dtype))

    class EmuMapping(MultiInstanceOctreeMapping):           # host logic unchanged; no CUDA objects
        def __init__(self, capacity=1 << 16):
            super().__init__(device="cpu", capacity=capacity)

        def _dev_ctx(self):
            return contextlib.nullcontext()

        def _read_back(self):
            self._host_counters = self._counters.clone()

            class Done:
                def synchronize(self):
                    pass

                def query(self):
                    return True
            self._pending = Done()
    return EmuMapping


@pytest.fixture()
def Mapping(emu, monkeypatch):
    return _mapping_class(monkeypatch, emu)


class Pair:
    """The emulated device map and the oracle fed the same scans."""

    def __init__(self, Mapping, background_pitch=0.02):
        self.ours = Mapping()
        self.trees, self.centres, self.boxes = {}, {}, {}
        self.server_trees = set()                # ids whose tree the server would have created
        self.bp = background_pitch

    def scan(self, label, pcd, T, class_ids, max_range=-1.0):
        self.ours.integrate_scan(label, pcd, T, class_ids, max_range=max_range,
                                 background_pitch=self.bp)
        osr.insert_scan(self.trees, self.centres, self.boxes, self.server_trees, label, pcd, T,
                        class_ids,
                        pitch_of=pitch_of, max_range=max_range, background_pitch=self.bp)

    def check(self):
        for i, tree in self.trees.items():
            assert self.ours.cells(i) == tree.cells, i
        got = self.ours.centres()
        assert set(got) == set(self.centres)
        for i, c in self.centres.items():
            assert_bitwise(got[i], c)
        got = self.ours.boxes()
        assert set(got) == set(self.trees) - {-1}
        for i in got:
            want = self.boxes.get(i, osr.DEFAULT_BBX)
            assert_bitwise(got[i], np.stack(want))

    def render(self, pcd, T, K):
        label, depth = self.ours.render(pcd, T, K)
        want = osr.render(self.trees, self.boxes, pcd, T, K)
        assert label.dtype == torch.int32 and depth.dtype == torch.float32
        assert np.array_equal(label.numpy(), want[0])
        assert_bitwise(depth.numpy(), want[1])
        return want


def views(seed, n, H=60, W=80, n_objects=4):
    from morefusion_b200 import synthetic
    return synthetic.make_rgbd_views(seed, n, H=H, W=W, n_objects=n_objects)


# ------------------------------------------------------------------ the oracle's castRay
def _random_tree(seed, res=0.01, n=400):
    rs = np.random.RandomState(seed)
    tree = oc.OcTree(res)
    for _ in range(n):
        k = tuple(int(v) for v in TREE_CENTRE + rs.randint(-12, 13, 3))
        tree.cells[k] = F32(rs.choice([-1.0, -0.4, 0.0, 0.85, 2.0]))
    return tree


TREE_CENTRE = np.array([32768 + 20, 32768 - 7, 32768 + 30])


def _rays(tree, seed, n=400):
    rs = np.random.RandomState(seed)
    c = (TREE_CENTRE - 32768 + 0.5) * tree.resolution
    origin = (c + rs.uniform(-0.3, 0.3, 3)).astype(F32)
    d = (c + rs.uniform(-0.15, 0.15, (n, 3)) - origin).astype(F32)
    d[:8, 1:] = 0                                               # axis-parallel
    d[8] = 0                                                    # zero direction
    rng = np.sqrt(((d.astype(np.float64)) ** 2).sum(1)) * rs.choice([0.6, 1.1, 2.0], n)
    rng[9:12] = 0.0                                             # no limit: to a hit or the key range
    return origin, d, rng


def test_cast_rays_equals_cast_ray():
    """The lockstep castRay against the one-ray restatement, start-in-occupied cell included."""
    tree = _random_tree(0)
    for seed in range(2):
        origin, d, rng = _rays(tree, seed, n=200)
        hit, end = osr.cast_rays(tree, origin, d, rng)
        for n in range(len(d)):
            h, e = osr.cast_ray(tree, origin, d[n], rng[n])
            assert h == hit[n], n
            if h:
                assert_bitwise(end[n], e)
        assert 30 < hit.sum() < len(d) - 30
    k = tree.coords_to_key(origin.astype(np.float64))
    tree.cells[k] = F32(0.0)                                    # log-odds 0 is occupied
    hit, end = osr.cast_rays(tree, origin, d, rng)
    assert hit.all() and (end == np.float32([tree.key_to_coord(a) for a in k])).all()
    assert osr.cast_ray(tree, origin, d[8], 0.0)[0]


def _slab(tree, origin, u):
    """Entry / exit distance along the unit float64 direction u of every occupied cell."""
    keys = np.array([k for k, lo in tree.cells.items() if lo >= 0], np.int64)
    lo = (keys - 32768).astype(np.float64) * tree.resolution
    hi = lo + tree.resolution
    o = origin.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (lo - o) / u, (hi - o) / u
    inside = (o >= lo) & (o < hi)
    t1 = np.where(u == 0, np.where(inside, -np.inf, np.inf), t1)
    t2 = np.where(u == 0, np.where(inside, np.inf, -np.inf), t2)
    return keys, np.maximum(np.minimum(t1, t2).max(1), 0.0), np.maximum(t1, t2).min(1)


def test_cast_ray_against_float64_slab_test():
    """A float64 slab test of every occupied cell against the ray: the cell castRay returns is
    crossed, within maxRange of its centre, and no occupied cell is crossed clearly before it
    (rays whose competing entry distances lie within 1e-6 m of each other are skipped)."""
    tree = _random_tree(1, n=600)
    tol = 1e-9
    checked = hits = 0
    for seed in range(4):
        origin, d, rng = _rays(tree, 10 + seed, n=300)
        hit, end = osr.cast_rays(tree, origin, d, rng)
        for n in range(9, len(d)):
            u = d[n].astype(np.float64) / np.linalg.norm(d[n].astype(np.float64))
            keys, t_in, t_out = _slab(tree, origin, u)
            crossed = t_out - t_in > tol
            if hit[n]:
                k = np.array(tree.coords_to_key(end[n].astype(np.float64)))
                j = np.flatnonzero((keys == k).all(1))
                assert len(j) == 1 and crossed[j[0]], n
                if rng[n] > 0:
                    assert np.linalg.norm(end[n].astype(np.float64) - origin) <= rng[n] + 1e-6
                e0 = t_in[j[0]]
                earlier = crossed & (t_in < e0 - tol)
                if (crossed & (np.abs(t_in - e0) < 1e-6) & ~(keys == k).all(1)).any():
                    continue
                assert not earlier.any(), n
                hits += 1
            else:
                reach = rng[n] - 2 * tree.resolution if rng[n] > 0 else np.inf
                ahead = crossed & (t_out < reach)
                if (crossed & (np.abs(t_out - reach) < 1e-6)).any():
                    continue
                assert not ahead.any(), n
            checked += 1
    assert checked > 500 and hits > 100


# ------------------------------------------------------------------ boxes and render vs the oracle
@pytest.mark.parametrize("seed,max_range", [(0, -1.0), (1, 1.0)])
def test_multiview_boxes_and_render_match_oracle(Mapping, seed, max_range):
    """A multi-view sequence, rendered after every scan; the single-point instance of view 0
    gets the empty box, a listed instance seen only on odd pixels and one never seen keep the
    default box; points beyond max_range widen the boxes."""
    f = views(seed, 3)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    classes[77] = 5                                              # only ever on odd pixels
    classes[78] = 6                                              # listed, never seen
    pair = Pair(Mapping)
    peek = f["peek_id"]
    rendered, n_depth = set(), 0
    for k, v in enumerate(f["views"]):
        pcd = pcd_of(v, f["K"])
        label = v["label"].copy()
        label[1::2, 1::2][np.random.RandomState(k).rand(*label[1::2, 1::2].shape) < 0.05] = 77
        pair.scan(label, pcd, v["sensor_to_world"], classes, max_range=max_range)
        pair.check()
        if k == 0:
            assert_bitwise(pair.ours.boxes()[peek], np.stack(EMPTY))
        want = pair.render(pcd, v["sensor_to_world"], f["K"])
        rendered |= set(np.unique(want[0]).tolist())
        n_depth += int((~np.isnan(want[1])).sum())
    boxes = pair.ours.boxes()
    for i in (77, 78):
        assert_bitwise(boxes[i], np.zeros((2, 3), F32))
    assert set(f["instance_ids"].tolist()) <= rendered and n_depth > 20
    if max_range > 0:                    # some object point beyond max_range widened a box
        beyond = False
        for v in f["views"]:
            w = osr.transform_f32(v["sensor_to_world"].astype(F32), pcd_of(v, f["K"])[0::2, 0::2].reshape(-1, 3))
            o = v["sensor_to_world"][:3, 3].astype(F32)
            far = np.linalg.norm((w - o).astype(np.float64), axis=1) > max_range
            lab = v["label"][0::2, 0::2].reshape(-1)
            beyond |= bool((far & (lab > 0)).any())
        assert beyond


def test_instance_listed_before_it_is_seen(Mapping):
    """Every id is listed from view 0.  `late` is not in view 0's labels: the server creates its
    tree in view 1, where its box is its own pushed points alone (not their union with the
    default box).  `odd_first` is in view 0's labels on one odd pixel only: its tree is created
    there with no listed point, so it keeps the default box, which view 1 then widens."""
    f = views(3, 3)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    lab1 = f["views"][1]["label"][0::2, 0::2]
    ids = sorted((i for i in classes if i != f["peek_id"]), key=lambda i: -(lab1 == i).sum())
    late, odd_first = ids[:2]
    pair = Pair(Mapping)
    for k, v in enumerate(f["views"]):
        pcd = pcd_of(v, f["K"])
        label = v["label"].copy()
        if k == 0:
            label[np.isin(label, [late, odd_first])] = -2
            label[1, 1] = odd_first
        pair.scan(label, pcd, v["sensor_to_world"], classes)
        pair.check()
        pair.render(pcd, v["sensor_to_world"], f["K"])
        boxes = pair.ours.boxes()
        if k == 0:
            assert late not in pair.server_trees and odd_first in pair.server_trees
            for i in (late, odd_first):
                assert_bitwise(boxes[i], np.zeros((2, 3), F32))
        if k == 1:
            w = osr.transform_f32(v["sensor_to_world"].astype(F32), pcd[0::2, 0::2].reshape(-1, 3))
            pts = w[(label[0::2, 0::2].reshape(-1) == late) & ~np.isnan(w).any(1)][1:]
            assert len(pts) > 10
            assert_bitwise(boxes[late], np.stack([pts.min(0), pts.max(0)]))
            union = np.stack([np.minimum(pts.min(0), 0), np.maximum(pts.max(0), 0)])
            assert not np.array_equal(union, boxes[late])       # the default box would stretch it
            lo, hi = boxes[odd_first]
            assert (lo <= 0).all() and (hi >= 0).all()


def test_box_pass_leaves_cells_and_centres_unchanged(Mapping, tmp_path_factory, monkeypatch):
    """The same scans through the scan without its box pass (tests/emu/mapping_server_emu.cpp):
    the hash table and the centres are identical, bit for bit."""
    f = views(2, 3)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    ours = Mapping()
    plain_lib = _build(tmp_path_factory, "mapping_server_emu",
                       ("integrate", "integrate_labelled", "update_points", "rehash",
                        "integrate_server"), without_boxes=("integrate_server",))
    for v in f["views"]:
        ours.integrate_scan(v["label"], pcd_of(v, f["K"]), v["sensor_to_world"], classes,
                            max_range=0.9)
    monkeypatch.undo()
    plain = _mapping_class(monkeypatch, plain_lib)()
    for v in f["views"]:
        plain.integrate_scan(v["label"], pcd_of(v, f["K"]), v["sensor_to_world"], classes,
                             max_range=0.9)
    assert torch.equal(ours._cells, plain._cells)
    assert torch.equal(ours._centres, plain._centres)
    assert torch.equal(ours._centre_set, plain._centre_set)
    assert (plain._boxes == -(1 << 31)).all()                    # the scan alone boxes nothing
    assert not (ours._boxes[:len(ours._pitch)] == -(1 << 31)).all()


def _planes(H=21, W=25):
    """An organised cloud of two fronto-parallel planes (camera frame): z = 0.5 in the centre
    (the occluder), z = 0.8 elsewhere; and a third at z = 1.5 seen in a second frame."""
    K = np.array([[30.0, 0, W / 2 - 0.3], [0, 30.0, H / 2 + 0.2], [0, 0, 1]])
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    centre = (np.abs(u - W / 2) < W / 5) & (np.abs(v - H / 2) < H / 5)

    def cloud(z):
        z = np.broadcast_to(np.asarray(z, np.float64), u.shape)
        return np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], -1).astype(F32)
    return K, centre, cloud


def test_occluder_nan_pixels_and_odd_size(Mapping):
    """An occluder (id 5) in front of a target (id 3) with a farther object (id 9) behind both:
    pixels with no depth cast to 1.1 x the z = 1 point with no box test, so the nearer occluder
    wins over the target and the object at 1.5 m is never reached; odd H and W."""
    K, centre, cloud = _planes()
    T = np.eye(4)
    T[:3, 3] = [0.013, -0.02, 0.004]
    pair = Pair(Mapping)
    classes = {3: 2, 5: 3, 9: 4}
    far = np.full(centre.shape, 9, np.int32)
    pair.scan(far, np.full(centre.shape + (3,), 1.5, F32) * cloud(1.0), T, classes)
    pair.scan(np.full(centre.shape, 3, np.int32), cloud(np.full(centre.shape, 0.8)), T, classes)
    label = np.where(centre, 5, 3).astype(np.int32)
    pcd = cloud(np.where(centre, 0.5, 0.8))
    pair.scan(label, pcd, T, classes)
    pair.check()
    want = pair.render(pcd, T, K)
    assert (want[0][centre] == 5).mean() > 0.5 and (want[0] == 3).any()
    nodepth = np.full_like(pcd, np.nan)
    lab, dep = pair.render(nodepth, T, K)
    even = np.zeros(centre.shape, bool)
    even[0::2, 0::2] = True
    assert set(np.unique(lab).tolist()) <= {5, 3, -2} and (lab == 5).any() and (lab == 3).any()
    assert (dep[even & ~np.isnan(dep)] < 1.0).all()
    # depth pixels: the far object's box holds its points, so it is rendered there
    lab, _ = pair.render(np.full(centre.shape + (3,), 1.5, F32) * cloud(1.0), T, K)
    assert (lab == 9).any()


def test_empty_map_and_labels_only_instance(Mapping):
    """An empty map renders nothing; an instance added only through integrate_labels has the
    default box: its depth pixels are skipped, its rays from pixels without depth are cast."""
    K, centre, cloud = _planes()
    T = np.eye(4)
    pair = Pair(Mapping)
    lab, dep = pair.ours.render(cloud(np.full(centre.shape, 0.8)), T, K)
    assert (lab.numpy() == -2).all() and np.isnan(dep.numpy()).all()
    assert pair.render(cloud(np.full(centre.shape, 0.8)), T, K)[0].min() == -2
    pcd = cloud(np.where(centre, 0.5, 0.8))
    pair.ours.initialize(50, pitch=0.005)
    pair.trees[50] = oc.OcTree(0.005)
    pair.server_trees.add(50)                    # a tree made outside the server's scan
    lab50 = np.where(centre, 50, -99)
    pair.ours.integrate_labels(lab50, pcd)
    pair.trees[50].insertPointCloud(pcd[centre], origin=(0, 0, 0))
    assert list(pair.ours.boxes()) == [50]
    assert_bitwise(pair.ours.boxes()[50], np.zeros((2, 3), F32))
    lab, _ = pair.render(pcd, T, K)
    assert (lab == -2).all()                                      # every depth pixel fails inBBX
    lab, _ = pair.render(np.full_like(pcd, np.nan), T, K)
    assert (lab == 50).any()
    # a later scan widens the default box: the union holds the origin
    pair.scan(np.where(centre, 50, -1).astype(np.int32), pcd, T, {50: 2})
    pair.check()
    lo, hi = pair.ours.boxes()[50]
    assert (lo <= 0).all() and (hi >= 0).all()
    pair.render(pcd, T, K)


def test_exact_tie_goes_to_the_lower_instance_id(Mapping):
    """Two instances with the same cells: every hit is an exact tie in distance, and the lower
    instance id (4, created after 9) wins every pixel."""
    K, centre, cloud = _planes()
    T = np.eye(4)
    pair = Pair(Mapping)
    pts = cloud(np.full(centre.shape, 0.6)).reshape(-1, 3).astype(np.float64)
    for i in (9, 4):
        pair.ours.initialize(i, pitch=0.004)
        pair.ours.update(i, pts)
        pair.trees[i] = oc.OcTree(0.004)
        pair.server_trees.add(i)
        pair.trees[i].updateNodes(pts, True)
    assert pair.ours.cells(4) == pair.ours.cells(9)
    lab, dep = pair.render(np.full((centre.shape) + (3,), np.nan, F32), T, K)
    assert (lab == 4).sum() > 100 and not (lab == 9).any()


def test_render_argument_checks(Mapping):
    m = Mapping()
    with pytest.raises(ValueError, match="H,W,3"):
        m.render(np.zeros((4, 3), F32), np.eye(4), np.eye(3))
    with pytest.raises(ValueError, match="finite"):
        m.render(np.zeros((4, 4, 3), F32), np.eye(4), np.full((3, 3), np.nan))
    lab, dep = m.render(np.zeros((0, 4, 3), F32), np.eye(4), np.eye(3))
    assert lab.shape == (0, 4) and dep.shape == (0, 4)
