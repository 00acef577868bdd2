"""GPU: point-to-point ICP (csrc/icp.cu) against the float64 restatement (oracle/icp.py) where its
kernels change path: voxel keys of 0 to 4 radix bytes per axis, sources on both sides of the
shared-memory limit (RUN_SMEM_POINTS = 4096), the cell list read back directly, a seed sweep, the
Horn solve through the kernel at the conditioning of tests/test_icp_emu.py, and the stop-rule,
far-query and key-overflow edges.  Every comparison has a wrong reference that must fail.  The
scene builders are in this file; the print-out gives the worst err / bound of each check."""

import numpy as np
import pytest
import torch

import test_icp_emu as te
from oracle import icp as oi

pytestmark = pytest.mark.gpu

VOXEL = 0.01
KEY_MAX = 2 ** 31 - 2


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _vds(x, voxel):
    from morefusion_b200.contrib.icp_registration import voxel_down_sample
    return [t.cpu().numpy() for t in voxel_down_sample(x, voxel)]


_DIFFER = [0]


def _passes(kmax):
    """Radix passes k_icp_sort runs for an axis whose largest key is kmax."""
    return next(b for b in range(5) if kmax >> (8 * b) == 0)


def _check_vds(clouds, voxel, shape=None):
    """Down-sample clouds (numpy [M,N,3], float32 or float64, non-finite rows allowed) and compare
    with the oracle on the finite rows: n, keys, counts exactly, means bitwise.  Returns the
    per-axis largest keys of each cloud."""
    x = torch.as_tensor(clouds, device="cuda")
    if shape is not None:
        x = x.reshape(shape)
    means, keys, counts, n = _vds(x, voxel)
    kmax = []
    for m, c in enumerate(clouds):
        c = c.reshape(-1, 3)
        fin = c[np.isfinite(c).all(1)]
        want, wkeys, wcounts = oi.voxel_down_sample(fin, voxel, return_counts=True)
        V = len(want)
        assert n[m] == V, (m, n[m], V)
        assert np.array_equal(keys[m, :V], wkeys) and np.array_equal(counts[m, :V], wcounts), m
        assert np.array_equal(_bits(means[m, :V]), _bits(want)), m
        # control: the sums taken in reverse row order are not always the same bits
        if V == 0:
            kmax.append(np.zeros(3, np.int64))
            continue
        _, inv = np.unique(oi.voxel_keys(fin, voxel)[0], axis=0, return_inverse=True)
        rev = np.zeros((V, 3))
        np.add.at(rev, inv.reshape(-1)[::-1], fin[::-1].astype(np.float64))
        _DIFFER[0] += int((_bits(rev / wcounts[:, None]) != _bits(means[m, :V])).any(1).sum())
        kmax.append(wkeys.max(0))
    return np.array(kmax)


def _byte_clouds(dtype, rs):
    """Two clouds of a 1 mm voxel whose keys need 0, 1, 2 (cloud 0) and 3, 4, 0 (cloud 1) radix
    passes on x, y, z: a dense 4 cm cluster with far outliers on the long axes, NaN and +-inf
    rows interleaved."""
    v = 2.0 ** -10
    out = []
    for ext in ((0.0, 0.2, 25.0), (1500.0, 20000.0, 0.0)):
        c = rs.uniform(0, 0.04, (3000, 3))
        for a in range(3):
            if ext[a] == 0.0:
                c[:, a] = 0.5
        far = np.zeros((6, 3)) + 0.02
        for a in range(3):
            if ext[a] > 0:
                far[:, a] = rs.uniform(0, ext[a], 6)
                far[0, a] = ext[a]
            else:
                far[:, a] = 0.5
        c = np.concatenate([c, far])
        c = c[rs.permutation(len(c))]
        bad = rs.choice(len(c), 200, replace=False)
        c[bad[:80], rs.randint(0, 3, 80)] = np.nan
        c[bad[80:140], rs.randint(0, 3, 60)] = np.inf
        c[bad[140:], rs.randint(0, 3, 60)] = -np.inf
        out.append(c)
    return np.stack(out).astype(dtype), v


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_voxel_down_sample_multi_byte_keys(dtype):
    rs = np.random.RandomState(0)
    clouds, v = _byte_clouds(dtype, rs)
    kmax = _check_vds(clouds, v)
    passes = [[_passes(int(k)) for k in km] for km in kmax]
    assert passes == [[0, 1, 2], [3, 4, 0]], (passes, kmax)
    # [M,H,W,3] input gives the same
    _check_vds(clouds, v, shape=(2, 18, 167, 3))
    print("kmax per axis:", kmax.tolist(), "passes:", passes)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_voxel_down_sample_sizes_and_edges(dtype):
    rs = np.random.RandomState(1)
    for N in (1, 511, 512, 513):
        c = rs.uniform(-0.1, 0.1, (3, N, 3))
        c[1, ::3, 1] = np.nan                       # NaN rows interleaved
        c[2] = np.nan                               # every row non-finite: n = 0
        if N > 1:
            c[2, -1, 0] = 0.0
            c[2, -1, 1:] = np.inf
        _check_vds(c.astype(dtype), VOXEL)
    # a 256^2 crop, every row finite
    crop = (rs.uniform(-0.15, 0.15, (2, 256, 256, 3)) + [0, 0, 0.7]).astype(dtype)
    _check_vds(crop.reshape(2, -1, 3), VOXEL, shape=(2, 256, 256, 3))
    # every point in one voxel; points on the faces of a dyadic voxel
    one = np.full((1, 700, 3), 0.3) + rs.uniform(0, 0.004, (1, 700, 3))
    _, _, counts, n = _vds(torch.as_tensor(one.astype(dtype), device="cuda"), VOXEL)
    assert n[0] == 1 and counts[0, 0] == 700
    _check_vds(one.astype(dtype), VOXEL)
    # float64 rows: the row-order sum is pinned, the reverse-order sum is other bits
    _DIFFER[0] = 0
    _check_vds(one, VOXEL)
    assert _DIFFER[0] == 1
    h = 2.0 ** -7
    faces = rs.randint(0, 8, (1, 4000, 3)) * (h / 2)   # on faces, centres and corners
    kmax = _check_vds(faces.astype(dtype), h)
    assert (kmax[0] == 4).all()


def test_voxel_down_sample_640x480():
    rs = np.random.RandomState(2)
    frame = rs.uniform(-0.4, 0.4, (1, 480, 640, 3)).astype(np.float32) + np.float32([0, 0, 1])
    frame[0, ::7, ::5] = np.nan
    _check_vds(frame.reshape(1, -1, 3), VOXEL, shape=(1, 480, 640, 3))


def test_key_overflow_is_refused():
    """A cloud spanning 2^31 - 1 voxels or more on an axis would merge voxels at the clamp; it is
    refused: n = -1, and register_batch gives that instance NaN and 0 iterations while the other
    instance is unchanged."""
    from morefusion_b200.contrib.icp_registration import ICPRegistration, ICPTarget, register_batch
    rs = np.random.RandomState(3)
    v = 2.0 ** -10
    ok = rs.uniform(0, 0.1, (400, 3))
    ok[1] = 0.0                                       # min_bound = -v / 2 on every axis
    huge = ok.copy()
    huge[0, 1] = (2.0 ** 31 + 8) * v                   # key 2^31 + 7 on y
    edge = ok.copy()
    edge[0, 1] = KEY_MAX * v - 0.25 * v                # the largest key that fits
    x = torch.as_tensor(np.stack([ok, huge, edge]), device="cuda")
    _, keys, _, n = _vds(x, v)
    assert n[1] == -1 and n[0] > 0
    assert keys[2, :n[2], 1].max() == KEY_MAX
    _check_vds(np.stack([ok, edge]), v)
    tgt = ICPTarget(ok, v, 2 * v)
    T, fit, rmse, it = [t.cpu().numpy() for t in register_batch(
        x[:2], [tgt, tgt], np.stack([np.eye(4)] * 2), voxel_size=v, max_iteration=5)]
    assert np.isnan(T[1]).all() and np.isnan(fit[1]) and np.isnan(rmse[1]) and it[1] == 0
    one = [t.cpu().numpy() for t in register_batch(x[:1], [tgt], np.eye(4)[None], voxel_size=v,
                                                    max_iteration=5)]
    for a, b in zip((T, fit, rmse, it), one):
        assert np.array_equal(a[:1], b)
    # a refused target: every instance registered to it is refused
    bad = ICPTarget(huge, v, 2 * v)
    T2, fit2, _, it2 = [t.cpu().numpy() for t in register_batch(x[:1], [bad], np.eye(4)[None],
                                                                voxel_size=v)]
    assert np.isnan(T2).all() and it2[0] == 0
    with pytest.raises(ValueError):
        ICPRegistration(huge, ok).register(voxel_size=v)


# ------------------------------------------------------------------------------- cell list

def _cell_list_oracle(points, h):
    keys, origin = oi.voxel_keys(points, h)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    return points[order], keys[order], order, origin


def _cell_list(points, n, h):
    from morefusion_b200 import _lib
    from morefusion_b200.functions.geometry import _util
    p = torch.as_tensor(np.ascontiguousarray(points, np.float64), device="cuda")
    N = p.shape[0]
    nd = torch.tensor([n], dtype=torch.int32, device="cuda")
    sp = torch.full((N, 3), np.nan, dtype=torch.float64, device="cuda")
    cells = torch.full((N, 3), -7, dtype=torch.int32, device="cuda")
    index = torch.full((N,), -7, dtype=torch.int32, device="cuda")
    origin = torch.empty(3, dtype=torch.float64, device="cuda")
    L = _lib.lib()
    nb = L.mf_icp_sort_workspace_bytes(1, N)
    ws = _util.workspace(nb, p.device)
    _lib.check(L.mf_icp_cell_list(_lib.ptr(p), _lib.ptr(nd), N, float(h), _lib.ptr(sp),
                                  _lib.ptr(cells), _lib.ptr(index), _lib.ptr(origin), _lib.ptr(ws),
                                  nb, _lib.stream()), "cell list")
    return [t.cpu().numpy() for t in (sp, cells, index, origin)]


def test_cell_list_matches_oracle():
    from morefusion_b200 import synthetic
    rs = np.random.RandomState(4)
    cad = synthetic.SyntheticYCBModels().get_pcd(5).astype(np.float64)
    big = np.concatenate([cad, cad * 40 + 3.0, rs.uniform(-30, 30, (500, 3))])
    most = 0
    for pts, n, h in ((cad, len(cad), 0.02), (cad, len(cad) - 37, 0.02), (big, len(big), 2.0 ** -12),
                      (big, len(big) - 1000, 2.0 ** -12), (cad[:1], 1, 0.02)):
        p = pts.copy()
        if n < len(p):
            p[n:] = np.nan                         # rows past the device count are never read
        sp, cells, index, origin = _cell_list(p, n, h)
        wp, wk, wo, worig = _cell_list_oracle(p[:n], h)
        assert np.array_equal(_bits(sp[:n]), _bits(wp)) and np.array_equal(cells[:n], wk)
        assert np.array_equal(index[:n], wo) and np.array_equal(_bits(origin), _bits(worig))
        assert (index[n:] == -7).all()
        most = max(most, max(_passes(int(k)) for k in wk.max(0)))
        # control: ties in reverse row order differ wherever equal keys exist
        if len(np.unique(wk, axis=0)) < n:
            unstable = np.lexsort((-np.arange(n), wk[:, 2], wk[:, 1], wk[:, 0]))
            assert not np.array_equal(index[:n], unstable)
    assert most >= 3


# ----------------------------------------------------------- register_batch path boundaries

def _surface(x, y):
    return 0.06 * np.sin(3.1 * x + 0.4) * np.cos(2.3 * y) + 0.03 * np.sin(7.0 * x * y)


def _rigid(rs, deg, t):
    T = np.eye(4)
    T[:3, :3] = te._axis_angle(rs.normal(size=3), np.deg2rad(deg))
    T[:3, 3] = rs.normal(size=3) / np.sqrt(3) * t
    return T


def plane_instance(n, seed):
    """A source of exactly n voxels at 1 cm (one jittered point per cell of a bumpy sheet; the
    first point, unjittered, puts min_bound on the cell corners), its target a denser sample of
    the same sheet moved by a true pose, and an init 2 mm / 1 degree off it."""
    rs = np.random.RandomState(seed)
    side = int(np.ceil(np.sqrt(n)))
    ij = np.stack(np.meshgrid(np.arange(side), np.arange(side), indexing="ij"), -1).reshape(-1, 2)[:n]
    jit = rs.uniform(0.05, 0.4, ij.shape)
    jit[0] = 0.0
    xy = (ij + 0.5 + jit) * VOXEL
    src = np.c_[xy, _surface(xy[:, 0], xy[:, 1]) * 0.2]
    dense = rs.uniform(0, side * VOXEL, (3 * n, 2))
    T_true = _rigid(rs, 10, 0.05)
    tgt = oi.transform(T_true, np.c_[dense, _surface(dense[:, 0], dense[:, 1]) * 0.2])
    init = T_true @ np.linalg.inv(_rigid(rs, 1, 0.002))
    return src, tgt, init


def _oracle(src, tgt, init, voxel=VOXEL, r=None, max_iteration=100, **kw):
    return oi.registration_icp_point_to_point(oi.voxel_down_sample(src, voxel),
                                              oi.voxel_down_sample(tgt, voxel),
                                              2 * voxel if r is None else r, init,
                                              max_iteration=max_iteration, **kw)


def _well_posed(res, margin=1e-9):
    return all(min(v, default=np.inf) > margin for v in res["margins"].values())


def _register(srcs, tgts, inits, dtype=np.float64, voxel=VOXEL, **kw):
    from morefusion_b200.contrib.icp_registration import ICPTarget, register_batch
    N = max(len(s) for s in srcs)
    x = np.full((len(srcs), N, 3), np.nan, dtype)
    for i, s in enumerate(srcs):
        x[i, :len(s)] = s
    r = kw.pop("max_distance", 2 * voxel)
    targets = [ICPTarget(t, voxel, r) for t in tgts]
    out = register_batch(torch.as_tensor(x, device="cuda"), targets, np.stack(inits),
                         voxel_size=voxel, max_distance=r, **kw)
    return [t.cpu().numpy() for t in out]


def _compare(res, T, fit, rmse, it, worst):
    assert it == res["iterations"] and fit == res["fitness"]
    err = np.abs(T - res["transformation"]).max()
    assert err <= 1e-9, err
    assert abs(rmse - res["inlier_rmse"]) <= 1e-9 * res["inlier_rmse"]
    worst[0] = max(worst[0], err / 1e-9)


# sources of n voxels and the seeds of their scenes, whose oracle margins all exceed 1e-9
SIZES = {4095: 4105, 4096: 4106, 4097: 4107, 10000: 1}


def test_register_across_shared_memory_limit():
    insts = {n: plane_instance(n, seed) for n, seed in SIZES.items()}
    res = {n: _oracle(*insts[n]) for n in SIZES}
    worst = [0.0]
    for n in SIZES:
        src, tgt, init = insts[n]
        assert len(oi.voxel_down_sample(src, VOXEL)) == n
        assert _well_posed(res[n]), (n, {k: min(v) for k, v in res[n]["margins"].items()})
        T, fit, rmse, it = _register([src], [tgt], [init])
        _compare(res[n], T[0], fit[0], rmse[0], it[0], worst)
        assert it[0] > 1
        # control: the oracle one iteration short differs
        short = _oracle(src, tgt, init, max_iteration=res[n]["iterations"] - 1)
        assert np.abs(T[0] - short["transformation"]).max() > 1e-9
    # a mixed batch, permuted: bitwise the single runs and a repeat
    order = [2, 3, 0, 1]
    srcs = [insts[list(SIZES)[k]][0] for k in order]
    tgts = [insts[list(SIZES)[k]][1] for k in order]
    inits = [insts[list(SIZES)[k]][2] for k in order]
    batch = _register(srcs, tgts, inits)
    again = _register(srcs, tgts, inits)
    for a, b in zip(batch, again):
        assert np.array_equal(a, b)
    for i, k in enumerate(order):
        one = _register([srcs[i]], [tgts[i]], [inits[i]])
        for a, b in zip(batch, one):
            assert np.array_equal(a[i], b[0]), (list(SIZES)[k], i)
    print(f"shared-memory boundary: worst |dT| / 1e-9 = {worst[0]:.3g}")


# ---------------------------------------------------------------------------- seed sweep

@pytest.mark.parametrize("M,seeds", [(8, range(100, 116)), (32, range(200, 204))])
def test_seed_sweep(M, seeds):
    from morefusion_b200 import synthetic
    worst, compared, total = [0.0], 0, 0
    for seed in seeds:
        s = synthetic.make_icp_scene(M, seed)
        init = np.linalg.inv(s["transform_init"])
        res = [_oracle(d, c, T0, max_iteration=100) for d, c, T0 in zip(s["pcd_depth"], s["pcd_cad"], init)]
        runs = [_register(s["pcd_depth"], s["pcd_cad"], init, dtype=dt) for dt in (np.float32, np.float64)]
        for a, b in zip(*runs):
            assert np.array_equal(a, b)                   # float32 and float64 sources alike
        T, fit, rmse, it = runs[0]
        for i, r in enumerate(res):
            total += 1
            if not _well_posed(r):
                continue
            compared += 1
            _compare(r, T[i], fit[i], rmse[i], it[i], worst)
    assert compared >= 0.75 * total, (compared, total)
    print(f"seed sweep M={M}: compared {compared}/{total}, worst |dT| / 1e-9 = {worst[0]:.3g}")


# ------------------------------------------------------------------- Horn through the kernel

def horn_instances(rs):
    """(family, source [K,3], target [K,3]) with well-separated points whose partners are exact
    transforms (or reflections), matched within r = 0.45 m at init = I: distinct z 1 m apart and
    small x, y, or a 1 m grid moved by a few degrees."""
    out = []
    for eps in (1e-3, 1e-6, 0.0):                         # near 180 degrees about ~z
        for _ in range(4):
            K = 6
            src = np.c_[rs.uniform(-0.05, 0.05, (K, 2)), np.arange(K) - 2.5]
            ax = np.array([0.0, 0.0, 1.0]) + rs.normal(size=3) * 1e-3
            R = te._axis_angle(ax, np.pi - eps * rs.uniform(-1, 1))
            out.append(("near180", src, src @ R.T + rs.normal(size=3) * 0.01))
    g = np.stack(np.meshgrid(np.arange(4.0), np.arange(4.0), indexing="ij"), -1).reshape(-1, 2)
    for refl in (False, True):                            # planar / noisy planar, reflected
        for noise in (0.0, 1e-4, 1e-7):
            src = np.c_[g + rs.uniform(-0.1, 0.1, g.shape), rs.normal(size=len(g)) * noise]
            R = te._axis_angle(rs.normal(size=3), np.deg2rad(1.5))
            dst = src @ R.T
            if refl:
                dst = dst * [1.0, 1.0, -1.0]
            out.append(("planar", src, dst))
    for gap in (1e-2, 1e-4, 1e-6):                         # small eigengap: nearly collinear
        t = np.arange(6.0)[:, None]
        src = t * [1.0, 0.0, 0.0] + rs.normal(size=(6, 3)) * [0, gap, gap]
        R = te._axis_angle(rs.normal(size=3), np.deg2rad(3))
        out.append(("gap", src, src @ R.T))
    return out


def _sigma(src, dst):
    return (dst - dst.mean(0)).T @ (src - src.mean(0)) / len(src)


def test_horn_through_the_kernel(tmp_path):
    """One iteration (max_iteration=1, init = I, so T is the update): T's rotation against the SVD
    route within the horn bound of tests/test_icp_emu.py with s1 replaced by (K + 4) sum |t||s| / K,
    which also covers sigma's rounding in the kernel's summation order; its translation within that
    times (1 + |s_mean|).  The kernel's rotation also equals horn_rotation on the host for the
    oracle's sigma within the same bound.  Two-point and collinear matches: a proper rotation
    attaining max tr(R^T sigma)."""
    emu = te.build_emu(tmp_path)
    rs = np.random.RandomState(5)
    cases = horn_instances(rs)
    r = 0.45
    srcs = [c[1] for c in cases]
    tgts = [c[2] for c in cases]
    # a voxel small enough that each point is its own voxel
    T, fit, _, it = _register(srcs, tgts, [np.eye(4)] * len(cases), voxel=2.0 ** -12,
                              max_distance=r, max_iteration=1)
    worst = {}
    for i, (fam, src, dst) in enumerate(cases):
        assert it[i] == 1 and fit[i] == 1.0, (fam, i)
        res = oi.registration_icp_point_to_point(src, dst, r, np.eye(4), max_iteration=1)
        sigma = _sigma(src, dst)
        s = np.linalg.svd(sigma, compute_uv=False)
        d = 1.0 if np.linalg.det(sigma) >= 0 else -1.0
        sabs = (np.abs(dst - dst.mean(0)).sum(1) * np.abs(src - src.mean(0)).sum(1)).sum() / len(src)
        bound = te.C_HORN * te.U53 * (len(src) + 4) * sabs / (s[1] + d * s[2])
        err = np.linalg.norm(T[i, :3, :3] - res["transformation"][:3, :3])
        assert err <= bound, (fam, err, bound)
        terr = np.abs(T[i, :3, 3] - res["transformation"][:3, 3]).max()
        assert terr <= bound * (1 + np.linalg.norm(src.mean(0))), (fam, terr)
        host = te.horn(emu, sigma * len(src))[0]
        assert np.linalg.norm(T[i, :3, :3] - host) <= bound, fam
        # controls: the transposed rotation and the SVD route without the det correction
        if bound < 1e-2 and fam != "near180":           # near 180 degrees R is nearly symmetric
            assert np.linalg.norm(T[i, :3, :3].T - res["transformation"][:3, :3]) > bound, fam
        if fam == "planar" and np.linalg.det(sigma) < -1e-30:
            assert np.linalg.norm(T[i, :3, :3] - oi.umeyama_rotation(sigma, False)) > bound
        worst[fam] = max(worst.get(fam, 0.0), err / bound)
    # rank 1: two points, and collinear points
    rk = []
    for K in (2, 2, 5, 5):
        a = rs.normal(size=3)
        src = np.arange(K)[:, None] * a / np.linalg.norm(a) * 0.9
        R = te._axis_angle(rs.normal(size=3), np.deg2rad(5))
        rk.append((src, src @ R.T + 0.01))
    T, _, _, it = _register([c[0] for c in rk], [c[1] for c in rk], [np.eye(4)] * len(rk),
                            voxel=2.0 ** -12, max_distance=r, max_iteration=1)
    for i, (src, dst) in enumerate(rk):
        R = T[i, :3, :3]
        assert np.abs(R.T @ R - np.eye(3)).max() <= 64 * te.U53
        assert abs(np.linalg.det(R) - 1) <= 64 * te.U53
        sigma = _sigma(src, dst)
        s1 = np.linalg.svd(sigma, compute_uv=False)[0]
        assert abs(np.trace(R.T @ sigma) - s1) <= te.C_HORN * te.U53 * (len(src) + 4) * s1
        worst["rank1"] = max(worst.get("rank1", 0.0), abs(np.trace(R.T @ sigma) - s1)
                             / (te.C_HORN * te.U53 * (len(src) + 4) * s1))
    print("horn through the kernel, worst err/bound:", {k: f"{v:.3g}" for k, v in worst.items()})


# --------------------------------------------------------------------- stop rules and limits

def test_stop_rules_and_limits():
    from morefusion_b200 import synthetic
    s = synthetic.make_icp_scene(4, 2)
    init = np.linalg.inv(s["transform_init"])
    d, c = s["pcd_depth"], s["pcd_cad"]
    for cap in (0, 1):
        T, fit, rmse, it = _register(d, c, init, max_iteration=cap)
        for i in range(4):
            r = _oracle(d[i], c[i], init[i], max_iteration=cap)
            assert it[i] == cap == r["iterations"] and fit[i] == r["fitness"]
            assert np.abs(T[i] - r["transformation"]).max() <= 1e-9
        if cap == 0:
            assert np.array_equal(T, init)
    # relative thresholds 0: every instance runs to the cap
    T, fit, rmse, it = _register(d, c, init, max_iteration=25, relative_fitness=0.0,
                                 relative_rmse=0.0)
    assert (it == 25).all()
    for i in range(4):
        r = _oracle(d[i], c[i], init[i], max_iteration=25, relative_fitness=0.0, relative_rmse=0.0)
        if _well_posed(r):
            assert np.abs(T[i] - r["transformation"]).max() <= 1e-9
    # an all-NaN source, a one-point target, an instance 1e3 m off and one 1e8 m off, in one batch
    base = _register(d, c, init)
    src = list(d) + [np.full((50, 3), np.nan, np.float32), d[1], d[1], d[2]]
    tgt = list(c) + [c[0], c[1][:1], c[1], c[2]]
    far = init.copy()
    inits = list(init) + [init[0], init[1], far[1].copy(), far[2].copy()]
    inits[6][:3, 3] += 1e3
    inits[7][:3, 3] += [1e8, -1e8, 1e8]
    T, fit, rmse, it = _register(src, tgt, inits)
    for a, b in zip((T, fit, rmse, it), base):
        assert np.array_equal(a[:4], b)                  # the others are unchanged
    assert fit[4] == 0 and rmse[4] == 0 and it[4] == 1 and np.array_equal(T[4], inits[4])
    for k in (6, 7):
        assert fit[k] == 0 and rmse[k] == 0 and it[k] == 1 and np.array_equal(T[k], inits[k])
    r = _oracle(d[1], c[1][:1], init[1])
    assert _well_posed(r)
    assert it[5] == r["iterations"] and fit[5] == r["fitness"]
    assert np.abs(T[5] - r["transformation"]).max() <= 1e-9


def test_icp_registration_640x480_cloud():
    """A 640x480 cloud (307 200 rows, NaN rows among them) through ICPRegistration."""
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib import ICPRegistration
    s = synthetic.make_icp_scene(1, 7)
    rs = np.random.RandomState(7)
    d = s["pcd_depth"][0]
    rows = np.concatenate([d, d[rs.randint(0, len(d), 307200 - len(d))] + rs.normal(0, 0.001, (307200 - len(d), 3))])
    rows = rows.astype(np.float32)
    rows[rs.choice(307200, 5000, replace=False)] = np.nan
    want, r = oi.icp_registration(rows[np.isfinite(rows).all(1)], s["pcd_cad"][0], s["transform_init"][0])
    got = ICPRegistration(rows.reshape(480, 640, 3), s["pcd_cad"][0], s["transform_init"][0]).register()
    if _well_posed(r):
        assert np.abs(got - want).max() <= 1e-9
    assert np.isfinite(got).all()
