"""CPU-only: the per-thread helpers of morefusion_b200/csrc/icp.cu run on the host
(tests/emu/icp_emu.cpp, g++ -DMF_HOST_EMU -ffp-contract=off; the .cu is built with -fmad=false,
so these are the device's results bit for bit) against float64 references:

  * horn_rotation, the rotation k_icp_run solves each iteration, against Umeyama's SVD route
    (oracle.icp.umeyama_rotation) over seeded cross-covariances at every conditioning;
  * nearest, the correspondence search, against brute force over cell lists built from the
    oracle's keys, at the exact-arithmetic edges of its rules;
  * cell_window, the window nearest loops over, which must end at every query.

The GPU runs of the same code are tests/test_icp_gpu.py and tests/test_icp_paths_gpu.py."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import icp as oi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U53 = 2.0 ** -53
INT_MAX = 2 ** 31 - 1
KEY_MAX = INT_MAX - 1

# Bound of horn_rotation against the SVD route: ||R - R_svd||_F <= C_HORN 2^-53 s1 / (s2 + d s3),
# d = sgn det(sigma), s the singular values of sigma.
#   Horn's 4x4 matrix N has eigenvalues s1 + s2 + d s3 >= s1 - s2 - d s3 >= ..., so its gap is
#   2 (s2 + d s3) and ||N||_F = 2 ||s|| <= 2 sqrt(3) s1.  Each Jacobi rotation is an orthogonal
#   similarity applied in floating point: c and s carry <= 6 roundings, every entry of the two
#   rotated rows and columns 3 more in each of the two passes, so it is exact for a matrix within
#   12 u ||N||_F of its input (u = 2^-53); V's columns take the same 12 u per rotation.  A sweep
#   has 6 rotations and the solves here end within JACOBI_SWEEPS sweeps (checked on every case by
#   _jacobi_sweeps, a float64 restatement of the loop that reproduces horn_rotation bit for bit),
#   so the backward error is ||E||_F <= 6 * JACOBI_SWEEPS * 12 u ||N||_F.  By Davis-Kahan the
#   quaternion turns by sin(theta) <= ||E|| / gap, and ||R(q) - R(q')||_F = 2 sqrt(2) sin(theta),
#   which gives 2 sqrt(2) * sqrt(3) * 72 * JACOBI_SWEEPS u s1 / (s2 + d s3), about 3530 u s1 / gap
#   with 10 sweeps.  The SVD side is the rotation of sigma + E', ||E'|| of a few u ||sigma||, and
#   that rotation moves by at most 2 ||E'|| / (s2 + d s3) (the sensitivity of the orthogonal
#   Procrustes factor), 2 * 10 * sqrt(3) u s1 / gap with 10 u per entry; the quaternion to R and
#   the normalisation add about 10 u.  C_HORN = 4096 covers the sum.
JACOBI_SWEEPS = 10
C_HORN = 4096


def build_emu(directory):
    """The host build of icp.cu's helpers, compiled into `directory`."""
    so = os.path.join(str(directory), "icp_emu.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17",
                    "-I" + os.path.join(ROOT, "tests", "emu"),
                    os.path.join(ROOT, "tests", "emu", "icp_emu.cpp"), "-o", so], check=True)
    lib = ctypes.CDLL(so)
    p, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.emu_horn_rotation.argtypes = [p, i, p]
    lib.emu_cell_window.argtypes = [p, i, d, d, d, p]
    lib.emu_nearest.argtypes = [p, i, p, p, p, i, p, d, d, d, p, p]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu(tmp_path_factory.mktemp("emu"))


def horn(emu, C):
    C = np.ascontiguousarray(np.asarray(C, np.float64).reshape(-1, 3, 3))
    R = np.empty_like(C)
    emu.emu_horn_rotation(C.ctypes.data, len(C), R.ctypes.data)
    return R


def window(emu, x, r, origin, h):
    x = np.ascontiguousarray(np.atleast_1d(np.asarray(x, np.float64)))
    out = np.empty((len(x), 2), np.int32)
    emu.emu_cell_window(x.ctypes.data, len(x), r, origin, h, out.ctypes.data)
    return out


# ------------------------------------------------------------------------------------- Horn

def _horn_matrix(C):
    """N of horn_rotation (S[a][b] = C[b][a])."""
    S = np.asarray(C, np.float64).T
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = S
    return np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
                     [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                     [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy],
                     [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])


def _quat_matrix(q):
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _jacobi_sweeps(C):
    """(R, sweeps): horn_rotation's cyclic Jacobi restated in Python floats (IEEE float64, no
    contraction), and the number of sweeps that rotated or zeroed an element."""
    A = [list(r) for r in _horn_matrix(C).tolist()]
    V = [[float(i == j) for j in range(4)] for i in range(4)]
    used = 0
    for sweep in range(50):
        off = 0.0
        for p in range(3):
            for q in range(p + 1, 4):
                off += abs(A[p][q])
        if off == 0.0:
            break
        used += 1
        for p in range(3):
            for q in range(p + 1, 4):
                apq = A[p][q]
                if apq == 0.0:
                    continue
                g = 100.0 * abs(apq)
                if sweep > 3 and abs(A[p][p]) + g == abs(A[p][p]) and abs(A[q][q]) + g == abs(A[q][q]):
                    A[p][q] = A[q][p] = 0.0
                    continue
                theta = (A[q][q] - A[p][p]) / (2.0 * apq)
                t = 1.0 / (abs(theta) + np.sqrt(theta * theta + 1.0))
                if theta < 0.0:
                    t = -t
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                for k in range(4):
                    akp, akq = A[k][p], A[k][q]
                    A[k][p] = c * akp - s * akq
                    A[k][q] = s * akp + c * akq
                for k in range(4):
                    apk, aqk = A[p][k], A[q][k]
                    A[p][k] = c * apk - s * aqk
                    A[q][k] = s * apk + c * aqk
                A[p][q] = A[q][p] = 0.0
                for k in range(4):
                    vkp, vkq = V[k][p], V[k][q]
                    V[k][p] = c * vkp - s * vkq
                    V[k][q] = s * vkp + c * vkq
    b = 0
    for k in range(1, 4):
        if A[k][k] > A[b][b]:
            b = k
    w, x, y, z = V[0][b], V[1][b], V[2][b], V[3][b]
    nq = np.sqrt(((w * w + x * x) + y * y) + z * z)
    w, x, y, z = w / nq, x / nq, y / nq, z / nq
    R = [1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y),
         2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x),
         2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]
    return np.array(R).reshape(3, 3), used


def _orth(rs, det):
    Q, Rq = np.linalg.qr(rs.normal(size=(3, 3)))
    Q = Q * np.sign(np.diag(Rq))
    if np.linalg.det(Q) * det < 0:
        Q[:, 2] = -Q[:, 2]
    return Q


def _axis_angle(axis, angle):
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def horn_cases(seed=0):
    """(family, sigma [3,3]) pairs: sigma = U diag(s) V^T at eigengaps 1 .. 1e-8 with det of both
    signs, planar and noisy-planar point sets (the SVD route's S[2] = -1 among them), rotations
    within 1e-3 rad of 180 degrees, scales 1e-6 and 1e3."""
    rs = np.random.RandomState(seed)
    out = []
    for gap in 10.0 ** -np.arange(9):
        for _ in range(120):
            d = 1.0 if rs.rand() < 0.5 else -1.0
            s1 = 1.0
            if d > 0:                      # s2 + s3 = gap
                s3 = rs.uniform(0, 0.5) * gap
                s = (s1, gap - s3, s3)
            else:                          # s2 - s3 = gap
                s3 = rs.uniform(0, 0.5)
                s = (s1, min(s1, s3 + gap), s3)
            U, V = _orth(rs, 1.0), _orth(rs, d)
            out.append(("gap", U @ np.diag(s) @ V.T))
    for _ in range(300):                   # planar and noisy-planar point sets
        n = rs.randint(3, 40)
        src = np.c_[rs.normal(size=(n, 2)), np.zeros(n)]
        if rs.rand() < 0.5:
            src[:, 2] = rs.normal(size=n) * 10.0 ** -rs.uniform(2, 8)
        R0 = _orth(rs, 1.0)
        dst = src @ R0.T + rs.normal(size=(n, 3)) * (10.0 ** -rs.uniform(1, 8) if rs.rand() < 0.5 else 0.0)
        if rs.rand() < 0.5:                # the reflected target: the unconstrained optimum is a reflection
            dst = dst @ np.diag([1.0, 1.0, -1.0])
        sigma = (dst - dst.mean(0)).T @ (src - src.mean(0)) / n
        out.append(("planar", sigma))
    for eps in (1e-3, 1e-5, 1e-8, 0.0):    # near 180 degrees
        for _ in range(40):
            R0 = _axis_angle(rs.normal(size=3), np.pi - eps * rs.uniform(-1, 1))
            V = _orth(rs, 1.0)
            s = np.sort(rs.uniform(0.05, 1.0, 3))[::-1]
            out.append(("near180", R0 @ V @ np.diag(s) @ V.T))
    for scale in (1e-6, 1e3):
        for _ in range(100):
            d = 1.0 if rs.rand() < 0.5 else -1.0
            s = np.sort(rs.uniform(0, 1, 3))[::-1] * scale
            out.append(("scale", _orth(rs, 1.0) @ np.diag(s) @ _orth(rs, d).T))
    return out


def horn_ratio(R, sigma):
    """||R - R_svd||_F over the bound."""
    s = np.linalg.svd(sigma, compute_uv=False)
    d = 1.0 if np.linalg.det(sigma) >= 0 else -1.0
    bound = C_HORN * U53 * s[0] / (s[1] + d * s[2])
    return np.linalg.norm(R - oi.umeyama_rotation(sigma)) / bound


def _proper(R, ulps=16):
    assert np.abs(R.T @ R - np.eye(3)).max() <= ulps * U53, R
    assert abs(np.linalg.det(R) - 1.0) <= ulps * U53, R


def test_horn_matches_umeyama_at_every_conditioning(emu):
    cases = horn_cases()
    sig = np.stack([c for _, c in cases])
    R = horn(emu, sig)
    worst = {}
    for (fam, sigma), r in zip(cases, R):
        ratio = horn_ratio(r, sigma)
        assert ratio <= 1.0, (fam, ratio, sigma)
        _proper(r)
        worst[fam] = max(worst.get(fam, 0.0), ratio)
    # coverage: both signs of det, the SVD route's reflection fix, gaps down to 1e-8
    dets = np.linalg.det(sig)
    assert (dets > 0).sum() > 100 and (dets < 0).sum() > 100
    flips = 0
    for _, sigma in cases:
        U, _, Vt = np.linalg.svd(sigma)
        flips += np.linalg.det(U) * np.linalg.det(Vt) < 0
    assert flips > 300
    print("horn worst err/bound:", {k: f"{v:.3g}" for k, v in sorted(worst.items())})


def test_horn_bound_assumptions_hold(emu):
    """The bound counts JACOBI_SWEEPS sweeps: the restatement that counts them reproduces
    horn_rotation bit for bit, and no case needs more."""
    cases = horn_cases()[::7]
    R = horn(emu, np.stack([c for _, c in cases]))
    most = 0
    for (_, sigma), r in zip(cases, R):
        Rp, used = _jacobi_sweeps(sigma)
        assert np.array_equal(Rp.view(np.uint64), r.view(np.uint64))
        most = max(most, used)
    assert most <= JACOBI_SWEEPS
    print("most Jacobi sweeps:", most)


def test_horn_controls_fail(emu):
    """Wrong references fail the bound: the SVD route without the det correction (on the cases
    that need it), R transposed, and the rotation of Horn's second eigenvector."""
    cases = horn_cases(1)
    sig = np.stack([c for _, c in cases])
    R = horn(emu, sig)
    n_det = n_t = 0
    for (fam, sigma), r in zip(cases, R):
        U, _, Vt = np.linalg.svd(sigma)
        if np.linalg.det(U) * np.linalg.det(Vt) < 0:
            bad = oi.umeyama_rotation(sigma, det_correction=False)
            assert horn_ratio(bad, sigma) > 1e3, fam
            n_det += 1
        if fam == "gap":                   # a generic rotation is not symmetric
            assert horn_ratio(r.T, sigma) > 1.0 or np.abs(r - r.T).max() < 1e-6
            n_t += horn_ratio(r.T, sigma) > 1.0
        w, v = np.linalg.eigh(_horn_matrix(sigma))
        assert horn_ratio(_quat_matrix(v[:, -2]), sigma) > 1.0, fam
    assert n_det > 300 and n_t > 1000


def test_horn_rank_one_and_zero(emu):
    """Rank 1 (two or collinear matches): no unique rotation, so a proper rotation attaining the
    maximum tr(R^T sigma) = s1 within C_HORN 2^-53 s1.  sigma = 0 gives exactly I."""
    rs = np.random.RandomState(3)
    sig = []
    for scale in (1e-6, 1.0, 1e3):
        for _ in range(100):
            u, v = rs.normal(size=3), rs.normal(size=3)
            sig.append(scale * np.outer(u / np.linalg.norm(u), v / np.linalg.norm(v)))
    for n in (2, 3, 7):                    # collinear point sets
        for _ in range(50):
            a, b = rs.normal(size=3), rs.normal(size=3)
            src = a + np.outer(rs.normal(size=n), b)
            R0 = _orth(rs, 1.0)
            dst = src @ R0.T + rs.normal(size=3)
            sig.append((dst - dst.mean(0)).T @ (src - src.mean(0)) / n)
    sig = np.stack(sig)
    R = horn(emu, sig)
    worst = 0.0
    for r, sigma in zip(R, sig):
        _proper(r)
        s1 = np.linalg.svd(sigma, compute_uv=False)[0]
        err = abs(np.trace(r.T @ sigma) - s1) / (C_HORN * U53 * s1)
        assert err <= 1.0, err
        worst = max(worst, err)
        # control: transposing the rotation loses the maximum on a generic rank-1 sigma
    bad = sum(abs(np.trace(r @ sigma) - np.linalg.svd(sigma, compute_uv=False)[0])
              > C_HORN * U53 * np.linalg.svd(sigma, compute_uv=False)[0] for r, sigma in zip(R, sig))
    assert bad > 0.9 * len(sig)
    print(f"rank-1 worst err/bound: {worst:.3g}")
    Z = horn(emu, np.zeros((3, 3, 3)))
    assert np.array_equal(Z, np.broadcast_to(np.eye(3), (3, 3, 3)))


# ------------------------------------------------------------------------------- cell list

def cell_list(points, h):
    """A cell list as mf_icp_cell_list builds it, from the oracle's keys: points sorted stably by
    (i, j, k) of floor((p - min_bound) / h), min_bound = min(p) - h / 2."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    keys, origin = oi.voxel_keys(p, h)
    order = np.lexsort((keys[:, 2], keys[:, 1], keys[:, 0]))
    assert keys.max() <= KEY_MAX
    return (np.ascontiguousarray(p[order]), np.ascontiguousarray(keys[order].astype(np.int32)),
            np.ascontiguousarray(order.astype(np.int32)), np.ascontiguousarray(origin))


def nearest(emu, q, cl, h, r, r2=None):
    pts, cells, index, origin = cl
    q = np.ascontiguousarray(np.asarray(q, np.float64).reshape(-1, 3))
    pos = np.empty(len(q), np.int32)
    d2 = np.empty(len(q))
    emu.emu_nearest(q.ctypes.data, len(q), pts.ctypes.data, cells.ctypes.data, index.ctypes.data,
                    len(pts), origin.ctypes.data, h, r, r * r if r2 is None else r2,
                    pos.ctypes.data, d2.ctypes.data)
    row = np.where(pos >= 0, index[np.maximum(pos, 0)], -1)
    return row, d2


def brute(q, target, r2, strict=True, lowest=True):
    """float64 brute force: the nearest row with d^2 < r2 (<= with strict=False), equidistant
    rows to the lowest (highest with lowest=False)."""
    q = np.asarray(q, np.float64).reshape(-1, 3)
    t = np.asarray(target, np.float64)
    dx, dy, dz = (q[:, None, a] - t[None, :, a] for a in range(3))
    d2 = (dx * dx + dy * dy) + dz * dz
    best = d2.min(1)
    if lowest:
        idx = d2.argmin(1)
    else:
        idx = len(t) - 1 - d2[:, ::-1].argmin(1)
    ok = best < r2 if strict else best <= r2
    return np.where(ok, idx, -1), best


def test_nearest_matches_brute_force(emu):
    """Random clouds on a dyadic lattice (exact distances, many ties) at several cell sizes."""
    rs = np.random.RandomState(0)
    for h, r, step in ((2.0 ** -6, 2.0 ** -6, 2.0 ** -9), (2.0 ** -5, 2.0 ** -6, 2.0 ** -8),
                       (2.0 ** -7, 2.0 ** -7, 2.0 ** -10)):
        t = rs.randint(-40, 40, (600, 3)) * step
        q = np.concatenate([rs.randint(-50, 50, (3000, 3)) * step, t[:200]])
        cl = cell_list(t, h)
        row, d2 = nearest(emu, q, cl, h, r)
        want, best = brute(q, t, r * r)
        assert np.array_equal(row, want)
        assert np.array_equal(d2[row >= 0], best[row >= 0])
        assert (row >= 0).sum() > 500 and (row < 0).sum() > 100


def test_nearest_exact_edges_and_controls(emu):
    """d^2 == r^2 is no match, the double below it is; equidistant targets in one cell and across
    cells go to the lowest row; queries below the origin and far above; the control rules fail."""
    h = r = 2.0 ** -6
    e = 2.0 ** -8
    # rows chosen so the lowest row of each tie sorts after the others in cell order
    t = np.array([[0.5, 0.5, 0.5],                 # 0
                  [0.5 + 3 * e, 0.5, 0.5],         # 1  same cell as 0
                  [0.5 + 4 * r + 2 * e, 0.5, 0.5],  # 2 the higher cell of a cross-cell tie
                  [0.5 + 4 * r - 2 * e, 0.5, 0.5],  # 3 the lower cell
                  [0.5 + 8 * r, 0.5, 0.5],          # 4 alone: a target at exactly r from a query
                  [0.0, 0.0, 0.0]])                 # 5 the minimum: cell (0, 0, 0) is near it
    cl = cell_list(t, h)
    q = np.array([[0.5 + 1.5 * e, 0.5, 0.5],       # equidistant to rows 0 and 1 (one cell)
                  [0.5 + 4 * r, 0.5, 0.5],          # equidistant to 2 and 3 (adjacent cells)
                  [0.5 + 8 * r - r, 0.5, 0.5],      # d^2 == r^2 to row 4
                  [-0.75 * h, 0.0, 0.0],            # below the origin on x: window clamped to 0
                  [-5.0, -5.0, -5.0],               # far below
                  [1e3, 1e3, 1e3]])                 # far above
    row, d2 = nearest(emu, q, cl, h, r)
    assert row.tolist() == [0, 2, -1, 5, -1, -1]
    assert row[1] < 3 and cl[1][cl[2] == 2][0, 0] > cl[1][cl[2] == 3][0, 0]   # 2 sorts after 3
    assert d2[2] == r * r
    want, _ = brute(q, t, r * r)
    assert np.array_equal(row, want)
    # the next double above d^2 as r2: d^2 is then the double below r2, a match
    row2, _ = nearest(emu, q[2:3], cl, h, r, np.nextafter(r * r, np.inf))
    assert row2[0] == 4
    # controls: <= in place of <, ties to the highest row
    assert not np.array_equal(row, brute(q, t, r * r, strict=False)[0])
    assert not np.array_equal(row, brute(q, t, r * r, lowest=False)[0])
    w = window(emu, q[3:, 0], r, cl[3][0], h)
    assert w[0].tolist() == [0, 0] and w[1].tolist() == [0, 0]
    assert w[2, 1] - w[2, 0] <= 2


def _old_window(x, r, origin, h):
    """The window before cell_window: cell_of of x - r and x + r, capped at INT_MAX only."""
    def cell_of(v):
        c = np.floor((v - origin) / h)
        return 0 if not c > 0 else (INT_MAX if c >= INT_MAX else int(c))
    return cell_of(x - r), cell_of(x + r)


def test_window_loop_ends_at_int_max(emu):
    """nearest loops `for (c = lo; c <= hi; ++c)`: with hi == INT_MAX, ++c overflows and the loop
    does not end.  The window before cell_window reaches INT_MAX for a query at origin +
    (2^31 - 1) h; cell_window never does, and a target at the largest key KEY_MAX is still found."""
    h = r = 2.0 ** -6
    origin = -h / 2
    xs = np.array([0.0, 1.0, 1e3, (2.0 ** 31 - 2) * h, (2.0 ** 31 - 1) * h, 2.0 ** 31 * h, 1e8,
                   1e12, 1e300, -1e8])
    w = window(emu, xs, r, origin, h)
    assert (w[:, 1] <= KEY_MAX).all() and (w[:, 0] <= w[:, 1]).all()
    old = np.array([_old_window(x, r, origin, h) for x in xs])
    assert (old[:, 1] == INT_MAX).sum() >= 5          # the old window: a loop that cannot end
    assert (w[old[:, 1] < INT_MAX] == old[old[:, 1] < INT_MAX]).all()   # unchanged elsewhere
    # a cloud with a target at key KEY_MAX on x, queried next to it and far beyond it
    t = np.array([[0.0, 0.0, 0.0], [KEY_MAX * h, 0.0, 0.0], [KEY_MAX * h, 4 * r, 0.0]])
    cl = cell_list(t, h)
    assert cl[1][:, 0].max() == KEY_MAX
    q = np.array([[KEY_MAX * h + 2.0 ** -8, 0.0, 0.0], [1e8, 0.0, 0.0], [1e8, 1e8, 1e8],
                  [KEY_MAX * h + 0.75 * h, 4 * r, 0.0]])
    assert _old_window(q[0, 0], r, cl[3][0], h)[1] == INT_MAX
    row, _ = nearest(emu, q, cl, h, r)
    want, _ = brute(q, t, r * r)
    assert row.tolist() == want.tolist() == [1, -1, -1, 2]
