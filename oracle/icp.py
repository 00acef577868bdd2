"""Float64 restatement of the two Open3D calls ``contrib.ICPRegistration`` makes
(morefusion/contrib/icp_registration.py:15-44): ``PointCloud.voxel_down_sample`` and
``registration_icp`` with ``TransformationEstimationPointToPoint(False)``.

TEST INFRASTRUCTURE ONLY.  Open3D is not installed and its source is not part of the reference
checkout, so this restates Open3D's published algorithm (``geometry::PointCloud::VoxelDownSample``,
``pipelines::registration::RegistrationICP``, ``GetRegistrationResultAndCorrespondences`` and
Eigen's ``umeyama``) rather than running it:

  * voxel_down_sample: min_bound = min(points) - voxel/2; a point's voxel is
    floor((p - min_bound) / voxel) (float64, correctly rounded); each occupied voxel gives the
    float64 mean of its points, summed in point order.  Open3D leaves the output order to an
    unordered map; here it is ascending (i, j, k).
  * registration_icp: source transformed by init; the correspondence of a source point is its
    nearest target point, kept when d^2 < max_distance^2 (strict), d^2 = dx^2 + dy^2 + dz^2 in
    that order, equidistant candidates to the lowest target index.  fitness = n_corr / n_source,
    inlier_rmse = sqrt(sum d^2 / n_corr), both 0 without a correspondence.  Each iteration takes
    the Umeyama update (no scaling, demeaned cross-covariance sigma = sum (t - t_mean)(s - s_mean)^T
    / n, R = U S V^T with S[2] = -1 when det(U) det(V) < 0; the identity without correspondences),
    T = update @ T, transforms the source points by the update, recomputes the correspondences and
    stops when |d fitness| < relative_fitness and |d rmse| < relative_rmse.

Rank of sigma: with one correspondence sigma is exactly 0 and the update is a pure translation
(U = V = I).  The kernel shares that rule (csrc/icp.cu).  With sigma of rank 1 (two, or collinear,
correspondences) the rotation is not determined by the matches; neither the kernel nor this
restatement is pinned to Eigen's choice there.  The tests check the kernel's rotation there by
its properties instead: a proper rotation that attains the maximum of tr(R^T sigma).
"""

import numpy as np


def voxel_keys(points, voxel_size):
    """(keys [N,3] int64, min_bound [3]) of float64 points."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    min_bound = p.min(0) - 0.5 * voxel_size
    return np.floor((p - min_bound) / voxel_size).astype(np.int64), min_bound


def voxel_down_sample(points, voxel_size, return_counts=False):
    """Means of the occupied voxels in ascending (i, j, k); with return_counts also the voxel keys
    [V,3] and the number of points of each voxel [V]."""
    if not voxel_size > 0:
        raise ValueError("voxel_size must be positive")
    p = np.asarray(points, np.float64).reshape(-1, 3)
    if len(p) == 0:
        out = np.zeros((0, 3))
        return (out, np.zeros((0, 3), np.int64), np.zeros(0, np.int64)) if return_counts else out
    keys, _ = voxel_keys(p, voxel_size)
    uniq, inv, counts = np.unique(keys, axis=0, return_inverse=True, return_counts=True)
    sums = np.zeros((len(uniq), 3))
    np.add.at(sums, inv.reshape(-1), p)                 # sequential, in point order
    means = sums / counts[:, None]
    return (means, uniq, counts) if return_counts else means


def transform(T, points):
    """T [4,4] applied to points [N,3]: ((T0 x + T1 y) + T2 z) + T3, row by row."""
    T = np.asarray(T, np.float64)
    p = np.asarray(points, np.float64)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3]
                     for r in range(3)], 1)


def correspondences(source, target, max_distance):
    """Per source point: index of its nearest target point (-1 beyond max_distance), d^2 of that
    point, and the gap between the best and the second-best candidate as a distance,
    sqrt(d^2_second) - sqrt(d^2_best) in metres (inf with one target)."""
    s = np.asarray(source, np.float64)
    t = np.asarray(target, np.float64)
    if len(s) == 0 or len(t) == 0:
        return (np.full(len(s), -1, np.int64), np.full(len(s), np.inf), np.full(len(s), np.inf))
    step = max(1, (1 << 24) // len(t))                 # rows per block: memory stays bounded
    if len(s) > step:
        parts = [correspondences(s[i:i + step], t, max_distance) for i in range(0, len(s), step)]
        return tuple(np.concatenate(x) for x in zip(*parts))
    dx = s[:, None, 0] - t[None, :, 0]
    dy = s[:, None, 1] - t[None, :, 1]
    dz = s[:, None, 2] - t[None, :, 2]
    d2 = (dx * dx + dy * dy) + dz * dz
    idx = d2.argmin(1)                                  # first minimum: the lowest index
    best = d2[np.arange(len(s)), idx]
    if len(t) > 1:
        part = np.partition(d2, 1, axis=1)
        gap = np.sqrt(part[:, 1]) - np.sqrt(part[:, 0])
    else:
        gap = np.full(len(s), np.inf)
    match = np.where(best < max_distance * max_distance, idx, -1)
    return match, best, gap


def umeyama_rotation(sigma, det_correction=True):
    """Umeyama's rotation of the cross-covariance sigma [3,3] = sum (t - t_mean)(s - s_mean)^T / n:
    R = U S V^T with S[2] = -1 when det(U) det(V) < 0; I for sigma = 0.  det_correction=False
    drops the S[2] rule (a wrong reference for the tests: it can return a reflection)."""
    sigma = np.asarray(sigma, np.float64)
    if not sigma.any():
        return np.eye(3)
    U, _, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if det_correction and np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    return U @ np.diag(S) @ Vt


def umeyama(src, dst):
    """Eigen::umeyama(src^T, dst^T, false) in float64: the rigid [4,4] with dst ~ R src + t."""
    T = np.eye(4)
    n = len(src)
    if n == 0:
        return T
    sm, dm = src.mean(0), dst.mean(0)
    sigma = (dst - dm).T @ (src - sm) / n
    R = umeyama_rotation(sigma)
    T[:3, :3] = R
    T[:3, 3] = dm - R @ sm
    return T


def _result(source, target, max_distance):
    match, best, gap = correspondences(source, target, max_distance)
    ok = match >= 0
    n = int(ok.sum())
    if n == 0:
        fit, rmse = 0.0, 0.0
    else:
        fit = n / len(source)
        rmse = float(np.sqrt(best[ok].sum() / n))
    r2 = max_distance * max_distance
    margin_d2 = float(np.abs(best - r2).min()) if len(best) else np.inf
    margin_nn = float(gap[ok].min()) if n else np.inf
    return match, fit, rmse, margin_d2, margin_nn


def registration_icp_point_to_point(source, target, max_distance, init=None, max_iteration=30,
                                    relative_fitness=1e-6, relative_rmse=1e-6):
    """Open3D's RegistrationICP, point to point without scaling.  Returns dict(transformation
    [4,4], fitness, inlier_rmse, iterations, margins) where margins lists, per correspondence
    search (the initial one, then one per iteration), the smallest |d^2 - max_distance^2|, the
    smallest best-to-second-best distance gap of a matched point, and, per iteration, how far
    |d fitness| and |d rmse| were from their thresholds."""
    src = np.asarray(source, np.float64).reshape(-1, 3)
    tgt = np.asarray(target, np.float64).reshape(-1, 3)
    T = np.eye(4) if init is None else np.array(init, np.float64).reshape(4, 4)
    pts = transform(T, src)
    match, fit, rmse, md2, mnn = _result(pts, tgt, max_distance)
    margins = dict(d2=[md2], nn=[mnn], fitness=[], rmse=[])
    it = 0
    for it in range(1, max_iteration + 1):
        ok = match >= 0
        update = umeyama(pts[ok], tgt[match[ok]])
        T = update @ T
        pts = transform(update, pts)
        fit0, rmse0 = fit, rmse
        match, fit, rmse, md2, mnn = _result(pts, tgt, max_distance)
        margins["d2"].append(md2)
        margins["nn"].append(mnn)
        margins["fitness"].append(abs(abs(fit0 - fit) - relative_fitness))
        margins["rmse"].append(abs(abs(rmse0 - rmse) - relative_rmse))
        if abs(fit0 - fit) < relative_fitness and abs(rmse0 - rmse) < relative_rmse:
            break
    return dict(transformation=T, fitness=fit, inlier_rmse=rmse, iterations=it, margins=margins)


def icp_registration(pcd_depth, pcd_cad, transform_init, iteration=100, voxel_size=0.01):
    """ICPRegistration(pcd_depth, pcd_cad, transform_init).register(iteration, voxel_size) with
    the wrapper's conventions: depth -> CAD, max_distance = 2 voxel_size, init = inv(transform),
    result = inv(T).  Returns (transform [4,4], the registration dict)."""
    src = voxel_down_sample(pcd_depth, voxel_size)
    tgt = voxel_down_sample(pcd_cad, voxel_size)
    r = registration_icp_point_to_point(src, tgt, 2 * voxel_size, np.linalg.inv(transform_init),
                                        max_iteration=iteration)
    return np.linalg.inv(r["transformation"]), r
