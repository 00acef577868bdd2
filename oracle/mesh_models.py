"""Float64 restatement of the per-class model data that ``YCBVideoModels`` derives from a CAD mesh
(morefusion/datasets/ycb_video/models.py:56-115): the solid voxel grid (binvox there), the signed
distance of points to the mesh (trimesh's ``nearest.signed_distance`` there) and the composition
of ``_get_sdf``.  csrc/mesh_models.cu computes these bit for bit, in the expression order below.

TEST INFRASTRUCTURE ONLY.  binvox and trimesh are not installed; these are the rules the kernels
follow, not a restatement of those tools (DESIGN.md section 4.22 lists what stays unpinned).

Grid of a mesh at dimension D
  * translate = the minimum of the vertices the faces reference, per axis; scale = the largest of
    the three extents (max - min); s = scale / D.  Voxel (i, j, k) (i along x) has its centre at
    translate + (idx + 0.5) s, per axis, and the half-size h = 0.5 s.
  * Surface: a voxel is filled if a face overlaps its closed box, by the Akenine-Moller
    separating-axis test in float64 (``tri_box_overlap``).  The voxels tested for a face are those
    whose index along each axis is in [floor((lo - t) / s) - 1, floor((hi - t) / s) + 1] (lo, hi
    the face's extent), clamped to [0, D).
  * Interior: a voxel is filled if its centre is inside by +z ray parity (``crossing``): the
    number of faces the upward ray from the centre crosses strictly above the centre is odd.  The
    columns tested for a face are those whose index along x and y is in
    [floor((lo - t) / s - 0.5) - 1, floor((hi - t) / s - 0.5) + 1], clamped to [0, D).
  * Both candidate ranges reach one voxel past every voxel the tests can accept, so they only
    bound the work.

+z ray parity of a point (px, py, pz) against a face
  * The face's vertex indices are sorted, i0 <= i1 <= i2 ("canonical order"); A, B, C are those
    vertices.  e(U, V; P) = (Vx - Ux)(Py - Uy) - (Vy - Uy)(Px - Ux).
  * area2 = e(A, B; C).  area2 == 0: no crossing.  sigma = sign(area2).
  * w0 = sigma e(B, C; P), w1 = sigma (-e(A, C; P)), w2 = sigma e(A, B; P): each edge is evaluated
    with its lower-index vertex first, then the sign is fixed, so two faces sharing an edge agree
    bit for bit on it.  The oriented edge directions are sigma (C - B), sigma (-(C - A)),
    sigma (B - A).
  * Inside iff every w_k > 0, or w_k == 0 and edge k is top-left: direction (dx, dy) with
    dy < 0, or dy == 0 and dx < 0.
  * Plane z = ((w0 Az + w1 Bz) + w2 Cz) / ((w0 + w1) + w2).  The face is crossed iff inside and
    z > pz.

Closest point (Ericson, Real-Time Collision Detection 5.1.5, ``ClosestPtPointTriangle``) with
a, b, c the canonical-order vertices; dot(u, v) = (ux vx + uy vy) + uz vz.  A face whose
cross(b - a, c - a) is exactly zero takes the nearest of its segments ab, bc, ca (first on a
tie), each t = clamp(dot(p - u, v - u) / dot(v - u, v - u), 0, 1) (0 when the segment has zero
length).  d^2 = (dx^2 + dy^2) + dz^2 of p - q.  The signed distance is sqrt of the smallest d^2
over the mesh's faces (the lowest face index on a tie), positive when the point is inside by
the parity rule and negative otherwise (-0.0 on the surface outside).
"""

import numpy as np


# ------------------------------------------------------------------------------------------------
# the mesh
# ------------------------------------------------------------------------------------------------
def grid_params(vertices, faces, dimension):
    """(translate [3], scale, s) of the mesh's grid."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    used = v[f.reshape(-1)]
    lo, hi = used.min(0), used.max(0)
    ext = hi - lo
    scale = max(max(ext[0], ext[1]), ext[2])
    return lo, scale, scale / dimension


def centres(translate, s, dimension):
    """[D] voxel centres along each axis: [3, D]."""
    idx = np.arange(dimension, dtype=np.float64) + 0.5
    return np.stack([translate[a] + idx * s for a in range(3)])


def canonical(vertices, faces):
    """[F,3,3] face vertices in canonical order (vertex indices sorted)."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    f = np.sort(np.asarray(faces, np.int64).reshape(-1, 3), axis=1)
    return v[f]


def bbox_diagonal(vertices, faces):
    """sqrt(sum(extents^2)) over the referenced vertices, as get_bbox_diagonal composes it."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    used = v[np.asarray(faces, np.int64).reshape(-1)]
    ext = used.max(0) - used.min(0)
    return np.sqrt((ext ** 2).sum())


# ------------------------------------------------------------------------------------------------
# separating axes
# ------------------------------------------------------------------------------------------------
def tri_box_overlap(a, b, c, centre, h):
    """Akenine-Moller's triangle / box test: does the face (a, b, c) [...,3] overlap the closed
    box of centre [...,3] and half-size h?  Broadcasts; returns bool [...]."""
    v0, v1, v2 = a - centre, b - centre, c - centre
    sep = np.zeros(np.broadcast(v0[..., 0], v1[..., 0]).shape, bool)
    for e in (v1 - v0, v2 - v1, v0 - v2):
        ex, ey, ez = e[..., 0], e[..., 1], e[..., 2]
        fx, fy, fz = np.abs(ex), np.abs(ey), np.abs(ez)
        for p, rad in (([ez * v[..., 1] - ey * v[..., 2] for v in (v0, v1, v2)], (fz + fy) * h),
                       ([ex * v[..., 2] - ez * v[..., 0] for v in (v0, v1, v2)], (fx + fz) * h),
                       ([ey * v[..., 0] - ex * v[..., 1] for v in (v0, v1, v2)], (fy + fx) * h)):
            lo = np.minimum(np.minimum(p[0], p[1]), p[2])
            hi = np.maximum(np.maximum(p[0], p[1]), p[2])
            sep |= (lo > rad) | (hi < -rad)
    for q in range(3):
        lo = np.minimum(np.minimum(v0[..., q], v1[..., q]), v2[..., q])
        hi = np.maximum(np.maximum(v0[..., q], v1[..., q]), v2[..., q])
        sep |= (lo > h) | (hi < -h)
    e0, e1 = v1 - v0, v2 - v1
    n = np.stack([e0[..., 1] * e1[..., 2] - e0[..., 2] * e1[..., 1],
                  e0[..., 2] * e1[..., 0] - e0[..., 0] * e1[..., 2],
                  e0[..., 0] * e1[..., 1] - e0[..., 1] * e1[..., 0]], -1)
    pos = n > 0
    vmin = np.where(pos, -h - v0, h - v0)
    vmax = np.where(pos, h - v0, -h - v0)
    dmin = (n[..., 0] * vmin[..., 0] + n[..., 1] * vmin[..., 1]) + n[..., 2] * vmin[..., 2]
    dmax = (n[..., 0] * vmax[..., 0] + n[..., 1] * vmax[..., 1]) + n[..., 2] * vmax[..., 2]
    sep |= (dmin > 0) | ~(dmax >= 0)
    return ~sep


# ------------------------------------------------------------------------------------------------
# +z ray parity
# ------------------------------------------------------------------------------------------------
def _edge(ux, uy, vx, vy, px, py):
    return (vx - ux) * (py - uy) - (vy - uy) * (px - ux)


def _top_left(dx, dy):
    return (dy < 0) | ((dy == 0) & (dx < 0))


def crossing(tri, px, py):
    """For canonical faces tri [...,3,3] and points (px, py) [...]: (inside [...] bool, plane z
    [...]), the rule of the module docstring.  z is only meaningful where inside."""
    A, B, C = tri[..., 0, :], tri[..., 1, :], tri[..., 2, :]
    ax, ay, bx, by, cx, cy = A[..., 0], A[..., 1], B[..., 0], B[..., 1], C[..., 0], C[..., 1]
    area2 = _edge(ax, ay, bx, by, cx, cy)
    sg = np.where(area2 < 0, -1.0, 1.0)
    w0 = sg * _edge(bx, by, cx, cy, px, py)
    w1 = sg * -_edge(ax, ay, cx, cy, px, py)
    w2 = sg * _edge(ax, ay, bx, by, px, py)
    d0 = (sg * (cx - bx), sg * (cy - by))
    d1 = (sg * -(cx - ax), sg * -(cy - ay))
    d2 = (sg * (bx - ax), sg * (by - ay))
    inside = np.broadcast_to(area2 != 0, w0.shape).copy()
    for w, d in ((w0, d0), (w1, d1), (w2, d2)):
        inside &= (w > 0) | ((w == 0) & _top_left(*d))
    with np.errstate(divide="ignore", invalid="ignore"):
        z = ((w0 * A[..., 2] + w1 * B[..., 2]) + w2 * C[..., 2]) / ((w0 + w1) + w2)
    return inside, z


# ------------------------------------------------------------------------------------------------
# the solid grid
# ------------------------------------------------------------------------------------------------
def _ranges(lo, hi, t, s, D, shift):
    a = np.floor((lo - t) / s - shift).astype(np.int64) - 1
    b = np.floor((hi - t) / s - shift).astype(np.int64) + 1
    return np.clip(a, 0, D - 1), np.clip(b, 0, D - 1)


def _pairs(lo, hi):
    """Every (face, offset) of per-face inclusive index boxes lo, hi [F,K]: (face [n], idx [n,K])."""
    n = np.maximum(hi - lo + 1, 0)
    vol = np.prod(n, axis=1)
    face = np.repeat(np.arange(len(lo)), vol)
    start = np.concatenate([[0], np.cumsum(vol)[:-1]])
    r = np.arange(vol.sum()) - np.repeat(start, vol)
    idx = np.empty((len(face), lo.shape[1]), np.int64)
    for q in range(lo.shape[1] - 1, -1, -1):
        nq = n[face, q]
        idx[:, q] = lo[face, q] + r % nq
        r //= nq
    return face, idx


def surface(tri, t, s, D, chunk=1 << 20):
    """bool [D,D,D]: the voxels some face overlaps."""
    out = np.zeros((D, D, D), bool)
    if len(tri) == 0:
        return out
    c = centres(t, s, D)
    lo, hi = _ranges(tri.min(1), tri.max(1), t, s, D, 0.0)
    face, idx = _pairs(lo, hi)
    h = 0.5 * s
    for q in range(0, len(face), chunk):
        fq, iq = face[q:q + chunk], idx[q:q + chunk]
        cen = np.stack([c[0][iq[:, 0]], c[1][iq[:, 1]], c[2][iq[:, 2]]], 1)
        hit = tri_box_overlap(tri[fq, 0], tri[fq, 1], tri[fq, 2], cen, h)
        out[iq[hit, 0], iq[hit, 1], iq[hit, 2]] = True
    return out


def column_crossings(tri, t, s, D, chunk=1 << 20):
    """int64 [D,D,D+1]: for each column (i, j), how many faces its ray crosses with n centres
    below the plane z (n = #{k : centre_k < z}), indexed by n."""
    hist = np.zeros((D, D, D + 1), np.int64)
    if len(tri) == 0:
        return hist
    c = centres(t, s, D)
    lo, hi = _ranges(tri[..., :2].min(1), tri[..., :2].max(1), t[:2], s, D, 0.5)
    face, idx = _pairs(lo, hi)
    for q in range(0, len(face), chunk):
        fq, iq = face[q:q + chunk], idx[q:q + chunk]
        inside, z = crossing(tri[fq], c[0][iq[:, 0]], c[1][iq[:, 1]])
        n = np.searchsorted(c[2], z[inside], side="left")
        np.add.at(hist, (iq[inside, 0], iq[inside, 1], n), 1)
    return hist


def interior(tri, t, s, D):
    """bool [D,D,D]: the centres inside by +z ray parity."""
    hist = column_crossings(tri, t, s, D)
    above = np.cumsum(hist[..., ::-1], axis=-1)[..., ::-1]      # above[k] = #crossings with n >= k
    return (above[..., 1:] % 2) == 1                            # voxel k: crossings with n > k


def voxelize_solid(vertices, faces, dimension=64):
    """The solid grid of one mesh: dict(matrix [D,D,D] bool, points [n,3] (filled centres in
    ascending (i, j, k)), translate [3], scale, pitch)."""
    D = int(dimension)
    t, scale, s = grid_params(vertices, faces, D)
    tri = canonical(vertices, faces)
    m = surface(tri, t, s, D) | interior(tri, t, s, D)
    c = centres(t, s, D)
    ijk = np.argwhere(m)
    pts = np.stack([c[0][ijk[:, 0]], c[1][ijk[:, 1]], c[2][ijk[:, 2]]], 1)
    return dict(matrix=m, points=pts, translate=t, scale=scale, pitch=s)


# ------------------------------------------------------------------------------------------------
# signed distance
# ------------------------------------------------------------------------------------------------
def _dot(u, v):
    return (u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1]) + u[..., 2] * v[..., 2]


def _seg_d2(p, u, v):
    d = v - u
    dd = _dot(d, d)
    with np.errstate(divide="ignore", invalid="ignore"):
        tt = np.where(dd > 0, _dot(p - u, d) / dd, 0.0)
    tt = np.minimum(np.maximum(tt, 0.0), 1.0)
    q = u + tt[..., None] * d
    r = p - q
    return _dot(r, r)


def closest_d2(p, a, b, c):
    """Squared distance from p to its closest point on face (a, b, c) [...,3], by Ericson's
    Voronoi regions; zero-area faces by their nearest segment."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ab, ac, ap = b - a, c - a, p - a
        d1, d2 = _dot(ab, ap), _dot(ac, ap)
        bp = p - b
        d3, d4 = _dot(ab, bp), _dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = p - c
        d5, d6 = _dot(ab, cp), _dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        v_ab = d1 / (d1 - d3)
        w_ac = d2 / (d2 - d6)
        w_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        denom = 1.0 / ((va + vb) + vc)
        v_f, w_f = vb * denom, vc * denom
        q = (a + ab * v_f[..., None]) + ac * w_f[..., None]
        cases = [
            ((d1 <= 0) & (d2 <= 0), a),
            ((d3 >= 0) & (d4 <= d3), b),
            ((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + v_ab[..., None] * ab),
            ((d6 >= 0) & (d5 <= d6), c),
            ((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + w_ac[..., None] * ac),
            ((va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0), b + w_bc[..., None] * (c - b)),
        ]
        for cond, qq in reversed(cases):
            q = np.where(cond[..., None], qq, q)
        r = p - q
        d2_face = _dot(r, r)
        n = np.stack([ab[..., 1] * ac[..., 2] - ab[..., 2] * ac[..., 1],
                      ab[..., 2] * ac[..., 0] - ab[..., 0] * ac[..., 2],
                      ab[..., 0] * ac[..., 1] - ab[..., 1] * ac[..., 0]], -1)
        degen = (n == 0).all(-1)
        s_ab, s_bc, s_ca = _seg_d2(p, a, b), _seg_d2(p, b, c), _seg_d2(p, c, a)
        seg = np.where(s_bc < s_ab, s_bc, s_ab)
        seg = np.where(s_ca < seg, s_ca, seg)
    return np.where(degen, seg, d2_face)


def signed_distance(vertices, faces, points, chunk=1 << 22):
    """(sdf [P] float64, nearest face [P] int64) of points [P,3] to one mesh."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    tri = canonical(vertices, faces)
    F, P = len(tri), len(p)
    best = np.full(P, np.inf)
    arg = np.full(P, -1, np.int64)
    odd = np.zeros(P, bool)
    step = max(1, chunk // max(F, 1))
    for q in range(0, P, step):
        pq = p[q:q + step]
        pp = pq[:, None, :]
        d2 = closest_d2(pp, tri[None, :, 0], tri[None, :, 1], tri[None, :, 2])
        i = d2.argmin(1)                                   # first minimum: the lowest face
        best[q:q + step] = d2[np.arange(len(pq)), i]
        arg[q:q + step] = i
        inside, z = crossing(tri[None], pq[:, 0:1], pq[:, 1:2])
        odd[q:q + step] = ((inside & (z > pq[:, 2:3])).sum(1) % 2) == 1
    d = np.sqrt(best)
    return np.where(odd, d, -d), arg


def column_parity_counts(vertices, faces, px, py):
    """How many faces the vertical line through each (px, py) crosses, at any z: even on a closed
    mesh under the half-open rule."""
    tri = canonical(vertices, faces)
    inside, _ = crossing(tri[None], np.asarray(px, np.float64).reshape(-1, 1),
                         np.asarray(py, np.float64).reshape(-1, 1))
    return inside.sum(1)


# ------------------------------------------------------------------------------------------------
# the composition of YCBVideoModels._get_sdf
# ------------------------------------------------------------------------------------------------
def get_sdf(vertices, faces, dimension=64):
    """(points, sdf) as _get_sdf composes them: the solid grid's points, down-sampled at the
    class pitch of dimension 32 (bbox diagonal / 32) by Open3D's rule (oracle/icp.py), and
    their signed distance."""
    from . import icp
    g = voxelize_solid(vertices, faces, dimension)
    pitch = 1.0 * bbox_diagonal(vertices, faces) / 32
    pts = icp.voxel_down_sample(g["points"], pitch)
    sdf, _ = signed_distance(vertices, faces, pts)
    return pts, sdf
