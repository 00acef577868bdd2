"""Meshes the mesh-model tests share: closed non-convex solids, an edge-aligned box, mixed
winding, degenerate faces and subdivided icospheres.  Each returns (vertices [V,3] float64,
faces [F,3] int32)."""

import numpy as np


def box(half=(0.05, 0.035, 0.0225), centre=(0.0, 0.0, 0.0)):
    from morefusion_b200 import synthetic
    v, f = synthetic.cad_mesh("box", np.asarray(half, np.float64))
    return v + np.asarray(centre, np.float64), f


def edge_aligned_box(D=16):
    """A box on whose D-grid columns run exactly through edges and vertices: z spans [0, 1] (the
    scale, s = 1 / D), x and y span [0, 7.5 s], so the far vertical edge and the far edges of the
    caps lie on column centres, and so does each cap's diagonal (x = y)."""
    s = 1.0 / D
    lo = np.array([0.0, 0.0, 0.0])
    hi = np.array([7.5 * s, 7.5 * s, 1.0])
    v = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = [t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))]
    return v, np.array(f, np.int32)


def torus(R=0.05, r=0.018, n_major=24, n_minor=12):
    u = 2 * np.pi * np.arange(n_major) / n_major
    w = 2 * np.pi * np.arange(n_minor) / n_minor
    uu, ww = np.meshgrid(u, w, indexing="ij")
    v = np.stack([(R + r * np.cos(ww)) * np.cos(uu), (R + r * np.cos(ww)) * np.sin(uu),
                  r * np.sin(ww)], -1).reshape(-1, 3)
    f = []
    for i in range(n_major):
        for j in range(n_minor):
            a = i * n_minor + j
            b = ((i + 1) % n_major) * n_minor + j
            c = ((i + 1) % n_major) * n_minor + (j + 1) % n_minor
            d = i * n_minor + (j + 1) % n_minor
            f += [(a, b, c), (a, c, d)]
    return v, np.array(f, np.int32)


def extruded_l(h=0.04):
    """An L-shaped prism: the outline (0,0) (0.06,0) (0.06,0.02) (0.02,0.02) (0.02,0.07) (0,0.07)
    extruded along z over [0, h], its caps fan-triangulated from their reflex corner."""
    p = np.array([[0, 0], [0.06, 0], [0.06, 0.02], [0.02, 0.02], [0.02, 0.07], [0, 0.07]], np.float64)
    n = len(p)
    v = np.concatenate([np.c_[p, np.zeros(n)], np.c_[p, np.full(n, h)]])
    f = []
    for i in range(n):
        j = (i + 1) % n
        f += [(i, j, n + j), (i, n + j, n + i)]
    cap = [(3, 4, 5), (3, 5, 0), (3, 0, 1), (3, 1, 2)]
    f += [(c, b, a) for a, b, c in cap]
    f += [(n + a, n + b, n + c) for a, b, c in cap]
    return v, np.array(f, np.int32)


def mixed_winding(v, f, seed=0):
    """The same mesh with a random half of its faces reversed."""
    rs = np.random.RandomState(seed)
    f = f.copy()
    flip = rs.uniform(size=len(f)) < 0.5
    f[flip] = f[flip][:, ::-1]
    return v, f


def with_degenerate(v, f):
    """The mesh plus zero-area faces: a repeated index, a collinear triple and an unused vertex
    far away that no face references."""
    v = np.concatenate([v, [(v[0] + v[1]) / 2, [9.0, 9.0, 9.0]]])
    m = len(v) - 2
    extra = np.array([[0, 0, 1], [0, m, 1], [2, 2, 2]], np.int32)
    return v, np.concatenate([f, extra]).astype(np.int32)


def icosphere(subdivisions, radius=0.05):
    """A closed icosphere: 20 * 4^subdivisions faces."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t],
         [0, 1, -t], [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4],
         [11, 10, 2], [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9],
         [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    v = [np.asarray(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdivisions):
        mid = {}

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        nf = []
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.asarray(v) * radius, np.asarray(f, np.int32)


def icosphere_faces(n_faces, radius=0.05):
    """An icosphere of about n_faces faces: the closest 20 * 4^k, then the faces of a
    latitude-longitude sphere when that is nearer (both closed)."""
    from morefusion_b200 import synthetic
    k = int(round(np.log(max(n_faces, 20) / 20.0) / np.log(4.0)))
    if abs(20 * 4 ** k - n_faces) <= 0.25 * n_faces:
        return icosphere(k, radius)
    n_around = int(round(np.sqrt(n_faces)))
    n_rings = max(3, int(round(n_faces / (2 * n_around))) + 1)
    return synthetic.cad_mesh("sphere", np.array([radius] * 3), n_around=n_around, n_rings=n_rings)


def all_cases():
    """name -> mesh of the fixed closed and special cases."""
    v, f = icosphere(2)
    return {
        "torus": torus(),
        "extruded_l": extruded_l(),
        "edge_aligned_box": edge_aligned_box(),
        "box_offset": box(centre=(0.3, -0.2, 0.1)),
        "mixed_winding": mixed_winding(v, f),
        "degenerate": with_degenerate(*torus(n_major=12, n_minor=8)),
    }


def sample_points(v, f, n, seed=0, margin=0.3):
    """Points in the mesh's bounding box widened by margin times its extent, plus its vertices
    and face centroids (on the surface)."""
    rs = np.random.RandomState(seed)
    used = v[f.reshape(-1)]
    lo, hi = used.min(0), used.max(0)
    ext = hi - lo
    p = rs.uniform(lo - margin * ext, hi + margin * ext, (n, 3))
    k = min(len(f), max(1, n // 8))
    cent = v[f[rs.choice(len(f), k, replace=False)]].mean(1)
    return np.concatenate([p, v[np.unique(f)][: n // 8], cent])
