"""Float64 NumPy restatement of the masks and depth of ``render_cad`` (morefusion/extra/
_pybullet.py:215-288): each pose of a CAD mesh rendered alone into a pinhole camera.  TEST
INFRASTRUCTURE ONLY; csrc/render_cad.cu is checked against it bit for bit.

Camera chain (pinned against the reference's own render_cad / render_camera / get_camera_image
under oracle/ref_harness/render_cad_stub.py):
  * fovy = 2 degrees(arctan(H / (2 fy))) (trimesh.scene.Camera(resolution=(W, H),
    focal=(fx, fy)).fov[1], datasets/rgbd_pose_estimation/base.py:99-101, :139-146);
  * the view matrix render_camera builds from inv(T_cad2cam) is diag(1, -1, -1, 1) T_cad2cam: a
    CAD point goes to the camera frame by T_cad2cam, OpenCV axes, then to OpenGL's eye frame;
  * computeProjectionMatrixFOV(fovy, aspect = W / H, near = 0.01, far = 1000): a symmetric
    frustum, so pixels are square with f = (H / 2) / tan(radians(fovy) / 2) and the principal
    point at the image centre.  The frame's fx, cx and cy are not used.

Rasterisation rules (pybullet's projection formula and its TinyRenderer rasteriser cannot be run
here; these rules are PARITY UNPINNED against them):
  * p' = ((r0 x + r1 y) + r2 z) + t (float64); u = (f X) / Z + W / 2, v = (f Y) / Z + H / 2;
    snapped to 1/256 pixel, s = rint(256 u).  Pixel (r, c) covers [c, c+1) x [r, r+1), rows top
    first; its centre is (256 c + 128, 256 r + 128) in snapped units.
  * A triangle with a vertex at Z < near, a non-finite vertex, or a snapped coordinate beyond
    +-2^30 is dropped whole (OpenGL would clip it).  No back-face culling: a triangle of negative
    area is reoriented (b and c swapped).  Zero area covers nothing.
  * A centre is covered when the three int64 edge functions e(b,c), e(c,a), e(a,b) with
    e(a, b; p) = (bx - ax)(py - ay) - (by - ay)(px - ax) are all >= 0, where 0 counts only on a
    top or left edge (direction (dx, dy) with dy < 0, or dy == 0 and dx > 0: the D3D / OpenGL
    fill rule in y-down coordinates).  Two triangles sharing an edge cover each centre on it once.
  * Depth at a covered centre, with w_a = e(b,c), w_b = e(c,a), w_c = e(a,b) and A2 = twice the
    snapped area (= w_a + w_b + w_c):
        z = float32(A2 / ((float64(w_a) * (1 / Z_a) + float64(w_b) * (1 / Z_b))
                          + float64(w_c) * (1 / Z_c)))
    (perspective-correct interpolation of 1/Z); the pixel keeps the smallest z of the triangles
    covering it.  NaN where nothing covers (get_camera_image, :233).  mask = covered, count =
    mask.sum().
"""

import math

import numpy as np

NEAR = 0.01
FAR = 1000.0
SNAP = 256
LIMIT = 1 << 30


def fovy_from_intrinsics(fy, height):
    """trimesh.scene.Camera(resolution=(W, H), focal=(fx, fy)).fov[1], in degrees."""
    return 2.0 * np.degrees(np.arctan(height / (2.0 * fy)))


def focal_from_fovy(fovy, height):
    """The square pixels' focal length of computeProjectionMatrixFOV's frustum (float64)."""
    return (height / 2.0) / math.tan(math.radians(fovy) / 2.0)


def view_matrix(T_cad2cam):
    """The OpenGL view matrix render_camera builds (:237-247), as a 4x4 acting on column
    vectors (pybullet reads the flattened matrix column-major)."""
    return np.diag([1.0, -1.0, -1.0, 1.0]) @ np.asarray(T_cad2cam, np.float64)


def projection_matrix(fovy, aspect, near=NEAR, far=FAR):
    """gluPerspective's matrix, which computeProjectionMatrixFOV is documented to build (the
    formula pybullet runs is not pinned here)."""
    t = 1.0 / math.tan(math.radians(fovy) / 2.0)
    return np.array([[t / aspect, 0, 0, 0], [0, t, 0, 0],
                     [0, 0, (far + near) / (near - far), 2 * far * near / (near - far)],
                     [0, 0, -1, 0]], np.float64)


def gl_pixel(view, proj, height, width, p):
    """(u, v) of CAD point p through view, projection and the viewport, rows top first."""
    c = proj @ (view @ np.r_[np.asarray(p, np.float64), 1.0])
    ndc = c[:3] / c[3]
    return (ndc[0] + 1.0) * width / 2.0, (1.0 - ndc[1]) * height / 2.0


def _floor256(a):
    return a >> 8


def _ceil256(a):
    return -((-a) >> 8)


def _top_left(dx, dy):
    return (dy < 0) | ((dy == 0) & (dx > 0))


def setup(vertices, faces, T, f, height, width):
    """The per-face records of one pose (k_rc_setup): a dict of arrays over the faces --
    ``valid`` (every vertex kept), ``keep`` (also non-zero area and a non-empty pixel box),
    snapped ``sx``/``sy`` [F,3] int64 oriented to positive area, ``iz`` [F,3] float64, ``a2``
    int64, ``tl`` [F,3] bool (edges b->c, c->a, a->b), pixel ``box`` [F,4] (c0, r0, c1, r1)."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    T = np.asarray(T, np.float64).reshape(4, 4)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    with np.errstate(all="ignore"):
        X = ((T[0, 0] * x + T[0, 1] * y) + T[0, 2] * z) + T[0, 3]
        Y = ((T[1, 0] * x + T[1, 1] * y) + T[1, 2] * z) + T[1, 3]
        Z = ((T[2, 0] * x + T[2, 1] * y) + T[2, 2] * z) + T[2, 3]
        su = np.rint(((f * X) / Z + 0.5 * width) * SNAP)
        sv = np.rint(((f * Y) / Z + 0.5 * height) * SNAP)
        iz = 1.0 / Z
        ok = ((Z >= NEAR) & np.isfinite(X) & np.isfinite(Y) & np.isfinite(Z)
              & (np.abs(su) <= LIMIT) & (np.abs(sv) <= LIMIT))
    su = np.where(ok, su, 0).astype(np.int64)
    sv = np.where(ok, sv, 0).astype(np.int64)
    valid = ok[fc].all(1) if len(fc) else np.zeros(0, bool)
    sx, sy, izf = su[fc].copy(), sv[fc].copy(), iz[fc].copy()
    a2 = (sx[:, 1] - sx[:, 0]) * (sy[:, 2] - sy[:, 0]) - (sy[:, 1] - sy[:, 0]) * (sx[:, 2] - sx[:, 0])
    neg = a2 < 0
    for a in (sx, sy, izf):
        a[neg, 1], a[neg, 2] = a[neg, 2].copy(), a[neg, 1].copy()
    a2 = np.abs(a2)
    c0 = np.maximum(_ceil256(sx.min(1) - SNAP // 2), 0)
    c1 = np.minimum(_floor256(sx.max(1) - SNAP // 2), width - 1)
    r0 = np.maximum(_ceil256(sy.min(1) - SNAP // 2), 0)
    r1 = np.minimum(_floor256(sy.max(1) - SNAP // 2), height - 1)
    keep = valid & (a2 != 0) & (c0 <= c1) & (r0 <= r1)
    tl = np.stack([_top_left(sx[:, 2] - sx[:, 1], sy[:, 2] - sy[:, 1]),
                   _top_left(sx[:, 0] - sx[:, 2], sy[:, 0] - sy[:, 2]),
                   _top_left(sx[:, 1] - sx[:, 0], sy[:, 1] - sy[:, 0])], 1)
    return dict(valid=valid, keep=keep, sx=sx, sy=sy, iz=izf, a2=a2, tl=tl,
                box=np.stack([c0, r0, c1, r1], 1))


def _edge(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def render_one(vertices, faces, T, f, height, width):
    """depth [H,W] float32 (NaN where nothing covers) and mask [H,W] bool of one pose."""
    s = setup(vertices, faces, T, f, height, width)
    depth = np.full((height, width), np.inf, np.float32)
    mask = np.zeros((height, width), bool)
    for i in np.flatnonzero(s["keep"]):
        c0, r0, c1, r1 = (int(t) for t in s["box"][i])
        (ax, bx, cx), (ay, by, cy) = s["sx"][i], s["sy"][i]
        px = np.arange(c0, c1 + 1, dtype=np.int64)[None, :] * SNAP + SNAP // 2
        py = np.arange(r0, r1 + 1, dtype=np.int64)[:, None] * SNAP + SNAP // 2
        wa = _edge(bx, by, cx, cy, px, py)
        wb = _edge(cx, cy, ax, ay, px, py)
        wc = _edge(ax, ay, bx, by, px, py)
        tl = s["tl"][i]
        inside = (((wa > 0) | ((wa == 0) & tl[0])) & ((wb > 0) | ((wb == 0) & tl[1]))
                  & ((wc > 0) | ((wc == 0) & tl[2])))
        if not inside.any():
            continue
        iza, izb, izc = s["iz"][i]
        den = (wa.astype(np.float64) * iza + wb.astype(np.float64) * izb) + wc.astype(np.float64) * izc
        with np.errstate(all="ignore"):
            z = (np.float64(s["a2"][i]) / den).astype(np.float32)
        win = depth[r0:r1 + 1, c0:c1 + 1]
        win[inside] = np.minimum(win[inside], z[inside])
        mask[r0:r1 + 1, c0:c1 + 1] |= inside
    depth[~mask] = np.nan
    return depth, mask


def render_cad(vertices, faces, Ts_cad2cam, f, height, width):
    """depth [N,H,W] float32, mask [N,H,W] bool and count [N] int64 of N poses [N,4,4]."""
    Ts = np.asarray(Ts_cad2cam, np.float64).reshape(-1, 4, 4)
    out = [render_one(vertices, faces, T, f, height, width) for T in Ts]
    depth = np.stack([d for d, _ in out]) if out else np.zeros((0, height, width), np.float32)
    mask = np.stack([m for _, m in out]) if out else np.zeros((0, height, width), bool)
    return depth, mask, mask.reshape(len(Ts), height * width).sum(1)


# ---------------------------------------------------------------------------------------------
# independent control: a float64 Moller-Trumbore ray test at every pixel centre
# ---------------------------------------------------------------------------------------------
def moller_trumbore_mask(vertices, faces, T, f, height, width, eps=1e-6):
    """(covered, decided) [H,W] bool: ``covered`` by a float64 Moller-Trumbore test of the ray
    through each pixel centre against every triangle the rules keep (every vertex valid), each
    rebuilt in the camera frame from its snapped projection at its vertices' depths; ``decided``
    where the centre lies farther than ``eps`` pixels from every snapped edge of those triangles
    (elsewhere the fill rule, not geometry, decides)."""
    s = setup(vertices, faces, T, f, height, width)
    cc, rr = np.meshgrid(np.arange(width) + 0.5, np.arange(height) + 0.5)
    d = np.stack([(cc - width / 2.0) / f, (rr - height / 2.0) / f, np.ones_like(cc)], -1)
    covered = np.zeros((height, width), bool)
    decided = np.ones((height, width), bool)
    for i in np.flatnonzero(s["valid"]):
        U, Vv, Z = s["sx"][i] / SNAP, s["sy"][i] / SNAP, 1.0 / s["iz"][i]
        P = np.stack([(U - width / 2.0) / f * Z, (Vv - height / 2.0) / f * Z, Z], 1)
        e1, e2 = P[1] - P[0], P[2] - P[0]
        h = np.cross(d, e2)
        a = h @ e1
        with np.errstate(all="ignore"):
            inv = 1.0 / a
            sv = -P[0]
            uu = inv * (h @ sv)
            q = np.cross(sv, e1)
            vv = inv * (d @ q)
            t = inv * (q @ e2)
        covered |= (a != 0) & (uu >= 0) & (vv >= 0) & (uu + vv <= 1) & (t > 0)
        for k in range(3):
            a0 = np.array([U[k], Vv[k]])
            b0 = np.array([U[(k + 1) % 3], Vv[(k + 1) % 3]])
            ab = b0 - a0
            L2 = ab @ ab
            ap = np.stack([cc - a0[0], rr - a0[1]], -1)
            tt = np.clip((ap @ ab) / L2, 0, 1) if L2 > 0 else np.zeros_like(cc)
            dist = np.linalg.norm(ap - tt[..., None] * ab, axis=-1)
            decided &= dist > eps
    return covered, decided
