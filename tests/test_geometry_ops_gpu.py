"""GPU: the standalone geometry operators (occupancy_grid_3d, max_voxelization_3d,
truncated_distance_function, pseudo_occupancy_voxelization, the transform operators) and their
closed-loop caller (contrib.OccupancyRegistration with optimizers.ChainerAdam) against float64
references, at the sizes their callers run.

Two kinds of claim, as in tests/test_loss_gpu.py and tests/test_train_backward_gpu.py:
  * bit-exact: against the fp32 oracle (oracle/voxel_ops.py, oracle/transforms.py) or an fp32
    NumPy restatement of the stated expression order (csrc/tdf.cu, voxelization.cu and
    transforms.cu are built with -fmad=false);
  * bounded: an fp32 result is held to c * 2^-24 * sum|terms| of a float64 reference fed with the
    kernel's own fp32 inputs, c taken from the rounding chain stated beside the comparison, and
    the same bound must reject a deliberately wrong reference (`control`).
Every bounded comparison prints its worst err / bound ratio."""

import math

import numpy as np
import pytest
import torch

from _bounds import U, check, control
from oracle import icc as oicc
from oracle import transforms as otf
from oracle import voxel_ops as vo

pytestmark = pytest.mark.gpu

F32 = np.float32
F64 = torch.float64
SQ3 = math.sqrt(3.0)


def cu(x, dev, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x), device=dev)
    return t if dtype is None else t.to(dtype)


def F():
    import morefusion_b200
    return morefusion_b200.functions


def abi():
    from morefusion_b200 import _lib
    return _lib


def t64(a):
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().double()
    return torch.as_tensor(np.asarray(a, dtype=np.float64))


def held(name, got, ref, tol):
    """`check` on host arrays, printing the worst err / bound ratio."""
    got = got.detach().cpu() if isinstance(got, torch.Tensor) else torch.as_tensor(np.asarray(got))
    worst = check(name, got, t64(ref), t64(tol))
    print(f"[err/bound] {name}: {worst:.3g}")
    return worst


def rejected(name, got, wrong, tol):
    got = got.detach().cpu() if isinstance(got, torch.Tensor) else torch.as_tensor(np.asarray(got))
    control(name, got, t64(wrong), t64(tol))


def c_chain(n):
    """Depth of the 256-thread block reduction over n terms (serial, butterfly, 8 warps)."""
    return -(-n // 256) + 5 + 8


# a YCB class at the grid size of the refinement: pitch of the 32^3 grid around the object
PITCH = F32(0.0063)
CENTRE = np.array([0.1, 0.2, 0.7])


def ycb_origin(dims, pitch=PITCH):
    return (CENTRE - float(pitch) * (np.array(dims) - 1) / 2.0).astype(F32)


# ================================================================== 1  occupancy_grid_3d
def occ_chunks(pts, pitch, origin, dims, chunk=256):
    """The oracle materialises [X, Y, Z, P]: run it over chunks of points."""
    for s in range(0, len(pts), chunk):
        m, aux = vo.occupancy_grid_3d_fwd(pts[s:s + chunk], pitch=pitch, origin=origin, dims=dims)
        yield s, m, aux


def occ_dmin(pts, pitch, origin, dims):
    """min_p of the oracle's fp32 distances [X, Y, Z] (a minimum is exact, so chunking is)."""
    dmin = np.full(dims, np.inf, F32)
    for _, _, aux in occ_chunks(pts, pitch, origin, dims):
        dmin = np.minimum(dmin, aux["dmin"])
    return dmin


def occ_grid_of(dmin, threshold):
    """The oracle's last two lines, applied to the chunk-wise minimum."""
    m = np.maximum(F32(threshold) - dmin, F32(0)).astype(F32)
    return np.minimum(m, F32(1))


def occ_tied_pairs(pts, dmin, pitch, origin, dims):
    """Every (voxel, point) whose fp32 distance equals the voxel's fp32 minimum -- the kernel's
    selection rule `d == dmin` -- sorted by voxel, then point: v, p, d [n], dd [n, 3] (fp32)."""
    V = int(np.prod(dims))
    vs, ps, ds, dds = [], [], [], []
    for s, _, aux in occ_chunks(pts, pitch, origin, dims):
        sel = (aux["d"] == dmin[..., None]).reshape(V, -1)
        v, j = np.nonzero(sel)
        vs.append(v)
        ps.append(j + s)
        ds.append(aux["d"].reshape(V, -1)[v, j])
        dds.append(np.stack([aux[k].reshape(V, -1)[v, j] for k in ("d0", "d1", "d2")], 1))
    v, p, d, dd = (np.concatenate(a) for a in (vs, ps, ds, dds))
    order = np.lexsort((p, v))
    return v[order], p[order], d[order], dd[order]


def occ_bwd_ref(gm, pairs, dmin, P, *, pitch, threshold, first_tie_only=False, gate=True,
                p_limit=None):
    """float64 gpoints [P, 3], sum|terms| [P, 3] and the number of terms per point.

    A term is gm[v] * dd / (d * pitch) for a tied minimum (v, p) of a voxel with
    0 < threshold - dmin <= 1, with the kernel's own fp32 d, dd, dmin and gm: the kernel rounds
    gd / d, (.) * dd and (.) / pitch, then adds the term to the point with an atomic.
    first_tie_only / gate=False / p_limit: the deliberately wrong references."""
    v, p, d, dd = pairs
    r = (F32(threshold) - dmin.reshape(-1)).astype(F32)
    active = (r > 0) & (r <= 1) if gate else (r > 0)
    keep = active[v]
    if p_limit is not None:
        keep &= p < p_limit
    if first_tie_only:
        first = np.ones(len(v), bool)
        first[1:] = v[1:] != v[:-1]
        keep &= first
    v, p, d, dd = v[keep], p[keep], d[keep].astype(np.float64), dd[keep].astype(np.float64)
    g = np.asarray(gm, np.float64).reshape(-1)[v]
    with np.errstate(invalid="ignore", divide="ignore"):
        terms = g[:, None] * dd / (d[:, None] * float(pitch))
    ref, absref = np.zeros((P, 3)), np.zeros((P, 3))
    np.add.at(ref, p, terms)
    np.add.at(absref, p, np.abs(terms))
    return ref, absref, np.bincount(p, minlength=P)


OCC_CASES = {
    # name: P, dims, threshold, geometry, controls
    "p0": dict(P=0, dims=(16, 16, 16), thr=1, geom="ycb"),
    "p1": dict(P=1, dims=(5, 5, 5), thr=1, geom="unit"),
    "p255": dict(P=255, dims=(7, 9, 11), thr=2, geom="ycb", controls=("gate",)),
    "p256": dict(P=256, dims=(16, 16, 16), thr=2.5, geom="ycb"),
    "p257": dict(P=257, dims=(16, 16, 16), thr=2, geom="ycb", controls=("tile", "gate")),
    "p600": dict(P=600, dims=(16, 16, 16), thr=2, geom="ycb", controls=("tile", "gate")),
    "p1000": dict(P=1000, dims=(32, 32, 32), thr=2, geom="ycb", controls=("tile", "gate")),
    "p4000": dict(P=4000, dims=(32, 32, 32), thr=1, geom="ycb", controls=("tile",)),
    "p1000_unit": dict(P=1000, dims=(7, 9, 11), thr=1, geom="unit", controls=("tile",)),
    # ties: a lattice midway between the voxel centres (8 points tie for a voxel), part of it
    # repeated in the second tile of 256
    "lattice": dict(P=300, dims=(5, 5, 5), thr=1, geom="lattice", controls=("tie", "tile")),
    # every point twice, 300 apart: each minimum is tied across two tiles
    "duplicates": dict(P=600, dims=(16, 16, 16), thr=2, geom="dup", controls=("tie", "tile", "gate")),
    # a point exactly on a voxel centre: d = 0, the gradient is 0/0 on both sides
    "on_centre": dict(P=42, dims=(5, 5, 5), thr=1, geom="centre"),
}


def occ_inputs(name):
    c = OCC_CASES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    P, dims = c["P"], c["dims"]
    D = np.array(dims, np.float64)
    if c["geom"] in ("ycb", "dup"):
        pitch, origin = PITCH, ycb_origin(dims)
        n = P // 2 if c["geom"] == "dup" else P
        # two voxels beyond the grid on every side: points partly outside
        pts = CENTRE + rs.uniform(-0.5, 0.5, (n, 3)) * (D + 3.0) * float(pitch)
        if c["geom"] == "dup":
            pts = np.concatenate([pts, pts])
    else:
        pitch, origin = F32(1), np.zeros(3, F32)
        if c["geom"] == "unit":
            pts = rs.uniform(-1.5, 1.0, (P, 3)) + rs.uniform(0, 1, (P, 3)) * D
        elif c["geom"] == "lattice":
            a = np.arange(-1, 5) + 0.5
            lat = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
            pts = np.concatenate([lat, lat[rs.permutation(len(lat))[:P - len(lat)]]])
        else:
            pts = np.concatenate([rs.uniform(-0.5, 4.5, (P - 2, 3)), [[2, 2, 2], [3, 1, 4]]])
    return np.ascontiguousarray(pts, F32), pitch, origin


@pytest.mark.parametrize("name", list(OCC_CASES))
def test_occupancy_grid_3d(cuda_device, name):
    """Forward: grid and the saved minimum distance bit-exact against the oracle, which takes
    min_p sqrt(s_p) where the kernel takes sqrt(min_p s_p).

    Backward bound.  Each term is three correctly rounded operations on the kernel's own fp32
    values (gd / d, * dd, / pitch: relative error <= 3u) and the n_p terms of a point are added by
    atomics in an unspecified order (any order: <= (n_p - 1) u sum|terms|), so
    |gpoints - ref| <= (n_p + 3) u sum|terms| per point, with a unit of margin for the
    second-order terms.  Run-to-run equality is not claimed (atomics)."""
    c = OCC_CASES[name]
    L = abi()
    pts, pitch, origin = occ_inputs(name)
    dims, thr, P = c["dims"], c["thr"], c["P"]
    o3 = [float(o) for o in origin]
    p_d = cu(pts, cuda_device).requires_grad_(True)
    grid = torch.empty(dims, dtype=torch.float32, device=cuda_device)
    dmin = torch.empty(dims, dtype=torch.float32, device=cuda_device)
    with torch.cuda.device(cuda_device):
        rc = L.lib().mf_occupancy_grid_3d_fwd(L.ptr(p_d), P, float(pitch), *o3, *dims, float(thr),
                                              L.ptr(grid), L.ptr(dmin), L.stream())
    L.check(rc, "occupancy_grid_3d")
    m = F().occupancy_grid_3d(p_d, pitch=pitch, origin=origin, dims=dims, threshold=thr)
    assert torch.equal(m.detach(), grid)
    if P == 0:
        assert bool(torch.isinf(dmin).all()) and float(grid.abs().max()) == 0.0
        m.sum().backward()
        assert tuple(p_d.grad.shape) == (0, 3)
        return
    dmin_ref = occ_dmin(pts, pitch, origin, dims)
    if P <= 256:        # one chunk: the oracle's own grid is the restated last two lines
        m_or, _ = vo.occupancy_grid_3d_fwd(pts, pitch=pitch, origin=origin, dims=dims, threshold=thr)
        assert np.array_equal(m_or, occ_grid_of(dmin_ref, thr))
    assert np.array_equal(dmin.cpu().numpy(), dmin_ref)
    assert np.array_equal(grid.cpu().numpy(), occ_grid_of(dmin_ref, thr))

    rs = np.random.RandomState(7)
    gm = rs.uniform(-1, 1, dims).astype(F32)
    m.backward(cu(gm, cuda_device))
    got = p_d.grad.cpu().numpy()
    pairs = occ_tied_pairs(pts, dmin_ref, pitch, origin, dims)
    kw = dict(pitch=pitch, threshold=thr)
    ref, absref, n = occ_bwd_ref(gm, pairs, dmin_ref, P, **kw)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)
    assert bool(nan.any()) == (name == "on_centre")
    got, ref, absref = (np.where(nan, 0.0, a) for a in (got, ref, absref))
    tol = (n + 3)[:, None] * U * absref
    held(f"occupancy_grid_3d bwd {name}", got, ref, tol)
    assert absref.sum() > 0
    for ctl in c.get("controls", ()):
        wrong = occ_bwd_ref(gm, pairs, dmin_ref, P, **kw, **{
            "tile": dict(p_limit=256), "tie": dict(first_tie_only=True), "gate": dict(gate=False),
        }[ctl])[0]
        rejected(f"occupancy_grid_3d bwd {name} / {ctl}", got, np.where(nan, 0.0, wrong), tol)


# ================================================================== 2  OccupancyRegistration
def quat_table64(qs):
    """quaternion_matrix's table on the scaled quaternion qs = q sqrt(2 / |q|^2), (w, x, y, z)."""
    w, x, y, z = qs.unbind(-1)
    R = torch.stack([1 - y * y - z * z, x * y - z * w, x * z + y * w,
                     x * y + z * w, 1 - x * x - z * z, y * z - x * w,
                     x * z - y * w, y * z + x * w, 1 - x * x - y * y], -1)
    return R.reshape(qs.shape[:-1] + (3, 3))


def quat_R64(q):
    """float64 rotation of q, normalised inside."""
    return quat_table64(q * torch.sqrt(2.0 / (q * q).sum(-1, keepdim=True)))


def unnormalised_R64(q):
    """The normalisation left out, q sqrt2 in the table: wrong unless |q| = 1."""
    return quat_table64(q * math.sqrt(2.0))


def link64(q, t, pts, target, *, pitch, origin, thr, sel=None, gate=True,
           penalty_over_occupied=False):
    """float64 restatement of OccupancyRegistrationLink.forward: quaternion -> matrix -> points ->
    the min / relu / minimum chain -> reward and penalty.  q, t are float64 leaves.

    sel = (v, p, r32): the tie set (every fp32 `d == dmin` pair, sorted by voxel) and the fp32
    threshold - dmin that decides the relu / minimum branches, so that the branch taken is the
    kernel's; each tied point receives the whole gradient, as F.min gives it.  sel = None: the
    float64 minimum and branches.  Returns loss and the graph's x [P, 3], m [V] (grads retained)."""
    dims = tuple(target.shape[1:])
    V = int(np.prod(dims))
    o = t64(np.asarray(origin, np.float64))
    x = pts @ quat_R64(q).T + t
    x.retain_grad()
    qv = (x - o) / float(pitch)
    ijk = torch.stack(torch.meshgrid(*(torch.arange(d, dtype=F64) for d in dims), indexing="ij"),
                      -1).reshape(V, 3)
    if sel is None:
        v = torch.arange(V)
        p = torch.cdist(ijk, qv.detach()).argmin(1)
    else:
        v, p = torch.as_tensor(sel[0]), torch.as_tensor(sel[1])
    d = (ijk[v] - qv[p]).norm(dim=1)
    first = torch.ones(len(v), dtype=torch.bool)
    first[1:] = v[1:] != v[:-1]
    zero = torch.zeros(V, dtype=F64)
    dmin = zero.index_add(0, v[first], d[first].detach()) + zero.index_add(0, v, d - d.detach())
    r = float(thr) - dmin
    rg = r.detach() if sel is None else t64(sel[2]).reshape(-1)
    m = torch.where(rg > 0, r, zero)
    if gate:
        m = torch.where(rg > 1, torch.ones_like(m), m)
    m.retain_grad()
    occupied = target[0].reshape(-1)
    unoccupied = (torch.maximum(target[1], target[2]) if target.shape[0] == 3 else target[1]).reshape(-1)
    reward = (occupied * m).sum() / occupied.sum()
    penalty = (unoccupied * m).sum() / (occupied.sum() if penalty_over_occupied else m.sum())
    return -reward + penalty, x, m


def registration_fixture(D, n_points, channels):
    """The box of test_model_api_gpu.py::test_occupancy_registration_recovers_translation: surface
    points, its occupied / unoccupied grids, a 1.5-voxel offset."""
    from morefusion_b200 import synthetic
    rs = np.random.RandomState(0)
    pitch = 0.16 / D
    half = np.array([0.04, 0.03, 0.02])
    pts = synthetic.surface_points("box", half, n_points, rs).astype(F32)
    origin = (-(D / 2.0 - 0.5) * pitch,) * 3
    ijk = np.stack(np.meshgrid(*(np.arange(D),) * 3, indexing="ij"), -1) * pitch + np.array(origin)
    d = synthetic.sdf_primitive("box", half, ijk)
    grids = [(np.abs(d) < 0.75 * pitch), (d < -1.5 * pitch)]
    if channels == 3:
        grids.append((ijk[..., 0] > 0.05) | (rs.rand(D, D, D) < 0.05))
    t0 = np.array([1.5, -1.0, 0.5], F32) * F32(pitch)
    return pts, np.stack(grids).astype(F32), pitch, origin, t0


@pytest.mark.parametrize("channels", [2, 3])
@pytest.mark.parametrize("D,n_points", [(16, 600), (32, 1000)])
def test_registration_link_forward_backward(cuda_device, D, n_points, channels):
    """One forward / backward of OccupancyRegistrationLink against float64.

    Loss, given the link's own fp32 grid: two ratios of sums over V = X Y Z voxels.  Any order of
    n additions is within (n - 1) u sum|terms|, each product and each division adds one rounding:
    |loss - ref| <= (2V + 3) u (|reward| + |penalty|).

    Gradients, against float64 autograd of the whole chain with the tie set and the branches taken
    from the fp32 distances.  First order in three error sources:
      * a voxel coordinate (x - o) / pitch of point p carries e_q = 16u (A_p + |o|) / pitch, with
        A_p = |R||p| + |t|: 4u A_p from the transform, <= 8u |p| from R, 2u (|x| + |o|) from the
        subtraction and division; it turns the unit vector of a pair by <= 2 sqrt3 e_q / d;
      * d loss / d grid is three ratios of the same grid sums, relative error
        rel = 3 ((V + 2) u + sqrt3 max(e_q) n_active / sum(grid)) (the grid's own error moves
        sum(grid));
      * the occupancy backward's chain, (n_p + 3) u per point (test_occupancy_grid_3d).
    That gives tol_gx per point; d translation sums it over P points (k_tp_bwd_T: ceil(P/256) + 13),
    gR sums gx (x) p (one more rounding), and d quaternion is k_quat_bwd's c = 26 on
    |J|^T |gR| plus |J|^T tol_gR (tests/test_loss_gpu.py).
    These are worst cases added up and are loose (err / bound around 1e-5 on an H100): this test
    shows that the stages are wired as the reference wires them, which the controls confirm it can
    see; the stages themselves are held to their own chains by the other tests of this file."""
    from morefusion_b200.contrib.occupancy_registration import OccupancyRegistrationLink
    f = F()
    pts, target, pitch, origin, t0 = registration_fixture(D, n_points, channels)
    q0 = np.array([0.98, 0.05, -0.08, 0.1], F32) * F32(1.3)      # not a unit quaternion
    thr = 2
    dims = (D, D, D)
    V = D ** 3
    link = OccupancyRegistrationLink(q0, t0).to(cuda_device)
    p_d, g_d = cu(pts, cuda_device), cu(target, cuda_device)
    loss = link(points_source=p_d, grid_target=g_d, pitch=pitch, origin=origin, threshold=thr)
    loss.backward()
    with torch.no_grad():    # the link's own intermediates (the kernels are deterministic)
        T = f.compose_transform(f.quaternion_matrix(link.quaternion[None])[:, :3, :3],
                                link.translation[None])
        x32 = f.transform_points(p_d, T)[0]
        grid32 = f.occupancy_grid_3d(x32, pitch=pitch, origin=origin, dims=dims, threshold=thr)

    # ---- loss, given the fp32 grid
    tg, m32 = t64(target), t64(grid32).reshape(-1)
    occ = tg[0].reshape(-1)
    un = (torch.maximum(tg[1], tg[2]) if channels == 3 else tg[1]).reshape(-1)
    reward, penalty = (occ * m32).sum() / occ.sum(), (un * m32).sum() / m32.sum()
    tol_loss = (2 * V + 3) * U * (reward.abs() + penalty.abs())
    tag = f"registration link D={D} C={channels}"
    held(f"{tag} loss", loss.reshape(1), (-reward + penalty).reshape(1), tol_loss.reshape(1))
    rejected(f"{tag} loss / penalty over occupied", loss.reshape(1),
             (-reward + (un * m32).sum() / occ.sum()).reshape(1), tol_loss.reshape(1))
    if channels == 3:
        rejected(f"{tag} loss / second unoccupied channel ignored", loss.reshape(1),
                 (-reward + (tg[1].reshape(-1) * m32).sum() / m32.sum()).reshape(1),
                 tol_loss.reshape(1))

    # ---- gradients: float64 autograd with the fp32 tie set
    o32 = np.asarray(origin, F32)
    x_np = x32.cpu().numpy()
    dmin32 = occ_dmin(x_np, F32(pitch), o32, dims)
    assert np.array_equal(grid32.cpu().numpy(), occ_grid_of(dmin32, thr))
    v, p, _, _ = occ_tied_pairs(x_np, dmin32, F32(pitch), o32, dims)
    r32 = (F32(thr) - dmin32).astype(F32)
    q64 = t64(q0).requires_grad_(True)
    tr64 = t64(t0).requires_grad_(True)
    kw = dict(pitch=float(F32(pitch)), origin=o32, thr=thr, sel=(v, p, r32))
    loss64, x64, m64 = link64(q64, tr64, t64(pts), tg, **kw)
    loss64.backward()

    P = n_points
    pitch_f = float(F32(pitch))
    R64 = quat_R64(q64.detach())
    A = t64(pts).abs() @ R64.abs().T + tr64.detach().abs()                       # [P, 3]
    e_q = 16 * U * (A.max(1).values + float(np.abs(o32).max())) / pitch_f        # [P]
    act = torch.as_tensor((r32.reshape(-1) > 0) & (r32.reshape(-1) <= 1))
    md = m64.detach()
    rel = 3 * ((V + 2) * U + SQ3 * float(e_q.max()) * float((md > 0).sum()) / float(md.sum()))
    vt, pt = torch.as_tensor(v), torch.as_tensor(p)
    keep = act[vt]
    vt, pt = vt[keep], pt[keep]
    ijk = torch.stack(torch.meshgrid(*(torch.arange(d, dtype=F64) for d in dims), indexing="ij"),
                      -1).reshape(V, 3)
    dvec = ijk[vt] - (x64.detach()[pt] - t64(o32)) / pitch_f
    d = dvec.norm(dim=1)
    w = m64.grad[vt].abs() / pitch_f
    term_abs = w[:, None] * dvec.abs() / d[:, None]
    n_p = torch.bincount(pt, minlength=P).double()
    tol_pair = (w * 2 * SQ3 * e_q[pt] / d)[:, None] + term_abs * (rel + (n_p[pt] + 3) * U)[:, None]
    zero = torch.zeros(P, 3, dtype=F64)
    tol_gx, abs_gx = zero.index_add(0, pt, tol_pair), zero.index_add(0, pt, term_abs)
    cP = c_chain(P)
    tol_gt = tol_gx.sum(0) + cP * U * abs_gx.sum(0)
    held(f"{tag} d translation", link.translation.grad, tr64.grad, tol_gt)
    pa = t64(pts).abs()
    abs_gR = abs_gx.T @ pa
    tol_gR = tol_gx.T @ pa + (cP + 1) * U * abs_gR
    J = torch.autograd.functional.jacobian(lambda z: quat_R64(z).reshape(9), q64.detach()).abs()
    tol_gq = J.T @ tol_gR.reshape(9) + 26 * U * (J.T @ abs_gR.reshape(9))
    held(f"{tag} d quaternion", link.quaternion.grad, q64.grad, tol_gq)

    # ---- the same bounds reject: saturated voxels (threshold - dmin > 1) passing gradient
    q_w, t_w = t64(q0).requires_grad_(True), t64(t0).requires_grad_(True)
    link64(q_w, t_w, t64(pts), tg, gate=False, **kw)[0].backward()
    rejected(f"{tag} d translation / no minimum(.,1) gate", link.translation.grad, t_w.grad, tol_gt)
    rejected(f"{tag} d quaternion / no minimum(.,1) gate", link.quaternion.grad, q_w.grad, tol_gq)


def adam64(p, m, v, g, t, *, alpha, beta1=0.9, beta2=0.999, eps=1e-8, eta=1.0, wd=0.0,
           m_new=None, v_new=None, torch_form=False):
    """float64 restatement of the rule in optimizers.ChainerAdam's docstring.  m_new / v_new:
    take the moments the step divides from the caller (the kernel's own fp32 ones)."""
    m1 = m + (1 - beta1) * (g - m)
    v1 = v + (1 - beta2) * (g * g - v)
    mm, vv = (m1 if m_new is None else m_new), (v1 if v_new is None else v_new)
    fix1, fix2 = 1 - beta1 ** t, 1 - beta2 ** t
    if torch_form:      # torch.optim.Adam: sqrt(v) / sqrt(1 - beta2^t) + eps
        step = alpha / fix1 * mm / (vv.sqrt() / math.sqrt(fix2) + eps)
    else:
        step = alpha * math.sqrt(fix2) / fix1 * mm / (vv.sqrt() + eps)
    return p - eta * (step + wd * p), m1, v1, step


@pytest.mark.parametrize("eta,wd", [(1.0, 0.0), (0.5, 0.0), (1.0, 1e-2), (0.7, 1e-3)])
def test_chainer_adam_vs_float64(cuda_device, eta, wd):
    """ChainerAdam step by step for 20 steps, two parameter groups with different alpha.

    Each step is checked from the optimizer's own fp32 state before it, so the bound is that
    step's roundings only: m' = m + fl(1 - beta1) (g - m) is a difference, a rounded constant, a
    product and a sum (c = 4 on |m| + (1 - beta1) |g - m|); v' has g g as well (c = 5); the
    parameter, from the fp32 m', v': alpha_t, product, sqrt, eps, sum, quotient, decay product,
    sum, eta product, difference (c = 10 on |p| + eta |step| + eta wd |p|).  torch.optim.Adam's
    form of the denominator must fail that bound (gradients down to 1e-6, where eps counts).
    Without weight decay the result also equals oracle/icc.py's restatement of the same rule, free
    running over the 20 steps, within 20 (|p| + 320 eta alpha) u: per step one rounding of p
    and <= 100 u on a step of at most 3.2 alpha."""
    from morefusion_b200.optimizers import ChainerAdam
    rs = np.random.RandomState(5)
    shapes, alphas = [(64,), (33,)], [0.01, 0.001]
    p0 = [rs.uniform(-1, 1, s).astype(F32) for s in shapes]
    params = [torch.nn.Parameter(cu(a, cuda_device)) for a in p0]
    opt = ChainerAdam([dict(params=[params[0]], alpha=alphas[0]),
                       dict(params=[params[1]], alpha=alphas[1])], eta=eta, weight_decay_rate=wd)
    orc = [oicc.ChainerAdam(s, a, eta=eta) for s, a in zip(shapes, alphas)]
    p_or = [a.copy() for a in p0]
    scale = [10.0 ** rs.uniform(-6, 0, s) for s in shapes]
    rows = {k: [] for k in ("m", "m_ref", "m_tol", "v", "v_ref", "v_tol", "p", "p_ref", "p_tol",
                            "p_wrong")}
    for t in range(1, 21):
        before = []
        for i, prm in enumerate(params):
            g = (rs.normal(size=shapes[i]) * scale[i]).astype(F32)
            st = opt.state[prm]
            zeros = torch.zeros(shapes[i], dtype=F64)
            before.append((t64(prm), t64(st["m"]) if st else zeros, t64(st["v"]) if st else zeros))
            prm.grad = cu(g, cuda_device)
            p_or[i] = orc[i].update(p_or[i], g)
        opt.step()
        for i, prm in enumerate(params):
            st = opt.state[prm]
            assert st["t"] == t
            p_b, m_b, v_b = before[i]
            g64 = t64(prm.grad)
            m_a, v_a = t64(st["m"]), t64(st["v"])
            kw = dict(alpha=alphas[i], eta=eta, wd=wd, m_new=m_a, v_new=v_a)
            p_ref, m_ref, v_ref, step = adam64(p_b, m_b, v_b, g64, t, **kw)
            p_wrong = adam64(p_b, m_b, v_b, g64, t, torch_form=True, **kw)[0]
            rows["m"].append(m_a), rows["m_ref"].append(m_ref)
            rows["m_tol"].append(4 * U * (m_b.abs() + 0.1 * (g64 - m_b).abs()))
            rows["v"].append(v_a), rows["v_ref"].append(v_ref)
            rows["v_tol"].append(5 * U * (v_b.abs() + 0.001 * (g64 * g64 + v_b)))
            rows["p"].append(t64(prm)), rows["p_ref"].append(p_ref), rows["p_wrong"].append(p_wrong)
            rows["p_tol"].append(10 * U * (p_b.abs() + eta * step.abs() + eta * wd * p_b.abs()))
    cat = {k: torch.cat(a) for k, a in rows.items()}
    tag = f"ChainerAdam eta={eta} wd={wd}"
    held(f"{tag} m", cat["m"], cat["m_ref"], cat["m_tol"])
    held(f"{tag} v", cat["v"], cat["v_ref"], cat["v_tol"])
    held(f"{tag} p", cat["p"], cat["p_ref"], cat["p_tol"])
    rejected(f"{tag} p / torch.optim.Adam's denominator", cat["p"], cat["p_wrong"], cat["p_tol"])
    if wd == 0.0:
        for i, prm in enumerate(params):
            tol = 20 * U * (np.abs(p_or[i]).astype(np.float64) + 320 * eta * alphas[i])
            held(f"{tag} vs oracle.icc.ChainerAdam, group {i}", prm, p_or[i], tol)


# |dt| (metres; the voxel is 0.01) and max |dR| allowed between the fp32 loop and its float64
# restatement after 10 iterations, and the translation error (0.0187 at the start) the 60
# iterations must reach.  Measured on an H100: 7.7e-10 and 4.6e-8 after 10 iterations, 1.7e-9 and
# 1.5e-7 after 20, 1.5e-5 and 4.9e-4 after 60 (the amplification described below); |t| = 0.0045
# at the end.
LOOP_TOL_T, LOOP_TOL_R, LOOP_FINAL_T = 1e-7, 2e-6, 0.006


def test_occupancy_registration_loop_vs_float64(cuda_device):
    """The 60 iterations of test_occupancy_registration_recovers_translation against the float64
    restatement (link64 + adam64) run on the host from the same initial (q, t), which are passed
    in: quaternion_from_matrix goes through LAPACK, whose last bits differ between CPUs.  Adam
    divides each gradient component by its own sqrt(v), so fp32 noise on a small component grows
    to O(alpha) with the iterations; the two loops are compared after 10 of them, where they
    still agree to a small fraction of a step (alpha = 0.01 for q, 0.001 for t), and the final
    translation error is held to a fixed value."""
    from morefusion_b200.contrib import OccupancyRegistration
    pts, target, pitch, origin, t0 = registration_fixture(16, 600, 2)
    q0 = np.array([1, 0, 0, 0], F32)
    T0 = np.eye(4, dtype=F32)
    T0[:3, 3] = t0
    alpha, thr = 0.01, 2
    reg = OccupancyRegistration(pts, target, pitch=pitch, origin=origin, threshold=thr,
                                transform_init=T0, gpu=cuda_device.index or 0, alpha=alpha)
    with torch.no_grad():
        reg._link.quaternion.copy_(cu(q0, cuda_device))
        reg._link.translation.copy_(cu(t0, cuda_device))
    got = list(reg.register_iterative(iteration=60))
    assert len(got) == 61

    q, t = t64(q0).requires_grad_(True), t64(t0).requires_grad_(True)
    state = {id(q): [torch.zeros(4, dtype=F64)] * 2, id(t): [torch.zeros(3, dtype=F64)] * 2}
    tg, p64 = t64(target), t64(pts)
    o32 = np.asarray(origin, F32)
    ref = []
    for k in range(1, 61):
        q.grad = t.grad = None
        link64(q, t, p64, tg, pitch=float(F32(pitch)), origin=o32, thr=thr)[0].backward()
        with torch.no_grad():
            for prm, a in ((q, alpha), (t, alpha * 0.1)):
                new, m1, v1, _ = adam64(prm, *state[id(prm)], prm.grad, k, alpha=a)
                prm.copy_(new)
                state[id(prm)] = [m1, v1]
        ref.append((quat_R64(q.detach()).numpy().copy(), t.detach().numpy().copy()))
    for k in (1, 2, 5, 10, 20, 60):
        dR = np.abs(got[k][:3, :3] - ref[k - 1][0]).max()
        dt = np.abs(got[k][:3, 3] - ref[k - 1][1]).max()
        print(f"[loop] iteration {k}: max|dR| {dR:.3g} max|dt| {dt:.3g} "
              f"|t| {np.linalg.norm(got[k][:3, 3]):.4g}")
    assert np.abs(got[10][:3, 3] - ref[9][1]).max() <= LOOP_TOL_T
    assert np.abs(got[10][:3, :3] - ref[9][0]).max() <= LOOP_TOL_R
    assert np.linalg.norm(ref[59][1]) < LOOP_FINAL_T
    assert np.linalg.norm(got[60][:3, 3]) < LOOP_FINAL_T


# ================================================================== 3  max_voxelization_3d
MAXVOX_SHAPES = {
    "model": dict(P=8000, C=144, B=8, dims=(32, 32, 32), sorted=True),
    "unsorted_noncubic": dict(P=5000, C=1, B=5, dims=(7, 9, 11), sorted=False),
    "collisions": dict(P=60000, C=5, B=2, dims=(16, 16, 16), sorted=True),
    "empty": dict(P=0, C=3, B=2, dims=(8, 8, 8), sorted=True),
}


def maxvox_inputs(shape, kind):
    s = MAXVOX_SHAPES[shape]
    rs = np.random.RandomState(11)
    P, C, B, dims = s["P"], s["C"], s["B"], s["dims"]
    origin = np.array([-1, -1, -1], F32)
    pitch = F32(2.0 / max(dims))
    pts = rs.uniform(-1.1, 1.1, (P, 3)).astype(F32)
    vals = rs.uniform(-1, 1, (P, C)).astype(F32)
    bi = rs.randint(0, B, P).astype(np.int32)
    if s["sorted"]:
        bi = np.sort(bi)
    inten = {
        "random": lambda: rs.uniform(-1, 1, P),
        "equal": lambda: np.full(P, 0.5),
        "ties": lambda: rs.randint(0, 5, P) / 4.0 - 0.5,            # -0.5 ... 0.5, zero included
        "negative": lambda: -rs.randint(1, 4, P) / 4.0,
        "signed_zero": lambda: np.where(rs.rand(P) < 0.5, 0.0, -0.0),
        "infinite": lambda: rs.choice([-np.inf, -1.0, -0.0, 0.0, 1.0, np.inf], P),
    }[kind]().astype(F32)
    return vals, pts, bi, inten, dict(batch_size=B, origin=origin, pitch=pitch, dimensions=dims)


@pytest.mark.parametrize("kind", ["random", "equal", "ties", "negative", "signed_zero", "infinite"])
@pytest.mark.parametrize("shape", list(MAXVOX_SHAPES))
def test_max_voxelization_vs_oracle(cuda_device, shape, kind):
    """Matrix, indices and gvalues bit-exact: the winner of a voxel is the largest intensity as
    `>` orders it (-0 == +0, the infinities included), the lowest point id among equals."""
    vals, pts, bi, inten, kw = maxvox_inputs(shape, kind)
    P = len(pts)
    want_m, want_i = vo.max_voxelization_3d_fwd(vals, pts, bi, inten, **kw)
    v = cu(vals, cuda_device).requires_grad_(True)
    y, ind = F().max_voxelization_3d(v, cu(pts, cuda_device), cu(bi, cuda_device),
                                     cu(inten, cuda_device), return_indices=True, **kw)
    assert np.array_equal(ind.cpu().numpy(), want_i)
    assert np.array_equal(y.detach().cpu().numpy(), want_m)
    if P == 0:
        assert tuple(y.shape) == (kw["batch_size"], vals.shape[1]) + kw["dimensions"]
        assert float(y.detach().abs().max()) == 0.0 and bool((ind == -1).all())
        return
    gy = np.random.RandomState(12).uniform(-1, 1, want_m.shape).astype(F32)
    y.backward(cu(gy, cuda_device))
    assert np.array_equal(v.grad.cpu().numpy(), vo.max_voxelization_3d_bwd(gy, want_i, P))
    if kind == "ties":      # the tie-break is visible: the highest id among equals is another grid
        rev = vo.max_voxelization_3d_fwd(vals[::-1], pts[::-1], bi[::-1], inten[::-1], **kw)[1]
        assert not np.array_equal(want_i, np.where(rev >= 0, P - 1 - rev, -1))


def test_max_voxelization_nan_intensity(cuda_device):
    """The reference's result with a NaN intensity depends on arrival order (`>` is false both
    ways: whichever point reaches the voxel first keeps it), so only the finite cases above are
    pinned to it.  The kernel defines the case: a NaN of either sign ranks above every number,
    the lowest id among NaNs wins -- the oracle's result with the NaNs replaced by +inf; voxels
    that hold no NaN are as if the NaN points were absent."""
    vals, pts, bi, inten, kw = maxvox_inputs("unsorted_noncubic", "ties")
    rs = np.random.RandomState(13)
    nan = rs.rand(len(inten)) < 0.05
    bits = inten.view(np.uint32).copy()
    bits[nan] = np.where(rs.rand(int(nan.sum())) < 0.5, 0x7fc00000, 0xffc00001).astype(np.uint32)
    inten = bits.view(F32)
    assert np.isnan(inten).sum() == nan.sum() > 0
    want_m, want_i = vo.max_voxelization_3d_fwd(vals, pts, bi, np.where(nan, F32(np.inf), inten), **kw)
    y, ind = F().max_voxelization_3d(cu(vals, cuda_device), cu(pts, cuda_device), cu(bi, cuda_device),
                                     cu(inten, cuda_device), return_indices=True, **kw)
    assert np.array_equal(ind.cpu().numpy(), want_i)
    assert np.array_equal(y.cpu().numpy(), want_m)


def test_max_voxelization_flags_and_losers_gradient(cuda_device):
    """Through the C ABI.  A batch index outside [0, B) drops the point and sets
    MF_FLAG_BAD_BATCH_INDEX, a NaN point sets MF_FLAG_NAN_POINTS; the public function raises
    ValueError("points include nan") and drops the bad batch index, both as
    average_voxelization_3d does.  The backward writes every element of gvalues: a point that wins
    no voxel has gradient exactly 0 on a buffer that held NaN."""
    L = abi()
    vals, pts, bi, inten, kw = maxvox_inputs("unsorted_noncubic", "ties")
    P, C = vals.shape
    B, dims, pitch = kw["batch_size"], kw["dimensions"], float(kw["pitch"])
    o3 = [float(o) for o in kw["origin"]]
    bad = np.arange(P) % 97 == 0
    bi_bad = np.where(bad, np.where(np.arange(P) % 2 == 0, -1, B), bi).astype(np.int32)
    far = np.where(bad[:, None], F32(50.0), pts)                 # the oracle's view: absent points
    want_m, want_i = vo.max_voxelization_3d_fwd(vals, far, bi, inten, **kw)

    def fwd(points, batch):
        d = [cu(a, cuda_device) for a in (vals, points, batch, inten)]
        matrix = torch.empty((B, C) + dims, dtype=torch.float32, device=cuda_device)
        indices = torch.empty((B,) + dims, dtype=torch.int32, device=cuda_device)
        flags = torch.zeros(1, dtype=torch.int32, device=cuda_device)
        ws = torch.empty(L.lib().mf_max_voxelization_3d_workspace_bytes(B, *dims),
                         dtype=torch.uint8, device=cuda_device)
        with torch.cuda.device(cuda_device):
            rc = L.lib().mf_max_voxelization_3d_fwd(
                *(L.ptr(a) for a in d), P, C, B, *o3, pitch, *dims, L.ptr(matrix), L.ptr(indices),
                L.ptr(ws), ws.numel(), L.ptr(flags), L.stream())
        L.check(rc, "max_voxelization_3d")
        return matrix, indices, int(flags.item())

    matrix, indices, flags = fwd(pts, bi_bad)
    assert flags == 4
    assert np.array_equal(indices.cpu().numpy(), want_i)
    assert np.array_equal(matrix.cpu().numpy(), want_m)
    pts_nan = pts.copy()
    pts_nan[5, 2] = np.nan
    assert fwd(pts_nan, bi)[2] == 1
    assert fwd(pts, bi)[2] == 0

    dev = [cu(a, cuda_device) for a in (vals, pts, bi_bad, inten)]
    y, ind = F().max_voxelization_3d(*dev, return_indices=True, **kw)
    assert np.array_equal(ind.cpu().numpy(), want_i) and np.array_equal(y.cpu().numpy(), want_m)
    avg = F().average_voxelization_3d(dev[0], dev[1], dev[2], **kw)
    avg_want = vo.average_voxelization_3d_fwd(vals, far, bi, **kw)[0]
    assert np.array_equal(avg.cpu().numpy(), avg_want)
    for op in (lambda p: F().max_voxelization_3d(dev[0], p, dev[2], dev[3], **kw),
               lambda p: F().average_voxelization_3d(dev[0], p, dev[2], **kw)):
        with pytest.raises(ValueError, match="points include nan"):
            op(cu(pts_nan, cuda_device))

    gy = np.random.RandomState(14).uniform(-1, 1, want_m.shape).astype(F32)
    gvalues = torch.full((P, C), float("nan"), dtype=torch.float32, device=cuda_device)
    with torch.cuda.device(cuda_device):
        rc = L.lib().mf_max_voxelization_3d_bwd(L.ptr(cu(gy, cuda_device)), L.ptr(indices), P, C, B,
                                                *dims, L.ptr(gvalues), L.stream())
    L.check(rc, "max_voxelization_3d backward")
    got = gvalues.cpu().numpy()
    assert np.array_equal(got, vo.max_voxelization_3d_bwd(gy, want_i, P))
    losers = np.setdiff1d(np.arange(P), want_i[want_i >= 0])
    assert len(losers) > 0 and np.all(got[losers] == 0)


# ================================================================== 4  TDF / pseudo-occupancy
TDF_CASES = {
    # name: P, dims, truncation / pitch, the kernel size it gives
    "ks1": dict(P=700, dims=(32, 32, 32), ratio=0.9, ks=1),
    "ks3": dict(P=5400, dims=(32, 32, 32), ratio=2.5, ks=3),
    "ks5_even_ceil": dict(P=20000, dims=(32, 32, 32), ratio=4.0, ks=5),
    "ks7": dict(P=700, dims=(20, 20, 20), ratio=6.5, ks=7),
    "ks3_even_ceil_noncubic": dict(P=5400, dims=(7, 9, 11), ratio=2.0, ks=3),
    "p1": dict(P=1, dims=(20, 20, 20), ratio=2.5, ks=3),
    "p0": dict(P=0, dims=(20, 20, 20), ratio=2.5, ks=3),
    # far outside (the float -> int conversions saturate), infinite and NaN points
    "wild": dict(P=700, dims=(32, 32, 32), ratio=2.5, ks=3, wild=True),
    # a lattice midway between voxel centres, every point twice: exact ties between points
    "ties": dict(P=432, dims=(5, 5, 5), ratio=2.0, ks=3, lattice=True),
}


def tdf_inputs(name):
    c = TDF_CASES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    P, dims = c["P"], c["dims"]
    if c.get("lattice"):
        pitch, origin = F32(1), np.zeros(3, F32)
        a = np.arange(-1, 5) + 0.5
        lat = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
        pts = np.concatenate([lat, lat[rs.permutation(len(lat))]])
    else:
        pitch, origin = PITCH, ycb_origin(dims)
        pts = CENTRE + rs.normal(0, 0.22, (P, 3)) * np.array(dims) * float(pitch)
    pts = np.ascontiguousarray(pts, F32)
    bad = np.zeros(P, bool)
    if c.get("wild"):
        rows = rs.permutation(P)[:48]
        vals = [1e9, -1e9, np.inf, -np.inf, np.nan, 3e4]
        for k, r in enumerate(rows):
            pts[r, k % 3] = vals[k % 6]
            if k >= 40:
                pts[r] = vals[k % 6]
        bad[rows] = True
    trunc = F32(F32(c["ratio"]) * pitch)
    assert vo.tdf_ksize(pitch, trunc) == c["ks"]
    return pts, pitch, origin, trunc, bad


def tdf_bwd_ref(gy, pts, ind, pitch, origin, dims, *, normalise=True):
    """float64 gpoints and sum|terms|: for every voxel a point wins, the unit vector from the voxel
    to the point times gtdf.  dd = f - voxel is taken in fp32 as the kernel takes it (its own
    input to the chain that is bounded); normalise=False is the wrong reference."""
    X, Y, Z = dims
    ind = ind.reshape(-1)
    hit = np.nonzero(ind >= 0)[0]
    pid = ind[hit]
    vox = np.stack([hit // (Y * Z), (hit // Z) % Y, hit % Z], 1).astype(F32)
    f = ((pts[pid] - origin[None]) / pitch).astype(F32)
    dd = (f - vox).astype(F32).astype(np.float64)
    n = np.sqrt((dd * dd).sum(1))
    keep = n > 0
    g = np.asarray(gy, np.float64).reshape(-1)[hit]
    with np.errstate(invalid="ignore", divide="ignore"):
        terms = (dd / n[:, None] if normalise else dd) * g[:, None]
    ref, absref = np.zeros((len(pts), 3)), np.zeros((len(pts), 3))
    np.add.at(ref, pid[keep], terms[keep])
    np.add.at(absref, pid[keep], np.abs(terms[keep]))
    return ref, absref


@pytest.mark.parametrize("name", list(TDF_CASES))
def test_truncated_distance_function(cuda_device, name):
    """tdf and winners bit-exact against the oracle; gpoints within (ks^3 + 5) u sum|terms| of
    float64: per term the norm of the fp32 dd (three products and two sums under a square root:
    <= 3.5u), the quotient and the product with gtdf (5.5u together, rounded down to 5 by the
    square root's halving), and at most ks^3 terms added in ascending voxel order -- a fixed
    order, so two runs are also bitwise equal.  Infinite and NaN points, and points whose voxel
    coordinate saturates the int conversion, win nothing and get a gradient of exactly 0."""
    c = TDF_CASES[name]
    pts, pitch, origin, trunc, bad = tdf_inputs(name)
    dims, P = c["dims"], c["P"]
    kw = dict(pitch=pitch, origin=origin, dims=dims, truncation=trunc)
    with np.errstate(all="ignore"):
        want_tdf, want_ind = vo.truncated_distance_function_fwd(pts, **kw)
    p_d = cu(pts, cuda_device).requires_grad_(True)
    tdf, ind = F().truncated_distance_function(p_d, return_indices=True, **kw)
    assert np.array_equal(ind.cpu().numpy(), want_ind)
    assert np.array_equal(tdf.detach().cpu().numpy(), want_tdf)
    gy = np.random.RandomState(21).uniform(-1, 1, dims).astype(F32)
    tdf.backward(cu(gy, cuda_device))
    if P == 0:
        assert tuple(p_d.grad.shape) == (0, 3) and np.all(want_ind == -1)
        return
    got = p_d.grad.cpu().numpy()
    ref, absref = tdf_bwd_ref(gy, pts, want_ind, pitch, origin, dims)
    tol = (c["ks"] ** 3 + 5) * U * absref
    held(f"truncated_distance_function bwd {name}", got, ref, tol)
    if P > 1:
        assert absref.sum() > 0
        rejected(f"truncated_distance_function bwd {name} / not normalised", got,
                 tdf_bwd_ref(gy, pts, want_ind, pitch, origin, dims, normalise=False)[0], tol)
    p2 = cu(pts, cuda_device).requires_grad_(True)
    F().truncated_distance_function(p2, **kw).backward(cu(gy, cuda_device))
    assert torch.equal(p2.grad, p_d.grad)
    if c.get("wild"):
        gone = bad & ~np.isfinite(pts).all(1) | (np.abs(pts) >= 1e9).any(1)
        assert gone.sum() >= 30
        assert not np.isin(want_ind, np.nonzero(gone)[0]).any()
        assert np.all(got[gone] == 0)
    if c.get("lattice"):
        # ties between points exist here: breaking them to the higher id is another grid
        rev = vo.truncated_distance_function_fwd(pts[::-1], **kw)[1]
        assert not np.array_equal(want_ind, np.where(rev >= 0, P - 1 - rev, -1))


@pytest.mark.parametrize("sdf_offset", [0.0, 0.02])
@pytest.mark.parametrize("threshold", [1, 2, 2.5, 4])
def test_pseudo_occupancy_voxelization(cuda_device, threshold, sdf_offset):
    """grid, surface and inside bit-exact against the oracle at the refinement's shape; then the
    same grid with every point out of reach: no winner, the largest inside-weight is 0 and the
    normalisation is 0/0 -- NaN by design, in the oracle's pattern."""
    rs = np.random.RandomState(22)
    P, dims = 5400, (32, 32, 32)
    origin = ycb_origin(dims)
    pts = (CENTRE + rs.normal(0, 0.03, (P, 3))).astype(F32)
    sdf = rs.uniform(-0.01, 0.03, P).astype(F32)
    kw = dict(pitch=PITCH, origin=origin, dims=dims, threshold=threshold, sdf_offset=sdf_offset)
    for points, reached in ((pts, True), ((pts + F32(10.0)).astype(F32), False)):
        with np.errstate(all="ignore"):
            r = vo.pseudo_occupancy_voxelization_fwd(points, sdf, **kw)
        assert bool((r["indices"] >= 0).any()) == reached
        assert bool(np.isnan(r["inside"]).all()) == (not reached)
        out = F().pseudo_occupancy_voxelization(cu(points, cuda_device), cu(sdf, cuda_device), **kw)
        for got, key in zip(out, ("grid", "surface", "inside")):
            assert np.array_equal(got.cpu().numpy(), r[key], equal_nan=True), key


# ================================================================== 5  transforms
def tp32(p, T):
    """((t0 x + t1 y) + t2 z) + t3 in separately rounded fp32 operations: [M, P, 3]."""
    x, y, z = p[None, :, 0], p[None, :, 1], p[None, :, 2]
    rows = [((T[:, r, 0, None] * x + T[:, r, 1, None] * y) + T[:, r, 2, None] * z)
            + T[:, r, 3, None] for r in range(3)]
    out = np.stack(rows, -1)
    assert out.dtype == F32
    return out


@pytest.mark.parametrize("P,M", [(1, 1), (255, 3), (257, 3), (500, 1000), (2000, 8), (17066, 1)])
def test_transform_points(cuda_device, P, M):
    """Forward bit-exact against the stated expression order.  gpoints[p] = sum_m R_m^T g[m, p]:
    per m three products and two sums, then one serial accumulation over m: c = M + 3.
    gT[m] = sum_p g[m, p] (x) [p, 1]: one product, then the 256-thread tree, c = ceil(P/256) + 14;
    its last row is exactly 0.  Both are fixed-order sums: two runs are bitwise equal."""
    rs = np.random.RandomState(31)
    pts = rs.uniform(-1, 1, (P, 3)).astype(F32)
    T = rs.uniform(-1, 1, (M, 4, 4)).astype(F32)
    go = rs.uniform(-1, 1, (M, P, 3)).astype(F32)

    def run():
        p_d = cu(pts, cuda_device).requires_grad_(True)
        T_d = cu(T, cuda_device).requires_grad_(True)
        out = F().transform_points(p_d, T_d)
        out.backward(cu(go, cuda_device))
        return out.detach(), p_d.grad, T_d.grad

    out, gp, gT = run()
    assert np.array_equal(out.cpu().numpy(), tp32(pts, T))
    assert np.array_equal(F().transform_points(cu(pts, cuda_device), cu(T[0], cuda_device)).cpu().numpy(),
                          tp32(pts, T)[0])
    p64, R64, g64 = t64(pts), t64(T)[:, :3, :3], t64(go)
    tag = f"transform_points P={P} M={M}"
    tol_p = (M + 3) * U * torch.einsum("mab,mpa->pb", R64.abs(), g64.abs())
    held(f"{tag} gpoints", gp, torch.einsum("mab,mpa->pb", R64, g64), tol_p)
    rejected(f"{tag} gpoints / R not transposed", gp, torch.einsum("mba,mpa->pb", R64, g64), tol_p)
    ph = torch.cat([p64, torch.ones(P, 1, dtype=F64)], 1)
    ref_T = torch.einsum("mpr,pk->mrk", g64, ph)
    tol_T = (c_chain(P) + 1) * U * torch.einsum("mpr,pk->mrk", g64.abs(), ph.abs())
    held(f"{tag} gT", gT[:, :3], ref_T, tol_T)
    assert float(gT[:, 3].abs().max()) == 0.0
    if P > 1:
        keep = min(256, P - 1)      # the first tile of the tree only (or all points but the last)
        rejected(f"{tag} gT / first {keep} points", gT[:, :3],
                 torch.einsum("mpr,pk->mrk", g64[:, :keep], ph[:keep]), tol_T)
    out2, gp2, gT2 = run()
    assert torch.equal(out, out2) and torch.equal(gp, gp2) and torch.equal(gT, gT2)


@pytest.mark.parametrize("P,M", [(300, 0), (0, 4), (0, 0)])
def test_transform_points_empty(cuda_device, P, M):
    """No transform or no point: shapes and zero gradients as the matmul formulation gives them,
    also on gradient buffers that held NaN (through the C ABI)."""
    L = abi()
    rs = np.random.RandomState(32)
    p_d = cu(rs.uniform(-1, 1, (P, 3)).astype(F32), cuda_device).requires_grad_(True)
    T_d = cu(rs.uniform(-1, 1, (M, 4, 4)).astype(F32), cuda_device).requires_grad_(True)
    out = F().transform_points(p_d, T_d)
    assert tuple(out.shape) == (M, P, 3)
    out.sum().backward()
    p2 = p_d.detach().clone().requires_grad_(True)
    T2 = T_d.detach().clone().requires_grad_(True)
    ph = torch.cat([p2, torch.ones(P, 1, device=cuda_device)], 1)
    torch.matmul(T2, ph.T).transpose(1, 2)[:, :, :3].sum().backward()
    for got, want in ((p_d.grad, p2.grad), (T_d.grad, T2.grad)):
        assert got.shape == want.shape and float(want.abs().sum()) == 0.0
        assert torch.equal(got, want)
    gp = torch.full((P, 3), float("nan"), device=cuda_device)
    gT = torch.full((M, 4, 4), float("nan"), device=cuda_device)
    go = torch.zeros((M, P, 3), device=cuda_device)
    with torch.cuda.device(cuda_device):
        rc = L.lib().mf_transform_points_bwd(L.ptr(go), L.ptr(p_d), P, L.ptr(T_d), M, L.ptr(gp),
                                             L.ptr(gT), L.stream())
    L.check(rc, "transform_points backward")
    assert float(gp.abs().sum()) == 0.0 and float(gT.abs().sum()) == 0.0


@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
@pytest.mark.parametrize("N", [1, 129, 100000])
def test_quaternion_matrix_compose_translation(cuda_device, N, scale):
    """quaternion_matrix forward within 12 u sum|terms| of float64 for |q| = 1e-3, 1, 1e3.  The
    chain: |q|^2 (four positive terms: 4u), 2 / n (5u), its square root (3.5u), q s (4.5u), a
    product of two of those (10u), two sums (12u); terms are 1 and the two products of a diagonal
    entry, the two products of an off-diagonal one.  The last row and column are exact.
    compose_transform and translation_matrix copy: bit-exact against the oracle.  A batched call
    and a call on one row give the same bits."""
    f = F()
    rs = np.random.RandomState(33)
    q = rs.normal(size=(N, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True) * scale).astype(F32)
    t = rs.uniform(-1, 1, (N, 3)).astype(F32)
    q_d, t_d = cu(q, cuda_device), cu(t, cuda_device)
    R = f.quaternion_matrix(q_d)
    q64 = t64(q)
    w, x, y, z = (q64 * torch.sqrt(2.0 / (q64 * q64).sum(1, keepdim=True))).unbind(1)
    a = {"xx": x * x, "yy": y * y, "zz": z * z, "xy": x * y, "xz": x * z, "yz": y * z,
         "xw": x * w, "yw": y * w, "zw": z * w}
    one = torch.ones(N, dtype=F64)
    absterms = torch.stack([one + a["yy"] + a["zz"], a["xy"].abs() + a["zw"].abs(), a["xz"].abs() + a["yw"].abs(),
                            a["xy"].abs() + a["zw"].abs(), one + a["xx"] + a["zz"], a["yz"].abs() + a["xw"].abs(),
                            a["xz"].abs() + a["yw"].abs(), a["yz"].abs() + a["xw"].abs(), one + a["xx"] + a["yy"]],
                           1).reshape(N, 3, 3)
    tol = 12 * U * absterms
    tag = f"quaternion_matrix N={N} |q|={scale:g}"
    held(tag, R[:, :3, :3], quat_R64(q64), tol)
    if scale == 1.0:
        rejected(f"{tag} / transposed", R[:, :3, :3], quat_R64(q64).transpose(1, 2), tol)
    else:       # the normalisation left out: q sqrt2 in place of q sqrt(2 / |q|^2)
        rejected(f"{tag} / not normalised", R[:, :3, :3], unnormalised_R64(q64), tol)
    last = torch.tensor([0.0, 0.0, 0.0, 1.0], device=cuda_device)
    assert bool((R[:, 3] == last).all()) and bool((R[:, :, 3] == last).all())

    T = f.compose_transform(R[:, :3, :3], t_d)
    Rn = R.cpu().numpy()
    assert np.array_equal(T.cpu().numpy(), otf.compose_transform(Rn[:, :3, :3], t))
    assert np.array_equal(f.translation_matrix(t_d).cpu().numpy(), otf.translation_matrix(t))
    assert torch.equal(f.transformation_matrix(q_d, t_d), T)
    for i in sorted({0, N // 2, N - 1}):
        assert torch.equal(f.quaternion_matrix(q_d[i]), R[i])
        assert torch.equal(f.compose_transform(R[i, :3, :3], t_d[i]), T[i])
        assert torch.equal(f.translation_matrix(t_d[i]), f.translation_matrix(t_d)[i])
        assert torch.equal(f.transformation_matrix(q_d[i], t_d[i]), T[i])


