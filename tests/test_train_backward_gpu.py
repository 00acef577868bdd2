"""GPU: the CUDA backward of the 3-D section (csrc/train.cu, csrc/gemm_train.cu and the forward
GEMM reused for dX) replayed stage by stage against float64 references.

Each stage's reference is computed from the kernel's OWN inputs to that stage (the bf16 / fp32
buffers the previous kernel wrote), so no model of how bf16 rounding propagates through the
network is needed and every stage is held to the precision of its own arithmetic:

  * fp32 accumulation:  |got - ref| <= c * 2^-24 * sum|terms|, with sum|terms| from the same
    float64 reference evaluated on absolute values and c fixed per stage from the length and
    order of the kernel's summation chain (commented beside each comparison);
  * bf16 stores:        the above plus half a bf16 ulp of the result;
  * masks, zero borders and pure re-layouts: exact.

Every stage also runs one deliberately wrong reference (missing K block, wrong parity, shifted
column offset, mask from the other activation, ...) through the same comparison and asserts
that it FAILS: the bound is tight enough to tell a subtly wrong kernel from a correct one.
The conv references are float64 matmuls through the space-to-depth identities of
tests/test_s2d_conv_math.py (no cuDNN, whose fp32 algorithm choice is not under our control).

The second half calls the mf_train_* kernels directly at shapes and values the model never
produces (tails, range ends, prefilled outputs, sentinels), and checks the optimizer."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff (round to nearest)
F64 = torch.float64
FEAT_LD = 1024


# ------------------------------------------------------------------ comparison helpers
def half_ulp_bf16(x):
    """Half a bf16 ulp of |x| (8 significant bits): 2^(floor(log2|x|) - 8), 0 at 0."""
    a = x.abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -126)))
    return torch.where(a > 0, torch.exp2(e - 8), torch.zeros_like(a))


def fp32_tol(absterms, c):
    return c * U * absterms


def bf16_tol(ref, absterms, c):
    """bf16 store of an fp32 result within c u sum|terms| of ref: rounding happens on the fp32
    value, whose magnitude may exceed |ref| by the fp32 error (next binade)."""
    d = c * U * absterms
    return d + half_ulp_bf16(ref.abs() + d)


def _ratio(got, ref, tol):
    err = (got.double() - ref).abs()
    bad = err > tol
    worst = float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0
    return bool(bad.any()), int(bad.sum()), worst


def check(name, got, ref, tol):
    bad, n, worst = _ratio(got, ref, tol)
    assert not bad, f"{name}: {n} elements outside the bound (worst err/bound {worst:.3g})"


def control(name, got, wrong, tol):
    """Negative control: the comparison must reject a deliberately wrong reference."""
    bad, _, _ = _ratio(got, wrong, tol)
    assert bad, f"{name}: negative control passed the bound (bound cannot see this error)"


def c_mma(K):
    """Chain length bound of a wgmma reduction of length K: one fp32 add per k16 step (K/16),
    at most K/512 split-K partial sums (>= 8 K blocks of 64 per split) and the 16-term tree
    inside the instruction (4); doubled because the tensor core's internal adds truncate
    (unit roundoff 2^-23, not 2^-24)."""
    return 2 * (-(-K // 16) + -(-K // 512) + 4)


# ------------------------------------------------------------------ layout helpers
def s2d_taps():
    return [(ad, ah, aw) for ad in (0, 1) for ah in (0, 1) for aw in (0, 1)]


def un_s2d_cl(xs, C):
    """[B,J,J,J,8C] s2d of the zero-padded grid -> channels-last [B,D,D,D,C] (ring dropped)."""
    B, J = xs.shape[:2]
    xp = xs.reshape(B, J, J, J, 2, 2, 2, C).permute(0, 1, 4, 2, 5, 3, 6, 7)
    return xp.reshape(B, 2 * J, 2 * J, 2 * J, C)[:, 1:-1, 1:-1, 1:-1]


def to_parity(dense):
    """[B,D,D,D,C] -> [8, B*(D/2)^3, C]: row (b, o) of parity r = voxel 2 o + 1 - r."""
    B, D, C = dense.shape[0], dense.shape[1], dense.shape[-1]
    rows = [dense[:, 1 - rd::2, 1 - rh::2, 1 - rw::2].reshape(-1, C)
            for rd in (0, 1) for rh in (0, 1) for rw in (0, 1)]
    return torch.stack(rows, 0)


def from_parity(par, B, D):
    C, Do = par.shape[-1], D // 2
    g = par.reshape(2, 2, 2, B, Do, Do, Do, C)
    dense = torch.empty(B, D, D, D, C, dtype=par.dtype, device=par.device)
    for rd in (0, 1):
        for rh in (0, 1):
            for rw in (0, 1):
                dense[:, 1 - rd::2, 1 - rh::2, 1 - rw::2] = g[rd, rh, rw]
    return dense


def wgrad_ref(dYp, Xs, Do, drop_block=None):
    """dWg[co, a*8C + k] = sum_(b,o) dY[(b,o), co] Xs[b, o + a, k]  (float64, packed K order).
    Returns (ref, sum|terms|).  drop_block: leave out one 64-voxel K block (negative control)."""
    Co = dYp.shape[-1]
    K8 = Xs.shape[-1]
    dY = dYp[:, 1:-1, 1:-1, 1:-1].to(F64).reshape(-1, Co)
    if drop_block is not None:
        dY = dY.clone()
        dY[drop_block * 64:(drop_block + 1) * 64] = 0
    ref = torch.empty(Co, 8 * K8, dtype=F64, device=dYp.device)
    ab = torch.empty_like(ref)
    for a, (ad, ah, aw) in enumerate(s2d_taps()):
        A = Xs[:, ad:ad + Do, ah:ah + Do, aw:aw + Do].to(F64).reshape(-1, K8)
        ref[:, a * K8:(a + 1) * K8] = dY.T @ A
        ab[:, a * K8:(a + 1) * K8] = dY.abs().T @ A.abs()
        del A
    return ref, ab


def dgrad_ref(dYp, Wg, C):
    """Channels-last dense input gradient [B,D,D,D,C] of the k4 s2 p1 conv through the s2d
    identity dXs[b, j] = sum_a dYp[b, j - a + 1] . Wg[:, a-block]; (ref, sum|terms|)."""
    B, Dp = dYp.shape[:2]
    J = Dp - 1
    K8 = 8 * C
    gx = torch.zeros(B, J, J, J, K8, dtype=F64, device=dYp.device)
    gxa = torch.zeros_like(gx)
    W = Wg.to(F64)
    for a, (ad, ah, aw) in enumerate(s2d_taps()):
        G = dYp[:, 1 - ad:1 - ad + J, 1 - ah:1 - ah + J, 1 - aw:1 - aw + J].to(F64)
        Wa = W[:, a * K8:(a + 1) * K8]
        gx += G @ Wa
        gxa += G.abs() @ Wa.abs()
        del G
    return un_s2d_cl(gx, C), un_s2d_cl(gxa, C)


def scatter_ref(g, points, C, D, divisor, *, floor=False):
    """Trilinear scatter (interpolate_voxel_grid backward) in float64: x = fl32(p / divisor),
    corner x0 = trunc(x) (C cast), out-of-grid corners skipped.  Returns (grid [B*D^3, C],
    sum|terms| grid, number of contributions per voxel)."""
    B, _, P = points.shape
    x = (points / divisor).permute(0, 2, 1).reshape(-1, 3)                     # fp32 division
    x0 = torch.floor(x) if floor else torch.trunc(x)
    l = (x - x0).to(F64)
    i0 = x0.long()
    g = g.to(F64)
    bidx = torch.arange(B, device=g.device).repeat_interleave(P)
    out = torch.zeros(B * D ** 3, C, dtype=F64, device=g.device)
    oab = torch.zeros_like(out)
    cnt = torch.zeros(B * D ** 3, 1, dtype=F64, device=g.device)
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                d = torch.tensor([dx, dy, dz], device=g.device)
                idx = i0 + d
                wt = torch.where(d.bool(), l, 1 - l).prod(1)
                ok = ((idx >= 0) & (idx < D)).all(1)
                flat = ((bidx * D + idx[:, 0]) * D + idx[:, 1]) * D + idx[:, 2]
                f = flat[ok]
                out.index_add_(0, f, wt[ok, None] * g[ok])
                oab.index_add_(0, f, (wt[ok, None] * g[ok]).abs())
                cnt.index_add_(0, f, torch.ones(int(ok.sum()), 1, dtype=F64, device=g.device))
    return out, oab, cnt


def voxel_of(points, D):
    """Voxel of each point with the voxeliser's rule (C roundf = half away from zero, then the
    (int) cast); -1 outside the grid.  Returns flat voxel index [B*P] within the object."""
    p = points.permute(0, 2, 1).reshape(-1, 3)
    t = torch.trunc(p)
    r = t + torch.where((p - t).abs() >= 0.5, torch.sign(p), torch.zeros_like(p))
    i = r.long()
    ok = ((i >= 0) & (i < D)).all(1)
    flat = (i[:, 0] * D + i[:, 1]) * D + i[:, 2]
    return torch.where(ok, flat, torch.full_like(flat, -1)), i


# ------------------------------------------------------------------ float64 stage references
def head4_draw(g_rot, g_trans, g_conf, raw8, pitch_per_point):
    """d raw (8 per point) of the pose epilogue + |terms| bound per component (float64)."""
    o = raw8.to(F64)
    g = g_rot.to(F64)
    nr = o[:, :4].norm(dim=1, keepdim=True)
    ne = nr + float(np.float32(1e-5))
    og = (o[:, :4] * g).sum(1, keepdim=True)
    oga = (o[:, :4] * g).abs().sum(1, keepdim=True)
    k2 = torch.where(nr > 0, og / (nr * ne * ne), torch.zeros_like(nr))
    k2a = torch.where(nr > 0, oga / (nr * ne * ne), torch.zeros_like(nr))
    d = torch.empty(o.shape[0], 8, dtype=F64, device=o.device)
    a = torch.empty_like(d)
    d[:, :4] = g / ne - o[:, :4] * k2
    a[:, :4] = g.abs() / ne + o[:, :4].abs() * k2a
    pt = pitch_per_point.to(F64)[:, None]
    d[:, 4:7] = g_trans.to(F64) * pt
    a[:, 4:7] = d[:, 4:7].abs()
    s = torch.sigmoid(o[:, 7])
    d[:, 7] = g_conf.to(F64) * s * (1 - s)
    # 1 - s cancels when s -> 1: its error is relative to s, not to 1 - s
    a[:, 7] = g_conf.to(F64).abs() * s
    return d, a


def head4_ref(d8, a8, hd3, W, fg_per_point):
    """dhd3 (masked by hd3 > 0) from d raw and the class rows of the bf16 head-4 weights.
    W = (w_rot [nfg*4,128], w_trans [nfg*3,128], w_conf [nfg,128]).  Returns (ref, |terms|)."""
    wr, wt, wc = [w.to(F64) for w in W]
    fg = fg_per_point
    rows = [wr.reshape(-1, 4, 128)[fg], wt.reshape(-1, 3, 128)[fg], wc.reshape(-1, 1, 128)[fg]]
    segs = [(0, 4), (4, 7), (7, 8)]
    h = hd3.to(F64)
    ref = torch.empty_like(h)
    ab = torch.empty_like(h)
    for s, ((lo, hi), Wr) in enumerate(zip(segs, rows)):
        ref[:, s * 128:(s + 1) * 128] = torch.einsum("nr,nrk->nk", d8[:, lo:hi], Wr)
        ab[:, s * 128:(s + 1) * 128] = torch.einsum("nr,nrk->nk", a8[:, lo:hi], Wr.abs())
    m = h > 0
    return ref * m, ab * m


def head4_wgrad_ref(d8, a8, hd3, fg_per_point, nfg):
    """dW4 rows fg*4.. / fg*3.. / fg of each head and db4: per-class sums over the points."""
    h = hd3.to(F64)
    out = {}
    for name, (lo, hi), seg in (("rot", (0, 4), 0), ("trans", (4, 7), 1), ("conf", (7, 8), 2)):
        n = hi - lo
        hs = h[:, seg * 128:(seg + 1) * 128]
        W = torch.zeros(nfg, n, 128, dtype=F64, device=h.device)
        Wa = torch.zeros_like(W)
        b = torch.zeros(nfg, n, dtype=F64, device=h.device)
        ba = torch.zeros_like(b)
        W.index_add_(0, fg_per_point, d8[:, lo:hi, None] * hs[:, None, :])
        Wa.index_add_(0, fg_per_point, a8[:, lo:hi, None] * hs.abs()[:, None, :])
        b.index_add_(0, fg_per_point, d8[:, lo:hi])
        ba.index_add_(0, fg_per_point, a8[:, lo:hi])
        out[name] = (W.reshape(nfg * n, 128), Wa.reshape(nfg * n, 128), b.reshape(-1), ba.reshape(-1))
    return out


def mask_pack_ref(dgrid, act_dense):
    """bf16(dgrid * (act > 0)) (exact: one RNE rounding of the fp32 value) and its column sum."""
    v = torch.where(act_dense.float() > 0, dgrid, torch.zeros_like(dgrid)).to(torch.bfloat16)
    return v


def point_mlp_ref(values, points, h1, d1, feat2, g2in, W1r, W1p, W2r, W2p, center, drop_direct=False):
    """Backward of the per-point MLP (k_point_mlp_bwd) in float64 from the kernel's inputs.
    Returns {name: (ref, |terms|)} for the weight / bias gradients and dvalues [B,32,P]."""
    B, _, P = values.shape
    xv = values.to(F64).permute(0, 2, 1).reshape(-1, 32)
    xp = (center - points.to(F64)).permute(0, 2, 1).reshape(-1, 3)
    h1 = h1.to(F64)
    g2 = torch.where(feat2 > 0, g2in, torch.zeros_like(g2in)).to(F64)
    direct = torch.zeros_like(h1) if drop_direct else d1.to(F64)
    W1r, W1p, W2r, W2p = [w.to(F64) for w in (W1r, W1p, W2r, W2p)]
    m1 = h1 > 0
    g1 = torch.cat([direct[:, :64] + g2[:, :128] @ W2r, direct[:, 64:] + g2[:, 128:] @ W2p], 1) * m1
    a1 = torch.cat([direct[:, :64].abs() + g2[:, :128].abs() @ W2r.abs(),
                    direct[:, 64:].abs() + g2[:, 128:].abs() @ W2p.abs()], 1) * m1
    out = {
        "conv2_rgb.weight": (g2[:, :128].T @ h1[:, :64], g2[:, :128].abs().T @ h1[:, :64].abs()),
        "conv2_pcd.weight": (g2[:, 128:].T @ h1[:, 64:], g2[:, 128:].abs().T @ h1[:, 64:].abs()),
        "conv2_rgb.bias": (g2[:, :128].sum(0), g2[:, :128].abs().sum(0)),
        "conv2_pcd.bias": (g2[:, 128:].sum(0), g2[:, 128:].abs().sum(0)),
        "conv1_rgb.weight": (g1[:, :64].T @ xv, a1[:, :64].T @ xv.abs()),
        "conv1_pcd.weight": (g1[:, 64:].T @ xp, a1[:, 64:].T @ xp.abs()),
        "conv1_rgb.bias": (g1[:, :64].sum(0), a1[:, :64].sum(0)),
        "conv1_pcd.bias": (g1[:, 64:].sum(0), a1[:, 64:].sum(0)),
    }
    dv = g1[:, :64] @ W1r
    dva = a1[:, :64] @ W1r.abs()
    out["values"] = (dv.reshape(B, P, 32).permute(0, 2, 1), dva.reshape(B, P, 32).permute(0, 2, 1))
    return out


def point_mlp_c(NP):
    """k_point_mlp_bwd: g1 = direct + up to 128 products (sequential, 130 roundings); weight /
    bias sums: 64 points per CTA in sequence then one atomic per CTA (NP/64); the centre
    offset of the pcd input is one more rounding."""
    return 130 + 64 + -(-NP // 64) + 2


# ------------------------------------------------------------------ the model run
def _model_and_batch(B, occ, dev, seed):
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib.singleview_3d.models import Model
    w = synthetic.init_weights(21, seed=1, with_occupancy=occ)
    model = Model(n_fg_class=21, with_occupancy=occ).to(dev).load_reference_weights(w)
    model.train()
    batch = synthetic.make_cnn_batch(B, 1000, seed=seed)
    # both ends of the class range; B = 2 and 16 repeat a class (atomics into the same head-4
    # rows from different objects)
    cid = batch["class_id"].copy()
    if B == 1:
        cid[:] = 21
    elif B == 2:
        cid[:] = 1
    else:
        cid[0], cid[1], cid[-1] = 1, 21, 1
    batch["class_id"] = cid.astype(np.int32)
    pts = batch["points"]
    for b in range(B):                        # grid edges: outside, upper faces, (-1, 0)
        pts[b, :, 0] = (-3.0, 10.0, 10.0)
        pts[b, :, 1] = (10.0, 40.0, 10.0)
        pts[b, :, 2] = (31.0, 31.0, 31.0)
        pts[b, :, 3] = (31.0, 12.0, 31.49)
        pts[b, :, 4] = (31.5, 12.0, 12.0)     # rounds to 32: dropped by the voxeliser
        pts[b, :, 5] = (-0.4, 5.0, 7.0)       # interp: x in (-1, 0), extrapolating weights
        pts[b, :, 6] = (-0.4, 5.0, 7.0)       # same voxel twice
    return model, batch


def _run_backward(B, occ, dev, seed=0):
    from morefusion_b200.contrib.singleview_3d.models import training
    model, batch = _model_and_batch(B, occ, dev, seed)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)   # noqa: E731
    values = t(batch["values"]).requires_grad_(True)
    points = t(batch["points"])
    rot, trans, conf = training.forward_features_with_grad(
        model, class_id=batch["class_id"], values=values, points=points, pitch=t(batch["pitch"]),
        origin=t(batch["origin"]),
        grid_nontarget_empty=t(batch["grid_nontarget_empty"]) if occ else None)
    gen = torch.Generator(device=dev).manual_seed(100 + B)
    g_rot = torch.randn(rot.shape, generator=gen, device=dev)
    g_trans = torch.randn(trans.shape, generator=gen, device=dev)
    g_conf = torch.randn(conf.shape, generator=gen, device=dev)
    torch.autograd.backward([rot, trans, conf], [g_rot, g_trans, g_conf])
    torch.cuda.synchronize()
    return model, batch, values, points, (g_rot, g_trans, g_conf)


@pytest.mark.parametrize("occ", [True, False])
@pytest.mark.parametrize("B", [1, 2, 16])
def test_backward_stage_replay(cuda_device, B, occ):
    from morefusion_b200.contrib.singleview_3d.models import training
    dev = cuda_device
    P, D, nfg = 1000, 32, 21
    NP = B * P
    Ct = 160 if occ else 144
    model, batch, values, points, (g_rot, g_trans, g_conf) = _run_backward(B, occ, dev)
    buf = model._work_buffers(B, P, dev)
    tb = training._train_buffers(model, B, P, dev)
    w = model._packed
    G = {n: p.grad for n, p in model.named_parameters() if n in training.flat_param_order(model)}
    cid = torch.as_tensor(batch["class_id"], device=dev).long()
    fg_pt = (cid - 1).repeat_interleave(P)
    pitch_pt = torch.as_tensor(batch["pitch"], device=dev).repeat_interleave(P)

    # ---- head 4 + pose epilogue
    d8, a8 = head4_draw(g_rot.reshape(NP, 4), g_trans.reshape(NP, 3), g_conf.reshape(NP),
                        tb["raw8"], pitch_pt)
    W4 = (w["conv4_rot/W"], w["conv4_trans/W"], w["conv4_conf/W"])
    ref, ab = head4_ref(d8, a8, buf["hd3"], W4, fg_pt)
    # c = 20: d raw is ~12 fp32 roundings deep (4-term dot / norm, sqrt, divisions, products;
    # expf's 2-ulp error enters through s) -> 16, then the <= 4-term row sum
    tol = bf16_tol(ref, ab, 20)
    check("dhd3", tb["dhd3"], ref, tol)
    wrong, _ = head4_ref(d8, a8, buf["hd3"], W4, (fg_pt + 1) % nfg)         # neighbouring class row
    control("dhd3 / class row + 1", tb["dhd3"], wrong, tol)
    n_cta = -(-P // 16)
    wg = head4_wgrad_ref(d8, a8, buf["hd3"], fg_pt, nfg)
    ncls = torch.bincount(cid - 1, minlength=nfg).max().item()
    # c: d raw (16) + 16 points summed per CTA + one atomic per CTA of every object of the class
    c4 = 16 + 16 + ncls * n_cta
    for h in ("rot", "trans", "conf"):
        W, Wa, b, ba = wg[h]
        check(f"conv4_{h}.weight", G[f"conv4_{h}.weight"].reshape(W.shape), W, fp32_tol(Wa, c4))
        check(f"conv4_{h}.bias", G[f"conv4_{h}.bias"], b, fp32_tol(ba, c4))
    # rows of classes not in the batch have sum|terms| = 0, so the checks above demand exact 0
    W, Wa, _, _ = wg["rot"]
    last = torch.arange(NP, device=dev) % P >= P - 8         # the last (partial) point tile
    Wd, _, _, _ = head4_wgrad_ref(d8 * (~last)[:, None], a8, buf["hd3"], fg_pt, nfg)["rot"]
    control("conv4_rot.weight / last point tile dropped", G["conv4_rot.weight"].reshape(W.shape), Wd,
            fp32_tol(Wa, c4))

    # ---- head layers 3, 2, 1: dW (TN GEMM over NP rows), db (colsum), dX (forward GEMM on W^T)
    c_col = 64 + 4 + -(-NP // 256)          # colsum: 64 rows per thread, 4 partials, atomic per CTA
    for layer, dz, x, n_out, k_in, dx, act in (
            (3, tb["dhd3"], buf["hd2"], 128, 256, tb["dhd2"], buf["hd2"]),
            (2, tb["dhd2"], buf["hd1"], 256, 640, tb["dhd1"], buf["hd1"])):
        dz64, x64 = dz.to(F64), x.to(F64)
        ref_dx = torch.zeros(NP, 3 * k_in, dtype=F64, device=dev)
        ab_dx = torch.zeros_like(ref_dx)
        for i, h in enumerate(("rot", "trans", "conf")):
            zi = dz64[:, i * n_out:(i + 1) * n_out]
            xi = x64[:, i * k_in:(i + 1) * k_in]
            ref = zi.T @ xi
            tol = fp32_tol(zi.abs().T @ xi.abs(), c_mma(NP))
            check(f"conv{layer}_{h}.weight", G[f"conv{layer}_{h}.weight"].reshape(ref.shape), ref, tol)
            if i == 0:
                short = zi[:NP - 64].T @ xi[:NP - 64]                        # last 64 rows dropped
                control(f"conv{layer}_rot.weight / last 64 rows", G[f"conv{layer}_{h}.weight"].reshape(ref.shape),
                        short, tol)
            check(f"conv{layer}_{h}.bias", G[f"conv{layer}_{h}.bias"], zi.sum(0), fp32_tol(zi.abs().sum(0), c_col))
            Wi = w[f"conv{layer}_{h}/W"].to(F64)                              # [n_out, k_in] bf16
            ref_dx[:, i * k_in:(i + 1) * k_in] = zi @ Wi
            ab_dx[:, i * k_in:(i + 1) * k_in] = zi.abs() @ Wi.abs()
        m = act > 0
        tol = bf16_tol(ref_dx, ab_dx, c_mma(n_out)) * m
        check(f"dhd{layer - 1} (masked)", dx, ref_dx * m, tol)
        # mask taken from the neighbouring head's activation (columns rotated by one head)
        control(f"dhd{layer - 1} / other head's mask", dx, ref_dx * torch.roll(m, k_in, 1), tol)
        if layer == 3:
            # dX column offset shifted by 8 (col_off bug in the grouped launch)
            control("dhd2 / col_off + 8", dx, torch.roll(ref_dx, 8, 1) * m, tol)
    dz64 = tb["dhd1"].to(F64)
    f64 = buf["feat"][:, :984].to(F64)
    ref = dz64.T @ f64
    tol = fp32_tol(dz64.abs().T @ f64.abs(), c_mma(NP))
    gw1 = torch.cat([G[f"conv1_{h}.weight"].reshape(640, 984) for h in ("rot", "trans", "conf")], 0)
    check("conv1_*.weight", gw1, ref, tol)
    control("conv1_*.weight / last 64 rows", gw1, dz64[:NP - 64].T @ f64[:NP - 64], tol)
    for i, h in enumerate(("rot", "trans", "conf")):
        zi = dz64[:, i * 640:(i + 1) * 640]
        check(f"conv1_{h}.bias", G[f"conv1_{h}.bias"], zi.sum(0), fp32_tol(zi.abs().sum(0), c_col))
    W1 = w["head1/W"][:, :984].to(F64)
    ref = dz64 @ W1
    tol = bf16_tol(ref, dz64.abs() @ W1.abs(), c_mma(1920))
    check("dfeat[:, :984]", tb["dfeat"][:, :984], ref, tol)
    assert torch.count_nonzero(tb["dfeat"][:, 984:]) == 0          # padding columns untouched
    control("dfeat / last K block dropped", tb["dfeat"][:, :984], dz64[:, :1856] @ W1[:1856], tol)

    # ---- trilinear scatters into the conv4 / conv3 output grids
    s4, s4a, n4 = scatter_ref(tb["dfeat"][:, 472:984], points, 512, 8, 4.0)
    # c = 4 + contributions: weight (3 products) and w*g roundings, then one fp32 atomic add per
    # contribution into the voxel
    tol4 = fp32_tol(s4a, 4 + n4)
    check("dgrid4", tb["dgrid4"].reshape(-1, 512), s4, tol4)
    s4w, _, _ = scatter_ref(tb["dfeat"][:, 480:992], points, 512, 8, 4.0)
    control("dgrid4 / col_off + 8", tb["dgrid4"].reshape(-1, 512), s4w, tol4)

    # ---- mask_pack 4: exact re-layout + bias gradient
    dY4 = tb["dY4p"]
    ref = mask_pack_ref(tb["dgrid4"].reshape(B, 8, 8, 8, 512), buf["h4"])
    assert torch.equal(dY4[:, 1:-1, 1:-1, 1:-1], ref), "dY4p interior"
    border = dY4.clone()
    border[:, 1:-1, 1:-1, 1:-1] = 0
    assert torch.count_nonzero(border) == 0, "dY4p border"
    wrong = mask_pack_ref(tb["dgrid4"].reshape(B, 8, 8, 8, 512), torch.roll(buf["h4"], 1, -1))
    assert not torch.equal(dY4[:, 1:-1, 1:-1, 1:-1], wrong), "mask_pack4 control (channel-shifted mask)"
    NV = B * 512
    # bias: each thread sums its grid-stride voxels (<= NV / (592 * 4) + 1), 4 voxel slots per
    # CTA, then one atomic per CTA (592)
    cb4 = -(-NV // (592 * 4)) + 1 + 4 + 592
    v = ref.to(F64).reshape(-1, 512)
    check("conv4.bias", G["conv4.bias"], v.sum(0), fp32_tol(v.abs().sum(0), cb4))
    control("conv4.bias / heaviest voxel dropped", G["conv4.bias"],
            v.sum(0) - v[v.abs().sum(1).argmax()], fp32_tol(v.abs().sum(0), cb4))

    # ---- conv4 weight gradient (K = B * 512 voxels) and input gradient (parity add into dgrid3)
    unpack = training.unpack_conv_k4s2_grad
    ref, ab = wgrad_ref(dY4, buf["x4"], 8)
    tol = unpack(fp32_tol(ab, c_mma(B * 512)), 512, 256)
    check("conv4.weight", G["conv4.weight"], unpack(ref, 512, 256), tol)
    heavy = int(dY4[:, 1:-1, 1:-1, 1:-1].float().abs().reshape(-1, 64 * 512).sum(1).argmax())
    refd, _ = wgrad_ref(dY4, buf["x4"], 8, drop_block=heavy)
    control("conv4.weight / one K block dropped", G["conv4.weight"], unpack(refd, 512, 256), tol)
    del ref, ab, refd, tol
    dg, dga = dgrad_ref(dY4, w["conv4/W"], 256)                              # [B,16,16,16,256]
    s3, s3a, n3 = scatter_ref(tb["dfeat"][:, 216:472], points, 256, 16, 2.0)
    ref3 = s3 + dg.reshape(-1, 256)
    # scatter as above; dgrad: wgmma chain over K = 8 taps x 512 channels; the final add of the
    # two partial results is one more rounding of |ref|
    tol3 = fp32_tol(s3a, 4 + n3) + fp32_tol(dga.reshape(-1, 256), c_mma(8 * 512)) + U * ref3.abs()
    check("dgrid3 (scatter + conv4 dgrad)", tb["dgrid3"].reshape(-1, 256), ref3, tol3)
    dg_wrong = dg.reshape(B, 16, 16, 16, 256)[:, torch.arange(16, device=dev) ^ 1]   # wrong x parity
    control("dgrid3 / wrong parity", tb["dgrid3"].reshape(-1, 256), s3 + dg_wrong.reshape(-1, 256), tol3)
    del dg, dga, s3, s3a, dg_wrong

    # ---- mask_pack 3 (mask from the s2d conv4 input = relu(conv3))
    dY3 = tb["dY3p"]
    h3 = un_s2d_cl(buf["x4"], 256)
    ref = mask_pack_ref(tb["dgrid3"].reshape(B, 16, 16, 16, 256), h3)
    assert torch.equal(dY3[:, 1:-1, 1:-1, 1:-1], ref), "dY3p interior"
    border = dY3.clone()
    border[:, 1:-1, 1:-1, 1:-1] = 0
    assert torch.count_nonzero(border) == 0, "dY3p border"
    wrong = mask_pack_ref(tb["dgrid3"].reshape(B, 16, 16, 16, 256), h3[:, torch.arange(16, device=dev) ^ 1])
    assert not torch.equal(dY3[:, 1:-1, 1:-1, 1:-1], wrong), "mask_pack3 control (wrong-parity mask)"
    NV = B * 4096
    cb3 = -(-NV // (592 * 8)) + 1 + 8 + 592
    v = ref.to(F64).reshape(-1, 256)
    check("conv3.bias", G["conv3.bias"], v.sum(0), fp32_tol(v.abs().sum(0), cb3))
    control("conv3.bias / heaviest voxel dropped", G["conv3.bias"],
            v.sum(0) - v[v.abs().sum(1).argmax()], fp32_tol(v.abs().sum(0), cb3))
    del h3, v, ref, wrong, border

    # ---- conv3 weight gradient (K = B * 4096 voxels; N = 8 Ct straddles tap boundaries)
    ref, ab = wgrad_ref(dY3, buf["x3"], 16)
    tol = unpack(fp32_tol(ab, c_mma(B * 4096)), 256, Ct)
    check("conv3.weight", G["conv3.weight"], unpack(ref, 256, Ct), tol)
    del ref, ab
    heavy = int(dY3[:, 1:-1, 1:-1, 1:-1].float().abs().reshape(-1, 64 * 256).sum(1).argmax())
    refd, _ = wgrad_ref(dY3, buf["x3"], 16, drop_block=heavy)
    control("conv3.weight / one K block dropped", G["conv3.weight"], unpack(refd, 256, Ct), tol)
    del refd, tol

    # ---- conv3 input gradient: bf16 parity rows [8, B*4096, Ct]
    dg, dga = dgrad_ref(dY3, w["conv3/W"], Ct)                              # [B,32,32,32,Ct]
    ref = to_parity(dg)
    tol = bf16_tol(ref, to_parity(dga), c_mma(8 * 256))
    check("dx3", tb["dx3"], ref, tol)
    control("dx3 / wrong parity", tb["dx3"], to_parity(dg[:, torch.arange(32, device=dev) ^ 1]), tol)
    del dg, dga, ref, tol
    dx3_dense = from_parity(tb["dx3"].to(F64), B, D)                          # what later stages read

    # ---- occupancy stencils (conv1_occ / conv2_occ) from channels 144..159 of dx3
    if occ:
        gne = torch.as_tensor(batch["grid_nontarget_empty"], device=dev).to(F64)[:, None]
        names = ("conv1_occ.weight", "conv1_occ.bias", "conv2_occ.weight", "conv2_occ.bias")
        named = dict(model.named_parameters())
        F, tg = torch.nn.functional, torch.nn.grad
        p64 = [named[n].detach().to(F64) for n in names]
        with torch.no_grad():
            # the stencil backward recomputes its forward in fp32: a pre-activation within
            # rounding of 0 may land on either side, so the ReLU masks are taken from that same
            # fp32 recompute; everything else is float64
            p32 = [named[n].detach().float() for n in names]
            h1_32 = F.relu(F.conv3d(gne.float(), p32[0], p32[1], padding=1))
            m1 = h1_32 > 0
            m2 = F.conv3d(h1_32, p32[2], p32[3], padding=2, dilation=2) > 0
            del h1_32

        def occ_grads(dense):
            h1 = F.conv3d(gne, p64[0], p64[1], padding=1) * m1
            g2 = dense.permute(0, 4, 1, 2, 3) * m2
            gh1 = tg.conv3d_input(h1.shape, p64[2], g2, padding=2, dilation=2) * m1
            return (tg.conv3d_weight(gne, p64[0].shape, gh1, padding=1), gh1.sum((0, 2, 3, 4)),
                    tg.conv3d_weight(h1, p64[2].shape, g2, padding=2, dilation=2), g2.sum((0, 2, 3, 4)))

        dense = dx3_dense[..., 144:160]
        refs = occ_grads(dense)
        # sum|terms|: the same backward on |dY|, |W|, with h1 replaced by the |terms| of its own
        # (recomputed, hence rounded) sum conv(x, |W1|) + |b1|
        h1a = F.conv3d(gne, p64[0].abs(), p64[1].abs(), padding=1) * m1
        g2a = dense.abs().permute(0, 4, 1, 2, 3) * m2
        gh1a = tg.conv3d_input(h1a.shape, p64[2].abs(), g2a, padding=2, dilation=2) * m1
        ab = (tg.conv3d_weight(gne, p64[0].shape, gh1a, padding=1), gh1a.sum((0, 2, 3, 4)),
              tg.conv3d_weight(h1a, p64[2].shape, g2a, padding=2, dilation=2), g2a.sum((0, 2, 3, 4)))
        # the stencil backward runs through torch's fp32 conv3d, where cuDNN may use TF32
        # (both operands rounded to 10 fraction bits: 2 * 2^-11 per product, in the recomputed
        # h1 as well) and an unknown blocked summation order: 2^-10 for each -> 2^-9 sum|terms|
        for n, r, a in zip(names, refs, ab):
            check(n, G[n], r, 2.0 ** -9 * a)
        wrongs = occ_grads(dx3_dense[:, torch.arange(32, device=dev) ^ 1][..., 144:160])
        control("conv2_occ.weight / wrong parity", G[names[2]], wrongs[2], 2.0 ** -9 * ab[2])
        del h1a, g2a, gh1a

    # ---- voxelisation backward: dfeat2 = direct + dX3(voxel) / count (counts from the points)
    flat, _ = voxel_of(points, D)
    bidx = torch.arange(B, device=dev).repeat_interleave(P)
    key = torch.where(flat >= 0, bidx * D ** 3 + flat, torch.full_like(flat, -1))
    cnt = torch.bincount(key[key >= 0], minlength=B * D ** 3).to(F64)
    inside = key >= 0
    ks = key.clamp_min(0)
    gvox = dx3_dense.reshape(-1, Ct)[ks, :144] * inside[:, None]
    c_pt = torch.where(inside, cnt[ks], torch.ones_like(cnt[ks]))[:, None]
    direct = tb["dfeat"][:, 72:216].to(F64)
    ref = direct + gvox / c_pt
    # 1/count, the product and the sum: 3 roundings
    tol = fp32_tol(direct.abs() + gvox.abs() / c_pt, 3)
    check("dfeat2", tb["dfeat2"], ref, tol)
    assert bool((cnt > 1).any()), "the batch must share voxels"
    control("dfeat2 / shared voxels not averaged", tb["dfeat2"], direct + gvox, tol)

    # ---- per-point MLP backward (+ the gradient into the 2-D extractor)
    feat2 = buf["feat2"]
    r = point_mlp_ref(values.detach(), points, buf["feat"][:, :72], tb["dfeat"][:, :72], feat2,
                      tb["dfeat2"], model.conv1_rgb.weight.detach().reshape(64, 32),
                      model.conv1_pcd.weight.detach().reshape(8, 3),
                      model.conv2_rgb.weight.detach().reshape(128, 64),
                      model.conv2_pcd.weight.detach().reshape(16, 8), D / 2.0 - 0.5)
    cm = point_mlp_c(NP)
    for n, (ref, ab) in r.items():
        got = values.grad if n == "values" else G[n].reshape(ref.shape)
        check(n, got, ref, fp32_tol(ab, cm))
    rw = point_mlp_ref(values.detach(), points, buf["feat"][:, :72], tb["dfeat"][:, :72], feat2,
                       tb["dfeat2"], model.conv1_rgb.weight.detach().reshape(64, 32),
                       model.conv1_pcd.weight.detach().reshape(8, 3),
                       model.conv2_rgb.weight.detach().reshape(128, 64),
                       model.conv2_pcd.weight.detach().reshape(16, 8), D / 2.0 - 0.5, drop_direct=True)
    control("values.grad / direct feat1 gradient dropped", values.grad, rw["values"][0],
            fp32_tol(r["values"][1], cm))


# ------------------------------------------------------------------ direct kernel calls: ABI edges
def _lib():
    from morefusion_b200 import _lib as lib
    return lib, lib.lib()


def _bf(x):
    return x.to(torch.bfloat16)


def test_head4_bwd_edges(cuda_device):
    """P = 37 (partial point tile), class ids 1 and nfg, a zero raw quaternion, prefilled
    (accumulated) weight / bias gradients and a row pitch ld > 384 whose pad must stay put."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(11)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)     # noqa: E731
    B, P, nfg, ld = 2, 37, 21, 392
    NP = B * P
    g_rot, g_trans, g_conf = rn(NP, 4), rn(NP, 3), rn(NP)
    raw8 = rn(NP, 8)
    raw8[5, :4] = 0                                                 # |o| = 0
    hd3 = _bf(rn(NP, ld))
    hd3[:, 384:] = 9.0                                              # pad columns (input side)
    W = [_bf(rn(nfg * k, 128) / 10) for k in (4, 3, 1)]
    cid = torch.tensor([1, nfg], dtype=torch.int32, device=dev)
    pitch = torch.tensor([0.01, 0.02], device=dev)
    dhd3 = torch.full((NP, ld), 5.0, dtype=torch.bfloat16, device=dev)
    pre = [rn(nfg * k, 128) for k in (4, 3, 1)] + [rn(nfg * k) for k in (4, 3, 1)]
    out = [p.clone() for p in pre]
    rc = L.mf_train_head4_bwd(*[lib.ptr(x) for x in (g_rot, g_trans, g_conf, raw8, hd3)], ld,
                              *[lib.ptr(x) for x in W], lib.ptr(cid), lib.ptr(pitch), B, P, nfg,
                              lib.ptr(dhd3), lib.ptr(out[0]), lib.ptr(out[3]), lib.ptr(out[1]),
                              lib.ptr(out[4]), lib.ptr(out[2]), lib.ptr(out[5]), lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    fg = (cid.long() - 1).repeat_interleave(P)
    d8, a8 = head4_draw(g_rot, g_trans, g_conf, raw8, pitch.repeat_interleave(P))
    ref, ab = head4_ref(d8, a8, hd3[:, :384], W, fg)
    check("dhd3", dhd3[:, :384], ref, bf16_tol(ref, ab, 20))
    assert bool((dhd3[:, 384:] == 5.0).all()), "dhd3 pad columns written"
    wg = head4_wgrad_ref(d8, a8, hd3[:, :384], fg, nfg)
    c = 16 + 16 + 3 + 1                        # d raw, 16-point CTA sum, 3 CTAs, + the prefill
    for i, h in enumerate(("rot", "trans", "conf")):
        Wr, Wa, b, ba = wg[h]
        check(f"dW {h}", out[i], pre[i].to(F64) + Wr, fp32_tol(Wa + pre[i].abs().to(F64), c))
        check(f"db {h}", out[3 + i], pre[3 + i].to(F64) + b, fp32_tol(ba + pre[3 + i].abs().to(F64), c))
    # the zero quaternion's d raw is g / eps-normalised without the projection term
    assert torch.isfinite(dhd3.float()).all()


@pytest.mark.parametrize("with_dvalues", [True, False])
def test_point_mlp_bwd_edges(cuda_device, with_dvalues):
    """B*P = 111 (not a multiple of the 64-point CTA), prefilled outputs (accumulate), and
    dvalues NULL / non-NULL."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(12)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)     # noqa: E731
    B, P, ldf, ldd = 3, 37, 80, 88
    NP = B * P
    values, points = rn(B, 32, P), rn(B, 3, P) * 8 + 15
    feat, dfeat = _bf(rn(NP, ldf)), _bf(rn(NP, ldd))
    feat2, g2 = rn(NP, 144), rn(NP, 144)
    Ws = [rn(64, 32) / 6, rn(8, 3) / 2, rn(128, 64) / 8, rn(16, 8) / 3]        # [out][in]
    shapes = [(64, 32), (64,), (8, 3), (8,), (128, 64), (128,), (16, 8), (16,)]
    pre = [rn(*s) for s in shapes]
    out = [p.clone() for p in pre]
    dv = torch.full((B, 32, P), 3.0, device=dev)
    rc = L.mf_train_point_mlp_bwd(lib.ptr(values), lib.ptr(points), lib.ptr(feat), ldf, lib.ptr(dfeat),
                                  ldd, lib.ptr(feat2), lib.ptr(g2), *[lib.ptr(w) for w in Ws], B, P,
                                  15.5, *[lib.ptr(o) for o in out],
                                  lib.ptr(dv) if with_dvalues else None, lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    r = point_mlp_ref(values, points, feat[:, :72], dfeat[:, :72], feat2, g2, *Ws, 15.5)
    cm = point_mlp_c(NP) + 1
    names = ["conv1_rgb.weight", "conv1_rgb.bias", "conv1_pcd.weight", "conv1_pcd.bias",
             "conv2_rgb.weight", "conv2_rgb.bias", "conv2_pcd.weight", "conv2_pcd.bias"]
    for n, o, p in zip(names, out, pre):
        ref, ab = r[n]
        check(n, o, p.to(F64) + ref, fp32_tol(ab + p.abs().to(F64), cm))
    if with_dvalues:
        check("dvalues", dv, r["values"][0], fp32_tol(r["values"][1], cm))
    else:
        assert bool((dv == 3.0).all())


@pytest.mark.parametrize("C,col_off", [(4, 12), (512, 472)])
def test_interp_bwd_edges(cuda_device, C, col_off):
    """Coordinates in (-1, 0) (truncation: extrapolating weights), exactly on D - 1 and beyond,
    C = 4 and 512, a non-zero column offset, accumulation into a non-zero grid."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(13)
    B, P, D, div = 2, 300, 8, 4.0
    pts = torch.rand(B, 3, P, generator=g, device=dev) * (D * div + 8) - 4
    pts[:, :, :20] = -torch.rand(B, 3, 20, generator=g, device=dev) * div * 0.99     # x in (-1, 0)
    pts[:, 0, 20:40] = (D - 1) * div                                                 # x = D - 1
    pts[:, :, 40:45] = (D - 1) * div
    ldg = col_off + C + 8
    gv = _bf(torch.randn(B * P, ldg, generator=g, device=dev))
    pre = torch.randn(B, D ** 3, C, generator=g, device=dev)
    grid = pre.clone()
    rc = L.mf_train_interp_bwd(lib.ptr(gv), ldg, col_off, lib.ptr(pts), B, P, C, D, div,
                               lib.ptr(grid), lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    s, sa, n = scatter_ref(gv[:, col_off:col_off + C], pts, C, D, div)
    pre64 = pre.to(F64).reshape(-1, C)
    tol = fp32_tol(sa + pre64.abs(), 4 + n)
    check("dgrid", grid.reshape(-1, C), pre64 + s, tol)
    s_fl, _, _ = scatter_ref(gv[:, col_off:col_off + C], pts, C, D, div, floor=True)
    control("dgrid / floor instead of trunc", grid.reshape(-1, C), pre64 + s_fl, tol)


@pytest.mark.parametrize("act_s2d", [0, 1])
@pytest.mark.parametrize("C", [160, 256])
def test_mask_pack_edges(cuda_device, C, act_s2d):
    """C = 160 (256 % (C/8) != 0: idle threads in the bias reduction), both activation layouts,
    dbias NULL and prefilled, and a sentinel border that must stay untouched."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(14)
    B, D = 2, 8
    dgrid = torch.randn(B, D ** 3, C, generator=g, device=dev)
    act = _bf(torch.randn(B, D, D, D, C, generator=g, device=dev))
    act[0, 0, 0, 0, :8] = 0.0
    act[0, 0, 0, 1, :8] = -0.0
    if act_s2d:
        xp = torch.nn.functional.pad(act.permute(0, 4, 1, 2, 3), (1, 1, 1, 1, 1, 1))
        J = D // 2 + 1
        act_in = xp.reshape(B, C, J, 2, J, 2, J, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(B, J, J, J, 8 * C).contiguous()
    else:
        act_in = act.contiguous()
    ref = mask_pack_ref(dgrid.reshape(B, D, D, D, C), act)
    v = ref.to(F64).reshape(-1, C)
    for with_bias in (True, False):
        out = torch.full((B, D + 2, D + 2, D + 2, C), -7.0, dtype=torch.bfloat16, device=dev)
        pre = torch.randn(C, generator=g, device=dev)
        db = pre.clone()
        rc = L.mf_train_mask_pack(lib.ptr(dgrid), lib.ptr(act_in), act_s2d, B, D, C, lib.ptr(out),
                                  lib.ptr(db) if with_bias else None, lib.stream())
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.equal(out[:, 1:-1, 1:-1, 1:-1], ref)
        border = out.clone()
        border[:, 1:-1, 1:-1, 1:-1] = -7.0
        assert bool((border == -7.0).all()), "border written"
        if with_bias:
            c = -(-B * D ** 3 // (592 * (256 // (C // 8)))) + 1 + 256 // (C // 8) + 592 + 1
            tol = fp32_tol(v.abs().sum(0) + pre.abs().to(F64), c)
            check("dbias", db, pre.to(F64) + v.sum(0), tol)
            control("dbias / last voxel dropped", db, pre.to(F64) + v[:-1].sum(0), tol)
        else:
            assert torch.equal(db, pre)
    wrong = mask_pack_ref(dgrid.reshape(B, D, D, D, C), act[:, torch.arange(D, device=dev) ^ 1])
    assert not torch.equal(out[:, 1:-1, 1:-1, 1:-1], wrong)


def test_vox_bwd_edges(cuda_device):
    """Dropped points (key -1), shared voxels (dup bit), voxels at 0 and D - 1 on every axis."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(15)
    B, P, D, C, ldp, ldg, col_off = 2, 50, 8, 144, 160, 232, 72
    V, Do = D ** 3, D // 2
    vox = torch.randint(0, D, (B, P, 3), generator=g, device=dev)
    vox[:, 0] = 0
    vox[:, 1] = D - 1
    vox[:, 2] = torch.tensor([0, D - 1, 0], device=dev)
    vox[:, 3] = torch.tensor([D - 1, 0, D - 1], device=dev)
    vox[:, 4] = vox[:, 1]                                   # shared with point 1
    vox[:, 5] = vox[:, 1]
    flat = (vox[..., 0] * D + vox[..., 1]) * D + vox[..., 2]
    key = flat + torch.arange(B, device=dev)[:, None] * V
    key[:, 6:9] = -1                                        # dropped
    keyf = key.reshape(-1)
    valid = keyf >= 0
    cnt = torch.bincount(keyf[valid], minlength=B * V)
    dup = valid & (cnt[keyf.clamp_min(0)] > 1)
    keys = torch.where(dup, keyf | 0x40000000, keyf).to(torch.int32)
    dx3 = _bf(torch.randn(8, B * Do ** 3, ldp, generator=g, device=dev))
    gd = _bf(torch.randn(B * P, ldg, generator=g, device=dev))
    out = torch.empty(B * P, C, device=dev)
    rc = L.mf_train_vox_bwd(lib.ptr(dx3), ldp, lib.ptr(keys), B, P, C, D, lib.ptr(gd), ldg, col_off,
                            lib.ptr(out), lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    dense = from_parity(dx3.to(F64), B, D).reshape(B * V, ldp)[:, :C]
    ks = keyf.clamp_min(0)
    c = torch.where(valid, cnt[ks], torch.ones_like(cnt[ks])).to(F64)[:, None]
    gv = dense[ks] * valid[:, None]
    direct = gd[:, col_off:col_off + C].to(F64)
    tol = fp32_tol(direct.abs() + gv.abs() / c, 3)
    check("dfeat2", out, direct + gv / c, tol)
    control("dfeat2 / wrong parity row", out,
            direct + from_parity(dx3.to(F64), B, D)[:, torch.arange(D, device=dev) ^ 1]
            .reshape(B * V, ldp)[ks, :C] * valid[:, None] / c, tol)


def test_relu_mask_colsum_edges(cuda_device):
    """M = 300 (not a multiple of 256), N = 72 (not a multiple of 64), ldx > N, +0 and -0
    activations (both masked), pad columns untouched, colsum accumulating into its output."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(16)
    M, N, ldx, lda = 300, 72, 88, 80
    x = _bf(torch.randn(M, ldx, generator=g, device=dev))
    act = _bf(torch.randn(M, lda, generator=g, device=dev))
    act[:5, :8] = 0.0
    act[5:10, :8] = -0.0
    x0 = x.clone()
    assert L.mf_train_relu_mask(lib.ptr(x), ldx, lib.ptr(act), lda, M, N, lib.stream()) == 0
    torch.cuda.synchronize()
    want = torch.where(act[:, :N].float() > 0, x0[:, :N], torch.zeros_like(x0[:, :N]))
    assert torch.equal(x[:, :N], want)
    assert torch.equal(x[:, N:], x0[:, N:])
    assert torch.count_nonzero(x[:10, :8]) == 0
    for Nc in (72, 70):
        pre = torch.randn(Nc + 2, generator=g, device=dev)
        out = pre.clone()
        assert L.mf_train_colsum(lib.ptr(x), ldx, M, Nc, lib.ptr(out), lib.stream()) == 0
        torch.cuda.synchronize()
        xs = x[:, :Nc].to(F64)
        c = 64 + 4 + -(-M // 256) + 1
        tol = fp32_tol(xs.abs().sum(0) + pre[:Nc].abs().to(F64), c)
        check("colsum", out[:Nc], pre[:Nc].to(F64) + xs.sum(0), tol)
        control("colsum / last row dropped", out[:Nc], pre[:Nc].to(F64) + xs[:-1].sum(0), tol)
        assert torch.equal(out[Nc:], pre[Nc:]), "columns beyond N written"


# ------------------------------------------------------------------ optimizer
def adam_ref(p, g, m, v, alpha_t, gscale, b1=0.9, b2=0.999, eps=1e-8):
    """Chainer's Adam (optimizers/adam.py, eta = 1) in float64 from the fp32 state, with the
    bound of the fused fp32 kernel: m, v each within 4 roundings of their |terms|, the update
    alpha_t m / (sqrt v + eps) within 8 more, p within one rounding of itself."""
    p, g, m, v = [t.to(F64) for t in (p, g, m, v)]
    g = g * gscale
    m2 = m + (1 - b1) * (g - m)
    v2 = v + (1 - b2) * (g * g - v)
    den = v2.sqrt() + eps
    upd = alpha_t * m2 / den
    p2 = p - upd
    em = 4 * U * (m.abs() + (1 - b1) * (g.abs() + m.abs()))
    ev = 4 * U * (v + (1 - b2) * (g * g + v))
    tol_m = em
    tol_v = ev
    # d upd <= alpha_t (em + |m2| (8 u + ev / (2 v2 (1 + eps / sqrt v2))) ) / den
    tol_p = U * p2.abs() + alpha_t * (em + m2.abs() * (8 * U + ev / (2 * v2.clamp_min(1e-300)))) / den
    return (p2, m2, v2), (tol_p, tol_m, tol_v)


@pytest.mark.parametrize("tail", [1, 2, 3])
def test_adam_kernel_tail_and_scale(cuda_device, tail):
    """mf_train_adam on n % 4 = tail elements (scalar tail loop) with grad_scale = 0.5, two
    steps, against float64 Chainer Adam; elements past n stay untouched."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(17 + tail)
    n = 4 * 37 + tail
    p = torch.randn(n + 4, generator=g, device=dev)
    m = torch.zeros(n + 4, device=dev)
    v = torch.zeros(n + 4, device=dev)
    p[n:] = m[n:] = v[n:] = 123.0
    import math
    for t in (1, 2):
        gr = torch.randn(n + 4, generator=g, device=dev)
        gr[n - 1] = 0.0
        alpha_t = float(np.float32(1e-3 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)))
        (pr, mr, vr), (tp, tm, tv) = adam_ref(p[:n], gr[:n], m[:n], v[:n], alpha_t, 0.5)
        rc = L.mf_train_adam(lib.ptr(p), lib.ptr(gr), lib.ptr(m), lib.ptr(v), n, alpha_t, 0.9, 0.999,
                             1e-8, 1.0, 0.5, lib.stream())
        assert rc == 0
        torch.cuda.synchronize()
        check(f"m t={t}", m[:n], mr, tm)
        check(f"v t={t}", v[:n], vr, tv)
        check(f"p t={t}", p[:n], pr, tp)
        assert bool((p[n:] == 123.0).all() and (m[n:] == 123.0).all() and (v[n:] == 123.0).all())
        if t == 1:
            # grad_scale dropped (m1 = (1 - b1) g instead of (1 - b1) g / 2): must be rejected
            control("adam / grad_scale ignored", m[:n], mr * 2, tm)


def test_trainer_adam_and_weight_refresh(cuda_device):
    """Two Trainer steps against float64 Chainer Adam (from flat_g as each step leaves it and the
    previous p, m, v), then the trained model's forward must be bit-identical to a fresh Model
    loaded with the updated parameters (the packed bf16 weights were rebuilt)."""
    from morefusion_b200.contrib.singleview_3d.models import Model, training
    dev = cuda_device
    model, batch = _model_and_batch(2, True, dev, seed=3)
    tr = training.Trainer(model, alpha=1e-3)
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)   # noqa: E731
    feats = dict(class_id=batch["class_id"], values=t(batch["values"]), points=t(batch["points"]),
                 pitch=t(batch["pitch"]), origin=t(batch["origin"]),
                 grid_nontarget_empty=t(batch["grid_nontarget_empty"]))
    def predict(**kw):
        return training.forward_features_with_grad(model, **feats)

    model.predict = predict
    q = np.tile(np.array([[1.0, 0, 0, 0]], np.float32), (2, 1))
    tt = (batch["points"].mean(2) * batch["pitch"][:, None] + batch["origin"]).astype(np.float32)
    with torch.no_grad():
        before = [x.clone() for x in model.forward_features(**feats)]
    for step in (1, 2):
        p0, m0, v0 = tr.flat_p.clone(), tr.flat_m.clone(), tr.flat_v.clone()
        np.random.seed(0)
        tr.step(class_id=batch["class_id"], rgb=None, pcd=None, quaternion_true=q, translation_true=tt)
        torch.cuda.synchronize()
        assert tr.t == step
        alpha_t = float(np.float32(tr.alpha_t()))
        (pr, mr, vr), (tp, tm, tv) = adam_ref(p0, tr.flat_g, m0, v0, alpha_t, 1.0 / tr.world)
        check(f"Trainer m t={step}", tr.flat_m, mr, tm)
        check(f"Trainer v t={step}", tr.flat_v, vr, tv)
        check(f"Trainer p t={step}", tr.flat_p, pr, tp)
        assert float((tr.flat_p - p0).abs().max()) > 0
    with torch.no_grad():
        got = model.forward_features(**feats)
        fresh = Model(n_fg_class=21, with_occupancy=True).to(dev)
        fresh.load_state_dict({k: v.detach().clone() for k, v in model.state_dict().items()})
        want = fresh.forward_features(**feats)
    for a, b, c in zip(got, want, before):
        assert torch.equal(a, b), "forward after the update differs from a fresh model's"
        assert not torch.equal(a, c), "the update did not change the forward"
