"""GPU: the CUDA backward of the singleview_pcd model (training.backward_pcd: csrc/posenet.cu, the
training kernels of csrc/train.cu / csrc/gemm_train.cu and the forward GEMM reused for dX)
replayed stage by stage against float64 references, as tests/test_train_backward_gpu.py does for
singleview_3d.

Each stage's reference is computed from the buffers the launch sequence itself read (the bf16 /
fp32 activations of the forward, the gradients the previous backward launch wrote), so every
stage is held to the precision of its own arithmetic: fp32 results within c * 2^-24 * sum|terms|
with c derived from the kernel's summation chain (commented beside each comparison), bf16 stores
within that plus half a bf16 ulp, masks and the mean's backward bit for bit.  Every stage also
runs a deliberately wrong reference (an off-by-one object or class row, a dropped tail, a shifted
column block, the wrong divisor or mask) through the same comparison and asserts that it fails.

The second half calls the three PoseNet backward entries directly at shapes the model never
produces, checks their rejections, and checks that two backward passes under a Trainer add up."""

import numpy as np
import pytest
import torch

from _bounds import check, control, fp32_tol
from test_train_backward_gpu import bf16_tol, c_mma, head4_draw, head4_ref, head4_wgrad_ref

pytestmark = pytest.mark.gpu

F64 = torch.float64
HEADS = ("rot", "trans", "conf")
PE = "posenet_extractor."
NFG = 21
MF_E_BADARG, MF_E_UNSUPPORTED = -1, -4
MLP = ("conv1_rgb", "conv1_pcd", "conv2_rgb", "conv2_pcd")


# ------------------------------------------------------------------ bounds and references
def c_gemm(K, tc):
    """Chain constant of the forward GEMM family's reduction over K, used for dX: the wgmma chain
    (c_mma) or, on the SIMT kernel, one fma per k in sequence (K roundings)."""
    return c_mma(K) if tc else K


def c_colsum(M):
    """mf_train_colsum: 64 rows per thread in sequence, the 4 row-group partials, then one atomic
    per 256-row block."""
    return 64 + 4 + -(-M // 256)


def c_point_mlp(NP):
    """k_posenet_mlp_bwd, parameter gradients: dz2 = dfeat + dfeat2 (1 rounding), dz1 = that
    + a 128-long fma chain (129), one fma per point over the CTA's 32 points, then one atomic per
    CTA (ceil(NP / 32))."""
    return 130 + 32 + -(-NP // 32)


C_DVALUES = 130 + 64        # dz1 (130) then the 64-long fma chain over conv1_rgb's outputs
C_H1 = 33                   # h1 recomputed in fp32: the bias then <= 32 fmas


def pool_bwd_host(dpooled, h4, P, divisor=None):
    """mf_posenet_pool_bwd on the host: bf16_rn(h4 > 0 ? fp32(dpooled[b]) / fp32(P) : +0), with
    IEEE fp32 division (posenet.cu is built without fast-math).  dpooled [B,N] fp32, h4 [B*P,N]."""
    g = torch.from_numpy(dpooled.cpu().numpy() / np.float32(divisor or P)).repeat_interleave(P, 0)
    return torch.where(h4.cpu().float() > 0, g, torch.zeros_like(g)).to(torch.bfloat16)


def bits(x):
    return x.cpu().contiguous().view(torch.int16)


def pcd_mlp_ref(values, pcd_c, feat12, dfeat, dfeat2, W, *, drop_direct=False, drop_dfeat2=False,
                x_pcd=None):
    """Backward of conv1_* / conv2_* (k_posenet_mlp_bwd) in float64 from its inputs: values
    [B,32,P], pcd_c [B,3,P], dfeat [NP,384], dfeat2 [NP,256] and W {name: ([out][in], bias)}.
    The ReLU masks are the forward's own (feat12 > 0, bf16), so a backward recompute that
    disagrees with the forward fails.  h1 is recomputed here in float64; the kernel's fp32
    recompute differs by <= C_H1 u |terms|, returned as ``h1_err`` and charged to the conv2
    weight gradients.  Returns {name: (ref, sum|terms|)} (+ 'values', + 'h1_err' terms)."""
    B, _, P = values.shape
    xv = values.to(F64).permute(0, 2, 1).reshape(-1, 32)
    xp = (pcd_c if x_pcd is None else x_pcd).to(F64).permute(0, 2, 1).reshape(-1, 3)
    (W1r, b1r), (W1p, b1p), (W2r, _), (W2p, _) = [(w.to(F64), b.to(F64)) for w, b in (W[n] for n in MLP)]
    m1, m2 = feat12[:, :128] > 0, feat12[:, 128:] > 0
    h1 = torch.cat([xv @ W1r.T + b1r, xp @ W1p.T + b1p], 1) * m1
    h1a = torch.cat([xv.abs() @ W1r.abs().T + b1r.abs(), xp.abs() @ W1p.abs().T + b1p.abs()], 1) * m1
    d2 = dfeat[:, 128:].to(F64) + (0 if drop_dfeat2 else dfeat2.to(F64))
    g2 = d2 * m2
    direct = torch.zeros_like(h1) if drop_direct else dfeat[:, :128].to(F64)
    g1 = (direct + torch.cat([g2[:, :128] @ W2r, g2[:, 128:] @ W2p], 1)) * m1
    a1 = (direct.abs() + torch.cat([g2[:, :128].abs() @ W2r.abs(), g2[:, 128:].abs() @ W2p.abs()], 1)) * m1
    ga = g2.abs()
    out = {
        "conv2_rgb.weight": (g2[:, :128].T @ h1[:, :64], ga[:, :128].T @ h1a[:, :64]),
        "conv2_pcd.weight": (g2[:, 128:].T @ h1[:, 64:], ga[:, 128:].T @ h1a[:, 64:]),
        "conv2_rgb.bias": (g2[:, :128].sum(0), ga[:, :128].sum(0)),
        "conv2_pcd.bias": (g2[:, 128:].sum(0), ga[:, 128:].sum(0)),
        "conv1_rgb.weight": (g1[:, :64].T @ xv, a1[:, :64].T @ xv.abs()),
        "conv1_pcd.weight": (g1[:, 64:].T @ xp, a1[:, 64:].T @ xp.abs()),
        "conv1_rgb.bias": (g1[:, :64].sum(0), a1[:, :64].sum(0)),
        "conv1_pcd.bias": (g1[:, 64:].sum(0), a1[:, 64:].sum(0)),
    }
    # |d dW2| from the kernel's rounded h1: sum over points of |g2| * C_H1 u |terms of h1|
    out["h1_err"] = {"conv2_rgb.weight": fp32_tol(ga[:, :128].T @ h1a[:, :64], C_H1),
                     "conv2_pcd.weight": fp32_tol(ga[:, 128:].T @ h1a[:, 64:], C_H1)}
    dv, dva = g1[:, :64] @ W1r, a1[:, :64] @ W1r.abs()
    out["values"] = (dv.reshape(B, P, 32).permute(0, 2, 1), dva.reshape(B, P, 32).permute(0, 2, 1))
    return out


def mlp_tol(r, name, c):
    ref, ab = r[name]
    return fp32_tol(ab, c) + r["h1_err"].get(name, 0)


# ------------------------------------------------------------------ the model run
def _class_ids(B):
    """Both ends of the class range and a repeated class (atomics from different objects into
    the same head-4 rows)."""
    if B == 1:
        return np.array([NFG], np.int32)
    cid = np.array([1 + (4 * i) % NFG for i in range(B)], np.int32)
    cid[0], cid[1], cid[-1] = 1, NFG, 1
    return cid


def _setup(B, P, centred, tc, trainer, dev):
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib.singleview_pcd.models import Model, training
    torch.manual_seed(0)
    model = Model(n_fg_class=NFG).to(dev).train()
    model.load_reference_weights(synthetic.init_weights_pcd(NFG, seed=2))
    model.use_tensor_cores = tc
    tr = training.Trainer(model, alpha=1e-3) if trainer else None
    g = torch.Generator().manual_seed(1000 * B + P)
    values = torch.log_softmax(torch.randn(B, 32, P, generator=g) * 2, dim=1)
    pcd = torch.randn(B, 3, P, generator=g) * 0.04 + torch.tensor([0.02, -0.01, 0.6])[None, :, None]
    inp = dict(class_id=_class_ids(B), values=values.to(dev).requires_grad_(True), pcd=pcd.to(dev),
               center=pcd.median(dim=2).values.to(dev) if centred else None)
    gen = torch.Generator(device=dev).manual_seed(100 + B)
    gs = [torch.randn(B, P, k, generator=gen, device=dev) for k in (4, 3)]
    gs.append(torch.randn(B, P, generator=gen, device=dev))
    return model, tr, inp, gs


def _pass(model, inp, gs):
    """forward_features_with_grad (the 2-D extractor bypassed) and the CUDA backward."""
    from morefusion_b200.contrib.singleview_pcd.models import training
    rot, trans, conf = training.forward_features_with_grad(model, **inp)
    torch.autograd.backward([rot, trans, conf], gs)
    torch.cuda.synchronize()


def _replay(model, inp, gs, tc):
    """Every stage of the forward's training buffers and of backward_pcd against float64.
    Returns {parameter name: (flat float64 reference, flat bound)} for every name of
    param_order, and prints each stage's worst err / bound."""
    from morefusion_b200.contrib.singleview_pcd.models import training
    values = inp["values"]
    dev = values.device
    B, _, P = values.shape
    NP = B * P
    buf = model._work_buffers(B, P, dev)
    tb = training._train_buffers(model, B, P, dev)
    w = model._pack()
    named = dict(model.named_parameters())
    G = {n: named[n].grad for n in training.param_order(model)}
    refs, ratios = {}, []

    def chk(name, got, ref, tol):
        ratios.append((name, check(name, got, ref, tol)))

    def keep(name, ref, tol):
        refs[name] = (ref.reshape(-1), tol.reshape(-1))

    cid = torch.as_tensor(inp["class_id"], device=dev).long()
    fg_pt = (cid - 1).repeat_interleave(P)
    nxt = P if B > 1 else 1             # rows of the next object (B = 1: of the next point)

    # ---- training forward: h4 = relu(conv4(h3)), stored only for the mean's ReLU mask
    h3 = buf["h3"].to(F64)
    W4, b4 = w["conv4/W"].to(F64), w["conv4/b"].to(F64)
    pre = h3 @ W4.T + b4
    ab = h3.abs() @ W4.abs().T + b4.abs()
    c4f = c_gemm(512, tc) + 1           # K = 512 chain, then the bias add of the epilogue
    ref = pre.clamp(min=0)
    tol = bf16_tol(ref, ab, c4f)
    chk("h4", tb["h4"], ref, tol)
    flip = (tb["h4"] > 0) != (pre > 0)
    assert bool((pre.abs() <= fp32_tol(ab, c4f))[flip].all()), "h4: ReLU mask differs beyond rounding"
    control("h4 / next object's rows", tb["h4"], ref.roll(nxt, 0), tol)
    # pooled (the other conv4 GEMM, OUT_OBJ_SUM_F32 + mf_posenet_pool): the chain above, 16 rows
    # per group in sequence, the object's ceil(P/16) + 1 groups in sequence, the division by P
    cpool = c4f + 16 + -(-P // 16) + 1 + 1
    pooled_ref = ref.reshape(B, P, 1024).mean(1)
    tol = fp32_tol(ab.reshape(B, P, 1024).mean(1), cpool)
    chk("pooled", buf["pooled"], pooled_ref, tol)
    control("pooled / x 1.01", buf["pooled"], pooled_ref * 1.01, tol)
    del h3, pre, ab, ref, flip, tol

    # ---- raw8: the class-selected conv4_{rot,trans,conf} pre-activations (k_head4_pose: one
    # 128-long fma chain then the bias add -> 129 roundings)
    hd3 = buf["hd3"].to(F64)

    def raw8_ref(fg):
        r, a = [], []
        for i, (h, k) in enumerate((("rot", 4), ("trans", 3), ("conf", 1))):
            Wh, bh = w[f"conv4_{h}/W"].to(F64), w[f"conv4_{h}/b"].to(F64)
            x = hd3[:, 128 * i:128 * (i + 1)]
            idx = fg[:, None] * k + torch.arange(k, device=dev)[None]
            r.append((x @ Wh.T + bh).gather(1, idx))
            a.append((x.abs() @ Wh.abs().T + bh.abs()).gather(1, idx))
        return torch.cat(r, 1), torch.cat(a, 1)

    ref, ab = raw8_ref(fg_pt)
    tol = fp32_tol(ab, 129)
    chk("raw8", tb["raw8"], ref, tol)
    control("raw8 / neighbouring class rows", tb["raw8"], raw8_ref((fg_pt + 1) % NFG)[0], tol)

    # ---- head 4 + pose epilogue, pitch 1 (trans = centred pcd + center + offset)
    g_rot, g_trans, g_conf = gs
    ones = torch.ones(NP, device=dev)
    d8, a8 = head4_draw(g_rot.reshape(NP, 4), g_trans.reshape(NP, 3), g_conf.reshape(NP), tb["raw8"], ones)
    W4h = (w["conv4_rot/W"], w["conv4_trans/W"], w["conv4_conf/W"])
    ref, ab = head4_ref(d8, a8, buf["hd3"], W4h, fg_pt)
    # c = 20: d raw is ~12 fp32 roundings deep (4-term dot / norm, sqrt, divisions, products;
    # expf's 2-ulp error enters through s) -> 16, then the <= 4-term row sum
    tol = bf16_tol(ref, ab, 20)
    chk("dhd3", tb["dhd3"], ref, tol)
    control("dhd3 / class row + 1", tb["dhd3"], head4_ref(d8, a8, buf["hd3"], W4h, (fg_pt + 1) % NFG)[0], tol)
    d8h, a8h = head4_draw(g_rot.reshape(NP, 4), g_trans.reshape(NP, 3), g_conf.reshape(NP), tb["raw8"],
                          ones * 0.5)
    control("dhd3 / pitch 0.5", tb["dhd3"], head4_ref(d8h, a8h, buf["hd3"], W4h, fg_pt)[0], tol)
    wg = head4_wgrad_ref(d8, a8, buf["hd3"], fg_pt, NFG)
    ncls = int(torch.bincount(cid - 1, minlength=NFG).max())
    # c: d raw (16) + 16 points summed per CTA + one atomic per CTA of every object of the class
    c4 = 16 + 16 + ncls * -(-P // 16)
    for h in HEADS:
        W, Wa, b, ba = wg[h]
        tw, tbias = fp32_tol(Wa, c4), fp32_tol(ba, c4)
        chk(f"conv4_{h}.weight", G[f"conv4_{h}.weight"].reshape(W.shape), W, tw)
        chk(f"conv4_{h}.bias", G[f"conv4_{h}.bias"], b, tbias)
        keep(f"conv4_{h}.weight", W, tw)
        keep(f"conv4_{h}.bias", b, tbias)
    W, Wa, _, _ = wg["trans"]
    control("conv4_trans.weight / pitch 0.5", G["conv4_trans.weight"].reshape(W.shape),
            head4_wgrad_ref(d8h, a8h, buf["hd3"], fg_pt, NFG)["trans"][0], fp32_tol(Wa, c4))
    del hd3, d8, a8, d8h, a8h, wg

    # ---- head layers 3, 2: dW (TN GEMM over NP rows), db (colsum), dX (forward GEMM on the
    # transposed weights; the reference uses the FORWARD pack, so a stale training pack fails)
    c_col = c_colsum(NP)
    for layer, dz, x, n_out, k_in, dx in ((3, tb["dhd3"], buf["hd2"], 128, 256, tb["dhd2"]),
                                          (2, tb["dhd2"], buf["hd1"], 256, 640, tb["dhd1"])):
        dz64, x64 = dz.to(F64), x.to(F64)
        ref_dx = torch.zeros(NP, 3 * k_in, dtype=F64, device=dev)
        ab_dx = torch.zeros_like(ref_dx)
        for i, h in enumerate(HEADS):
            zi, xi = dz64[:, i * n_out:(i + 1) * n_out], x64[:, i * k_in:(i + 1) * k_in]
            ref = zi.T @ xi
            tol = fp32_tol(zi.abs().T @ xi.abs(), c_mma(NP))
            chk(f"conv{layer}_{h}.weight", G[f"conv{layer}_{h}.weight"].reshape(ref.shape), ref, tol)
            keep(f"conv{layer}_{h}.weight", ref, tol)
            if i == 0:
                control(f"conv{layer}_rot.weight / last 64 rows", G[f"conv{layer}_{h}.weight"].reshape(ref.shape),
                        zi[:NP - 64].T @ xi[:NP - 64], tol)
            tol = fp32_tol(zi.abs().sum(0), c_col)
            chk(f"conv{layer}_{h}.bias", G[f"conv{layer}_{h}.bias"], zi.sum(0), tol)
            keep(f"conv{layer}_{h}.bias", zi.sum(0), tol)
            Wi = w[f"conv{layer}_{h}/W"].to(F64)                              # [n_out, k_in] bf16
            ref_dx[:, i * k_in:(i + 1) * k_in] = zi @ Wi
            ab_dx[:, i * k_in:(i + 1) * k_in] = zi.abs() @ Wi.abs()
        m = x > 0
        tol = bf16_tol(ref_dx, ab_dx, c_gemm(n_out, tc)) * m
        chk(f"dhd{layer - 1} (masked)", dx, ref_dx * m, tol)
        control(f"dhd{layer - 1} / other head's mask", dx, ref_dx * torch.roll(m, k_in, 1), tol)
        if layer == 3:
            control("dhd2 / col_off + 8", dx, torch.roll(ref_dx, 8, 1) * m, tol)
    del dz64, x64, ref_dx, ab_dx, m, tol

    # ---- layer 1: the [feat1|feat2] columns per point, the feat3 columns per object
    dz1 = tb["dhd1"].to(F64)
    f12 = buf["feat12"].to(F64)
    gw1_ref = torch.empty(1920, 1408, dtype=F64, device=dev)
    gw1_tol = torch.empty_like(gw1_ref)
    ref = dz1.T @ f12
    tol = fp32_tol(dz1.abs().T @ f12.abs(), c_mma(NP))
    chk("gw1[:, :384]", tb["gw1"][:, :384], ref, tol)
    control("gw1[:, :384] / last 64 rows", tb["gw1"][:, :384], dz1[:NP - 64].T @ f12[:NP - 64], tol)
    gw1_ref[:, :384], gw1_tol[:, :384] = ref, tol
    # seg: each object's 256-row blocks (c_colsum's chain within a block) added in sequence
    tol = fp32_tol(dz1.abs().reshape(B, P, 1920).sum(1), 64 + 4 + -(-P // 256))
    chk("seg", tb["seg"], dz1.reshape(B, P, 1920).sum(1), tol)
    shifted = torch.cat([dz1[16:], dz1.new_zeros(16, 1920)]).reshape(B, P, 1920).sum(1)
    control("seg / object rows shifted by 16", tb["seg"], shifted, tol)
    s64, pl = tb["seg"].to(F64), buf["pooled"].to(F64)
    # dW1b, db1: one fma (add) per object in sequence (B), then the += into the zeroed buffer
    ref = s64.T @ pl
    tol = fp32_tol(s64.abs().T @ pl.abs(), B + 1)
    chk("gw1[:, 384:]", tb["gw1"][:, 384:], ref, tol)
    wrong = s64.T @ pl.roll(1, 0) if B > 1 else torch.zeros_like(ref)
    control("gw1[:, 384:] / pooled of the next object" if B > 1 else "gw1[:, 384:] / object dropped",
            tb["gw1"][:, 384:], wrong, tol)
    gw1_ref[:, 384:], gw1_tol[:, 384:] = ref, tol
    gb1_ref, gb1_tol = s64.sum(0), fp32_tol(s64.abs().sum(0), B + 1)
    chk("gb1", tb["gb1"], gb1_ref, gb1_tol)
    # dpooled: one sequential fma chain over the 1920 rows
    W1b = w["head1/W"][:, 384:].to(F64)
    tol = fp32_tol(s64.abs() @ W1b.abs(), 1920)
    chk("dpooled", tb["dpooled"], s64 @ W1b, tol)
    control("dpooled / W1b columns shifted by 8", tb["dpooled"], s64 @ W1b.roll(8, 1), tol)
    W1a = w["head1/W"][:, :384].to(F64)
    tol = fp32_tol(dz1.abs() @ W1a.abs(), c_gemm(1920, tc))           # fp32 output, no bias
    chk("dfeat", tb["dfeat"], dz1 @ W1a, tol)
    control("dfeat / last K block dropped", tb["dfeat"], dz1[:, :1856] @ W1a[:1856], tol)
    for i, h in enumerate(HEADS):
        rows = slice(i * 640, (i + 1) * 640)
        assert torch.equal(G[f"conv1_{h}.weight"].reshape(640, 1408), tb["gw1"][rows]), h
        assert torch.equal(G[f"conv1_{h}.bias"], tb["gb1"][rows]), h
        keep(f"conv1_{h}.weight", gw1_ref[rows], gw1_tol[rows])
        keep(f"conv1_{h}.bias", gb1_ref[rows], gb1_tol[rows])
    del dz1, f12, gw1_ref, gw1_tol, s64, W1a, W1b, shifted, wrong

    # ---- the mean's backward, bit for bit
    want = pool_bwd_host(tb["dpooled"], tb["h4"], P)
    assert torch.equal(bits(tb["dz4"]), bits(want)), "dz4"
    assert not torch.equal(bits(tb["dz4"]), bits(pool_bwd_host(tb["dpooled"], tb["h4"], P, NP if B > 1 else P - 1))), \
        "dz4 control (wrong divisor)"
    assert not torch.equal(bits(tb["dz4"]), bits(pool_bwd_host(tb["dpooled"], tb["h4"].roll(nxt, 0), P))), \
        "dz4 control (next object's mask)"
    del want

    # ---- conv4, conv3: as the heads; conv3 reads feat2 = feat12[:, 128:], its dX (dfeat2) is
    # fp32 and unmasked (the point-MLP backward masks it)
    for n, dz, x, n_out, dx, act in (("conv4", tb["dz4"], buf["h3"], 1024, tb["dh3"], buf["h3"]),
                                     ("conv3", tb["dh3"], buf["feat12"][:, 128:], 512, tb["dfeat2"], None)):
        z, xx = dz.to(F64), x.to(F64)
        ref = z.T @ xx
        tol = fp32_tol(z.abs().T @ xx.abs(), c_mma(NP))
        got = G[PE + n + ".weight"].reshape(ref.shape)
        chk(n + ".weight", got, ref, tol)
        keep(PE + n + ".weight", ref, tol)
        if n == "conv4":
            control("conv4.weight / last 64 rows", got, z[:NP - 64].T @ xx[:NP - 64], tol)
        else:
            control("conv3.weight / feat12[:, :256]", got, z.T @ buf["feat12"][:, :256].to(F64), tol)
        tol = fp32_tol(z.abs().sum(0), c_col)
        chk(n + ".bias", G[PE + n + ".bias"], z.sum(0), tol)
        keep(PE + n + ".bias", z.sum(0), tol)
        Wf = w[n + "/W"].to(F64)
        ref, ab = z @ Wf, z.abs() @ Wf.abs()
        if act is not None:
            m = act > 0
            tol = bf16_tol(ref, ab, c_gemm(n_out, tc)) * m
            chk("dh3 (masked)", dx, ref * m, tol)
            control("dh3 / unmasked", dx, ref, tol)
        else:
            tol = fp32_tol(ab, c_gemm(n_out, tc))
            chk("dfeat2", dx, ref, tol)
            control("dfeat2 / last 64 rows of K", dx, z[:, :n_out - 64] @ Wf[:n_out - 64], tol)
    del z, xx, ref, ab, tol

    # ---- conv1_* / conv2_* and the gradient to values
    pe = model.posenet_extractor
    Wm = {n: (getattr(pe, n).weight.detach()[:, :, 0], getattr(pe, n).bias.detach()) for n in MLP}
    args = (values.detach(), buf["pcd_c"], buf["feat12"], tb["dfeat"], tb["dfeat2"], Wm)
    r = pcd_mlp_ref(*args)
    cm = c_point_mlp(NP)
    for n in (f"{m}.{k}" for m in MLP for k in ("weight", "bias")):
        ref = r[n][0]
        tol = mlp_tol(r, n, cm)
        chk(n, G[PE + n].reshape(ref.shape), ref, tol)
        keep(PE + n, ref, tol)
    tol_v = fp32_tol(r["values"][1], C_DVALUES)
    chk("values.grad", values.grad, r["values"][0], tol_v)
    rw = pcd_mlp_ref(*args, drop_dfeat2=True)
    control("conv2_pcd.weight / dfeat2 dropped", G[PE + "conv2_pcd.weight"].reshape(128, 64),
            rw["conv2_pcd.weight"][0], mlp_tol(r, "conv2_pcd.weight", cm))
    rw = pcd_mlp_ref(*args, drop_direct=True)
    control("values.grad / direct dfeat dropped", values.grad, rw["values"][0], tol_v)
    if inp["center"] is not None:
        rw = pcd_mlp_ref(*args, x_pcd=inp["pcd"])
        control("conv1_pcd.weight / uncentred pcd", G[PE + "conv1_pcd.weight"].reshape(64, 3),
                rw["conv1_pcd.weight"][0], mlp_tol(r, "conv1_pcd.weight", cm))
    assert set(refs) == set(training.param_order(model))
    print(f"\nB={B} P={P} {'tc' if tc else 'simt'}: worst err/bound per stage")
    for name, ratio in ratios:
        print(f"  {name:28s} {ratio:.3g}")
    return refs


@pytest.mark.parametrize("B,P,centred,tc,trainer", [
    (1, 1000, True, True, False),
    (8, 1000, True, True, True),        # the checks read flat_g through the Trainer's views
    (8, 1000, True, False, False),      # the SIMT GEMM for every forward GEMM and dX
    (16, 1000, True, True, False),
    (3, 1003, False, True, False),      # objects straddle 16-row groups, 32-point CTAs, 256-row blocks
], ids=["B1", "B8-trainer", "B8-simt", "B16", "B3-P1003-uncentred"])
def test_backward_stage_replay(cuda_device, B, P, centred, tc, trainer):
    from morefusion_b200.contrib.singleview_pcd.models import training
    model, tr, inp, gs = _setup(B, P, centred, tc, trainer, cuda_device)
    _pass(model, inp, gs)
    if tr is not None:
        named = dict(model.named_parameters())
        for n in training.param_order(model):
            assert named[n].grad.data_ptr() == tr.flat_g[tr.offs[n][0]:].data_ptr(), n
    log = model.launch_log
    assert any(e[0] == ("tc" if tc else "simt") for e in log)
    assert not any(e[0] == ("simt" if tc else "tc") for e in log), log
    _replay(model, inp, gs, tc)


def test_trainer_accumulates_two_backward_passes(cuda_device):
    """Two backward passes without zero_grad() under a Trainer: every gradient of param_order is
    the sum of two passes.  The stage inputs of the two passes are identical (the forward and the
    backward's intermediate buffers are deterministic; asserted), so the sum of two separate
    passes is 2x the float64 reference of one pass.  Each pass lands within its stage bound tol
    of that reference; the second pass's roundings act on partial sums up to twice as large, so
    the two together are within tol + 2 tol."""
    from morefusion_b200.contrib.singleview_pcd.models import training
    model, tr, inp, gs = _setup(2, 1000, True, True, True, cuda_device)
    tr.zero_grad()
    _pass(model, inp, gs)
    refs = _replay(model, inp, gs, True)
    tb = training._train_buffers(model, 2, 1000, cuda_device)
    first = {k: tb[k].clone() for k in ("raw8", "dhd1", "seg", "dpooled", "dz4", "dfeat", "dfeat2")}
    _pass(model, inp, gs)
    for k, v in first.items():
        assert torch.equal(tb[k], v), f"{k} differs between the passes"
    named = dict(model.named_parameters())
    bad = []                            # every parameter that does not add up, not just the first
    for n in training.param_order(model):
        ref, tol = refs[n]
        try:
            check(f"{n} after two passes", named[n].grad.reshape(-1), 2 * ref, 3 * tol)
        except AssertionError as e:
            bad.append(str(e))
    assert not bad, "\n".join(bad)
    for h in HEADS:
        for k in ("weight", "bias"):
            n = f"conv1_{h}.{k}"
            ref, tol = refs[n]
            control(f"{n} / one pass only", named[n].grad.reshape(-1), ref, 3 * tol)


# ------------------------------------------------------------------ direct kernel calls
def _lib():
    from morefusion_b200 import _lib as lib
    return lib, lib.lib()


@pytest.mark.parametrize("B,P,N", [(1, 16, 1024), (3, 1003, 200), (2, 17, 8)])
def test_pool_bwd_direct(cuda_device, B, P, N):
    """B*P*N = 16384, 601800, 272 (the last two not a multiple of the 256-thread CTA); h4 with
    +0, -0, NaN and negative values (all masked to +0); a sentinel past the last element."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(21 + P)
    NP = B * P
    dpooled = torch.randn(B, N, generator=g, device=dev) * 3
    h4 = torch.randn(NP, N, generator=g, device=dev).to(torch.bfloat16)
    h4[0, :4] = 0.0
    h4[1, :4] = -0.0
    h4[2, :4] = float("nan")
    h4[3, :4] = -1.5
    out = torch.full((NP * N + 16,), 5.0, dtype=torch.bfloat16, device=dev)
    assert L.mf_posenet_pool_bwd(lib.ptr(dpooled), lib.ptr(h4), B, P, N, lib.ptr(out), lib.stream()) == 0
    torch.cuda.synchronize()
    got = out[:NP * N].reshape(NP, N)
    assert torch.equal(bits(got), bits(pool_bwd_host(dpooled, h4, P)))
    assert bool((bits(got[:4, :4]) == 0).all()), "masked entries are not +0"
    assert bool((out[NP * N:] == 5.0).all()), "written past the end"
    assert not torch.equal(bits(got), bits(pool_bwd_host(dpooled, h4, P, P + 1)))


@pytest.mark.parametrize("rows,ldw,B", [(1920, 1408, 1), (1920, 1408, 33), (7, 1024, 33), (7, 1030, 1)])
def test_obj_bias_bwd_direct(cuda_device, rows, ldw, B):
    """The model's shape (rows 1920, W at column 384 of a 1408 pitch) and rows = 7; B = 1 and
    33; dW of pitch 1500 whose columns 1024..1499 hold sentinels; prefilled dW and db (+=), db
    NULL; dpooled overwritten, with a sentinel past it."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(rows + B)
    K, lddw = 1024, 1500
    s = torch.randn(B, rows, generator=g, device=dev)
    pooled = torch.rand(B, K, generator=g, device=dev)
    Wfull = (torch.randn(rows, ldw, generator=g, device=dev) / 32).to(torch.bfloat16)
    W = Wfull[:, ldw - K:]
    pre_dW = torch.randn(rows, lddw, generator=g, device=dev)
    pre_dW[:, K:] = 9.0
    pre_db = torch.randn(rows, generator=g, device=dev)
    s64, p64, W64 = s.to(F64), pooled.to(F64), W.to(F64)
    # dW, db: B fmas / adds in sequence, then the += onto the prefill
    tol_w = fp32_tol(s64.abs().T @ p64 + pre_dW[:, :K].abs().to(F64), B + 1)
    tol_b = fp32_tol(s64.abs().sum(0) + pre_db.abs().to(F64), B + 1)
    tol_x = fp32_tol(s64.abs() @ W64.abs(), rows)                       # rows fmas in sequence
    for with_db in (True, False):
        dW, db = pre_dW.clone(), pre_db.clone()
        dp = torch.full((B * K + 8,), 7.0, device=dev)
        assert L.mf_posenet_obj_bias_bwd(lib.ptr(s), lib.ptr(pooled), lib.ptr(W), ldw, rows, K, B, lib.ptr(dW),
                                         lddw, lib.ptr(db) if with_db else None, lib.ptr(dp), lib.stream()) == 0
        torch.cuda.synchronize()
        ref_w = pre_dW[:, :K].to(F64) + s64.T @ p64
        check("dW", dW[:, :K], ref_w, tol_w)
        control("dW / last object dropped", dW[:, :K], pre_dW[:, :K].to(F64) + s64[:-1].T @ p64[:-1], tol_w)
        assert bool((dW[:, K:] == 9.0).all()), "dW columns past K written"
        if with_db:
            check("db", db, pre_db.to(F64) + s64.sum(0), tol_b)
        else:
            assert torch.equal(db, pre_db)
        check("dpooled", dp[:B * K].reshape(B, K), s64 @ W64, tol_x)
        control("dpooled / W columns shifted by 8", dp[:B * K].reshape(B, K), s64 @ W64.roll(8, 1), tol_x)
        assert bool((dp[B * K:] == 7.0).all()), "dpooled written past the end"


def _mlp_weights(dev, g):
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)     # noqa: E731
    return {"conv1_rgb": (rn(64, 32) / 6, rn(64) * 0.1), "conv1_pcd": (rn(64, 3) * 2, rn(64) * 0.1),
            "conv2_rgb": (rn(128, 64) / 8, rn(128) * 0.1), "conv2_pcd": (rn(128, 64) / 8, rn(128) * 0.1)}


@pytest.mark.parametrize("with_dvalues", [True, False])
@pytest.mark.parametrize("B,P", [(1, 17), (3, 1003)])
def test_point_mlp_bwd_direct(cuda_device, B, P, with_dvalues):
    """B*P = 17 and 3009 (CTAs of 32 points straddle objects, a partial last CTA), prefilled
    parameter gradients (added to), dvalues NULL (the parameter gradients unchanged) or not.  The
    activations come from mf_posenet_point_mlp on the same inputs, as in the model."""
    lib, L = _lib()
    dev = cuda_device
    g = torch.Generator(device=dev).manual_seed(31 + B * P)
    NP = B * P
    Wm = _mlp_weights(dev, g)
    values = torch.randn(B, 32, P, generator=g, device=dev)
    pcd = torch.randn(B, 3, P, generator=g, device=dev) * 0.5
    feat12 = torch.zeros(NP, 384, dtype=torch.bfloat16, device=dev)
    pcd_c = torch.empty(B, 3, P, device=dev)
    fwd = []
    for n in MLP:
        fwd += [Wm[n][0].t().contiguous(), Wm[n][1]]
    assert L.mf_posenet_point_mlp(lib.ptr(values), lib.ptr(pcd), None, *[lib.ptr(t) for t in fwd], B, P,
                                  lib.ptr(feat12), 384, lib.ptr(pcd_c), lib.stream()) == 0
    dfeat = torch.randn(NP, 384, generator=g, device=dev)
    dfeat2 = torch.randn(NP, 256, generator=g, device=dev)
    names = [f"{n}.{k}" for n in MLP for k in ("weight", "bias")]
    pre = [torch.randn(*(Wm[n.split(".")[0]][0 if n.endswith("weight") else 1].shape), generator=g, device=dev)
           for n in names]
    out = [p.clone() for p in pre]
    dv = torch.full((B * 32 * P + 8,), 3.0, device=dev)
    bwd = []
    for n in MLP:
        bwd += [Wm[n][0].contiguous(), Wm[n][1]]
    assert L.mf_posenet_point_mlp_bwd(lib.ptr(values), lib.ptr(pcd_c), *[lib.ptr(t) for t in bwd], B, P,
                                      lib.ptr(dfeat), lib.ptr(dfeat2), *[lib.ptr(o) for o in out],
                                      lib.ptr(dv) if with_dvalues else None, lib.stream()) == 0
    torch.cuda.synchronize()
    assert bool((feat12 > 0).any()) and bool((feat12 == 0).any())          # both sides of every mask
    r = pcd_mlp_ref(values, pcd_c, feat12, dfeat, dfeat2, Wm)
    cm = c_point_mlp(NP) + 1                                               # + the prefill
    for n, o, p in zip(names, out, pre):
        ref = r[n][0]
        check(n, o, p.to(F64) + ref, mlp_tol(r, n, cm) + fp32_tol(p.abs().to(F64), cm))
    rw = pcd_mlp_ref(values, pcd_c, feat12, dfeat, dfeat2, Wm, drop_dfeat2=True)
    control("conv2_rgb.weight / dfeat2 dropped", out[4], pre[4].to(F64) + rw["conv2_rgb.weight"][0],
            mlp_tol(r, "conv2_rgb.weight", cm) + fp32_tol(pre[4].abs().to(F64), cm))
    if with_dvalues:
        tol = fp32_tol(r["values"][1], C_DVALUES)
        check("dvalues", dv[:B * 32 * P].reshape(B, 32, P), r["values"][0], tol)
        rw = pcd_mlp_ref(values, pcd_c, feat12, dfeat, dfeat2, Wm, drop_direct=True)
        control("dvalues / direct dfeat dropped", dv[:B * 32 * P].reshape(B, 32, P), rw["values"][0], tol)
        assert bool((dv[B * 32 * P:] == 3.0).all()), "dvalues written past the end"
    else:
        assert bool((dv == 3.0).all()), "dvalues written although NULL"


def test_posenet_bwd_rejections(cuda_device):
    """B <= 0 (and B > 65535 for the per-object bias, whose grid has one row per object), P <= 0,
    N or rows <= 0, each required NULL pointer and K != 1024: rejected before any launch, so the
    prefilled outputs stay as they were."""
    lib, L = _lib()
    dev = cuda_device
    p, st = lib.ptr, lib.stream()
    f = lambda *s: torch.full(s, 7.0, device=dev)                  # noqa: E731
    # ---- pool_bwd
    dpooled, h4 = f(2, 64), torch.ones(32, 64, dtype=torch.bfloat16, device=dev)
    dz = torch.full((32, 64), 7.0, dtype=torch.bfloat16, device=dev)
    for B, P, N in ((0, 16, 64), (-1, 16, 64), (2, 0, 64), (2, -3, 64), (2, 16, 0), (2, 16, -1)):
        assert L.mf_posenet_pool_bwd(p(dpooled), p(h4), B, P, N, p(dz), st) == MF_E_BADARG, (B, P, N)
    for i in range(3):
        a = [p(dpooled), p(h4), p(dz)]
        a[i] = None
        assert L.mf_posenet_pool_bwd(a[0], a[1], 2, 16, 64, a[2], st) == MF_E_BADARG, i
    # ---- obj_bias_bwd
    s, pooled = f(2, 8), f(2, 1024)
    W = torch.ones(8, 1024, dtype=torch.bfloat16, device=dev)
    dW, db, dp = f(8, 1024), f(8), f(2, 1024)
    ok = [p(s), p(pooled), p(W), 1024, 8, 1024, 2, p(dW), 1024, p(db), p(dp), st]
    for i, v in ((6, 0), (6, -1), (6, 65536), (4, 0), (4, -2)):
        a = list(ok)
        a[i] = v
        assert L.mf_posenet_obj_bias_bwd(*a) == MF_E_BADARG, (i, v)
    for i in (0, 1, 2, 7, 10):
        a = list(ok)
        a[i] = None
        assert L.mf_posenet_obj_bias_bwd(*a) == MF_E_BADARG, i
    for K in (512, 1023, 1032):
        a = list(ok)
        a[5] = K
        assert L.mf_posenet_obj_bias_bwd(*a) == MF_E_UNSUPPORTED, K
    # ---- point_mlp_bwd
    B, P = 2, 16
    ins = [f(B, 32, P), f(B, 3, P), f(64, 32), f(64), f(64, 3), f(64), f(128, 64), f(128), f(128, 64), f(128)]
    grads = [f(B * P, 384), f(B * P, 256)]
    outs = [f(64, 32), f(64), f(64, 3), f(64), f(128, 64), f(128), f(128, 64), f(128), f(B, 32, P)]
    ok = [p(t) for t in ins] + [B, P] + [p(t) for t in grads + outs] + [st]
    for i, v in ((10, 0), (10, -1), (11, 0), (11, -5)):
        a = list(ok)
        a[i] = v
        assert L.mf_posenet_point_mlp_bwd(*a) == MF_E_BADARG, (i, v)
    for i in [*range(10), *range(12, 22)]:                          # all but dvalues (optional)
        a = list(ok)
        a[i] = None
        assert L.mf_posenet_point_mlp_bwd(*a) == MF_E_BADARG, i
    torch.cuda.synchronize()
    assert bool((dz == 7.0).all()), "pool_bwd launched"
    for t in (dW, db, dp, *outs):
        assert bool((t == 7.0).all()), "a rejected call wrote its output"
