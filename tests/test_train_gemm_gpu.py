"""GPU: the training-side wgmma GEMMs (csrc/gemm_train.cu) against plain PyTorch fp32
references of the same operations (torch.matmul / torch.nn.grad.conv3d_*), bf16 operands."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def L():
    from morefusion_b200 import _lib
    return _lib, _lib.lib()


def bf(x):
    return x.to(torch.bfloat16)


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("M,N,K,groups", [(8000, 1920, 984, 1), (8000, 256, 640, 3), (8000, 128, 256, 3),
                                          (500, 128, 64, 1)])
def test_gemm_tn(cuda_device, M, N, K, groups):
    """out[g][n, k] = sum_m dZ[m, g*N + n] * X[m, g*K + k]: both operands MN-major."""
    lib, l = L()
    torch.manual_seed(0)
    ldz = groups * N
    ldx = (groups * K + 63) // 64 * 64
    dZ = bf(torch.randn(M, ldz, device=cuda_device))
    X = bf(torch.randn(M, ldx, device=cuda_device))
    out = torch.full((groups, N, K), 7.0, device=cuda_device)
    rc = l.mf_train_gemm_tn(lib.ptr(dZ), ldz, lib.ptr(X), ldx, M, N, K, lib.ptr(out), K, groups,
                            N, K, N * K, 0, lib.stream())
    assert rc == 0
    for g in range(groups):
        want = dZ[:, g * N:(g + 1) * N].float().T @ X[:, g * K:(g + 1) * K].float()
        assert rel_err(out[g], want) < 2e-3, (g, rel_err(out[g], want))
    # accumulate = 1 adds on top
    rc = l.mf_train_gemm_tn(lib.ptr(dZ), ldz, lib.ptr(X), ldx, M, N, K, lib.ptr(out), K, groups,
                            N, K, N * K, 1, lib.stream())
    assert rc == 0
    want = 2 * (dZ[:, :N].float().T @ X[:, :K].float())
    assert rel_err(out[0], want) < 2e-3


def s2d_pack(x):
    """[B,C,D,D,D] fp32 -> bf16 [B,J,J,J,8*C] with J = D/2+1 (cnn.cu layout: xpad padded by 1)."""
    B, C, D = x.shape[:3]
    J = D // 2 + 1
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1, 1, 1))                  # [B,C,D+2,...]
    xp = xp.reshape(B, C, J, 2, J, 2, J, 2)                               # b c jd rd jh rh jw rw
    xp = xp.permute(0, 2, 4, 6, 3, 5, 7, 1)                               # b jd jh jw rd rh rw c
    return bf(xp.reshape(B, J, J, J, 8 * C)).contiguous()


def pad_cl(dy):
    """[B,C,Do,Do,Do] -> bf16 channels-last [B,Do+2,Do+2,Do+2,C] with a zero border."""
    return bf(torch.nn.functional.pad(dy, (1, 1, 1, 1, 1, 1)).permute(0, 2, 3, 4, 1)).contiguous()


@pytest.mark.parametrize("B,Ci,Co,D", [(2, 160, 256, 32), (2, 256, 512, 16)])
def test_conv_wgrad(cuda_device, B, Ci, Co, D):
    lib, l = L()
    from morefusion_b200.contrib.singleview_3d.models.model import pack_conv_k4s2_weight
    torch.manual_seed(1)
    Do = D // 2
    x = bf(torch.randn(B, Ci, D, D, D, device=cuda_device)).float()
    dy = bf(torch.randn(B, Co, Do, Do, Do, device=cuda_device)).float()
    want = torch.nn.grad.conv3d_weight(x, (Co, Ci, 4, 4, 4), dy, stride=2, padding=1)
    want = pack_conv_k4s2_weight(want).float()                            # [Co, 64*Ci], tap-major
    out = torch.full((Co, 64 * Ci), 3.0, device=cuda_device)
    dyp, xs = pad_cl(dy), s2d_pack(x)                 # keep the operands alive across the launch
    rc = l.mf_train_conv_wgrad(lib.ptr(dyp), lib.ptr(xs), B, Do, Co, 8 * Ci,
                               lib.ptr(out), 0, lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert rel_err(out, want) < 1e-2, rel_err(out, want)                  # `want` is bf16-rounded


def pack_dgrad_weight(W):
    """OIDHW [Co,Ci,4,4,4] -> bf16 [8][Ci][8*Co]: Wd[r][ci][a*Co+co] = W[co][ci][2a+r]."""
    Co, Ci = W.shape[:2]
    W = W.reshape(Co, Ci, 2, 2, 2, 2, 2, 2)                # co ci ad rd ah rh aw rw
    W = W.permute(3, 5, 7, 1, 2, 4, 6, 0)                  # rd rh rw ci ad ah aw co
    return bf(W.reshape(8, Ci, 8 * Co)).contiguous()


@pytest.mark.parametrize("B,Ci,Co,D,epi", [(2, 256, 512, 16, 1), (2, 160, 256, 32, 2)])
def test_conv_dgrad(cuda_device, B, Ci, Co, D, epi):
    lib, l = L()
    torch.manual_seed(2)
    Do = D // 2
    W = bf(torch.randn(Co, Ci, 4, 4, 4, device=cuda_device) / 30).float()
    dy = bf(torch.randn(B, Co, Do, Do, Do, device=cuda_device)).float()
    want = torch.nn.grad.conv3d_input((B, Ci, D, D, D), W, dy, stride=2, padding=1)
    want_cl = want.permute(0, 2, 3, 4, 1).contiguous()                    # [B,D,D,D,Ci]
    Wd = pack_dgrad_weight(W)
    dyp = pad_cl(dy)                                  # keep alive across the launches
    if epi == 1:
        out = torch.ones(B, D, D, D, Ci, device=cuda_device)               # accumulated into
        rc = l.mf_train_conv_dgrad(lib.ptr(dyp), lib.ptr(Wd), B, Do, Co, Ci, 1, lib.ptr(out),
                                   Ci, 0, lib.stream())
        assert rc == 0
        assert rel_err(out - 1.0, want_cl) < 1e-2
    else:
        M = B * Do ** 3
        out = torch.zeros(8, M, Ci, dtype=torch.bfloat16, device=cuda_device)
        rc = l.mf_train_conv_dgrad(lib.ptr(dyp), lib.ptr(Wd), B, Do, Co, Ci, 2, lib.ptr(out),
                                   Ci, M * Ci, lib.stream())
        assert rc == 0
        got = torch.zeros_like(want_cl)
        o = out.float().reshape(2, 2, 2, B, Do, Do, Do, Ci)
        for rd in range(2):
            for rh in range(2):
                for rw in range(2):
                    got[:, 1 - rd::2, 1 - rh::2, 1 - rw::2] = o[rd, rh, rw]    # x = 2 o + 1 - r
        assert rel_err(got, want_cl) < 1.5e-2


# ------------------------------------------------------------------ per-rank batch sizes, derived bounds
# float64 references through the s2d identities and the derived fp32 / bf16 bounds of
# test_train_backward_gpu.py (c_mma: chain length of a wgmma reduction; sum|terms| from the
# same reference on absolute values).  B = 1 / 2 are the per-rank batches of 16- / 8-GPU runs,
# B = 16 the single-GPU batch; the split-K factor of the wgrad depends on B (conv4 at B = 1
# runs unsplit: plain stores).
CONV_SHAPES = [(160, 256, 32), (144, 256, 32), (256, 512, 16)]     # (Ci, Co, D): conv3 +/- occupancy, conv4


@pytest.mark.parametrize("Ci,Co,D", CONV_SHAPES)
@pytest.mark.parametrize("B", [1, 2, 8, 16])
def test_conv_wgrad_batches(cuda_device, B, Ci, Co, D):
    from test_train_backward_gpu import F64, c_mma, check, control, fp32_tol, wgrad_ref
    from morefusion_b200.contrib.singleview_3d.models.training import unpack_conv_k4s2_grad as unpack
    lib, l = L()
    g = torch.Generator(device=cuda_device).manual_seed(B * 1000 + Ci)
    Do = D // 2
    x = bf(torch.randn(B, Ci, D, D, D, generator=g, device=cuda_device)).float()
    dy = bf(torch.randn(B, Co, Do, Do, Do, generator=g, device=cuda_device)).float()
    dyp, xs = pad_cl(dy), s2d_pack(x)
    del x, dy
    ref, ab = wgrad_ref(dyp, xs, Do)
    c = c_mma(B * Do ** 3)
    out = torch.full((Co, 64 * Ci), 3.0, device=cuda_device)
    assert l.mf_train_conv_wgrad(lib.ptr(dyp), lib.ptr(xs), B, Do, Co, 8 * Ci, lib.ptr(out), 0,
                                 lib.stream()) == 0
    torch.cuda.synchronize()
    tol = unpack(fp32_tol(ab, c), Co, Ci)
    check("wgrad", unpack(out, Co, Ci), unpack(ref, Co, Ci), tol)
    # accumulate = 1 onto a prefilled output (one more rounding per element: the prefill add)
    pre = torch.randn(Co, 64 * Ci, generator=g, device=cuda_device)
    out = pre.clone()
    assert l.mf_train_conv_wgrad(lib.ptr(dyp), lib.ptr(xs), B, Do, Co, 8 * Ci, lib.ptr(out), 1,
                                 lib.stream()) == 0
    torch.cuda.synchronize()
    tol = unpack(fp32_tol(ab + pre.abs().to(F64), c + 1), Co, Ci)
    check("wgrad accumulate", unpack(out, Co, Ci), unpack(pre.to(F64) + ref, Co, Ci), tol)
    # (a lost O(1) prefill is below the worst-case bound of a 65536-term chain at B = 16;
    # a product added twice, e.g. a split-K partial stored and accumulated, is not)
    control("wgrad accumulate / added twice", unpack(out, Co, Ci), unpack(pre.to(F64) + 2 * ref, Co, Ci), tol)


@pytest.mark.parametrize("Ci,Co,D", CONV_SHAPES)
@pytest.mark.parametrize("B", [1, 2, 8, 16])
def test_conv_dgrad_batches(cuda_device, B, Ci, Co, D):
    """conv3 shapes through the bf16 parity-row epilogue (Ci = 144: a partial 256-wide N tile),
    conv4 through the fp32 parity-add epilogue onto a prefilled grid; row pitch ldo > Ci and
    gaps between the parity groups hold a sentinel that must survive."""
    from test_train_backward_gpu import F64, U, bf16_tol, c_mma, check, control, dgrad_ref, fp32_tol, to_parity
    from morefusion_b200.contrib.singleview_3d.models.model import pack_conv_k4s2_weight
    lib, l = L()
    g = torch.Generator(device=cuda_device).manual_seed(B * 1000 + Ci + 1)
    Do = D // 2
    W = bf(torch.randn(Co, Ci, 4, 4, 4, generator=g, device=cuda_device) / 30).float()
    dy = bf(torch.randn(B, Co, Do, Do, Do, generator=g, device=cuda_device)).float()
    dyp, Wd = pad_cl(dy), pack_dgrad_weight(W)
    ref, ab = dgrad_ref(dyp, pack_conv_k4s2_weight(W), Ci)                  # [B,D,D,D,Ci]
    c = c_mma(8 * Co)
    ldo = Ci + 32
    if Co == 512:                                                         # epilogue 1 (conv4)
        pre = torch.randn(B, D, D, D, ldo, generator=g, device=cuda_device)
        out = pre.clone()
        assert l.mf_train_conv_dgrad(lib.ptr(dyp), lib.ptr(Wd), B, Do, Co, Ci, 1, lib.ptr(out), ldo,
                                     0, lib.stream()) == 0
        torch.cuda.synchronize()
        want = pre[..., :Ci].to(F64) + ref
        tol = fp32_tol(ab, c) + U * want.abs()
        check("dgrad parity-add", out[..., :Ci], want, tol)
        assert torch.equal(out[..., Ci:], pre[..., Ci:]), "columns beyond Ci written"
        control("dgrad parity-add / wrong parity", out[..., :Ci],
                pre[..., :Ci].to(F64) + ref[:, torch.arange(D, device=cuda_device) ^ 1], tol)
    else:                                                                 # epilogue 2 (conv3)
        M = B * Do ** 3
        stride = M * ldo + 64
        out = torch.full((8 * stride,), -5.0, dtype=torch.bfloat16, device=cuda_device)
        assert l.mf_train_conv_dgrad(lib.ptr(dyp), lib.ptr(Wd), B, Do, Co, Ci, 2, lib.ptr(out), ldo,
                                     stride, lib.stream()) == 0
        torch.cuda.synchronize()
        rows = out.reshape(8, stride)[:, :M * ldo].reshape(8, M, ldo)
        want = to_parity(ref)
        check("dgrad parity rows", rows[..., :Ci], want, bf16_tol(want, to_parity(ab), c))
        assert bool((rows[..., Ci:] == -5.0).all()), "pad columns written"
        assert bool((out.reshape(8, stride)[:, M * ldo:] == -5.0).all()), "group gap written"
        control("dgrad parity rows / wrong parity", rows[..., :Ci],
                to_parity(ref[:, torch.arange(D, device=cuda_device) ^ 1]),
                bf16_tol(want, to_parity(ab), c))


@pytest.mark.parametrize("M,N,K,groups", [(8000, 256, 640, 3), (8000, 128, 256, 3), (1000, 1920, 984, 1),
                                          (16000, 128, 256, 3)])
def test_gemm_tn_accumulate_all_groups(cuda_device, M, N, K, groups):
    """TN with accumulate = 1 onto prefilled outputs, every group checked; the output has a row
    pitch ldo > K and a gap between groups, both holding a sentinel that must survive."""
    from test_train_backward_gpu import F64, c_mma, check, control, fp32_tol
    lib, l = L()
    g = torch.Generator(device=cuda_device).manual_seed(M + N)
    ldz = groups * N
    ldx = (groups * K + 63) // 64 * 64
    dZ = bf(torch.randn(M, ldz, generator=g, device=cuda_device))
    X = bf(torch.randn(M, ldx, generator=g, device=cuda_device))
    ldo = K + 12
    gstride = N * ldo + 36
    buf = torch.full((groups * gstride,), 7.0, device=cuda_device)
    view = buf.reshape(groups, gstride)[:, :N * ldo].reshape(groups, N, ldo)
    pre = torch.randn(groups, N, K, generator=g, device=cuda_device)
    view[..., :K] = pre
    rc = l.mf_train_gemm_tn(lib.ptr(dZ), ldz, lib.ptr(X), ldx, M, N, K, lib.ptr(buf), ldo, groups,
                            N, K, gstride, 1, lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    for i in range(groups):
        z = dZ[:, i * N:(i + 1) * N].to(F64)
        x = X[:, i * K:(i + 1) * K].to(F64)
        want = pre[i].to(F64) + z.T @ x
        tol = fp32_tol(z.abs().T @ x.abs() + pre[i].abs().to(F64), c_mma(M) + 1)
        check(f"tn accumulate group {i}", view[i, :, :K], want, tol)
        if i == groups - 1:
            control("tn accumulate / last 64 rows", view[i, :, :K],
                    pre[i].to(F64) + z[:M - 64].T @ x[:M - 64], tol)
    assert bool((view[..., K:] == 7.0).all()), "pad columns written"
    assert bool((buf.reshape(groups, gstride)[:, N * ldo:] == 7.0).all()), "group gap written"
