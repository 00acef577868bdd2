"""GPU: wgmma GEMM kernel vs torch fp32 reference of the same op (bf16 operands, fp32
accumulate) and vs the SIMT kernel, for the linear (heads) and implicit-conv (s2d) modes."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _call(kind, A, W, bias, out, M, N, K, **kw):
    from morefusion_b200 import _lib
    from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
    from morefusion_b200.functions.geometry import _util
    L = _lib.lib()
    gp = GemmParams(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(out), M, N, K,
                    kw.get("mode", 0), kw.get("lda", 0), W.shape[1], kw.get("Do", 0),
                    kw.get("Ci8", 0), kw.get("relu", 1), kw.get("out_mode", 0), kw.get("ldo", N),
                    kw.get("col_off", 0))
    if kind == "tc":
        ws = _util.workspace(L.mf_gemm_bf16_tc_workspace_bytes(M, N), A.device)
        rc = L.mf_gemm_bf16_tc(ctypes.byref(gp), _lib.ptr(ws), ws.numel(), _lib.stream())
    elif kind in ("sk", "one_shot"):
        # stream-K: caller-owned flag words (zeroed once, reused across calls) + slots
        sync = kw["sync"] if "sync" in kw else None
        ws = torch.empty(L.mf_gemm_bf16_tc_workspace_bytes(M, N), dtype=torch.uint8, device=A.device)
        ws.fill_(0x7F)                       # garbage in the slots must not matter
        rc = L.mf_gemm_bf16_tc_ex(ctypes.byref(gp), 1, _lib.ptr(ws), ws.numel(), _lib.ptr(sync), None,
                                  1 if kind == "one_shot" else 0, _lib.stream())
    else:
        rc = L.mf_gemm_bf16_simt(ctypes.byref(gp), _lib.stream())
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 128), (8000, 1920, 984),
                                   (8000, 256, 640), (1000, 128, 256), (4096, 512, 2048),
                                   (4096, 512, 8192), (2304, 256, 4096)])   # last two: split-K
def test_tc_linear(cuda_device, M, N, K):
    torch.manual_seed(0)
    A = torch.randn(M, K, device=cuda_device).to(torch.bfloat16)
    W = (torch.randn(N, K, device=cuda_device) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=cuda_device)
    out = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
    rc = _call("tc", A, W, bias, out, M, N, K, lda=K)
    assert rc == 0
    ref = torch.relu(A.float() @ W.float().T + bias)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2 * max(1.0, ref.abs().max().item()), err
    # fp32 output, no relu
    out32 = torch.zeros(M, N, device=cuda_device)
    rc = _call("tc", A, W, bias, out32, M, N, K, lda=K, relu=0, out_mode=1)
    assert rc == 0
    ref = A.float() @ W.float().T + bias
    torch.testing.assert_close(out32, ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("Do,Ci,Co,B", [(16, 160, 256, 2), (8, 256, 512, 2), (8, 256, 512, 8)])
def test_tc_conv_s2d(cuda_device, Do, Ci, Co, B):
    """conv k4 s2 p1 through the s2d implicit GEMM == torch conv3d on the same bf16 operands."""
    from morefusion_b200.contrib.singleview_3d.models.model import pack_conv_k4s2_weight
    torch.manual_seed(1)
    D = 2 * Do
    x = torch.randn(B, Ci, D, D, D, device=cuda_device).to(torch.bfloat16)
    Wc = (torch.randn(Co, Ci, 4, 4, 4, device=cuda_device) / (Ci * 64) ** 0.5)
    bias = torch.randn(Co, device=cuda_device)
    # s2d layout of the zero-padded input
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1, 1, 1))
    J = Do + 1
    X = xp.reshape(B, Ci, J, 2, J, 2, J, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(B, J, J, J, 8 * Ci).contiguous()
    Wg = pack_conv_k4s2_weight(Wc)
    M, N, K = B * Do ** 3, Co, 64 * Ci
    ref = torch.relu(torch.nn.functional.conv3d(x.float(), Wc.to(torch.bfloat16).float(), bias, stride=2, padding=1))
    ref = ref.permute(0, 2, 3, 4, 1).reshape(M, N)
    for kind in ("simt", "tc"):
        out = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
        rc = _call(kind, X, Wg, bias, out, M, N, K, mode=1, Do=Do, Ci8=8 * Ci)
        assert rc == 0, kind
        err = (out.float() - ref).abs().max().item()
        assert err <= 2e-2 * max(1.0, ref.abs().max().item()), (kind, err)
    # s2d output mode (conv3 -> conv4 input): compare with the row-major result re-laid out
    if Do == 16:
        J2 = Do // 2 + 1
        out2 = torch.zeros(B, J2, J2, J2, 8 * N, device=cuda_device, dtype=torch.bfloat16)
        rc = _call("tc", X, Wg, bias, out2, M, N, K, mode=1, Do=Do, Ci8=8 * Ci, out_mode=2)
        assert rc == 0
        h = out.reshape(B, Do, Do, Do, N).permute(0, 4, 1, 2, 3)
        hp = torch.nn.functional.pad(h, (1, 1, 1, 1, 1, 1))
        want = hp.reshape(B, N, J2, 2, J2, 2, J2, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(B, J2, J2, J2, 8 * N)
        assert torch.equal(out2, want.contiguous())


@pytest.mark.parametrize("M,N,K", [(4096, 512, 8192), (8000, 512, 2048), (32768, 256, 2048),
                                   (2304, 256, 4096), (640, 256, 16384)])
def test_tc_stream_k_linear(cuda_device, M, N, K):
    """Stream-K scheduling (equal K-block ranges per SM, partial accumulators parked in the
    workspace, reduction in the owning CTA's epilogue) against the fp32 reference, three calls
    on the same flag words (the kernel must leave them zero)."""
    torch.manual_seed(0)
    A = torch.randn(M, K, device=cuda_device).to(torch.bfloat16)
    W = (torch.randn(N, K, device=cuda_device) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=cuda_device)
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    ref = torch.relu(A.float() @ W.float().T + bias)
    for _ in range(3):
        out = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
        rc = _call("sk", A, W, bias, out, M, N, K, lda=K, sync=sync)
        assert rc == 0
        err = (out.float() - ref).abs().max().item()
        assert err <= 2e-2 * max(1.0, ref.abs().max().item()), err
        assert int(sync.abs().sum()) == 0
    one = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
    assert _call("one_shot", A, W, bias, one, M, N, K, lda=K, sync=None) == 0
    # same products, different fp32 summation split: within one bf16 ulp of the one-shot kernel
    torch.testing.assert_close(out.float(), one.float(), rtol=2 ** -7, atol=2e-2)


@pytest.mark.parametrize("Do,Ci,Co,B", [(16, 160, 256, 8), (8, 256, 512, 8), (16, 160, 256, 3)])
def test_tc_stream_k_conv_s2d(cuda_device, Do, Ci, Co, B):
    """conv3 / conv4 shapes of the model (256 and 64 tiles on 132 SMs) under stream-K, in both
    output layouts, against the whole-tile schedule of the same kernel."""
    from morefusion_b200.contrib.singleview_3d.models.model import pack_conv_k4s2_weight
    torch.manual_seed(1)
    D, J = 2 * Do, Do + 1
    x = torch.randn(B, Ci, D, D, D, device=cuda_device).to(torch.bfloat16)
    Wc = (torch.randn(Co, Ci, 4, 4, 4, device=cuda_device) / (Ci * 64) ** 0.5)
    bias = torch.randn(Co, device=cuda_device)
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1, 1, 1))
    X = xp.reshape(B, Ci, J, 2, J, 2, J, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(B, J, J, J, 8 * Ci).contiguous()
    Wg = pack_conv_k4s2_weight(Wc)
    M, N, K = B * Do ** 3, Co, 64 * Ci
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    ref = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
    assert _call("tc", X, Wg, bias, ref, M, N, K, mode=1, Do=Do, Ci8=8 * Ci) == 0
    for _ in range(2):
        out = torch.zeros(M, N, device=cuda_device, dtype=torch.bfloat16)
        assert _call("sk", X, Wg, bias, out, M, N, K, mode=1, Do=Do, Ci8=8 * Ci, sync=sync) == 0
        torch.testing.assert_close(out.float(), ref.float(), rtol=2 ** -7, atol=2e-2)
        assert int(sync.abs().sum()) == 0
    if Do == 16:
        J2 = Do // 2 + 1
        out2 = torch.zeros(B, J2, J2, J2, 8 * N, device=cuda_device, dtype=torch.bfloat16)
        assert _call("sk", X, Wg, bias, out2, M, N, K, mode=1, Do=Do, Ci8=8 * Ci, out_mode=2, sync=sync) == 0
        h = out.reshape(B, Do, Do, Do, N).permute(0, 4, 1, 2, 3)
        hp = torch.nn.functional.pad(h, (1, 1, 1, 1, 1, 1))
        want = hp.reshape(B, N, J2, 2, J2, 2, J2, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(B, J2, J2, J2, 8 * N)
        assert torch.equal(out2, want.contiguous())


@pytest.mark.parametrize("M,N,K", [(8000, 256, 640), (8000, 128, 256), (1000, 256, 640)])
def test_tc_stream_k_grouped_heads(cuda_device, M, N, K):
    """The three pose heads as one grouped stream-K launch (short K: 4-10 K blocks per tile):
    column-offset outputs into one buffer, compared with per-head fp32 references."""
    from morefusion_b200 import _lib
    from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
    L = _lib.lib()
    torch.manual_seed(2)
    A = torch.randn(M, 3 * K, device=cuda_device).to(torch.bfloat16)
    Ws = [(torch.randn(N, K, device=cuda_device) / K ** 0.5).to(torch.bfloat16) for _ in range(3)]
    bs = [torch.randn(N, device=cuda_device) for _ in range(3)]
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    ws = torch.empty(L.mf_gemm_bf16_tc_workspace_bytes(M, N), dtype=torch.uint8, device=cuda_device)
    for rep in range(2):
        out = torch.zeros(M, 3 * N, device=cuda_device, dtype=torch.bfloat16)
        arr = (GemmParams * 3)()
        views = [A[:, i * K:] for i in range(3)]
        for i in range(3):
            arr[i] = GemmParams(_lib.ptr(views[i]), _lib.ptr(Ws[i]), _lib.ptr(bs[i]), _lib.ptr(out), M, N, K,
                                0, 3 * K, K, 0, 0, 1, 0, 3 * N, i * N)
        rc = L.mf_gemm_bf16_tc_ex(arr, 3, _lib.ptr(ws), ws.numel(), _lib.ptr(sync), None, 0, _lib.stream())
        torch.cuda.synchronize()
        assert rc == 0
        for i in range(3):
            ref = torch.relu(A[:, i * K:(i + 1) * K].float() @ Ws[i].float().T + bs[i])
            got = out[:, i * N:(i + 1) * N].float()
            assert (got - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
        assert int(sync.abs().sum()) == 0


@pytest.mark.parametrize("M", [1000, 16000])
def test_tc_backward_dx_shapes(cuda_device, M):
    """The forward kernel at the shapes the training backward uses it for (dX = dZ W^T), with
    bias = NULL and no ReLU, bf16 stores within the derived bound of test_train_backward_gpu:
      head 1   (M, 992, 1920), ldo = 1024: the last N tile is 224 wide; columns 984..991 come
               from the zero pad rows of W^T, 992..1023 must keep their sentinel;
      layer 2  grouped (M, 640, 256) x 3 with col_off = i * 640 into ldo = 1920;
      layer 3  (M, 256, 128), ldo = 384: columns 256..383 keep their sentinel."""
    from morefusion_b200 import _lib
    from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
    from test_train_backward_gpu import F64, bf16_tol, c_mma, check, control
    L = _lib.lib()
    g = torch.Generator(device=cuda_device).manual_seed(M)
    rn = lambda *s: torch.randn(*s, generator=g, device=cuda_device)     # noqa: E731
    S = -3.0
    # head 1
    A = rn(M, 1920).to(torch.bfloat16)
    W = torch.zeros(992, 1920, device=cuda_device, dtype=torch.bfloat16)
    W[:984] = (rn(984, 1920) / 40).to(torch.bfloat16)
    out = torch.full((M, 1024), S, device=cuda_device, dtype=torch.bfloat16)
    assert _call("tc", A, W, None, out, M, 992, 1920, lda=1920, relu=0, ldo=1024) == 0
    ref = A.to(F64) @ W.to(F64).T
    tol = bf16_tol(ref, A.to(F64).abs() @ W.to(F64).abs().T, c_mma(1920))
    check("head1 dX", out[:, :992], ref, tol)
    assert torch.count_nonzero(out[:, 984:992]) == 0
    assert bool((out[:, 992:] == S).all()), "columns past N written"
    control("head1 dX / last K block dropped", out[:, :992], A[:, :1856].to(F64) @ W[:, :1856].to(F64).T, tol)
    # layer 2: three heads grouped, column offsets into one 1920-wide row (one sentinel row below)
    dz = rn(M, 768).to(torch.bfloat16)
    Ws = [(rn(640, 256) / 16).to(torch.bfloat16) for _ in range(3)]
    out = torch.full((M + 1, 1920), S, device=cuda_device, dtype=torch.bfloat16)
    views = [dz[:, i * 256:] for i in range(3)]
    arr = (GemmParams * 3)()
    for i in range(3):
        arr[i] = GemmParams(_lib.ptr(views[i]), _lib.ptr(Ws[i]), None, _lib.ptr(out), M, 640, 256,
                            0, 768, 256, 0, 0, 0, 0, 1920, i * 640)
    ws = torch.empty(L.mf_gemm_bf16_tc_workspace_bytes(M, 640), dtype=torch.uint8, device=cuda_device)
    assert L.mf_gemm_bf16_tc_grouped(arr, 3, _lib.ptr(ws), ws.numel(), _lib.stream()) == 0
    torch.cuda.synchronize()
    for i in range(3):
        z = dz[:, i * 256:(i + 1) * 256].to(F64)
        ref = z @ Ws[i].to(F64).T
        tol = bf16_tol(ref, z.abs() @ Ws[i].to(F64).abs().T, c_mma(256))
        check(f"layer2 dX head {i}", out[:M, i * 640:(i + 1) * 640], ref, tol)
        if i == 1:
            control("layer2 dX / col_off + 8", out[:M, i * 640:(i + 1) * 640], torch.roll(ref, 8, 1), tol)
    assert bool((out[M] == S).all())
    # layer 3: K = 128 (two K blocks), ldo = 384
    dz = rn(M, 128).to(torch.bfloat16)
    W = (rn(256, 128) / 11).to(torch.bfloat16)
    out = torch.full((M, 384), S, device=cuda_device, dtype=torch.bfloat16)
    assert _call("tc", dz, W, None, out, M, 256, 128, lda=128, relu=0, ldo=384) == 0
    ref = dz.to(F64) @ W.to(F64).T
    tol = bf16_tol(ref, dz.to(F64).abs() @ W.to(F64).abs().T, c_mma(128))
    check("layer3 dX", out[:, :256], ref, tol)
    assert bool((out[:, 256:] == S).all())
    control("layer3 dX / relu applied", out[:, :256], ref.clamp_min(0), tol)
