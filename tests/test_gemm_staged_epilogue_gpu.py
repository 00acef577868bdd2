"""GPU: the staged bf16 epilogue of the wgmma GEMM (csrc/conv3d_tc.cu, staged_epilogue).

conv3 and conv4 write their bf16 tiles through a shared-memory staging buffer and TMA stores:
conv3 into the space-to-depth layout of conv4's input (four parity boxes per 64-channel slice),
conv4 row-major.  The s2d result is held bit for bit against the row-major result of the same
call rearranged on the host, with a sentinel in the zero ring and around the buffer; the
row-major one against a contiguous run with a pitch wider than N and a column offset.  Outputs a
TMA store cannot take (fp32, split-K slices) keep the register epilogue; bf16 outputs that are
not 16-byte aligned are declined before any launch."""

import ctypes

import pytest
import torch

from test_train_backward_gpu import F64, bf16_tol, c_mma, check

pytestmark = pytest.mark.gpu

S = -3.0                  # sentinel
GUARD = 4096              # sentinel elements before and after the output buffer
OUT_BF16, OUT_F32, OUT_S2D_BF16 = 0, 1, 2


def _lib():
    from morefusion_b200 import _lib as lib
    return lib, lib.lib()


def _params(A, W, bias, out, M, N, K, *, mode, lda=0, Do=0, Ci8=0, out_mode=OUT_BF16, ldo=None, col_off=0):
    from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
    lib, _ = _lib()
    return GemmParams(lib.ptr(A), lib.ptr(W), lib.ptr(bias), out, M, N, K, mode, lda, K, Do, Ci8, 1,
                      out_mode, N if ldo is None else ldo, col_off)


def _run(gp, M, N, dev, sync=None):
    lib, L = _lib()
    ws = torch.empty(L.mf_gemm_bf16_tc_workspace_bytes(M, N), dtype=torch.uint8, device=dev)
    ws.fill_(0x7F)
    rc = L.mf_gemm_bf16_tc_ex(ctypes.byref(gp), 1, lib.ptr(ws), ws.numel(),
                              lib.ptr(sync) if sync is not None else None, None, 0, lib.stream())
    return rc, ws


def _conv_case(B, Do, Ci, Co, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    J = Do + 1
    X = torch.randn(B, J, J, J, 8 * Ci, generator=g, device=dev).to(torch.bfloat16)
    K = 64 * Ci
    W = (torch.randn(Co, K, generator=g, device=dev) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(Co, generator=g, device=dev)
    return X, W, bias


def _guarded(n, dev):
    """A flat bf16 buffer of GUARD + n + GUARD sentinels and its middle n elements."""
    buf = torch.full((n + 2 * GUARD,), S, dtype=torch.bfloat16, device=dev)
    return buf, buf[GUARD:GUARD + n]


def _to_s2d(rows, B, N):
    """Row-major conv3 output [B*16^3, N] -> s2d layout [B, 9, 9, 9, 8 N] of the zero-padded 18^3
    grid, the ring (padded coordinate 0 or 17) left at the sentinel."""
    P = torch.full((B, 18, 18, 18, N), S, dtype=rows.dtype, device=rows.device)
    P[:, 1:17, 1:17, 1:17] = rows.reshape(B, 16, 16, 16, N)
    return P.reshape(B, 9, 2, 9, 2, 9, 2, N).permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(B, 9, 9, 9, 8 * N)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _conv3_pair(X, W, bias, B, Ci, dev, sync):
    """conv3 row-major and into s2d from the same inputs; returns (rows, s2d buffer with guards)."""
    lib, _ = _lib()
    M, N, K = B * 4096, 256, 64 * Ci
    rows = torch.full((M, N), S, dtype=torch.bfloat16, device=dev)
    rc, _ = _run(_params(X, W, bias, lib.ptr(rows), M, N, K, mode=1, Do=16, Ci8=8 * Ci), M, N, dev, sync)
    assert rc == 0, rc
    buf, x4 = _guarded(B * 729 * 8 * N, dev)
    rc, _ = _run(_params(X, W, bias, lib.ptr(x4), M, N, K, mode=1, Do=16, Ci8=8 * Ci, out_mode=OUT_S2D_BF16),
                 M, N, dev, sync)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return rows, buf


@pytest.mark.parametrize("Ci", [160, 144])
@pytest.mark.parametrize("B", [1, 2, 3, 8, 16])
def test_conv3_s2d_equals_row_major(cuda_device, B, Ci):
    """Every interior parity slot of x4 holds the row-major result of the same call, bit for bit;
    the zero ring and the guard elements around x4 keep the sentinel; flag words end at zero."""
    dev = cuda_device
    X, W, bias = _conv_case(B, 16, Ci, 256, dev, seed=B * 10 + Ci)
    sync = torch.zeros(2048, dtype=torch.int32, device=dev)
    rows, buf = _conv3_pair(X, W, bias, B, Ci, dev, sync)
    assert int(sync.abs().sum()) == 0, "stream-K flag words left raised"
    assert bool((rows != S).any()), "row-major output not written"
    want = _to_s2d(rows, B, 256).reshape(-1)
    got = buf[GUARD:GUARD + want.numel()]
    bad = (_bits(got) != _bits(want)).nonzero()
    assert bad.numel() == 0, f"B={B} Ci={Ci}: {bad.numel()} s2d elements differ, first at {bad[:4].flatten().tolist()}"
    assert bool((buf[:GUARD] == S).all()) and bool((buf[GUARD + want.numel():] == S).all()), \
        "elements outside x4 written"


def test_conv3_s2d_graph_replays_bit_identical(cuda_device):
    """conv3 into s2d at B = 1 (stream-K over the pairs): CUDA-graph replays give the bits of the
    eager launch and leave every flag word zero."""
    dev = cuda_device
    lib, _ = _lib()
    B, Ci = 1, 160
    X, W, bias = _conv_case(B, 16, Ci, 256, dev, seed=5)
    sync = torch.zeros(2048, dtype=torch.int32, device=dev)
    _, eager = _conv3_pair(X, W, bias, B, Ci, dev, sync)
    M, N, K = B * 4096, 256, 64 * Ci
    buf, x4 = _guarded(B * 729 * 8 * N, dev)
    gp = _params(X, W, bias, lib.ptr(x4), M, N, K, mode=1, Do=16, Ci8=8 * Ci, out_mode=OUT_S2D_BF16)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rc, keep = _run(gp, M, N, dev, sync)
        assert rc == 0, rc
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            rc, keep = _run(gp, M, N, dev, sync)
            assert rc == 0, rc
    torch.cuda.synchronize()
    x4.fill_(S)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    del keep
    assert torch.equal(_bits(buf), _bits(eager))
    assert int(sync.abs().sum()) == 0


def test_conv4_pitch_and_column_offset(cuda_device):
    """conv4 (B = 8, stream-K) row-major into a buffer of pitch ldo > N at a non-zero column
    offset: the written columns equal a contiguous run bit for bit, every other column and the
    guard elements keep the sentinel; eager launches and CUDA-graph replays agree."""
    dev = cuda_device
    lib, _ = _lib()
    B, Ci, N = 8, 256, 512
    M, K = B * 512, 64 * Ci
    X, W, bias = _conv_case(B, 8, Ci, N, dev, seed=11)
    sync = torch.zeros(2048, dtype=torch.int32, device=dev)
    flat = torch.full((M, N), S, dtype=torch.bfloat16, device=dev)
    rc, _ = _run(_params(X, W, bias, lib.ptr(flat), M, N, K, mode=1, Do=8, Ci8=8 * Ci), M, N, dev, sync)
    assert rc == 0, rc
    ldo, col_off = N + 72, 40
    buf, out = _guarded(M * ldo, dev)
    gp = _params(X, W, bias, ctypes.c_void_p(out.data_ptr()), M, N, K, mode=1, Do=8, Ci8=8 * Ci,
                 ldo=ldo, col_off=col_off)
    rc, _ = _run(gp, M, N, dev, sync)
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert int(sync.abs().sum()) == 0
    o = out.view(M, ldo)
    assert torch.equal(_bits(o[:, col_off:col_off + N]), _bits(flat))
    assert bool((o[:, :col_off] == S).all()) and bool((o[:, col_off + N:] == S).all()), "pad columns written"
    assert bool((buf[:GUARD] == S).all()) and bool((buf[GUARD + M * ldo:] == S).all())
    eager = buf.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rc, keep = _run(gp, M, N, dev, sync)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            rc, keep = _run(gp, M, N, dev, sync)
    torch.cuda.synchronize()
    buf.fill_(S)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    del keep
    assert torch.equal(_bits(buf), _bits(eager))
    assert int(sync.abs().sum()) == 0


def _linear_case(M, N, K, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    A = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g, device=dev) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device=dev)
    ref = (A.to(F64) @ W.to(F64).T + bias.to(F64)).clamp_min(0)
    ab = A.to(F64).abs() @ W.to(F64).abs().T + bias.abs().to(F64)
    return A, W, bias, ref, bf16_tol(ref, ab, c_mma(K) + 2)


@pytest.mark.parametrize("K", [2048, 4096])
def test_register_path_outputs(cuda_device, K):
    """Outputs that keep the register epilogue, against float64: fp32 at a pitch wider than N and
    a column offset (pad columns untouched), and bf16 when K is split into slices (3 tiles and
    64 K blocks without the flag words: K = 4096)."""
    dev = cuda_device
    lib, _ = _lib()
    M, N = 384, 256
    A, W, bias, ref, tol = _linear_case(M, N, K, dev, seed=K)
    ldo, col_off = N + 16, 8
    o32 = torch.full((M, ldo), S, dtype=torch.float32, device=dev)
    rc, _ = _run(_params(A, W, bias, ctypes.c_void_p(o32.data_ptr()), M, N, K, mode=0, lda=K, out_mode=OUT_F32,
                         ldo=ldo, col_off=col_off), M, N, dev)
    assert rc == 0, rc
    o16 = torch.full((M, N), S, dtype=torch.bfloat16, device=dev)
    rc, _ = _run(_params(A, W, bias, lib.ptr(o16), M, N, K, mode=0, lda=K), M, N, dev)
    assert rc == 0, rc
    torch.cuda.synchronize()
    check(f"K={K} fp32 out, ldo > N, col_off {col_off}", o32[:, col_off:col_off + N], ref, tol)
    assert bool((o32[:, :col_off] == S).all()) and bool((o32[:, col_off + N:] == S).all())
    check(f"K={K} bf16 out", o16, ref, tol)


def test_misaligned_bf16_output_declined(cuda_device):
    """A bf16 output whose column offset is not a multiple of 8 elements is declined (the model
    then runs its SIMT GEMM) and nothing is written."""
    dev = cuda_device
    M, N, K = 256, 256, 512
    A, W, bias, _, _ = _linear_case(M, N, K, dev, seed=4)
    o = torch.full((M, N + 8), S, dtype=torch.bfloat16, device=dev)
    rc, _ = _run(_params(A, W, bias, ctypes.c_void_p(o.data_ptr()), M, N, K, mode=0, lda=K, ldo=N + 8,
                         col_off=4), M, N, dev)
    torch.cuda.synchronize()
    assert rc == -4, rc
    assert bool((o == S).all())
