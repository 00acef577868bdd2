"""GPU: the CTA-pair schedule of the wgmma GEMM (csrc/conv3d_tc.cu) at the conv3 / conv4 shapes.

The implicit-GEMM convolutions run as clusters of two CTAs on m-tiles 2i and 2i + 1 of the same
n-tile: each CTA loads half of the W tile and multicasts it into both, and K is walked channel
block by channel block with the 8 cell offsets innermost.  Linear GEMMs, whose m-tile count can
be odd, keep one CTA per tile.  Every result is held against a float64 reference with the derived
bound of tests/test_train_backward_gpu.py, with as many extra adds as the scheduler of
tests/test_cnn_forward_stages_gpu.py::gemm_parts allows."""

import ctypes

import pytest
import torch

from test_cnn_forward_stages_gpu import gemm_parts, s2d_conv
from test_train_backward_gpu import F64, bf16_tol, c_mma, check, control

pytestmark = pytest.mark.gpu

S = -3.0                  # sentinel around the output
CONVS = [("conv3", 16, 160, 256), ("conv3_no_occupancy", 16, 144, 256), ("conv4", 8, 256, 512)]


def _lib():
    from morefusion_b200 import _lib as lib
    return lib


def pair_parts(M, N, K, n_sm):
    """Most K pieces per tile under the pair schedule: the same choice between stream-K, split-K
    and whole tiles as gemm_parts, but stream-K cuts units = tile pairs x K blocks into one range
    per cluster (n_sm // 2 of them)."""
    BN = 256 if N >= 256 else 128
    kb = -(-K // 64)
    tiles = -(-M // 128) * -(-N // BN)
    waves = -(-tiles // n_sm)
    if kb >= 32 and N % 32 == 0 and tiles / (waves * n_sm) < 0.95:
        units, G = tiles // 2, n_sm // 2
        W = units * kb
        lo = [W * c // G for c in range(G + 1)]
        rng = [(lo[c], lo[c + 1]) for c in range(G) if lo[c] < lo[c + 1]]
        return max(sum(1 for a, b in rng if a < (u + 1) * kb and b > u * kb) for u in range(units))
    return gemm_parts(M, N, K, n_sm)


def _conv_case(B, Do, Ci, Co, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    J = Do + 1
    X = torch.randn(B, J, J, J, 8 * Ci, generator=g, device=dev).to(torch.bfloat16)
    K = 64 * Ci
    Wg = (torch.randn(Co, K, generator=g, device=dev) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(Co, generator=g, device=dev)
    return X, Wg, bias


def _gemm(X, Wg, bias, out, M, N, K, *, mode, Do=0, Ci8=0, lda=0, sync=None, one_shot=0):
    """out: a row-major [M, N] bf16 view; ReLU + bias as the model's layers."""
    from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
    lib = _lib()
    L = lib.lib()
    ws = torch.empty(L.mf_gemm_bf16_tc_workspace_bytes(M, N), dtype=torch.uint8, device=X.device)
    ws.fill_(0x7F)                               # garbage in the stream-K slots must not matter
    gp = GemmParams(lib.ptr(X), lib.ptr(Wg), lib.ptr(bias), lib.ptr(out), M, N, K, mode, lda, K, Do,
                    Ci8, 1, 0, N, 0)
    rc = L.mf_gemm_bf16_tc_ex(ctypes.byref(gp), 1, lib.ptr(ws), ws.numel(),
                              lib.ptr(sync) if sync is not None else None, None, one_shot, lib.stream())
    assert rc == 0, rc
    return ws


def _sentinel_out(M, N, dev):
    full = torch.full((M + 2, N), S, device=dev, dtype=torch.bfloat16)
    return full, full[1:M + 1]


def _swap_halves(t, BN=256):
    """Columns with the two 128-wide halves of every 256-wide n-tile exchanged."""
    N = t.shape[-1]
    idx = torch.arange(N, device=t.device)
    idx = (idx // BN) * BN + (idx % BN + BN // 2) % BN
    return t[..., idx]


@pytest.mark.parametrize("name,Do,Ci,Co", CONVS)
@pytest.mark.parametrize("B", [1, 2, 3, 8, 16])
def test_pair_conv_vs_float64(cuda_device, name, Do, Ci, Co, B):
    """conv3 (Ci = 160 with occupancy, 144 without) and conv4 at the batch sizes the model and
    training run, with the stream-K flag words (as the model) and one-shot, against float64."""
    n_sm = _lib().lib().mf_device_sm_count(cuda_device.index or 0)
    X, Wg, bias = _conv_case(B, Do, Ci, Co, cuda_device, seed=B * 100 + Ci)
    M, N, K = B * Do ** 3, Co, 64 * Ci
    parts = gemm_parts(M, N, K, n_sm)
    assert pair_parts(M, N, K, n_sm) <= parts, "the pair schedule sums a tile from more pieces"
    ref = s2d_conv(X, Wg, Do).reshape(M, N).add_(bias.to(F64))
    ab = s2d_conv(X.abs(), Wg.abs(), Do).reshape(M, N).add_(bias.abs().to(F64))
    # wgmma chain over K, one add per further K piece of the tile, the bias in the epilogue
    tol = bf16_tol(ref.clamp_min(0), ab, c_mma(K) + parts + 1)
    del ab
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    for one_shot in (0, 1):
        full, out = _sentinel_out(M, N, cuda_device)
        _gemm(X, Wg, bias, out, M, N, K, mode=1, Do=Do, Ci8=8 * Ci, sync=sync, one_shot=one_shot)
        torch.cuda.synchronize()
        check(f"{name} B={B} one_shot={one_shot} ({parts} K pieces per tile)", out, ref.clamp_min(0), tol)
        assert bool((full[0] == S).all()) and bool((full[M + 1] == S).all()), "rows outside the output written"
        assert int(sync.abs().sum()) == 0, "stream-K flag words left raised"
    control(f"{name} B={B} / W halves swapped", out, _swap_halves(ref.clamp_min(0)), tol)


def test_pair_conv_replays_bit_identical(cuda_device):
    """conv4 at B = 8 (stream-K over the pairs): two launches in a row and a CUDA-graph replay on
    the same flag words give the same bits and leave every flag word zero."""
    X, Wg, bias = _conv_case(8, 8, 256, 512, cuda_device, seed=7)
    M, N, K = 8 * 512, 512, 16384
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    outs = []
    for _ in range(2):
        full, out = _sentinel_out(M, N, cuda_device)
        _gemm(X, Wg, bias, out, M, N, K, mode=1, Do=8, Ci8=2048, sync=sync)
        torch.cuda.synchronize()
        assert int(sync.abs().sum()) == 0
        outs.append(full)
    assert torch.equal(outs[0], outs[1])
    full, out = _sentinel_out(M, N, cuda_device)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        keep = _gemm(X, Wg, bias, out, M, N, K, mode=1, Do=8, Ci8=2048, sync=sync)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            keep = _gemm(X, Wg, bias, out, M, N, K, mode=1, Do=8, Ci8=2048, sync=sync)
    torch.cuda.synchronize()
    out.fill_(0)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    del keep
    assert torch.equal(full, outs[0])
    assert int(sync.abs().sum()) == 0


def test_odd_m_tiles_keep_single_ctas(cuda_device):
    """A linear GEMM with 63 m-tiles (M = 8000), long K and the stream-K flags: a pair schedule
    would leave the last m-tile unwritten (its sentinel) or read past the end."""
    g = torch.Generator(device=cuda_device).manual_seed(3)
    M, N, K = 8000, 256, 2048
    A = torch.randn(M, K, generator=g, device=cuda_device).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g, device=cuda_device) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device=cuda_device)
    sync = torch.zeros(2048, dtype=torch.int32, device=cuda_device)
    full, out = _sentinel_out(M, N, cuda_device)
    _gemm(A, W, bias, out, M, N, K, mode=0, lda=K, sync=sync)
    torch.cuda.synchronize()
    ref = A.to(F64) @ W.to(F64).T + bias.to(F64)
    ab = A.to(F64).abs() @ W.to(F64).abs().T + bias.abs().to(F64)
    n_sm = _lib().lib().mf_device_sm_count(cuda_device.index or 0)
    tol = bf16_tol(ref.clamp_min(0), ab, c_mma(K) + gemm_parts(M, N, K, n_sm) + 1)
    check("linear M=8000", out, ref.clamp_min(0), tol)
    assert bool((full[0] == S).all()) and bool((full[M + 1] == S).all())
    assert int(sync.abs().sum()) == 0
