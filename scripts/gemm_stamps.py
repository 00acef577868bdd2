"""Per-role clock stamps of the persistent wgmma GEMM (CTA 0) for the model's GEMM shapes.

Prints, per work unit of CTA 0: producer span, consumer unit start, first operands, main loop end,
epilogue start and end, in SM cycles.  Also times each shape by CUDA-graph replay.  The conv3 /
conv4 shapes (B = 8, s2d implicit GEMM, with the stream-K flag words as the model passes them)
are timed like the others; their stamps come from a run without the flag words."""
import ctypes
import json
import sys

import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from morefusion_b200 import _lib
from morefusion_b200.contrib.singleview_3d.models.model import GemmParams
from morefusion_b200.functions.geometry import _util

dev = torch.device("cuda:0")
L = _lib.lib()
B_CONV = 8
SHAPES = [("head1", 8000, 1920, 984), ("head1_pitch1024", 8000, 1920, 984),
          ("head2", 8000, 512, 640), ("head3", 8000, 256, 512), ("head4", 8000, 128, 256),
          ("big", 32768, 2048, 1024),
          # name, M, N, K, Do, input channels (conv3 with the 16 occupancy channels)
          ("conv3", B_CONV * 4096, 256, 64 * 160, 16, 160), ("conv4", B_CONV * 512, 512, 64 * 256, 8, 256)]
if len(sys.argv) > 1:
    SHAPES = [s for s in SHAPES if s[0] in sys.argv[1:]]
for name, M, N, K, *conv in SHAPES:
    torch.manual_seed(0)
    sync = None
    if conv:
        Do, Ci = conv
        J = Do + 1
        A = torch.randn(B_CONV, J, J, J, 8 * Ci, device=dev).to(torch.bfloat16)   # s2d input
        W = (torch.randn(N, K, device=dev) / K ** 0.5).to(torch.bfloat16)
        ld = K
        sync = torch.zeros(2048, dtype=torch.int32, device=dev)
    else:
        ld = 1024 if name.endswith("pitch1024") else K
        A = torch.randn(M, ld, device=dev).to(torch.bfloat16)
        W = (torch.randn(N, ld, device=dev) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
    if conv:
        gp = GemmParams(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(out), M, N, K, 1, 0, K, Do,
                        8 * Ci, 1, 0, N, 0)
    else:
        gp = GemmParams(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(out), M, N, K, 0, ld, ld, 0,
                        0, 1, 0, N, 0)
    ws = _util.workspace(max(16, L.mf_gemm_bf16_tc_workspace_bytes(M, N)), dev)
    stamps = torch.zeros(16 * 8, dtype=torch.int64, device=dev)

    def call():
        if sync is not None:
            rc = L.mf_gemm_bf16_tc_ex(ctypes.byref(gp), 1, _lib.ptr(ws), ws.numel() * ws.element_size(),
                                      _lib.ptr(sync), None, 0, _lib.stream())
        else:
            rc = L.mf_gemm_bf16_tc(ctypes.byref(gp), _lib.ptr(ws), ws.numel(), _lib.stream())
        assert rc == 0, rc

    call()
    torch.cuda.synchronize()
    # timing (graph replay, stamps off)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        call()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(20):
                call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    torch.cuda.synchronize()
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 20
    tf = 2.0 * M * N * K / us / 1e6
    rc = L.mf_gemm_bf16_tc_ex(ctypes.byref(gp), 1, _lib.ptr(ws), ws.numel(), None, _lib.ptr(stamps), 0,
                              _lib.stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    st = stamps.cpu().view(16, 8)
    t0 = int(st[0, 0])
    rows = []
    for it in range(16):
        if int(st[it, 0]) == 0:
            break
        r = [int(x) - t0 for x in st[it]]
        rows.append(r)
    print(json.dumps({"shape": name, "M": M, "N": N, "K": K, "us": round(us, 2),
                      "TFLOPs": round(tf, 1)}))
    print("  unit: prod_begin prod_end | mma_buf_free mma_first_ops mma_commit | "
          "epi_ready epi_drained epi_stored   (SM cycles from CTA-0 start)")
    for i, r in enumerate(rows):
        print("  %2d: %7d %7d | %7d %7d %7d | %7d %7d %7d" % (i, *r))
