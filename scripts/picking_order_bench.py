#!/usr/bin/env python
"""Time the picking-order scene render at 640x480: ``geometry._render_instances_batch`` of 8, 32
and 64 synthetic primitives (the three classes' meshes packed once, objects crowded into the
image centre so that they overlap), by CUDA events around many calls after warm-up; and a full
``SelectPickingOrder`` call on the same scenes (host packing, upload, render, the one host read and
the graph), as the median of a host clock.  Prints one JSON line with the card's name and power
limit read in the same run.

    python scripts/picking_order_bench.py [--iters 200] [--calls 50] [--out DIR]
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from morefusion_b200 import geometry, synthetic  # noqa: E402
from morefusion_b200.contrib import SelectPickingOrder  # noqa: E402

H, W = 480, 640
CLASSES = (1, 2, 3)


def _time_events(fn, iters, warmup=10):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _scene(rs, n, f):
    """n poses in the camera frame at 0.5-1.2 m, centres in the middle half of the image."""
    Ts = []
    for _ in range(n):
        q = rs.normal(size=4)
        T = np.eye(4)
        T[:3, :3] = geometry.quaternion_matrix(q / np.linalg.norm(q))[:3, :3]
        z = rs.uniform(0.5, 1.2)
        T[:3, 3] = ((rs.uniform(0.25, 0.75) * W - W / 2) / f * z,
                    (rs.uniform(0.25, 0.75) * H - H / 2) / f * z, z)
        Ts.append(T)
    return np.array(Ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("picking_order_bench needs a CUDA device")
    dev = torch.device("cuda")
    K = synthetic.CAMERA_K
    fovy = geometry.fovy_from_intrinsics(K[1, 1], H)
    f = geometry.focal_from_fovy(fovy, H)
    models = synthetic.SyntheticYCBModels()
    res = dict(gpu=None, height=H, width=W, iters=a.iters, calls=a.calls)
    for n in (8, 32, 64):
        rs = np.random.RandomState(n)
        cls = np.array(CLASSES)[rs.randint(0, len(CLASSES), n)]
        ids = rs.permutation(1000)[:n]
        T_cad2cam = _scene(rs, n, f)
        v, fc, off, mesh = geometry._pack_cads([models.get_cad(int(c)) for c in cls])
        d_v = torch.tensor(v, device=dev)
        d_f = torch.tensor(fc, device=dev)
        d_T = torch.tensor(T_cad2cam, device=dev)
        ms = _time_events(lambda: geometry._render_instances_batch(
            d_v, d_f, off, mesh, d_T, ids, f=f, height=H, width=W), a.iters)
        _, _, whole, occluded = geometry._render_instances_batch(d_v, d_f, off, mesh, d_T, ids, f=f,
                                                                 height=H, width=W)
        # the camera at the world origin: T_cad2base = T_cad2cam
        sel = SelectPickingOrder(models, int(cls[0]))
        times, cycles = [], 0
        for i in range(a.warmup + a.calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                sel(ids, cls, T_cad2cam, np.eye(4), K, H, W)
            except ValueError:                  # interpenetrating objects can occlude each other
                cycles += 1
            torch.cuda.synchronize()
            if i >= a.warmup:
                times.append(time.perf_counter() - t0)
        res[f"render_{n}_ms"] = round(ms, 4)
        res[f"select_{n}_ms_median"] = round(1e3 * float(np.median(times)), 3)
        res[f"select_{n}_cycle"] = cycles > 0
        res[f"occluded_pairs_{n}"] = int((occluded > 0).sum().item())
        res[f"covered_px_{n}"] = int(whole.sum().item())
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    res["gpu"] = q[0] if q else torch.cuda.get_device_name()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "picking_order_bench.json"), "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
