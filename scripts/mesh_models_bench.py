#!/usr/bin/env python
"""Time csrc/mesh_models.cu on closed subdivided icospheres: ``signed_distance`` at
P in {1k, 5k, 20k} points x F in {1k, 10k, 100k} faces, and ``voxelize_solid`` at D = 64 and 128,
with CUDA events around the launch sequences (the meshes and points already on the device).

    python scripts/mesh_models_bench.py [--reps 20] [--out DIR]

Prints one JSON line: the GPU's name and power limit (queried, never set), and per case the
median, minimum and maximum milliseconds over the repetitions."""

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = out[0].split(", ")
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts = np.asarray(ts)
    return dict(median_ms=float(np.median(ts)), min_ms=float(ts.min()), max_ms=float(ts.max()))


def main():
    import _mesh_cases as mc
    from morefusion_b200 import geometry
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_models_bench needs a CUDA device")
    name, power = gpu_info()
    res = dict(gpu=name, power_limit=power, reps=a.reps, signed_distance=[], voxelize_solid=[])
    for F in (1000, 10000, 100000):
        v, f = mc.icosphere_faces(F)
        dv = torch.as_tensor(v, device="cuda")
        df = torch.as_tensor(f, device="cuda")
        off = [0, len(f)]
        for P in (1000, 5000, 20000):
            rs = np.random.RandomState(P)
            p = torch.as_tensor(rs.uniform(-0.07, 0.07, (P, 3)), device="cuda")
            tag = torch.zeros(P, dtype=torch.int32, device="cuda")
            t = timed(lambda: geometry._signed_distance_batch(dv, df, off, p, tag), a.reps)
            pairs = P * len(f)
            res["signed_distance"].append(dict(P=P, F=int(len(f)), **t,
                                               pairs_per_s=pairs / (t["median_ms"] * 1e-3)))
        for D in (64, 128):
            t = timed(lambda: geometry._voxelize_solid_batch(dv, df, off, D), a.reps)
            res["voxelize_solid"].append(dict(D=D, F=int(len(f)), **t))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mesh_models_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
