#!/usr/bin/env python
"""Time the CAD render at 640x480: ``geometry._render_cad_batch`` of 8 synthetic instances (the
three primitives at poses like make_pose_frame's) and of 8 poses of a random 10^5-triangle mesh
(the triangle counts of YCB's textured_simple.obj are not known here), by CUDA events around
many launches; and ``get_example`` of a make_pose_frame with and without ``with_visibility``, as
the median of a host clock around work that ends in a device synchronise.  Prints one JSON line
with the card's name and power limit read in the same run.

    python scripts/render_cad_bench.py [--iters 200] [--frames 20] [--out DIR]
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

from morefusion_b200 import datasets, geometry, synthetic  # noqa: E402

H, W = 480, 640


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


def _instances(rs, n, f):
    Ts = []
    for _ in range(n):
        q = rs.normal(size=4)
        T = np.eye(4)
        T[:3, :3] = geometry.quaternion_matrix(q / np.linalg.norm(q))[:3, :3]
        z = rs.uniform(0.6, 0.8)
        T[:3, 3] = ((rs.uniform(0.2, 0.8) * W - W / 2) / f * z,
                    (rs.uniform(0.2, 0.8) * H - H / 2) / f * z, z)
        Ts.append(T)
    return np.array(Ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_cad_bench needs a CUDA device")
    dev = torch.device("cuda")
    rs = np.random.RandomState(0)
    fovy = geometry.fovy_from_intrinsics(synthetic.CAMERA_K[1, 1], H)
    f = geometry.focal_from_fovy(fovy, H)
    models = synthetic.SyntheticYCBModels()

    def packed(meshes):
        vs, fs, off, base = [], [], [0], 0
        for v, fc in meshes:
            vs.append(v)
            fs.append(fc + base)
            base += len(v)
            off.append(off[-1] + len(fc))
        return (torch.tensor(np.concatenate(vs), device=dev),
                torch.tensor(np.concatenate(fs).astype(np.int32), device=dev), np.array(off))

    cads = [models.get_cad(c) for c in (1, 2, 3)]
    v, fc, off = packed([(c.vertices, c.faces) for c in cads])
    mesh = torch.tensor(np.arange(8) % 3, dtype=torch.int32, device=dev)
    Ts = torch.tensor(_instances(rs, 8, f), device=dev)
    ms_prims = _time_events(lambda: geometry._render_cad_batch(v, fc, off, mesh, Ts, f=f, height=H,
                                                               width=W), a.iters)
    n_faces = 100000
    sv = rs.uniform(-0.06, 0.06, (50000, 3))
    sv = sv[np.argsort(sv[:, 0])]
    c0 = rs.randint(0, len(sv), n_faces)
    sf = np.stack([c0, (c0 + rs.randint(1, 60, n_faces)) % len(sv),
                   (c0 + rs.randint(1, 60, n_faces)) % len(sv)], 1)
    v2, f2, off2 = packed([(sv, sf)])
    mesh2 = torch.zeros(8, dtype=torch.int32, device=dev)
    ms_soup = _time_events(lambda: geometry._render_cad_batch(v2, f2, off2, mesh2, Ts, f=f,
                                                              height=H, width=W), max(a.iters // 4, 10))
    frames = [synthetic.make_pose_frame(s, n_objects=8) for s in range(a.frames + a.warmup)]

    class Frames(datasets.RGBDPoseEstimationDatasetBase):
        def get_frame(self, index):
            return frames[index]

    per_frame = {}
    for vis in (False, True, False, True):                     # alternate, keep the second pass
        ds = Frames(models, device="cuda", with_visibility=vis)
        times = []
        for i in range(a.warmup + a.frames):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ds.get_example(i)
            torch.cuda.synchronize()
            if i >= a.warmup:
                times.append(time.perf_counter() - t0)
        per_frame[vis] = 1e3 * float(np.median(times))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    res = dict(gpu=q[0] if q else torch.cuda.get_device_name(), height=H, width=W,
               render_8_primitives_ms=round(ms_prims, 4),
               primitive_faces=[int(len(c.faces)) for c in cads],
               render_8_poses_1e5_faces_ms=round(ms_soup, 4),
               get_example_ms_median=round(per_frame[False], 3),
               get_example_visibility_ms_median=round(per_frame[True], 3), frames=a.frames)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "render_cad_bench.json"), "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
