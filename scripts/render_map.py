"""Time the occupancy server's render (``MultiInstanceOctreeMapping.render``) and the cost of the box
pass ``integrate_scan`` gained with it.

    python scripts/render_map.py [--parent-root DIR] [--out FILE]

Render: the 10-view synthetic sequence (640x480, 8 instances); after each scan the frame is
rendered (3 warm-up calls, then --reps calls timed one by one with CUDA events); the median and
p90 over all timed calls, and the host time of the oracle's render per frame.

Box pass: with --parent-root (a built checkout of the commit before the box pass), integrate_scan
per frame of the same sequence in this tree and in that one, each in a fresh process, alternated,
three runs of each; a run warms up on one pass of the sequence and times a second pass on a
fresh map.

Prints one JSON record with the GPU's name and power limit read in the same call."""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pcd_of(view, K):
    z = view["depth"].astype(np.float64)
    H, W = z.shape
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    return np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z], -1).astype(np.float32)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        import torch
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def time_scans(root):
    """integrate_scan per frame (ms) of the 10-view sequence, with the package from `root`."""
    sys.path.insert(0, root)
    import torch
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib import MultiInstanceOctreeMapping
    f = synthetic.make_rgbd_views(0, 10, n_objects=8)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    frames = [(torch.as_tensor(v["label"], device="cuda"),
               torch.as_tensor(pcd_of(v, f["K"]), device="cuda"), v["sensor_to_world"])
              for v in f["views"]]
    out = []
    for timed in (False, True):
        m = MultiInstanceOctreeMapping()
        for lab, pcd, T in frames:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            m.integrate_scan(lab, pcd, T, classes, max_range=synthetic.VIEWS_MAX_RANGE,
                             background_pitch=0.01)
            b.record()
            torch.cuda.synchronize()
            if timed:
                out.append(a.elapsed_time(b))
    return out


def time_render(reps):
    sys.path.insert(0, ROOT)
    import torch
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib import MultiInstanceOctreeMapping
    from morefusion_b200.contrib.singleview_3d.models.model import YCB_VOXEL_PITCH_32
    from oracle import octomap_server_render as osr
    f = synthetic.make_rgbd_views(0, 10, n_objects=8)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    m = MultiInstanceOctreeMapping()
    trees, centres, boxes, server_trees = {}, {}, {}, set()
    times, oracle_s, mismatches = [], [], 0
    for v in f["views"]:
        pcd = pcd_of(v, f["K"])
        d_pcd = torch.as_tensor(pcd, device="cuda")
        T = v["sensor_to_world"]
        m.integrate_scan(torch.as_tensor(v["label"], device="cuda"), d_pcd, T, classes,
                         max_range=synthetic.VIEWS_MAX_RANGE, background_pitch=0.01)
        osr.insert_scan(trees, centres, boxes, server_trees, v["label"], pcd, T, classes,
                        pitch_of=lambda c: YCB_VOXEL_PITCH_32[c],
                        max_range=synthetic.VIEWS_MAX_RANGE, background_pitch=0.01)
        for _ in range(3):
            label, depth = m.render(d_pcd, T, f["K"])
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            m.render(d_pcd, T, f["K"])
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        t0 = time.perf_counter()
        want = osr.render(trees, boxes, pcd, T, f["K"])
        oracle_s.append(time.perf_counter() - t0)
        mismatches += int((label.cpu().numpy() != want[0]).sum())
        mismatches += int((depth.cpu().numpy().view(np.uint32) != want[1].view(np.uint32)).sum())
    return times, oracle_s, mismatches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-root", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--scan-only", default=None, help=argparse.SUPPRESS)   # child process
    args = ap.parse_args()
    if args.scan_only:
        print(json.dumps(time_scans(args.scan_only)))
        return
    name, power = gpu_info()
    times, oracle_s, mismatches = time_render(args.reps)
    rec = dict(gpu=name, power_limit=power, frame="640x480", instances=8, views=10,
               render_ms_median=float(np.median(times)), render_ms_p90=float(np.percentile(times, 90)),
               render_calls_timed=len(times), oracle_render_s_per_frame=float(np.mean(oracle_s)),
               render_mismatched_pixels=mismatches)
    if args.parent_root:
        runs = {"this": [], "parent": []}
        for _ in range(3):
            for key, root in (("this", ROOT), ("parent", os.path.abspath(args.parent_root))):
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--scan-only", root],
                                     capture_output=True, text=True, check=True).stdout
                runs[key].append(float(np.mean(json.loads(out.strip().splitlines()[-1]))))
        rec.update(integrate_scan_ms_per_frame_this=runs["this"],
                   integrate_scan_ms_per_frame_parent=runs["parent"])
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
