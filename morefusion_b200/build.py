"""Build libmorefusion_sm90a.so in-tree with nvcc (sm_90a only).

    python -m morefusion_b200.build [--force] [-j N]

nvcc cross-compiles without a GPU.  The .so lands in morefusion_b200/lib/ (git-ignored).  No torch headers are involved: the library is a
plain C ABI (include/morefusion_b200.h).
"""

import argparse
import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libmorefusion_sm90a.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-O3",
          "--expt-relaxed-constexpr", "-Xptxas", "-v"]
# translation units whose arithmetic must be bit-identical to the oracle's non-contracted
# float32 NumPy: no FMA contraction.
SOURCES = {
    "voxelization.cu": ["-fmad=false"],
    "interpolate.cu": ["-fmad=false"],
    "tdf.cu": ["-fmad=false"],
    "transforms.cu": ["-fmad=false"],
    "icc.cu": ["-fmad=false"],
    "loss.cu": ["-fmad=false"],
    "cnn.cu": [],
    "conv3d_tc.cu": [],
    "gemm_train.cu": [],
    "train.cu": [],
    "frontend.cu": ["-fmad=false"],
    "mapping.cu": ["-fmad=false"],
    "object_mapping.cu": ["-fmad=false"],
    "extractor_tail.cu": [],
    "precise.cu": [],
    "posenet.cu": [],
    "icp.cu": ["-fmad=false"],
    "occupancy_registration.cu": ["-fmad=false"],
    "icp_link.cu": ["-fmad=false"],
    "pose_metrics.cu": ["-fmad=false"],
    "training_examples.cu": ["-fmad=false"],
    "render_cad.cu": ["-fmad=false"],
    "mesh_models.cu": ["-fmad=false"],
}


def nvcc():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found")
    return p


def _digest(paths, flags):
    h = hashlib.sha1()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(flags).encode())
    return h.hexdigest()


def _compile_one(src, extra, force, log):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    stamp = obj + ".sha1"
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "morefusion_b200.h"))
    flags = ARCH + COMMON + extra
    dig = _digest([path] + headers, flags)
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False, ""
    cmd = [nvcc()] + flags + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return obj, True, r.stderr


def build(force=False, jobs=None, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = [(s, e) for s, e in SOURCES.items() if os.path.exists(os.path.join(CSRC, s))]
    jobs = jobs or min(8, len(srcs))
    objs, rebuilt = [], False
    logs = []
    with concurrent.futures.ThreadPoolExecutor(jobs) as ex:
        futs = [ex.submit(_compile_one, s, e, force, verbose) for s, e in srcs]
        for f in futs:
            obj, did, log = f.result()
            objs.append(obj)
            rebuilt |= did
            if did:
                logs.append(log)
    if verbose:
        for l in logs:
            sys.stderr.write(l)
    if rebuilt or not os.path.exists(LIB):
        cmd = [nvcc()] + ARCH + ["-shared", "--cudart", "shared", "-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("-j", type=int, default=None)
    ap.add_argument("-v", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.j, a.v))


if __name__ == "__main__":
    main()
