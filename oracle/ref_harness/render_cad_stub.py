#!/usr/bin/env python
"""Run the reference's own ``render_cad`` / ``render_camera`` / ``get_camera_image``
(morefusion/extra/_pybullet.py:215-288), taken from the reference checkout, under a ``pybullet``
stand-in that records the arguments they pass, and write them to
tests/golden/render_cad/camera_chain.npz.

TEST INFRASTRUCTURE ONLY.  Needs the reference checkout (MOREFUSION_REFERENCE):

    python -m oracle.ref_harness.render_cad_stub

The stand-in records computeProjectionMatrixFOV's keywords (fov, aspect, nearVal, farVal) and
getCameraImage's (width, height, viewMatrix); its camera image is empty.  ``add_model`` (the mesh
load) is a no-op: the pinned part is the camera chain, not the rasteriser.
camera_chain.npz, per case of CASES: ``<case>/Ts`` [N,4,4] (inputs), ``<case>/view`` [N,16] (the
flattened view matrices), ``<case>/proj`` [N,4] (fov, aspect, near, far), ``<case>/size`` [N,2]
(width, height); ``<case>/fovy_hw`` (fovy, height, width).
"""

import ast
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.ref_harness import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "render_cad")
CASES = {"vga": (480, 640, 3), "odd": (5, 7, 2), "tall": (100, 50, 2)}


def case_inputs(name):
    """(Ts [N,4,4], fovy, height, width) of a case, regenerated from its name."""
    H, W, n = CASES[name]
    rs = np.random.RandomState(sum(map(ord, name)))
    Ts = []
    for _ in range(n):
        q = rs.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        T = np.eye(4)
        T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
        T[:3, 3] = rs.uniform(-0.2, 0.2, 3) + [0, 0, 0.8]
        Ts.append(T)
    fy = rs.uniform(300, 1100) * H / 480
    fovy = 2.0 * np.degrees(np.arctan(H / (2.0 * fy)))
    return np.array(Ts), float(fovy), H, W


def _functions():
    path = os.path.join(shim.REF_ROOT, "morefusion", "extra", "_pybullet.py")
    text = open(path).read()
    g = dict(np=np, add_model=lambda *a, **k: None)
    for node in ast.parse(text).body:
        if isinstance(node, ast.FunctionDef) and node.name in (
                "get_camera_image", "render_camera", "render_cad"):
            exec(ast.get_source_segment(text, node), g)
    return g


def record(Ts, fovy, height, width):
    """The reference's render_cad(cad, Ts, fovy, height, width) under the recording stand-in:
    (view [N,16], proj [N,4], size [N,2])."""
    calls = {"proj": [], "image": []}
    pb = types.ModuleType("pybullet")
    pb.DIRECT = 2
    pb.ER_BULLET_HARDWARE_OPENGL = 131072
    pb.connect = lambda *a, **k: 0
    pb.disconnect = lambda *a, **k: None

    def projection(fov, aspect, nearVal, farVal):
        calls["proj"].append((fov, aspect, nearVal, farVal))
        return ("projection", len(calls["proj"]))

    def image(width, height, viewMatrix, projectionMatrix, renderer=None):
        calls["image"].append((width, height, np.asarray(viewMatrix, np.float64)))
        return (width, height, np.zeros((height, width, 4), np.uint8),
                np.ones((height, width), np.float32), np.full((height, width), -1))

    pb.computeProjectionMatrixFOV = projection
    pb.getCameraImage = image
    keep = sys.modules.get("pybullet")
    sys.modules["pybullet"] = pb
    try:
        _functions()["render_cad"]("cad.obj", Ts, fovy=fovy, height=height, width=width)
    finally:
        if keep is None:
            sys.modules.pop("pybullet")
        else:
            sys.modules["pybullet"] = keep
    view = np.stack([v for _, _, v in calls["image"]])
    size = np.array([(w, h) for w, h, _ in calls["image"]], np.int64)
    return view, np.array(calls["proj"], np.float64), size


def main():
    out = {}
    for name in CASES:
        Ts, fovy, H, W = case_inputs(name)
        view, proj, size = record(Ts, fovy, H, W)
        out.update({f"{name}/Ts": Ts, f"{name}/view": view, f"{name}/proj": proj,
                    f"{name}/size": size, f"{name}/fovy_hw": np.array([fovy, H, W])})
    os.makedirs(OUT, exist_ok=True)
    np.savez(os.path.join(OUT, "camera_chain.npz"), **out)


if __name__ == "__main__":
    main()
