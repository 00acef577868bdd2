"""CPU: oracle/render_cad.py's camera chain against the arguments the reference's own
``render_cad`` / ``render_camera`` / ``get_camera_image`` (extra/_pybullet.py:215-288) pass to
pybullet, recorded under oracle/ref_harness/render_cad_stub.py into
tests/golden/render_cad/camera_chain.npz, and -- where the reference checkout is present --
recorded afresh on further poses and image sizes."""

import os

import numpy as np
import pytest

from oracle import render_cad as orc
from oracle.ref_harness import render_cad_stub as stub

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "render_cad", "camera_chain.npz")


def _check(Ts, fovy, H, W, view, proj, size):
    """The recorded view matrices are the oracle's (pybullet reads them column-major), and the
    projection and image-size arguments are the oracle's camera: fovy, W / H, 0.01, 1000."""
    assert len(view) == len(Ts)
    for T, v, p, s in zip(Ts, view, proj, size):
        np.testing.assert_allclose(v.reshape(4, 4).T, orc.view_matrix(T), rtol=0, atol=1e-12)
        assert p[0] == fovy and p[1] == 1.0 * W / H
        assert p[2] == orc.NEAR and p[3] == orc.FAR
        assert tuple(s) == (W, H)
        # through gluPerspective and the viewport, the recorded chain lands where the oracle's
        # projection does
        P = orc.projection_matrix(p[0], p[1], p[2], p[3])
        f = orc.focal_from_fovy(fovy, H)
        for x in ((0.0, 0.0, 0.0), (0.03, -0.02, 0.05)):
            c = T[:3, :3] @ np.asarray(x) + T[:3, 3]
            u, vv = orc.gl_pixel(v.reshape(4, 4).T, P, H, W, x)
            np.testing.assert_allclose([u, vv], [f * c[0] / c[2] + W / 2, f * c[1] / c[2] + H / 2],
                                       rtol=0, atol=1e-8)


@pytest.mark.parametrize("case", sorted(stub.CASES))
def test_camera_chain_equals_fixture(case):
    z = np.load(GOLDEN)
    Ts, fovy, H, W = stub.case_inputs(case)
    assert np.array_equal(z[case + "/Ts"], Ts)
    assert np.array_equal(z[case + "/fovy_hw"], [fovy, H, W])
    _check(Ts, fovy, H, W, z[case + "/view"], z[case + "/proj"], z[case + "/size"])


@pytest.mark.parametrize("H,W,fy", [(480, 640, 1066.778), (1, 1, 3.0), (33, 47, 20.0)])
def test_camera_chain_reference_direct(H, W, fy):
    from oracle.ref_harness import shim
    if not shim.reference_available():
        pytest.skip("reference checkout not present")
    rs = np.random.RandomState(H)
    Ts = []
    for _ in range(4):
        q, _ = np.linalg.qr(rs.normal(size=(3, 3)))
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = q * np.sign(np.linalg.det(q)), rs.uniform(-0.3, 0.3, 3) + [0, 0, 1]
        Ts.append(T)
    Ts = np.array(Ts)
    fovy = orc.fovy_from_intrinsics(fy, H)
    _check(Ts, fovy, H, W, *stub.record(Ts, fovy, H, W))
    # one pose [4,4] is rendered as a batch of one
    view, proj, size = stub.record(Ts[0], fovy, H, W)
    _check(Ts[:1], fovy, H, W, view, proj, size)
