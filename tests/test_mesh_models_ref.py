"""CPU-only: the model-data composition of YCBVideoModels (tests/golden/mesh_models, written by
oracle/ref_harness/gen_mesh_models.py from the reference's own methods) against
oracle/mesh_models.py, and against a fresh run of those methods when the reference checkout is
present; the oracle's rules on constructed cases; the OBJ reader; and what ``MeshModels`` does
without a GPU (pitches, the sdf.npz cache, missing directories)."""

import hashlib
import json
import os

import numpy as np
import pytest

import _mesh_cases as mc
from oracle import mesh_models as omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh_models")


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def golden():
    data = np.load(os.path.join(GOLDEN, "cases.npz"))
    return {k: data[k] for k in data.files}


def case_names(golden):
    return sorted({k.split("/")[0] for k in golden} - {"cache"})


def test_digest(golden):
    want = json.load(open(os.path.join(GOLDEN, "digest.json")))
    got = {k: hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest() for k, v in golden.items()}
    assert got == want


def test_golden_composition_is_the_oracle(golden):
    names = case_names(golden)
    assert len(names) >= 5
    for name in names:
        v, f = golden[f"{name}/vertices"], golden[f"{name}/faces"]
        pts, sdf = omm.get_sdf(v, f)
        assert np.array_equal(bits(pts), bits(golden[f"{name}/points"])), name
        assert np.array_equal(bits(sdf), bits(golden[f"{name}/sdf"])), name
        # the reference writes what it returns
        assert np.array_equal(bits(golden[f"{name}/written_points"]), bits(pts))
        assert np.array_equal(bits(golden[f"{name}/written_sdf"]), bits(sdf))
        diag = omm.bbox_diagonal(v, f)
        assert bits(diag) == bits(golden[f"{name}/bbox_diagonal"])
        assert bits(1.0 * diag / 32) == bits(golden[f"{name}/pitch32"])
        assert (sdf > 0).any() and np.isfinite(sdf).all()


def test_mesh_models_pitch_and_cache_without_gpu(golden, tmp_path):
    from morefusion_b200.datasets import MeshModels
    names = case_names(golden)
    meshes = {i + 1: (golden[f"{n}/vertices"], golden[f"{n}/faces"]) for i, n in enumerate(names)}
    files = {}
    for c in meshes:
        files[c] = str(tmp_path / f"{c}.npz")
        n = names[c - 1]
        np.savez_compressed(files[c], points=golden[f"{n}/points"], sdf=golden[f"{n}/sdf"])
    models = MeshModels(meshes, {c: np.zeros((4, 3)) for c in meshes}, [2], sdf_files=files)
    for c, n in enumerate(names, 1):
        assert bits(models.get_bbox_diagonal(c)) == bits(golden[f"{n}/bbox_diagonal"])
        assert bits(models.get_voxel_pitch(32, c)) == bits(golden[f"{n}/pitch32"])
        pts, sdf = models.get_sdf(c)                # read from the cache, as _get_sdf reads it
        assert np.array_equal(bits(pts), bits(golden[f"{n}/points"]))
    # the reference returns an existing sdf.npz as it is; MeshModels does the same
    f = str(tmp_path / "cached.npz")
    np.savez_compressed(f, points=golden["cache/points"], sdf=golden["cache/sdf"])
    m = MeshModels({1: meshes[1]}, {1: np.zeros((1, 3))}, sdf_files={1: f})
    p, s = m.get_sdf(1)
    assert np.array_equal(p, golden["cache/points"]) and np.array_equal(s, golden["cache/sdf"])
    assert m.class_ids_symmetric.size == 0 and models.class_ids_symmetric.tolist() == [2]


def test_reference_composition():
    from oracle.ref_harness import shim
    if not shim.reference_available():
        pytest.skip("reference checkout not present")
    import tempfile
    from oracle.ref_harness import gen_mesh_models as gen
    data = np.load(os.path.join(GOLDEN, "cases.npz"))
    meshes = gen.cases()
    with tempfile.TemporaryDirectory() as tmp:
        got = gen.run(meshes, os.path.join(tmp, "m"))
        cache = gen.run_cache(os.path.join(tmp, "c"))
    for name, arrays in got.items():
        for k, a in arrays.items():
            assert np.array_equal(bits(a), bits(data[f"{name}/{k}"])), (name, k)
    assert np.array_equal(cache[2], data["cache/points"]) and np.array_equal(cache[3], data["cache/sdf"])


def test_box_sdf_against_primitive():
    from morefusion_b200 import synthetic
    kind, half = synthetic._primitive(3)
    assert kind == "box"
    v, f = synthetic.cad_mesh(kind, half)
    rs = np.random.RandomState(0)
    p = rs.uniform(-1.6, 1.6, (3000, 3)) * half
    got, _ = omm.signed_distance(v, f, p)
    want = synthetic.sdf_primitive(kind, half, p)
    ulp = np.spacing(np.float64(np.abs(half).max()))
    assert np.abs(got - want).max() <= 8 * ulp
    assert (np.sign(got) == np.sign(want))[np.abs(want) > 1e-12].all()


def test_columns_through_edges_and_vertices_oracle():
    D = 16
    v, f = mc.edge_aligned_box(D)
    s = 1.0 / D
    c = (np.arange(D) + 0.5) * s
    xs, ys = np.meshgrid(c, c, indexing="ij")
    px = np.concatenate([xs.reshape(-1), v[:, 0], c[:8]])
    py = np.concatenate([ys.reshape(-1), v[:, 1], c[:8]])
    n = omm.column_parity_counts(v, f, px, py)
    assert (n % 2 == 0).all()
    assert (n[-8:-1] == 2).all()                   # along the caps' shared diagonal (x = y)
    g = omm.voxelize_solid(v, f, D)
    # the grid is the box: x, y in [0, 7.5 s] fill columns 0..7, the whole height
    assert g["matrix"][:8, :8].all() and not g["matrix"][8:].any() and not g["matrix"][:, 8:].any()


def test_read_obj(tmp_path):
    from morefusion_b200.datasets import read_obj
    p = tmp_path / "m.obj"
    p.write_text("# comment\nmtllib m.mtl\no thing\nv 0 0 0\nv 1 0 0 1.0\nv 1 1 0\nv 0 1 0\n"
                 "vt 0 0\nvn 0 0 1\nusemtl x\ns off\nf 1 2 3\nf 1/1 3/1 4/1\nf 1//1 2//1 4//1\n"
                 "f 1/1/1 2/1/1 3/1/1 4/1/1\nf -4 -3 -2\ng group\n\n")
    v, f = read_obj(str(p))
    assert v.dtype == np.float64 and v.shape == (4, 3)
    assert f.dtype == np.int32
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 3], [0, 1, 2], [0, 2, 3], [0, 1, 2]]
    bad = tmp_path / "bad.obj"
    bad.write_text("v 0 0 0\nf 1 2 3\n")
    with pytest.raises(ValueError):
        read_obj(str(bad))


def test_from_directory(tmp_path):
    from morefusion_b200.datasets import MeshModels
    with pytest.raises(FileNotFoundError):
        MeshModels.from_directory(str(tmp_path / "missing"), ["__background__", "a"])
    v, f = mc.box()
    d = tmp_path / "a"
    d.mkdir()
    lines = ([f"v {float(x)!r} {float(y)!r} {float(z)!r}" for x, y, z in v]
             + [f"f {a + 1} {b + 1} {c + 1}" for a, b, c in f])
    (d / "textured_simple.obj").write_text("\n".join(lines) + "\n")
    np.savetxt(d / "points.xyz", v)
    m = MeshModels.from_directory(str(tmp_path), ["__background__", "a"], [1])
    assert np.array_equal(m.get_cad(1).vertices, v) and np.array_equal(m.get_cad(1).faces, f)
    assert np.array_equal(m.get_pcd(1), v)
    assert bits(m.get_voxel_pitch(32, 1)) == bits(1.0 * omm.bbox_diagonal(v, f) / 32)
    with pytest.raises(FileNotFoundError):
        MeshModels.from_directory(str(tmp_path), ["__background__", "a", "b"])
    with pytest.raises(ValueError):
        MeshModels({1: (v, np.zeros((0, 3), np.int32))}, {})
