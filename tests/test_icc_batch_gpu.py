"""Batched ICC refinement (`k_icc_run` through `ICCBatch` / `_run`) at the batch sizes and group
sizes the benchmark runs.

The invariant: at a fixed group size G (CTAs per scene) every cross-CTA reduction of a scene runs
in an order fixed by G alone (per-CTA `partials` / `slots` rows, the P4 totals, the P5 block tree,
per-warp `sAcc` in order of first occurrence), the key and max phases are order-free atomics, and
the point ids in a scene's keys are all shifted by the same offset.  So every scene of a batch
must be BIT-IDENTICAL to that scene run alone at the same G: loss history, final q / t, Adam m / v
and the last iteration's gradients.  Across different G the fp64 sums change order; they are sums
of exactly representable fp32 terms rounded once to fp32, so there the kernel is compared with the
float64-summing oracle (`oracle/icc.py`) to about one ulp instead of bitwise.

Every comparison also runs one deliberately wrong reference that it must reject."""

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import icc as oicc
from oracle import transforms as otf
from oracle import voxel_ops as vo

pytestmark = pytest.mark.gpu
F32 = np.float32
N_ITER = 10
# group sizes of the open-loop sweep: 1, around the barrier's sub-group count kBarSub = 24 and its
# double, and the device maximum (appended at run time)
GROUPS = (1, 2, 3, 7, 8, 9, 23, 24, 25, 47, 48, 49)


# ------------------------------------------------------------------ helpers
def max_group(S):
    """mf_icc_max_group_size(S): (SMs x co-resident CTAs per SM) // S on the current device."""
    from morefusion_b200 import _lib
    return int(_lib.lib().mf_icc_max_group_size(int(S)))


def make_scene(n_pts, pitch, *, D=16, seed=0, kind="ball", isolated=False, dead=False):
    """N = len(n_pts) balls (or boxes) of exactly n_pts[i] random points with the analytic sdf
    (positive inside), grid pitch pitch[i], on a line with neighbours overlapping by ~10 % of
    their radii, so every object collides with the next one.  `isolated` moves object 1 half a
    metre away (the other-object grids of both objects are then NaN and skipped); `dead` makes
    every sdf <= -0.03, so that sdf + sdf_offset <= 0 for any offset <= 0.02 and the loss is NaN."""
    rs = np.random.RandomState(seed)
    N = len(n_pts)
    pitch = np.asarray(pitch, F32)
    points, sdf, T0, origin, gt, gne = [], [], [], [], [], []
    x = 0.0
    ijk = np.stack(np.meshgrid(*(np.arange(D),) * 3, indexing="ij"), -1).astype(F32)
    for i in range(N):
        p = float(pitch[i])
        r = p * D * 0.3
        if i > 0:
            x += 0.9 * (r + float(pitch[i - 1]) * D * 0.3)
        c = np.array([x + (0.5 if isolated and i == 1 else 0.0), rs.uniform(-0.2, 0.2) * r, 0.6], F32)
        if kind == "ball":
            v = rs.normal(size=(n_pts[i], 3))
            v /= np.linalg.norm(v, axis=1, keepdims=True)
            pts = v * (r * rs.uniform(size=n_pts[i]) ** (1 / 3))[:, None]
            s = r - np.linalg.norm(pts, axis=1)
        else:
            half = r * np.array([1.0, 0.75, 0.5])
            pts = rs.uniform(-half, half, (n_pts[i], 3))
            s = (half - np.abs(pts)).min(1)
        if dead:
            s = -np.abs(s) - 0.03
        points.append(pts.astype(F32))
        sdf.append(s.astype(F32))
        ang = rs.uniform(-0.3, 0.3, 3)
        q = np.array([1.0, *ang]) / np.linalg.norm([1.0, *ang])
        T = np.eye(4)
        T[:3, :3] = otf.quaternion_matrix_fwd(q[None].astype(F32))[0][0, :3, :3]
        T[:3, 3] = c + rs.normal(0, 0.5 * p, 3)
        T0.append(T.astype(F32))
        o = (c - p * (D / 2.0 - 0.5)).astype(F32)
        origin.append(o)
        dist = np.linalg.norm(ijk * F32(p) + o - c, axis=-1)
        gt.append(((dist < r) & (dist > r - 1.5 * p) & (ijk[..., 2] * p + o[2] < c[2])).astype(F32))
        gne.append(((dist > r + p) & (rs.uniform(size=dist.shape) < 0.7)).astype(F32))
    return dict(points=points, sdf=sdf, pitch=pitch, origin=np.stack(origin),
                grid_target=np.stack(gt), grid_nontarget_empty=np.stack(gne),
                transform_init=np.stack(T0), voxel_dim=D)


def initial_pose(sc):
    from morefusion_b200.geometry import quaternion_from_matrix, translation_from_matrix
    q = np.stack([quaternion_from_matrix(np.asarray(T)) for T in sc["transform_init"]]).astype(F32)
    t = np.stack([translation_from_matrix(np.asarray(T)) for T in sc["transform_init"]]).astype(F32)
    return q, t


def on_device(sc, dev):
    """The scene with its arrays on the device once, so that batches of hundreds of copies only
    concatenate; q0 / t0 are the initial parameters as ICCBatch computes them."""
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)   # noqa: E731
    out = dict(sc, points=[t(p) for p in sc["points"]], sdf=[t(s) for s in sc["sdf"]],
               pitch=t(sc["pitch"]), origin=t(sc["origin"]),
               grid_target=t(np.asarray(sc["grid_target"], F32)),
               grid_nontarget_empty=t(np.asarray(sc["grid_nontarget_empty"], F32)))
    if "q0" not in out:
        out["q0"], out["t0"] = initial_pose(sc)
    return out


def np_args(sc):
    return (sc["points"], sc["sdf"], sc["pitch"], sc["origin"], np.asarray(sc["grid_target"], F32),
            np.asarray(sc["grid_nontarget_empty"], F32))


def run(scenes, G, n_iter, update=True, *, D=16, thr=2, off=0.02, q=None, t=None):
    """One `_run` launch over `scenes` (device scenes of `on_device`) at group size G from
    (q, t) (default: every scene's q0 / t0) and zero Adam state.  Returns numpy arrays of the
    loss history [S, n_iter], last-iteration grads [Ntot, 7], final q / t and Adam m / v, and
    the scenes' object offsets."""
    from morefusion_b200.contrib.iterative_collision_check_link import (_Problem, _run,
                                                                       chainer_adam_alpha)
    dev = scenes[0]["points"][0].device
    prob = _Problem(scenes, D, dev)
    qd = torch.tensor(np.concatenate([s["q0"] for s in scenes]) if q is None else q, device=dev)
    td = torch.tensor(np.concatenate([s["t0"] for s in scenes]) if t is None else t, device=dev)
    adam = torch.zeros(14 * prob.Ntot, dtype=torch.float32, device=dev)
    steps = range(1, n_iter + 1) if update else ()
    loss, grads = _run(prob, qd, td, adam, n_iter=n_iter, update=update,
                       alpha_q=[chainer_adam_alpha(0.01, s) for s in steps],
                       alpha_t=[chainer_adam_alpha(0.001, s) for s in steps],
                       voxel_threshold=thr, sdf_offset=off, group_size=G)
    n = prob.Ntot
    a = adam.cpu().numpy()
    return dict(loss=loss.cpu().numpy(), grads=grads.cpu().numpy(), q=qd.cpu().numpy(),
                t=td.cpu().numpy(), mq=a[:4 * n].reshape(n, 4), mt=a[4 * n:7 * n].reshape(n, 3),
                vq=a[7 * n:11 * n].reshape(n, 4), vt=a[11 * n:].reshape(n, 3),
                off=prob.scene_obj_off.cpu().numpy())


FIELDS = ("loss", "grads", "q", "t", "mq", "mt", "vq", "vt")


def scene_of(res, s):
    o0, o1 = res["off"][s], res["off"][s + 1]
    return {k: (res[k][s] if k == "loss" else res[k][o0:o1]) for k in FIELDS}


def bits_equal(a, b):
    """Bit-for-bit equal float32 arrays; NaN matches NaN (payloads aside)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    if a.shape != b.shape:
        return False
    nan = np.isnan(a)
    return bool(np.array_equal(nan, np.isnan(b))
                and np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan]))


def differing(x, y):
    return [k for k in FIELDS if not bits_equal(x[k], y[k])]


def ulps(a, b):
    """Distance in float32 ulps (units in the last place), +0 == -0."""
    def ordered(x):
        i = np.asarray(x, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def open_loop_errors(res, ref):
    """Deviation of one `update=0, n_iter=1` launch from oracle.icc.icc_forward_backward:
    (loss relative error, worst gt ulps vs float32(gsum), worst gq error / row max |gq|,
    number of the 7N gradient components bit-equal to the oracle)."""
    g = res["grads"]
    dl = abs(float(res["loss"][0, 0]) - float(ref["loss"])) / abs(float(ref["loss"]))
    gt_ref = ref["gsum"][:, [3, 7, 11]].astype(F32)
    du = int(ulps(g[:, 4:], gt_ref).max())
    dq = float((np.abs(g[:, :4] - ref["gq"]) / np.abs(ref["gq"]).max(1, keepdims=True)).max())
    n_eq = int((g[:, 4:] == gt_ref).sum() + (g[:, :4] == ref["gq"]).sum())
    return dl, du, dq, n_eq


def meets_open_loop_bars(err):
    """loss rtol 3e-7; gt within 1 fp32 ulp of float32(gsum); gq within 1e-6 of its row max."""
    dl, du, dq, _ = err
    return dl <= 3e-7 and du <= 1 and dq <= 1e-6


def oracle_poses(sc, n_steps=3, **kw):
    """(q, t) at the initial pose and after `n_steps` oracle Adam steps, with the oracle's
    forward-backward at both."""
    q, t = initial_pose(sc) if "q0" not in sc else (sc["q0"].copy(), sc["t0"].copy())
    oq, ot = oicc.ChainerAdam(q.shape, 0.01), oicc.ChainerAdam(t.shape, 0.001)
    out = []
    for k in range(n_steps + 1):
        r = oicc.icc_forward_backward(q, t, *np_args(sc), **kw)
        if k in (0, n_steps):
            out.append((q.copy(), t.copy(), r))
        oq.update(q, r["gq"])
        ot.update(t, r["gt"])
    return out


def pose_err(q, t, q_ref, t_ref):
    T = otf.transformation_matrix(q, t)
    Tr = otf.transformation_matrix(q_ref, t_ref)
    return (float(np.abs(T[:, :3, :3] - Tr[:, :3, :3]).max()),
            float(np.abs(T[:, :3, 3] - Tr[:, :3, 3]).max()))


def hetero_scenes(dev):
    """Scenes of 1, 2 (isolated pair), 3, 8 and 32 objects and a 3-object scene with NaN loss,
    per-object point counts 1, 31, 33, 256, 257 and 5400, every object its own pitch; ordered so
    that the first four already mix a 32-object, a 1-object and the NaN scene."""
    rs = np.random.RandomState(1234)
    P = lambda n: rs.uniform(0.004, 0.009, n).astype(F32)                  # noqa: E731
    s32 = make_scene([(31, 33, 256, 257)[i % 4] for i in range(32)], P(32), seed=1)
    s1 = make_scene([257], P(1), seed=2)
    dead = make_scene([256, 257, 31], P(3), seed=3, dead=True)
    s3 = make_scene([1, 256, 5400], P(3), seed=4)
    s8 = make_scene([33, 257, 31, 256, 5400, 1, 256, 33], P(8), seed=5, kind="box")
    s2 = make_scene([31, 33], P(2), seed=6, isolated=True)
    return [on_device(s, dev) for s in (s32, s1, dead, s3, s8, s2)]


# ------------------------------------------------------------------ 1. batch == single scene at G
def test_batch_equals_single_scene_at_the_batch_group_size(cuda_device):
    H = hetero_scenes(cuda_device)
    n_sm = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    cap = max_group(1)                       # co-resident CTAs: S = cap runs at G = 1
    assert max_group(cap) == 1 and max_group(cap + 1) == 0
    alone = {}
    sweep = []
    for S in sorted({4, 8, 16, n_sm // 4, n_sm // 2, n_sm, cap}):
        G = max_group(S)
        idx = [i % len(H) for i in range(S)]
        res = run([H[i] for i in idx], G, N_ITER)
        for s, i in enumerate(idx):
            if (i, G) not in alone:
                alone[(i, G)] = scene_of(run([H[i]], G, N_ITER), 0)
            assert not differing(scene_of(res, s), alone[(i, G)]), \
                (S, G, s, i, differing(scene_of(res, s), alone[(i, G)]))
        # wrong reference: a scene against its neighbour's single run
        assert not bits_equal(res["loss"][0], alone[(idx[1], G)]["loss"])
        sweep.append((S, G))
        # the NaN scene really is NaN, its neighbours are finite
        assert np.isnan(res["loss"][2]).all() and np.isfinite(res["loss"][[0, 1, 3]]).all()
    print("batch sweep (S, G):", sweep)
    assert [g for _, g in sweep][-1] == 1

    # the reversed batch gives the reversed results; two runs at the same G are bit-identical
    S = 8
    G = max_group(S)
    fwd = run([H[i % 6] for i in range(S)], G, N_ITER)
    rev = run([H[i % 6] for i in reversed(range(S))], G, N_ITER)
    again = run([H[i % 6] for i in range(S)], G, N_ITER)
    for s in range(S):
        assert not differing(scene_of(fwd, s), scene_of(rev, S - 1 - s)), s
        assert not differing(scene_of(fwd, s), scene_of(again, s)), s
    assert not bits_equal(fwd["loss"][3], rev["loss"][3])       # wrong reference: unreversed

    # IterativeCollisionCheckLink.refine at group_size = G == ICCBatch == run()
    from morefusion_b200.contrib import IterativeCollisionCheckLink
    from morefusion_b200.contrib.iterative_collision_check_link import ICCBatch
    sc = H[3]
    G = max_group(4)
    link = IterativeCollisionCheckLink(sc["transform_init"], voxel_dim=16, sdf_offset=0.02)
    link = link.to(cuda_device)
    link.group_size = G
    with torch.no_grad():
        link.quaternion.copy_(torch.from_numpy(sc["q0"]))
        link.translation.copy_(torch.from_numpy(sc["t0"]))
    hl = link.refine(sc["points"], sc["sdf"], sc["pitch"], sc["origin"], sc["grid_target"],
                     sc["grid_nontarget_empty"], n_iter=N_ITER).cpu().numpy()
    batch = ICCBatch([sc], voxel_dim=16, sdf_offset=0.02, device=cuda_device)
    batch.quaternion.copy_(torch.from_numpy(sc["q0"]))
    batch.translation.copy_(torch.from_numpy(sc["t0"]))
    batch.group_size = G
    hb = batch.refine(n_iter=N_ITER).cpu().numpy()
    ref = scene_of(run([sc], G, N_ITER), 0)
    assert bits_equal(hl, hb[0]) and bits_equal(hb[0], ref["loss"])
    for x, y in ((link.quaternion.detach(), batch.quaternion), (link.translation.detach(), batch.translation),
                 (link._adam_state, batch.adam_state)):
        assert bits_equal(x.cpu().numpy(), y.cpu().numpy())
    assert bits_equal(batch.quaternion.cpu().numpy(), ref["q"])
    assert bits_equal(batch.translation.cpu().numpy(), ref["t"])


def test_bench_scenes_batched_at_n_sm_for_100_iterations(cuda_device):
    """The `icc` record's largest batch: make_icc_scene(N=8, seed=10..13) repeated to n_sm scenes,
    100 iterations, against every scene alone at the same G."""
    from morefusion_b200 import synthetic
    scenes = [on_device(synthetic.make_icc_scene(N=8, seed=10 + i), cuda_device) for i in range(4)]
    n_sm = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    G = max_group(n_sm)
    res = run([scenes[i % 4] for i in range(n_sm)], G, 100, D=32)
    alone = [scene_of(run([sc], G, 100, D=32), 0) for sc in scenes]
    for s in range(n_sm):
        assert not differing(scene_of(res, s), alone[s % 4]), (s, differing(scene_of(res, s), alone[s % 4]))
    assert differing(scene_of(res, 0), alone[1])                # wrong reference: the neighbour
    print(f"bench scenes: S={n_sm} G={G} bit-identical to the single-scene runs")


# ------------------------------------------------------------------ 2. every G vs the oracle
def test_every_group_size_against_the_oracle_open_loop(cuda_device):
    from morefusion_b200 import synthetic
    sc = synthetic.make_icc_scene(N=8, seed=3, kinds=("box",))
    poses = oracle_poses(sc, sdf_offset=0.02)
    dsc = on_device(sc, cuda_device)
    Gmax = max_group(1)
    worst = {}
    for G in GROUPS + (Gmax,):
        for k, (q, t, ref) in enumerate(poses):
            res = run([dsc], G, 1, update=False, D=32, q=q, t=t)
            err = open_loop_errors(res, ref)
            assert meets_open_loop_bars(err), (G, k, err)
            w = worst.get(G, (0.0, 0, 0.0, 7 * 8 * 2))
            worst[G] = (max(w[0], err[0]), max(w[1], err[1]), max(w[2], err[2]), min(w[3], err[3]))
        if G == Gmax:
            # wrong reference: the kernel at the second pose against the oracle at the first
            assert not meets_open_loop_bars(open_loop_errors(res, poses[0][2]))
    for G, (dl, du, dq, n_eq) in worst.items():
        print(f"G={G:4d}: loss rel {dl:.2g}, gt {du} ulp, gq {dq:.2g} of row max, "
              f">= {n_eq}/56 components bit-equal to the oracle")


# ------------------------------------------------------------------ 3. closed loop vs fixtures
def _fixture_scene(name):
    from oracle.ref_harness import gen_icc_closed_loop as gen
    g = golden("icc_closed_loop_" + name)
    if name == "ref3":
        off = np.r_[0, np.cumsum(g["sizes"])]
        sc = dict(points=[g["points"][off[i]:off[i + 1]] for i in range(3)],
                  sdf=[g["sdf"][off[i]:off[i + 1]] for i in range(3)], pitch=g["pitch"],
                  origin=g["origin"], grid_target=g["grid_target"].astype(F32),
                  grid_nontarget_empty=g["grid_nontarget_empty"].astype(F32),
                  transform_init=g["transform_init"])
    else:
        sc = gen.scene(name)
    assert gen.inputs_checksum(sc) == str(g["inputs_sha1"]), "inputs differ from the fixture's"
    sc["q0"], sc["t0"] = g["q0"], g["t0"]
    return sc, g


def test_closed_loop_batches_against_the_fixtures(cuda_device):
    from morefusion_b200.contrib.iterative_collision_check_link import ICCBatch
    names = ("ref3", "seed3", "seed4")
    fx = {n: _fixture_scene(n) for n in names}
    dsc = {n: on_device(fx[n][0], cuda_device) for n in names}
    n_sm = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    for S in (3, 4, n_sm):
        order = [names[i % 3] for i in range(S)]
        batch = ICCBatch([dsc[n] for n in order], sdf_offset=0.02, device=cuda_device)
        off = batch.prob.scene_obj_off.cpu().numpy()
        for s, n in enumerate(order):
            batch.quaternion[off[s]:off[s + 1]] = torch.from_numpy(fx[n][1]["q0"]).to(cuda_device)
            batch.translation[off[s]:off[s + 1]] = torch.from_numpy(fx[n][1]["t0"]).to(cuda_device)
        hist = batch.refine(n_iter=100).cpu().numpy()
        q, t = batch.quaternion.cpu().numpy(), batch.translation.cpu().numpy()
        exact = []
        for s, n in enumerate(order):
            g = fx[n][1]
            qs, ts = q[off[s]:off[s + 1]], t[off[s]:off[s + 1]]
            dR, dt = pose_err(qs, ts, g["q"], g["t"])
            assert dR <= 1e-4 and dt <= 1e-4, (S, s, n, dR, dt)
            np.testing.assert_allclose(hist[s], g["loss"], rtol=1e-4, atol=1e-5)
            exact.append(bits_equal(qs, g["q"]) and bits_equal(ts, g["t"]) and bits_equal(hist[s], g["loss"]))
        # wrong reference: seed3's result against seed4's fixture
        s3 = order.index("seed3")
        dR, dt = pose_err(q[off[s3]:off[s3 + 1]], t[off[s3]:off[s3 + 1]], fx["seed4"][1]["q"],
                          fx["seed4"][1]["t"])
        assert dR > 1e-4 or dt > 1e-4
        print(f"closed loop S={S} G={max_group(S)}: {sum(exact)}/{S} scenes bit-identical to their fixture")


# ------------------------------------------------------------------ 4. non-default arguments
def ks_jump_pitch():
    """A pitch at which voxel_threshold 3 gives ks = 5: ceilf(fl(3 p) / p) = 4 in fp32."""
    for p in np.arange(0.0060, 0.0070, 1e-7).astype(F32):
        if vo.tdf_ksize(p, F32(F32(3) * p)) == 5:
            return p
    raise AssertionError("no ks-jump pitch in [6, 7) mm")


CONFIGS = {
    "thr1": dict(thr=1, D=16, off=0.02, pitch=(0.0063, 0.0087, 0.0064)),
    "thr3_ks5": dict(thr=3, D=20, off=0.02, pitch=None),
    "thr4": dict(thr=4, D=16, off=0.0, pitch=(0.0055, 0.0071, 0.0048)),
    "thr2.5_d20": dict(thr=2.5, D=20, off=0.02, pitch=(0.0061, 0.0052, 0.0077)),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_non_default_arguments_against_the_oracle(cuda_device, name):
    cfg = CONFIGS[name]
    thr, D, off = cfg["thr"], cfg["D"], cfg["off"]
    pitch = cfg["pitch"]
    if pitch is None:
        pj = ks_jump_pitch()
        pitch = (F32(0.0066), pj, F32(0.0058))
        ks = [vo.tdf_ksize(p, F32(F32(3) * F32(p))) for p in pitch]
        assert ks == [3, 5, 3], ks
        print(f"ks-jump pitch {float(pj)!r}: ks {ks}")
    sc = make_scene([300, 400, 350], pitch, D=D, seed=11)
    kw = dict(voxel_dim=D, voxel_threshold=thr, sdf_offset=off)
    poses = oracle_poses(sc, **kw)
    dsc = on_device(sc, cuda_device)
    Gmax = max_group(1)
    worst = 0
    for G in GROUPS + (Gmax,):
        for q, t, ref in poses:
            err = open_loop_errors(run([dsc], G, 1, update=False, D=D, thr=thr, off=off, q=q, t=t), ref)
            assert meets_open_loop_bars(err), (G, err)
            worst = max(worst, err[1])
    # wrong reference
    q, t, _ = poses[0]
    res = run([dsc], Gmax, 1, update=False, D=D, thr=thr, off=off, q=q, t=t)
    if name == "thr3_ks5":
        wrong = oicc.icc_forward_backward(q, t, *np_args(sc), voxel_dim=D, voxel_threshold=2, sdf_offset=off)
    else:
        wrong = oicc.icc_forward_backward(q, t, *np_args(sc), voxel_dim=D, voxel_threshold=thr,
                                          sdf_offset=0.02 - off)
    assert not meets_open_loop_bars(open_loop_errors(res, wrong))
    # closed loop, 10 iterations
    q_ref, t_ref, h_ref = oicc.icc_refine(sc["transform_init"], *np_args(sc), n_iter=N_ITER,
                                          return_history=True, q0=poses[0][0], t0=poses[0][1], **kw)
    for G in (Gmax, 4):
        res = run([dsc], G, N_ITER, D=D, thr=thr, off=off)
        dR, dt = pose_err(res["q"], res["t"], q_ref, t_ref)
        assert dR <= 1e-4 and dt <= 1e-4, (G, dR, dt)
        np.testing.assert_allclose(res["loss"][0], h_ref, rtol=1e-4, atol=1e-5)
    print(f"{name}: open loop worst gt {worst} ulp over G in {GROUPS + (Gmax,)}")


# ------------------------------------------------------------------ 5. launch chunking and reuse
def _contact3(dev):
    g = golden("icc_forward_contact3")
    sc = dict(points=[g[f"points_{i}"] for i in range(3)], sdf=[g[f"sdf_{i}"] for i in range(3)],
              pitch=g["pitch"], origin=g["origin"], grid_target=g["grid_target"],
              grid_nontarget_empty=g["grid_nontarget_empty"], transform_init=g["transform_init"])
    assert int(g["voxel_dim"]) == 16 and int(g["voxel_threshold"]) == 2
    assert float(g["sdf_offset"]) == F32(0.02)
    return sc, on_device(sc, dev)


def test_refine_chunking_matches_one_launch_and_the_oracle(cuda_device):
    from morefusion_b200.contrib import IterativeCollisionCheckLink
    sc, dsc = _contact3(cuda_device)
    args = (dsc["points"], dsc["sdf"], dsc["pitch"], dsc["origin"], dsc["grid_target"],
            dsc["grid_nontarget_empty"])

    def link():
        lk = IterativeCollisionCheckLink(sc["transform_init"], voxel_dim=16, sdf_offset=0.02)
        lk = lk.to(cuda_device)
        with torch.no_grad():
            lk.quaternion.copy_(torch.from_numpy(dsc["q0"]))
            lk.translation.copy_(torch.from_numpy(dsc["t0"]))
        return lk

    def state(lk, hist):
        a = lk._adam_state.cpu().numpy()
        return dict(loss=hist, q=lk.quaternion.detach().cpu().numpy(),
                    t=lk.translation.detach().cpu().numpy(), adam=a)

    one = link()
    s130 = state(one, one.refine(*args, n_iter=130).cpu().numpy())
    two = link()
    h = [two.refine(*args, n_iter=64).cpu().numpy(), two.refine(*args, n_iter=66).cpu().numpy()]
    s64_66 = state(two, np.concatenate(h))
    single = link()
    h, at128 = [], None
    for k in range(130):
        if k == 128:
            at128 = state(single, None)
        h.append(single.refine(*args, n_iter=1).cpu().numpy())
    s1x130 = state(single, np.concatenate(h))
    assert one._adam_t == two._adam_t == single._adam_t == 130
    for other in (s64_66, s1x130):
        for k in ("loss", "q", "t", "adam"):
            assert bits_equal(s130[k], other[k]), k

    # the oracle loop, Chainer Adam driven directly for its m and v
    q, t = dsc["q0"].copy(), dsc["t0"].copy()
    oq, ot = oicc.ChainerAdam(q.shape, 0.01), oicc.ChainerAdam(t.shape, 0.001)
    hist = []
    for _ in range(130):
        r = oicc.icc_forward_backward(q, t, *np_args(sc), voxel_dim=16, sdf_offset=0.02)
        hist.append(float(r["loss"]))
        oq.update(q, r["gq"])
        ot.update(t, r["gt"])
    N = q.shape[0]
    a = s130["adam"]
    dR, dt = pose_err(s130["q"], s130["t"], q, t)
    assert dR <= 1e-4 and dt <= 1e-4, (dR, dt)
    np.testing.assert_allclose(s130["q"], q, rtol=0, atol=1e-4)
    np.testing.assert_allclose(s130["loss"], hist, rtol=1e-4, atol=1e-5)
    for got, ref in ((a[:4 * N], oq.m), (a[4 * N:7 * N], ot.m), (a[7 * N:11 * N], oq.v),
                     (a[11 * N:], ot.v)):
        np.testing.assert_allclose(got.reshape(ref.shape), ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())
    print(f"refine(130) vs oracle: |dR| {dR:.3g} |dt| {dt:.3g}")

    # the launch boundary: from the kernel's own state after 128 steps, the oracle's steps 129 and
    # 130 must reproduce the chunked refine's last two steps; the same steps counted from 128
    # (Adam's step count off by one from step 129 on) must not.  The gradients at one pose agree
    # to <= 1 ulp (test_every_group_size_against_the_oracle_open_loop), so two Adam steps from one
    # state may move q and t (|q| = 1) apart by a few ulps: 2e-7.  alpha_t of steps 128 and 129
    # differ by 0.37 %.
    def branch(first_step):
        q, t = at128["q"].copy(), at128["t"].copy()
        a = at128["adam"]
        oq, ot = oicc.ChainerAdam(q.shape, 0.01), oicc.ChainerAdam(t.shape, 0.001)
        oq.m, ot.m = a[:4 * N].reshape(N, 4).copy(), a[4 * N:7 * N].reshape(N, 3).copy()
        oq.v, ot.v = a[7 * N:11 * N].reshape(N, 4).copy(), a[11 * N:].reshape(N, 3).copy()
        oq.t = ot.t = first_step - 1
        for _ in range(2):
            r = oicc.icc_forward_backward(q, t, *np_args(sc), voxel_dim=16, sdf_offset=0.02)
            oq.update(q, r["gq"])
            ot.update(t, r["gt"])
        return max(np.abs(q - s130["q"]).max(), np.abs(t - s130["t"]).max())
    right, wrong = branch(129), branch(128)
    print(f"steps 129-130 from the kernel's state: {right:.3g} (step count 129), "
          f"{wrong:.3g} (step count 128)")
    assert right <= 2e-7 < wrong, (right, wrong)


def test_bench_and_chain_reuse_of_a_batch(cuda_device):
    from morefusion_b200.contrib.iterative_collision_check_link import ICCBatch
    sc, dsc = _contact3(cuda_device)
    alt = make_scene([464, 464, 464], sc["pitch"], D=16, seed=21)
    alt2 = make_scene([200, 300, 250], (0.0058, 0.0064, 0.0071), D=16, seed=22)
    scenes = [dsc, on_device(alt, cuda_device), on_device(alt2, cuda_device)]

    def fresh(scs):
        b = ICCBatch(scs, voxel_dim=16, sdf_offset=0.02, device=cuda_device)
        b.quaternion.copy_(torch.from_numpy(np.concatenate([s["q0"] for s in scs])))
        b.translation.copy_(torch.from_numpy(np.concatenate([s["t0"] for s in scs])))
        return b

    def snap(b, hist):
        off = b.prob.scene_obj_off.cpu().numpy()
        q, t, a = (x.cpu().numpy() for x in (b.quaternion, b.translation, b.adam_state))
        return [dict(loss=hist[s], q=q[off[s]:off[s + 1]], t=t[off[s]:off[s + 1]]) for s in range(len(off) - 1)], a

    b = fresh(scenes)
    q0, t0 = b.quaternion.clone(), b.translation.clone()
    first, a_first = snap(b, b.refine(n_iter=N_ITER).cpu().numpy())

    def reset():
        b.quaternion.copy_(q0)
        b.translation.copy_(t0)
        b.adam_state.zero_()
        b.adam_t = 0
    # bench pattern
    reset()
    again, a_again = snap(b, b.refine(n_iter=N_ITER).cpu().numpy())
    assert bits_equal(a_first, a_again)
    for x, y in zip(first, again):
        assert all(bits_equal(x[k], y[k]) for k in x)

    # chain pattern: scene 1's target and non-target grids rewritten in place
    new = dict(alt, grid_target=np.roll(alt["grid_target"], 1, axis=1),
               grid_nontarget_empty=np.roll(alt["grid_nontarget_empty"], -1, axis=2))
    off = b.prob.scene_obj_off.cpu().numpy()
    V = 16 ** 3
    b.prob.grid_target[off[1]:off[2]] = torch.from_numpy(new["grid_target"].reshape(-1, V)).to(cuda_device)
    b.prob.gne[off[1]:off[2]] = torch.from_numpy(new["grid_nontarget_empty"].reshape(-1, V)).to(cuda_device)
    reset()
    chained, _ = snap(b, b.refine(n_iter=N_ITER).cpu().numpy())
    f = fresh([scenes[0], on_device(new, cuda_device), scenes[2]])
    ref, _ = snap(f, f.refine(n_iter=N_ITER).cpu().numpy())
    for s in range(3):
        assert all(bits_equal(chained[s][k], ref[s][k]) for k in ref[s]), s
        if s != 1:
            assert all(bits_equal(chained[s][k], first[s][k]) for k in ref[s]), s
    # wrong reference: scene 1 before its grids were rewritten
    assert not bits_equal(chained[1]["loss"], first[1]["loss"])


def test_over_capacity_batches_are_refused(cuda_device):
    from morefusion_b200.contrib.iterative_collision_check_link import ICCBatch
    big = make_scene([1] * 33, np.full(33, 0.006, F32), D=16, seed=31)
    with pytest.raises(ValueError):
        ICCBatch([big], voxel_dim=16, device=cuda_device)
    tiny = on_device(make_scene([1], [0.006], D=16, seed=32), cuda_device)
    cap = max_group(1)
    b = ICCBatch([tiny] * (cap + 1), voxel_dim=16, device=cuda_device)
    q = b.quaternion.clone()
    with pytest.raises(ValueError):
        b.refine(n_iter=1)
    assert b.adam_t == 0 and torch.equal(b.quaternion, q)
    ok = ICCBatch([tiny] * cap, voxel_dim=16, device=cuda_device)     # at capacity it runs
    assert ok.refine(n_iter=1).shape == (cap, 1)
