"""GPU parity: 3D-CNN section of singleview_3d.Model (CUDA, bf16 operands / fp32 accumulate)
vs the torch-CPU oracle.  Tolerances: against the oracle run with bf16-rounded operands at the
same points (tight) and against the pure fp32 oracle (bf16-level)."""

import numpy as np
import pytest
import torch

from oracle import cnn as ocnn

pytestmark = pytest.mark.gpu
F32 = np.float32


def make_inputs(B, P=1000, seed=0):
    rs = np.random.RandomState(seed)
    values = rs.normal(0, 1, (B, 32, P)).astype(F32)
    # surface-like cloud in the voxel frame, a few points outside the grid
    c = rs.uniform(12, 20, (B, 3, 1))
    d = rs.normal(size=(B, 3, P))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    points = (c + d * rs.uniform(6, 11, (B, 1, P))).astype(F32)
    points[:, :, :5] = rs.uniform(-3, 35, (B, 3, 5))
    gne = (rs.uniform(size=(B, 32, 32, 32)) < 0.4)
    class_id = (np.arange(B) % 21 + 1).astype(np.int32)
    pitch = np.array([0.0063 + 0.0005 * i for i in range(B)], F32)
    origin = rs.uniform(-0.2, 0.6, (B, 3)).astype(F32)
    return dict(values=values, points=points, grid_nontarget_empty=gne, class_id=class_id,
                pitch=pitch, origin=origin)


def run_cuda(w, inp, dev, with_occ=True, tc=True):
    from morefusion_b200.contrib.singleview_3d.models import Model
    m = Model(n_fg_class=21, with_occupancy=with_occ).to(dev)
    m.load_reference_weights(w)
    m.use_tensor_cores = tc
    rot, trans, conf = m.forward_features(
        class_id=torch.as_tensor(inp["class_id"], device=dev),
        values=torch.as_tensor(inp["values"], device=dev),
        points=torch.as_tensor(inp["points"], device=dev),
        pitch=inp["pitch"], origin=inp["origin"],
        grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=dev))
    torch.cuda.synchronize()
    return m, rot.cpu().numpy(), trans.cpu().numpy(), conf.cpu().numpy()


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("with_occ", [True, False])
def test_cnn_forward_vs_oracle(cuda_device, with_occ, tc):
    B = 2
    w = ocnn.init_weights(21, seed=1, with_occupancy=with_occ)
    inp = make_inputs(B)
    m, rot, trans, conf = run_cuda(w, inp, cuda_device, with_occ, tc)
    ref = ocnn.forward(w, n_fg_class=21, bf16=True, **inp)
    # concat feature [B*P,984] (bf16 storage) vs oracle feat
    feat = m._wbufs[(B, 1000, cuda_device)]["feat"][:, :984].float().cpu().numpy()
    want = ref["feat"].transpose(0, 2, 1).reshape(B * 1000, 984)
    err = np.abs(feat - want)
    scale = np.abs(want).max()
    assert err.max() <= 0.02 * scale, (err.max(), scale)
    assert np.mean(err) <= 2e-3 * scale
    # final poses: tight vs bf16-rounded oracle
    # normalised quaternions amplify bf16 noise where the raw head output is small:
    # 99.9% of components within 2e-2, all within 0.1
    drot = np.abs(rot - ref["rot"])
    assert np.mean(drot <= 2e-2) >= 0.999 and drot.max() <= 0.1, (np.mean(drot <= 2e-2), drot.max())
    np.testing.assert_allclose(conf, ref["conf"], rtol=0, atol=2e-2)
    np.testing.assert_allclose(trans, ref["trans"], rtol=0, atol=2e-2 * float(inp["pitch"].max()) * 8)
    assert np.mean(np.abs(rot - ref["rot"])) < 2e-3
    # bf16-level vs the reference's fp32 arithmetic
    ref32 = ocnn.forward(w, n_fg_class=21, bf16=False, **inp)
    assert np.mean(np.abs(rot - ref32["rot"])) < 1e-2
    assert np.mean(np.abs(conf - ref32["conf"])) < 1e-2
    # argmax-confidence pose (what the callers consume, demo.py:85 / evaluate.py:86)
    k = conf.argmax(1)
    k32 = ref32["conf"].argmax(1)
    for b in range(B):
        q, q32 = rot[b, k[b]], ref32["rot"][b, k[b]]
        assert abs(abs(float(q @ q32)) - 1) < 5e-3
        assert ref32["conf"][b, k[b]] >= ref32["conf"][b, k32[b]] - 2e-2


def test_fused_voxelize_equals_operator_composition(cuda_device):
    """The fused voxelise->s2d path (sparse clear + leader scatter + occupancy stencil writing
    in place) produces bit-identical conv3 input to average_voxelization_3d + occ convs + pack,
    across consecutive calls with different inputs (exercises the sparse re-zeroing)."""
    from morefusion_b200.contrib.singleview_3d.models import Model
    B = 3
    w = ocnn.init_weights(21, seed=2)
    m = Model(n_fg_class=21, with_occupancy=True).to(cuda_device).load_reference_weights(w)

    def x3_of(inp, fused):
        m.fused_voxelize = fused
        m.forward_features(
            class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
            values=torch.as_tensor(inp["values"], device=cuda_device),
            points=torch.as_tensor(inp["points"], device=cuda_device),
            pitch=inp["pitch"], origin=inp["origin"],
            grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device))
        torch.cuda.synchronize()
        return m._wbufs[(B, 1000, cuda_device)]["x3"].clone()

    def same(x, ref):
        x = x.reshape(B, 17, 17, 17, 8, 160).float()
        ref = ref.reshape(B, 17, 17, 17, 8, 160).float()
        # 144 averaged feature channels: bit-identical
        assert torch.equal(x[..., :144], ref[..., :144])
        # 16 occupancy channels: tensor-core (bf16 operand) stencil vs the fp32 SIMT stencil
        torch.testing.assert_close(x[..., 144:], ref[..., 144:], rtol=0,
                                   atol=0.02 * float(ref[..., 144:].abs().max()))

    a, b, c = make_inputs(B, seed=5), make_inputs(B, seed=6), make_inputs(B, seed=7)
    ref_a, ref_b, ref_c = x3_of(a, False), x3_of(b, False), x3_of(c, False)
    same(x3_of(a, True), ref_a)     # dense -> fused transition (full clear)
    same(x3_of(b, True), ref_b)     # sparse clear of a's voxels
    same(x3_of(c, True), ref_c)
    assert torch.equal(x3_of(a, False), ref_a)    # and back


@pytest.mark.parametrize("B,P,spread", [(2, 1000, 6.0), (3, 37, 2.0), (1, 5000, 9.0), (2, 4096, 30.0)])
def test_voxelize_s2d_sorted_and_search_paths_bit_exact(cuda_device, B, P, spread):
    """mf_cnn_voxelize_s2d (sort-based for P <= 4096, search-based above) against a sequential
    restatement of average_voxelization_3d (average_voxelization_3d.py:43-118: fp32 sums in
    ascending point order, IEEE divide) + bf16 rounding + the s2d layout; clustered points (most
    voxels shared), NaN and out-of-grid points, two consecutive calls (sparse re-zeroing)."""
    from morefusion_b200 import _lib
    L = _lib.lib()
    D, C, Ct = 32, 144, 160
    J = D // 2 + 1
    rs = np.random.RandomState(B * 1000 + P)
    X = torch.zeros(B, J, J, J, 8 * Ct, dtype=torch.bfloat16, device=cuda_device)
    prev = torch.full((2 * B * P,), -1, dtype=torch.int32, device=cuda_device)
    for call in range(2):
        pts = (15.5 + rs.randn(B, 3, P) * spread).astype(np.float32)
        pts[0, :, 3] = np.nan
        pts[-1, 0, 5] = 40.0
        feat = rs.rand(B * P, C).astype(np.float32)
        ft, pt = torch.as_tensor(feat, device=cuda_device), torch.as_tensor(pts, device=cuda_device)
        _lib.check(L.mf_cnn_voxelize_s2d(_lib.ptr(ft), _lib.ptr(pt), B, P, C, D, Ct, _lib.ptr(prev),
                                         _lib.ptr(X), _lib.stream()), "voxelize_s2d")
        torch.cuda.synchronize()
        want = np.zeros((B, J, J, J, 8, Ct), np.float32)
        for b in range(B):
            ijk = np.round(pts[b]).T                      # round-half-away == roundf for these values
            sums, cnt = {}, {}
            for p in range(P):
                v = ijk[p]
                if np.isnan(pts[b, :, p]).any() or (v < 0).any() or (v >= D).any():
                    continue
                k = tuple(int(t) for t in v)
                sums[k] = feat[b * P + p].copy() if k not in sums else (sums[k] + feat[b * P + p]).astype(np.float32)
                cnt[k] = cnt.get(k, 0) + 1
            for (x, y, z), sm in sums.items():
                px, py, pz = x + 1, y + 1, z + 1
                r = ((px & 1) << 2) | ((py & 1) << 1) | (pz & 1)
                want[b, px >> 1, py >> 1, pz >> 1, r, :C] = sm / np.float32(cnt[(x, y, z)])
        got = X.reshape(B, J, J, J, 8, Ct).float().cpu().numpy()
        ref = torch.as_tensor(want).to(torch.bfloat16).float().numpy()
        assert np.array_equal(got, ref), (call, np.abs(got - ref).max())
        keys = prev[:B * P].cpu().numpy()
        assert (keys[3] == -1) and (keys[(B - 1) * P + 5] == -1)


@pytest.mark.parametrize("as_bytes", [False, True])
def test_fused_occ_kernel_bit_identical_to_two_kernel_path(cuda_device, as_bytes):
    """conv1_occ + conv2_occ in one kernel (conv1 evaluated per consumer slab in shared memory)
    writes the same bits into the conv3 input as conv1 -> global bf16 -> conv2, for float and
    byte occupancy grids (boundary slabs x = 0, 1, 30, 31 included: B x 32 CTAs cover them all)."""
    from morefusion_b200.contrib.singleview_3d.models import Model
    B = 3
    w = ocnn.init_weights(21, seed=3)
    inp = make_inputs(B, seed=9)
    m = Model(n_fg_class=21, with_occupancy=True).to(cuda_device).load_reference_weights(w)
    gne = torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device)
    if as_bytes:
        gne = (gne > 0.5).to(torch.uint8)

    def x3_of(fused):
        m.fused_occ = fused
        m.forward_features(
            class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
            values=torch.as_tensor(inp["values"], device=cuda_device),
            points=torch.as_tensor(inp["points"], device=cuda_device),
            pitch=inp["pitch"], origin=inp["origin"], grid_nontarget_empty=gne)
        torch.cuda.synchronize()
        return m._wbufs[(B, 1000, cuda_device)]["x3"].clone()

    ref = x3_of(False)
    got = x3_of(True)
    assert float(ref.reshape(B, -1, 160)[..., 144:].float().abs().max()) > 0
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("B", [1, 3, 8])
def test_fused_heads_launch_bit_identical_to_three_launches(cuda_device, B):
    """Head layers 1-3 as one persistent launch with tile-level dependencies (mf_cnn_heads_tc):
    same tiles, same K order, same epilogue as the three grouped launches -> identical bits in
    hd1 / hd2 / hd3 and in the poses; repeated calls exercise the epoch counters."""
    from morefusion_b200.contrib.singleview_3d.models import Model
    w = ocnn.init_weights(21, seed=5)
    m = Model(n_fg_class=21, with_occupancy=True).to(cuda_device).load_reference_weights(w)

    def run(inp, fused):
        m.fused_heads = fused
        out = m.forward_features(
            class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
            values=torch.as_tensor(inp["values"], device=cuda_device),
            points=torch.as_tensor(inp["points"], device=cuda_device),
            pitch=inp["pitch"], origin=inp["origin"],
            grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device))
        torch.cuda.synchronize()
        buf = m._wbufs[(B, 1000, cuda_device)]
        return [o.clone() for o in out] + [buf[k].clone() for k in ("hd1", "hd2", "hd3")]

    for seed in (21, 22, 23):
        inp = make_inputs(B, seed=seed)
        ref = run(inp, False)
        got = run(inp, True)
        assert any(k[0] == "tc" for k in m.launch_log)
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
    ep = int(m._wbufs[(B, 1000, cuda_device)]["hd_sync"][0])
    assert ep == 3, ep            # one epoch per fused launch


def test_fused_head4_and_concurrent_branches_equal_sequential(cuda_device):
    """Last head layer fused with class selection + pose epilogue, and the two-stream branch
    overlap, give the same poses as the sequential grouped-GEMM + k_pose composition (fp32
    accumulation order differs between the tensor-core GEMM and the fused dot products)."""
    from morefusion_b200.contrib.singleview_3d.models import Model
    B = 3
    w = ocnn.init_weights(21, seed=4)
    inp = make_inputs(B, seed=11)
    m = Model(n_fg_class=21, with_occupancy=True).to(cuda_device).load_reference_weights(w)

    def run(fused, conc):
        m.fused_head4, m.concurrent_branches = fused, conc
        out = m.forward_features(
            class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
            values=torch.as_tensor(inp["values"], device=cuda_device),
            points=torch.as_tensor(inp["points"], device=cuda_device),
            pitch=inp["pitch"], origin=inp["origin"],
            grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device))
        torch.cuda.synchronize()
        return [o.clone() for o in out]

    base = run(False, False)
    conc = run(False, True)
    for a, b in zip(base, conc):                      # same kernels, only the schedule differs
        assert torch.equal(a, b)
    fused = run(True, True)
    # raw head outputs are O(1); fp32 summation-order differences only
    torch.testing.assert_close(fused[1], base[1], rtol=0, atol=1e-5)     # trans
    torch.testing.assert_close(fused[2], base[2], rtol=0, atol=1e-5)     # conf
    drot = (fused[0] - base[0]).abs()
    assert float(drot.max()) <= 1e-3 and float(drot.mean()) <= 1e-5, (drot.max(), drot.mean())


def test_runner_graph_equals_forward_features(cuda_device):
    """The serving entry (pinned host blob -> one H2D copy -> captured CUDA graphs -> one D2H
    copy) returns exactly what forward_features computes for the same batch, across batches, at
    B = 2 and at B = 8 (the batch bench.py times through this runner)."""
    from morefusion_b200.contrib.singleview_3d.models import Model
    w = ocnn.init_weights(21, seed=6)
    m = Model(n_fg_class=21, with_occupancy=True).to(cuda_device).load_reference_weights(w)
    for B in (2, 8):
        runner = m.make_runner(B, 1000, cuda_device, graph=True)
        for seed in (21, 22, 23):
            inp = make_inputs(B, seed=seed)
            runner.load_host(inp)
            runner.run()
            host = runner.download()
            torch.cuda.synchronize()
            got = [host[k].clone() for k in ("rot", "trans", "conf")]
            want = m.forward_features(
                class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
                values=torch.as_tensor(inp["values"], device=cuda_device),
                points=torch.as_tensor(inp["points"], device=cuda_device),
                pitch=inp["pitch"], origin=inp["origin"],
                grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device))
            torch.cuda.synchronize()
            for k, a, b in zip(("rot", "trans", "conf"), got, want):
                assert torch.equal(a, b.cpu()), (B, seed, k)
            # the end-to-end graph (both copies inside, `values` copied under the occupancy
            # branch): scribble over the device inputs and the host outputs first
            runner.in_blob.fill_(0x55)
            runner.host_out_blob.zero_()
            host = runner.run_e2e()
            torch.cuda.synchronize()
            for k, b in zip(("rot", "trans", "conf"), want):
                assert torch.equal(host[k], b.cpu()), (B, seed, k, "e2e")


@pytest.mark.parametrize("D,C,s2d", [(8, 512, 0), (8, 64, 0), (8, 48, 0), (16, 256, 0), (16, 256, 1)])
def test_interp_cl_equals_public_operator(cuda_device, D, C, s2d):
    """Internal channels-last bf16 gather (slab-staged for small grids, direct otherwise, s2d or
    row-major) == the public interpolate_voxel_grid on the same bf16-rounded grid, up to the
    final bf16 rounding of the output."""
    import morefusion_b200 as mf
    from morefusion_b200 import _lib
    B, P = 3, 1000
    torch.manual_seed(D + C + s2d)
    grid = torch.randn(B, C, D, D, D, device=cuda_device).to(torch.bfloat16)
    div = 32.0 / D
    pts = torch.rand(B, 3, P, device=cuda_device) * 36.0 - 2.0          # some outside the grid
    if s2d:
        J = D // 2 + 1
        xp = torch.nn.functional.pad(grid, (1, 1, 1, 1, 1, 1))
        G = xp.reshape(B, C, J, 2, J, 2, J, 2).permute(0, 2, 4, 6, 3, 5, 7, 1).reshape(
            B, J, J, J, 8 * C).contiguous()
    else:
        G = grid.permute(0, 2, 3, 4, 1).contiguous()
    feat = torch.zeros(B * P, C + 16, device=cuda_device, dtype=torch.bfloat16)
    L = _lib.lib()
    _lib.check(L.mf_cnn_interp_cl(_lib.ptr(G), s2d, _lib.ptr(pts), B, P, C, D, div, _lib.ptr(feat),
                                  C + 16, 8, _lib.stream()), "interp_cl")
    torch.cuda.synchronize()
    p_flat = (pts / div).permute(0, 2, 1).reshape(B * P, 3).contiguous()
    bi = torch.arange(B, device=cuda_device, dtype=torch.int32).repeat_interleave(P)
    want = mf.functions.interpolate_voxel_grid(grid.float(), p_flat, bi)
    got = feat[:, 8:8 + C].float()
    assert torch.all(feat[:, :8] == 0) and torch.all(feat[:, 8 + C:] == 0)
    torch.testing.assert_close(got, want, rtol=2 ** -7, atol=1e-6)


@pytest.mark.parametrize("B", [2, 8])
@pytest.mark.parametrize("with_occ", [True, False])
def test_cnn_precise_mode_meets_north_star_tolerance(cuda_device, with_occ, B):
    """Model.precision = "bf16x3" (every GEMM operand split hi + lo, three wgmma GEMMs per
    product, fp32 everywhere else): poses within 1e-4 abs of the reference's fp32 arithmetic
    (oracle/cnn.py, bf16=False) -- north_star's R/t tolerance -- on every one of the B*P
    per-point predictions, and the bf16 throughput mode bounded against the same oracle."""
    w = ocnn.init_weights(21, seed=1, with_occupancy=with_occ)
    inp = make_inputs(B)
    ref32 = ocnn.forward(w, n_fg_class=21, bf16=False, **inp)
    from morefusion_b200.contrib.singleview_3d.models import Model
    m = Model(n_fg_class=21, with_occupancy=with_occ).to(cuda_device).load_reference_weights(w)
    m.precision = "bf16x3"
    args = dict(class_id=torch.as_tensor(inp["class_id"], device=cuda_device),
                values=torch.as_tensor(inp["values"], device=cuda_device),
                points=torch.as_tensor(inp["points"], device=cuda_device),
                pitch=inp["pitch"], origin=inp["origin"],
                grid_nontarget_empty=torch.as_tensor(inp["grid_nontarget_empty"], device=cuda_device))
    rot, trans, conf = (x.cpu().numpy() for x in m.forward_features(**args))
    d_rot = np.abs(rot - ref32["rot"]).max()
    d_trans = np.abs(trans - ref32["trans"]).max()
    d_conf = np.abs(conf - ref32["conf"]).max()
    print(f"bf16x3 vs fp32 oracle: max|d rot|={d_rot:.3g} max|d trans|={d_trans:.3g} max|d conf|={d_conf:.3g}")
    # translation and confidence: 1e-4 at every one of the B*P points.  The quaternion is
    # o / (|o| + 1e-5): where the raw head output o is short, the normalisation amplifies ANY
    # fp32-level difference by 1/|o| (two fp32 implementations with different summation orders
    # differ by the same amount there), so the per-point bar is 1e-4 on >= 99.5 % of the points
    # and 3e-4 everywhere, and the pose the callers consume -- the argmax-confidence point of
    # every object (demo.py:85, evaluate.py:86) -- must meet 1e-4 on the rotation MATRIX and t.
    assert d_trans <= 1e-4 and d_conf <= 1e-4, (d_trans, d_conf)
    dq = np.abs(rot - ref32["rot"]).max(axis=2)
    assert np.mean(dq <= 1e-4) >= 0.995 and d_rot <= 3e-4, (np.mean(dq <= 1e-4), d_rot)
    from oracle import transforms as otf
    k = ref32["conf"].argmax(1)
    assert np.array_equal(conf.argmax(1), k)
    ar = np.arange(B)
    R = otf.quaternion_matrix_fwd(rot[ar, k])[0][:, :3, :3]
    R32 = otf.quaternion_matrix_fwd(ref32["rot"][ar, k])[0][:, :3, :3]
    assert np.abs(R - R32).max() <= 1e-4 and np.abs(trans[ar, k] - ref32["trans"][ar, k]).max() <= 1e-4
    # throughput mode: a max-error bound (not only a mean) against the same fp32 oracle
    m.precision = "bf16"
    rot, trans, conf = (x.cpu().numpy() for x in m.forward_features(**args))
    b_rot, b_trans, b_conf = (np.abs(rot - ref32["rot"]).max(), np.abs(trans - ref32["trans"]).max(),
                              np.abs(conf - ref32["conf"]).max())
    print(f"bf16   vs fp32 oracle: max|d rot|={b_rot:.3g} max|d trans|={b_trans:.3g} max|d conf|={b_conf:.3g}")
    assert b_rot <= 0.15 and b_trans <= 5e-3 and b_conf <= 5e-2, (b_rot, b_trans, b_conf)
