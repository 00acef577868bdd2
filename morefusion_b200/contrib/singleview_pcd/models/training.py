"""Training of the singleview_pcd model on the sm_90a kernels: chainer's reverse pass through
examples/ycb_video/singleview_pcd/contrib/models/model.py:115-153 (heads, pose) and :315-330
(PoseNetExtractor) as one CUDA launch sequence behind a torch.autograd.Function.

Backward, in launch order (bf16 gradients where they feed a GEMM, fp32 parameter gradients):
  * layer 4 + pose: mf_train_head4_bwd (pitch 1: d offset = d trans);
  * layers 3, 2 of each head: dW (mf_train_gemm_tn), db (mf_train_colsum), dX on the forward GEMM
    with transposed weights, ReLU mask;
  * layer 1: dW1a = dZ1^T [feat1|feat2]; s_b = column sums of dZ1 over each object's rows
    (mf_posenet_obj_colsum, one launch);
    dW1b = sum_b s_b pooled_b, db1 = sum_b s_b, dpooled_b = W1b^T s_b (mf_posenet_obj_bias_bwd);
    d[feat1|feat2] = dZ1 W1a;
  * the mean: dZ4 = relu'(h4) dpooled_b / P (mf_posenet_pool_bwd); conv4 and conv3 as the heads;
    d feat2 adds the heads' path and conv3's path;
  * conv1_* / conv2_*: mf_posenet_point_mlp_bwd, to the four weights and to ``values``.

Data-parallel training uses the Trainer shared with singleview_3d (contrib/_training.py): it makes
the parameters and their gradients views into flat buffers, ``backward_pcd`` writes the gradients
straight into those views and announces the buckets of ``train_layout`` as it finishes them, and
the 2-D extractor's gradients (torch autograd) form the last bucket.
"""

import torch

from .... import _lib
from ... import _training
from ..._pose_model import OUT_F32
from .model import FEAT12, HEADS

_PE = "posenet_extractor."


def param_order(model):
    """Names of the parameters the CUDA backward produces gradients for."""
    names = []
    for layer in (4, 3, 2, 1):
        for h in HEADS:
            names += [f"conv{layer}_{h}.weight", f"conv{layer}_{h}.bias"]
    for n in ("conv4", "conv3", "conv2_rgb", "conv2_pcd", "conv1_rgb", "conv1_pcd"):
        names += [_PE + n + ".weight", _PE + n + ".bias"]
    return names


def train_layout(model):
    """What the shared Trainer needs from this model: ``param_order`` (the order in which
    backward_pcd finishes the gradients) and the buckets backward_pcd announces through
    ``_on_bucket``: the four layers of the heads, PoseNet's conv4 and conv3, the point MLP."""
    order = param_order(model)
    return order, [("heads", order[0], "conv1_conf.bias"),
                   ("conv4+conv3", _PE + "conv4.weight", _PE + "conv3.bias"),
                   ("point_mlp", _PE + "conv2_rgb.weight", order[-1])]


Trainer = _training.Trainer


def _train_pack(model):
    """Transposed bf16 weights of the dX GEMMs and [out][in] fp32 point-MLP weights."""
    def build():
        bf = torch.bfloat16
        t = lambda W: W.detach()[:, :, 0].t().to(bf).contiguous()       # noqa: E731
        pe = model.posenet_extractor
        p = {}
        p["head1/Wt"] = torch.cat([getattr(model, f"conv1_{h}").weight.detach()[:, :FEAT12, 0] for h in HEADS],
                                  0).t().to(bf).contiguous()                              # [384, 1920]
        for h in HEADS:
            for layer in (2, 3):
                p[f"conv{layer}_{h}/Wt"] = t(getattr(model, f"conv{layer}_{h}").weight)
        p["conv4/Wt"] = t(pe.conv4.weight)                                              # [512, 1024]
        p["conv3/Wt"] = t(pe.conv3.weight)                                              # [256, 512]
        for n in ("conv1_rgb", "conv1_pcd", "conv2_rgb", "conv2_pcd"):
            m = getattr(pe, n)
            p[n + "/W"] = m.weight.detach()[:, :, 0].float().contiguous()
            p[n + "/b"] = m.bias.detach().float().contiguous()
        return p
    return model._derived("train", model._section_params(), build)


def _train_buffers(model, B, P, dev):
    key = ("train", B, P, dev)
    if key not in model._wbufs:
        bf, f32 = torch.bfloat16, torch.float32
        z = lambda *s, dt=bf: torch.zeros(*s, dtype=dt, device=dev)     # noqa: E731
        NP = B * P
        model._wbufs[key] = dict(
            raw8=z(NP, 8, dt=f32), h4=z(NP, 1024), dhd3=z(NP, 384), dhd2=z(NP, 768), dhd1=z(NP, 1920),
            gw1=z(1920, 1408, dt=f32), gb1=z(1920, dt=f32), seg=z(B, 1920, dt=f32),
            dpooled=z(B, 1024, dt=f32), dz4=z(NP, 1024), dh3=z(NP, 512), dfeat=z(NP, FEAT12, dt=f32),
            dfeat2=z(NP, 256, dt=f32))
    return model._wbufs[key]


class _PoseNetPcd(torch.autograd.Function):
    """values -> (rot, trans, conf) through the CUDA forward; backward = the launch sequence above.
    The activations live in the model's work buffers: run backward before the next forward of
    the same batch shape."""

    @staticmethod
    def forward(ctx, model, class_id, pcd, center, values, *params):
        B, _, P = values.shape
        tb = _train_buffers(model, B, P, values.device)
        values = values.detach().contiguous().float()
        rot, trans, conf = model._forward(class_id=class_id, values=values, pcd=pcd, center=center, tb=tb)
        ctx.model, ctx.values, ctx.class_id = model, values, class_id
        ctx.needs_values = ctx.needs_input_grad[4]
        return rot, trans, conf

    @staticmethod
    def backward(ctx, g_rot, g_trans, g_conf):
        model = ctx.model
        grads = backward_pcd(model, ctx.values, ctx.class_id, g_rot.contiguous().float(),
                             g_trans.contiguous().float(), g_conf.contiguous().float(), ctx.needs_values)
        dvalues = grads.pop("values", None)
        names = param_order(model)
        if getattr(model, "_train_grad_views", None) is not None:
            # Trainer mode: the gradients are already in the flat buffer that the parameters'
            # .grad views alias -- returning them would make autograd add them again
            return (None, None, None, None, dvalues) + (None,) * len(names)
        return (None, None, None, None, dvalues) + tuple(grads[n] for n in names)


def forward_features_with_grad(model, *, class_id, values, pcd, center=None):
    named = dict(model.named_parameters())
    return _PoseNetPcd.apply(model, class_id, pcd, center, values, *[named[n] for n in param_order(model)])


def _out_grads(model):
    """fp32 gradient destinations: the Trainer's views into the flat gradient buffer (zeroed by
    the Trainer) if there is one, else fresh zero tensors."""
    tg = getattr(model, "_train_grad_views", None)
    if tg is not None:
        return dict(tg)
    named = dict(model.named_parameters())
    return {n: torch.zeros_like(named[n], dtype=torch.float32) for n in param_order(model)}


def backward_pcd(model, values, class_id, g_rot, g_trans, g_conf, needs_values=False, on_bucket=None):
    """The backward launch sequence.  Returns {parameter name: fp32 gradient} (+ 'values').
    ``on_bucket`` (default ``model._on_bucket``, set by a Trainer) is called with each bucket's
    name of ``train_layout`` once the bucket's last gradient is enqueued."""
    L, s, ptr, chk = _lib.lib(), _lib.stream, _lib.ptr, _lib.check
    B, _, P = values.shape
    dev = values.device
    NP, nfg = B * P, model._n_fg_class
    w = model._pack()
    tw = _train_pack(model)
    buf = model._work_buffers(B, P, dev)
    tb = _train_buffers(model, B, P, dev)
    G = _out_grads(model)
    on_bucket = on_bucket or getattr(model, "_on_bucket", None)
    cid = torch.as_tensor(class_id, device=dev).to(torch.int32).contiguous()
    with torch.cuda.device(dev):
        for k in ("gw1", "gb1", "seg"):
            tb[k].zero_()
        # ---- layer 4 of the heads + pose epilogue
        chk(L.mf_train_head4_bwd(
            ptr(g_rot), ptr(g_trans), ptr(g_conf), ptr(tb["raw8"]), ptr(buf["hd3"]), 384,
            ptr(w["conv4_rot/W"]), ptr(w["conv4_trans/W"]), ptr(w["conv4_conf/W"]), ptr(cid),
            ptr(buf["pitch"]), B, P, nfg, ptr(tb["dhd3"]),
            ptr(G["conv4_rot.weight"]), ptr(G["conv4_rot.bias"]), ptr(G["conv4_trans.weight"]),
            ptr(G["conv4_trans.bias"]), ptr(G["conv4_conf.weight"]), ptr(G["conv4_conf.bias"]), s()),
            "head4_bwd")
        # ---- layers 3, 2 of each head
        for layer, dz, x, n_out, k_in, dx in ((3, tb["dhd3"], buf["hd2"], 128, 256, tb["dhd2"]),
                                              (2, tb["dhd2"], buf["hd1"], 256, 640, tb["dhd1"])):
            for i, h in enumerate(HEADS):
                chk(L.mf_train_gemm_tn(ptr(dz[:, i * n_out:]), dz.shape[1], ptr(x[:, i * k_in:]), x.shape[1],
                                       NP, n_out, k_in, ptr(G[f"conv{layer}_{h}.weight"]), k_in, 1, 0, 0, 0,
                                       1, s()), "gemm_tn")
                chk(L.mf_train_colsum(ptr(dz[:, i * n_out:]), dz.shape[1], NP, n_out,
                                      ptr(G[f"conv{layer}_{h}.bias"]), s()), "colsum")
                model._gemm(L, dz[:, i * n_out:], tw[f"conv{layer}_{h}/Wt"], None, dx, NP, k_in, n_out,
                            lda=dz.shape[1], relu=0, ldo=dx.shape[1], col_off=i * k_in)
            chk(L.mf_train_relu_mask(ptr(dx), dx.shape[1], ptr(x), x.shape[1], NP, dx.shape[1], s()),
                "relu_mask")
        # ---- layer 1: [feat1|feat2] columns per point, feat3 columns per object
        dz1 = tb["dhd1"]
        chk(L.mf_train_gemm_tn(ptr(dz1), 1920, ptr(buf["feat12"]), FEAT12, NP, 1920, FEAT12, ptr(tb["gw1"]),
                               1408, 1, 0, 0, 0, 1, s()), "gemm_tn")
        chk(L.mf_posenet_obj_colsum(ptr(dz1), 1920, B, P, 1920, ptr(tb["seg"]), s()), "obj_colsum")
        chk(L.mf_posenet_obj_bias_bwd(ptr(tb["seg"]), ptr(buf["pooled"]), ptr(w["head1/W"][:, FEAT12:]), 1408,
                                      1920, 1024, B, ptr(tb["gw1"][:, FEAT12:]), 1408, ptr(tb["gb1"]),
                                      ptr(tb["dpooled"]), s()), "obj_bias_bwd")
        model._gemm(L, dz1, tw["head1/Wt"], None, tb["dfeat"], NP, FEAT12, 1920, lda=1920, relu=0,
                    out_mode=OUT_F32, ldo=FEAT12)
        # added like every other gradient: under a Trainer the destinations are .grad views that a
        # second backward before zero_grad() accumulates into (gw1 / gb1 are zeroed above)
        for i, h in enumerate(HEADS):
            G[f"conv1_{h}.weight"].view(640, 1408).add_(tb["gw1"][i * 640:(i + 1) * 640])
            G[f"conv1_{h}.bias"].add_(tb["gb1"][i * 640:(i + 1) * 640])
        if on_bucket:
            on_bucket("heads")
        # ---- the mean over the points, conv4, conv3
        chk(L.mf_posenet_pool_bwd(ptr(tb["dpooled"]), ptr(tb["h4"]), B, P, 1024, ptr(tb["dz4"]), s()),
            "pool_bwd")
        for n, dz, x, ldx, n_out, k_in, dx, act, out_mode in (
                ("conv4", tb["dz4"], buf["h3"], 512, 1024, 512, tb["dh3"], buf["h3"], None),
                ("conv3", tb["dh3"], buf["feat12"][:, 128:], FEAT12, 512, 256, tb["dfeat2"], None, OUT_F32)):
            chk(L.mf_train_gemm_tn(ptr(dz), n_out, ptr(x), ldx, NP, n_out, k_in, ptr(G[_PE + n + ".weight"]),
                                   k_in, 1, 0, 0, 0, 1, s()), "gemm_tn")
            chk(L.mf_train_colsum(ptr(dz), n_out, NP, n_out, ptr(G[_PE + n + ".bias"]), s()), "colsum")
            model._gemm(L, dz, tw[n + "/Wt"], None, dx, NP, k_in, n_out, lda=n_out, relu=0, ldo=k_in,
                        **({} if out_mode is None else dict(out_mode=out_mode)))
            if act is not None:
                chk(L.mf_train_relu_mask(ptr(dx), k_in, ptr(act), k_in, NP, k_in, s()), "relu_mask")
        if on_bucket:
            on_bucket("conv4+conv3")
        # ---- conv1_* / conv2_*
        dvalues = torch.empty_like(values) if needs_values else None
        pg = lambda n, k: ptr(G[_PE + n + "." + k])       # noqa: E731
        chk(L.mf_posenet_point_mlp_bwd(
            ptr(values), ptr(buf["pcd_c"]), ptr(tw["conv1_rgb/W"]), ptr(tw["conv1_rgb/b"]),
            ptr(tw["conv1_pcd/W"]), ptr(tw["conv1_pcd/b"]), ptr(tw["conv2_rgb/W"]), ptr(tw["conv2_rgb/b"]),
            ptr(tw["conv2_pcd/W"]), ptr(tw["conv2_pcd/b"]), B, P, ptr(tb["dfeat"]), ptr(tb["dfeat2"]),
            pg("conv1_rgb", "weight"), pg("conv1_rgb", "bias"), pg("conv1_pcd", "weight"), pg("conv1_pcd", "bias"),
            pg("conv2_rgb", "weight"), pg("conv2_rgb", "bias"), pg("conv2_pcd", "weight"), pg("conv2_pcd", "bias"),
            ptr(dvalues), s()), "posenet_point_mlp_bwd")
        if on_bucket:
            on_bucket("point_mlp")
    if needs_values:
        G["values"] = dvalues
    return G
