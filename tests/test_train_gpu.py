"""GPU: the training step of the 3-D section (forward + CUDA backward, csrc/train.cu +
csrc/gemm_train.cu) against the differentiable fp32 oracle oracle/cnn_train.py: loss and every
parameter gradient (model.py:93-141, :239-273 backward; loss :377-441), at B=2 and B=8.

Bars (bf16 operands / bf16 stored activations and activation gradients, fp32 accumulation, vs an
all-fp32 oracle): loss within 2 %; per parameter tensor, relative L2 error of the gradient
<= 6 % and cosine similarity >= 0.998 (DESIGN.md section 3 states the same bars).  The tight,
per-kernel checks of the backward are in test_train_backward_gpu.py."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
F32 = np.float32


def _setup(B, dev, seed=0):
    from morefusion_b200 import synthetic
    from morefusion_b200.contrib.singleview_3d.models import Model
    w = synthetic.init_weights(21, seed=1)
    model = Model(n_fg_class=21, with_occupancy=True).to(dev).load_reference_weights(w)
    batch = synthetic.make_cnn_batch(B, 1000, seed=seed)
    rs = np.random.RandomState(seed + 7)
    q_true = rs.normal(size=(B, 4)).astype(F32)
    q_true /= np.linalg.norm(q_true, axis=1, keepdims=True)
    # true translation near the object's points (camera frame)
    cam = batch["points"] * batch["pitch"][:, None, None] + batch["origin"][:, :, None]
    t_true = cam.mean(axis=2).astype(F32)
    models = synthetic.SyntheticYCBModels()
    cad = [models.get_pcd(int(c))[rs.permutation(2000)[:500]] for c in batch["class_id"]]
    sym = [bool(int(c) in models.class_ids_symmetric) for c in batch["class_id"]]
    return w, model, batch, q_true, t_true, cad, sym


def _loss(F, rot, trans, conf, q_true, t_true, cad, sym, lam=0.015):
    """Model.loss (model.py:377-441) with the CAD samples fixed (the reference draws them with
    np.random.permutation inside the loss)."""
    dev = rot.device
    B = rot.shape[0]
    loss = 0
    for i in range(B):
        T_pred = F.transformation_matrix(rot[i], trans[i])
        T_true = F.transformation_matrix(torch.as_tensor(q_true[i], device=dev),
                                         torch.as_tensor(t_true[i], device=dev))
        add = F.average_distance(torch.as_tensor(cad[i], device=dev), T_true, T_pred, symmetric=sym[i])
        c = conf[i]
        keep = c.detach() > 0
        loss = loss + torch.mean(add[keep] * c[keep] - lam * torch.log(c[keep]))
    return loss / B


@pytest.mark.parametrize("B", [2, 8])
def test_training_step_gradients_vs_oracle(cuda_device, B):
    import morefusion_b200 as mf
    from morefusion_b200.contrib.singleview_3d.models import training
    from oracle import cnn_train as ct
    w, model, batch, q_true, t_true, cad, sym = _setup(B, cuda_device)
    want_loss, want, _ = ct.loss_and_grads(w, batch, quaternion_true=q_true, translation_true=t_true,
                                           cad_points=cad, symmetric=sym)
    dev = cuda_device
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)   # noqa: E731
    model.train()
    values = t(batch["values"]).requires_grad_(True)
    rot, trans, conf = training.forward_features_with_grad(
        model, class_id=batch["class_id"], values=values, points=t(batch["points"]),
        pitch=t(batch["pitch"]), origin=t(batch["origin"]),
        grid_nontarget_empty=t(batch["grid_nontarget_empty"]))
    loss = _loss(mf.functions, rot, trans, conf, q_true, t_true, cad, sym)
    loss.backward()
    assert abs(float(loss) - want_loss) <= 2e-2 * abs(want_loss) + 1e-4, (float(loss), want_loss)
    named = dict(model.named_parameters())
    worst = {}
    for name in training.flat_param_order(model):
        key = name.replace(".weight", "/W").replace(".bias", "/b")
        g = named[name].grad.detach().float().cpu().numpy().reshape(-1)
        r = want[key].reshape(-1)
        nr = np.linalg.norm(r)
        rel = np.linalg.norm(g - r) / max(nr, 1e-12)
        cos = float(g @ r / max(np.linalg.norm(g) * nr, 1e-20))
        worst[name] = (rel, cos)
    bad = {k: v for k, v in worst.items() if not (v[0] <= 6e-2 and v[1] >= 0.998)}
    print("worst rel", max(v[0] for v in worst.values()), "min cos", min(v[1] for v in worst.values()))
    assert not bad, bad
    assert values.grad is not None and torch.isfinite(values.grad).all()


def test_trainer_single_gpu_step_decreases_loss(cuda_device):
    """Trainer (flat buffers, fused Adam) on one rank: a few steps on a fixed batch reduce the
    loss and keep parameters / gradients finite; parameters are views into the flat buffer."""
    from morefusion_b200.contrib.singleview_3d.models import training
    w, model, batch, q_true, t_true, cad, sym = _setup(2, cuda_device, seed=3)
    model.train()
    tr = training.Trainer(model, alpha=1e-4)
    dev = cuda_device
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=dev)   # noqa: E731
    # feed the 3-D section directly (no images): patch predict to use the synthetic features
    def predict(**kw):
        return training.forward_features_with_grad(
            model, class_id=batch["class_id"], values=t(batch["values"]), points=t(batch["points"]),
            pitch=t(batch["pitch"]), origin=t(batch["origin"]),
            grid_nontarget_empty=t(batch["grid_nontarget_empty"]))
    model.predict = predict
    losses = []
    for _ in range(6):
        np.random.seed(0)
        loss = tr.step(class_id=batch["class_id"], rgb=None, pcd=None, quaternion_true=q_true,
                       translation_true=t_true)
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert torch.isfinite(tr.flat_p).all() and torch.isfinite(tr.flat_g).all()
    assert model.conv3.weight.data_ptr() == tr.flat_p[tr.offs["conv3.weight"][0]:].data_ptr()
