"""One SGD training step (posecnn_b200/train.py, BASELINE configs[4]) against torch fp32 autograd of the reference graph
(tests/train_ref.py reference_grads) and tf.train.MomentumOptimizer + l2 regularisation (train.py:481, 633).
Stated tolerance: the forward runs on BF16 / FP16 tensor-core operands and the backward propagates 16-bit gradients, so parameter
gradients are compared by relative L2 norm per tensor (limits in tests/train_ref.py limits(), every value printed)."""
import pytest
import torch

from tests.train_ref import compare_grads, make_inputs, make_net, reference_grads, rel_l2, synthetic_pose_targets

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def test_training_step_matches_fp32_autograd(cuda):
    from posecnn_b200.train import Trainer
    net = make_net(cuda)
    args, _, _ = make_inputs(cuda)
    data, gt, centers, meta, ext, gtp, pts, sym = args
    lr, mu, wd, vw_, wi, margin = 0.01, 0.9, 1e-4, 1.0, 10.0, 0.01
    tr = Trainer(net, lr=lr, momentum=mu, weight_decay=wd, vertex_w=vw_, vertex_w_inside=wi, margin=margin)
    A = tr.forward(data, gt, centers, meta, ext, gtp, pts, sym)
    assert A["rows"] >= 9
    tw, wt = synthetic_pose_targets(A, pts, sym, margin)
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    P, ref = reference_grads(net, A, args, tw, wt, True, vw_, wi, margin)
    Pf, reff = reference_grads(net, A, args, tw, wt, False, vw_, wi, margin)
    # forward parity of the training graph: tight against the 16-bit-rounded restatement, stated bf16 tolerance against pure fp32
    assert rel_l2(A["score"].permute(0, 3, 1, 2), ref["score"]) < 5e-3
    assert rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), ref["vertex"]) < 5e-3
    assert rel_l2(A["score"].permute(0, 3, 1, 2), reff["score"]) < 3e-2
    assert rel_l2(tr.dense_vertex_pred(A).permute(0, 3, 1, 2), reff["vertex"]) < 3e-2
    for r_ in (ref, reff):
        assert abs(A["cls_out"][0].item() - r_["loss_cls"]) < 3e-2 * max(1.0, abs(r_["loss_cls"]))
        assert abs(vw_ * A["vtx_out"][0].item() - r_["loss_vertex"]) < 3e-2 * max(1.0, abs(r_["loss_vertex"]))
        assert abs(A["loss_pose"].item() - r_["loss_pose"]) < 3e-2 * max(1e-3, abs(r_["loss_pose"]))
    assert set(grads) == set(tr.master)
    compare_grads(tr, grads, P, Pf, list(grads))
    # the update: accum = grad + wd * w (first step), w -= lr * accum; tensor-core copies refreshed
    before = {k: v.clone() for k, v in tr.master.items()}
    tr.update(grads)
    for name in ("conv3_2/w", "fc7/w", "score/b", "conv1_1/w"):
        want = before[name] - lr * (grads[name] + wd * before[name])
        assert torch.allclose(tr.master[name], want, rtol=1e-5, atol=1e-7), name
    assert torch.equal(tr.tc["conv3_2/w"], tr.master["conv3_2/w"].to(torch.bfloat16))
    assert torch.equal(tr.tc["fc7/w"], tr.master["fc7/w"].to(torch.float16))
    assert torch.equal(tr.fc_t["fc7"], tr.tc["fc7/w"].t().contiguous())
    # a second full step runs (momentum path) and the loss is finite; exported params feed the inference network
    out = tr.step(data, gt, centers, meta, ext, gtp, pts, sym)
    assert torch.isfinite(out["loss"]).all()
    tr.export_params()
    assert torch.allclose(net.params["conv3_2/weights"].permute(3, 0, 1, 2).reshape(256, -1), tr.master["conv3_2/w"])
