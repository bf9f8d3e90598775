"""The VERTEX_REG_3D training target restated in numpy float32 (lib/gt_synthesize_layer/minibatch.py:595-600, _scale_vertmap
:605-616), with `centers` as the presence table of the device entry points: a pixel labelled c in 1..C-1 is weighted iff
centers[b, c, 2] > 0; and torch fp32 autograd of the object-coordinate training graph (no pose head) on those targets."""
import numpy as np
import torch
import torch.nn.functional as F

from tests import ref_network as R
from tests.train_ref import MEANS, _ste


def scale_coeffs(extents):
    """(a, b) [C,3] float32: vmin = -e / 2, vmax = e / 2, a = 1 / (vmax - vmin), b = -1 * vmin / (vmax - vmin); 0 where vmax <= vmin."""
    e = np.asarray(extents, np.float32)
    vmin, vmax = -e / np.float32(2), e / np.float32(2)
    span = vmax - vmin
    ok = span > 0
    safe = np.where(ok, span, np.float32(1))
    a = np.where(ok, np.float32(1) / safe, np.float32(0)).astype(np.float32)
    b = np.where(ok, (np.float32(-1) * vmin) / safe, np.float32(0)).astype(np.float32)
    return a, b


def vertex_targets_3d(label, vertmap, centers, extents, w_inside):
    """(targets, weights) [B,H,W,3C] float32; the target is a * v rounded, then + b rounded (two float32 operations)."""
    label = np.asarray(label)
    vertmap = np.asarray(vertmap, np.float32)
    B, H, W = label.shape
    C = centers.shape[1]
    a, b = scale_coeffs(extents)
    t = np.zeros((B, H, W, 3 * C), np.float32)
    w = np.zeros((B, H, W, 3 * C), np.float32)
    for n in range(B):
        for c in range(1, C):
            m = label[n] == c
            if not m.any() or not centers[n, c, 2] > 0:
                continue
            t[n][m, 3 * c:3 * c + 3] = (vertmap[n][m] * a[c]).astype(np.float32) + b[c]
            w[n][m, 3 * c:3 * c + 3] = np.float32(w_inside)
    return t, w


def presence_table(cls_indexes, num_classes):
    """centers [B,C,3] with z = 1 for the classes listed in each frame (the only column the 3-D target reads)."""
    cen = np.zeros((len(cls_indexes), num_classes, 3), np.float32)
    for n, listed in enumerate(cls_indexes):
        for c in np.asarray(listed).astype(int).flatten():
            cen[n, c] = (0.0, 0.0, 1.0)
    return cen


def coord_reference_grads(net, inputs, vertex_targets, sim16, vertex_w=1.0):
    """torch fp32 autograd of loss_cls + vertex_w * loss_vertex of an object-coordinate network (COLOR, no pose head: the reference
    builds Hough voting, RoiPool and fc6-fc8 under vertex_reg_2d, vgg16_convs.py:165-200) on the inputs tuple of Trainer.step and
    the materialised 3-D targets (targets, weights) [B,H,W,3C] numpy float32.  Returns the parameters (with .grad) and a dict of the
    losses and outputs.  sim16 as in tests/train_ref.reference_grads: False = the reference's op order in pure fp32, True = this
    implementation's op order (1x1 before the x8 up-sampling) with every stored activation and tensor-core weight rounded to bf16."""
    data, gt = inputs[0], inputs[1]
    P = {k: v.detach().clone().requires_grad_(True) for k, v in net.params.items()}
    C = net.num_classes
    r16 = (lambda y: _ste(y, torch.bfloat16)) if sim16 else (lambda y: y)
    x = r16((data.float() - torch.tensor(MEANS, device=data.device)).permute(0, 3, 1, 2))
    feats = {}
    for item in R.VGG_CFG:
        if isinstance(item, str):
            x = F.max_pool2d(x, 2)
        else:
            x = r16(R.conv(x, r16(P[f"{item[0]}/weights"]), P[f"{item[0]}/biases"]))
            feats[item[0]] = x
    c4, c5 = feats["conv4_3"], feats["conv5_3"]
    s5 = r16(R.conv(c5, r16(P["score_conv5/weights"]), P["score_conv5/biases"]))
    s4 = r16(R.conv(c4, r16(P["score_conv4/weights"]), P["score_conv4/biases"]))
    v5 = r16(R.conv(c5, r16(P["score_conv5_vertex/weights"]), P["score_conv5_vertex/biases"], False))
    v4 = r16(R.conv(c4, r16(P["score_conv4_vertex/weights"]), P["score_conv4_vertex/biases"], False))
    if sim16:
        add_s, add_v = r16(s4 + R.deconv(s5, 4, 2)), r16(v4 + R.deconv(v5, 4, 2))
        zs, zv = torch.zeros(C, device=data.device), torch.zeros(3 * C, device=data.device)
        lr_s = r16(R.conv(add_s, r16(P["score/weights"]), zs, False))
        lr_v = r16(R.conv(add_v, r16(P["vertex_pred/weights"]), zv, False))
        score = torch.relu(R.deconv(lr_s, 16, 8) + P["score/biases"][None, :, None, None])
        vertex = R.deconv(lr_v, 16, 8) + P["vertex_pred/biases"][None, :, None, None]
        prob = F.softmax(score, 1)
    else:
        score, _, prob, vertex = R.heads_from_scores(P, s4, s5, v4, v5)
    g = gt.long()
    pg = prob.detach().gather(1, g.clamp(min=0)[:, None])[:, 0]
    sel = (g >= 0) & ((g > 0) | (pg < net.threshold_label))
    logp = F.log_softmax(score, 1).gather(1, g.clamp(min=0)[:, None])[:, 0]
    loss_cls = -(logp * sel).sum() / (sel.sum() + 1e-10)
    vt, vw = (torch.from_numpy(a).to(data.device).permute(0, 3, 1, 2) for a in vertex_targets)
    diff = vw * (vertex - vt)
    sl1 = torch.where(diff.abs() < 1, 0.5 * diff * diff, diff.abs() - 0.5)
    loss_vertex = sl1.sum() / (vw.sum() + 1e-10)
    (loss_cls + vertex_w * loss_vertex).backward()
    return P, dict(loss_cls=loss_cls.item(), loss_vertex=(vertex_w * loss_vertex).item(), score=score.detach(), vertex=vertex.detach())
