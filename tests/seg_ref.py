"""Shared harness of the segmentation-network tests: the network with O(1) logits, and torch fp32 autograd of its training graph
(lib/networks/vgg16_convs.py:79-149, loss = loss_cross_entropy_single_frame on the Hardlabel selection, lib/fcn/train.py:455-465,
518-521) restated on oracle/ref_network.py, in the reference's op order or in this implementation's with its 16-bit roundings."""
import torch
import torch.nn.functional as F

from tests import ref_network as R
from tests.train_ref import MEANS, _ste


def make_seg_net(cuda, fmt="COLOR", C=10, is_train=True, seed=0, score_scale=0.02):
    """A seeded segmentation network (vertex_reg_2d = vertex_reg_3d = False); `score` scaled by score_scale (O(1) logits)."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    net = vgg16_convs(input_format=fmt, num_classes=C, device=cuda, is_train=is_train, vertex_reg_2d=False,
                      vertex_reg_3d=False).init_random(seed=seed, bias_std=0.02)
    net.params["score/weights"] *= score_scale
    net.prepare()
    return net


def seg_reference_grads(net, data, gt, sim16, depth_blob=None):
    """torch autograd of loss_cls on the segmentation graph.  sim16=False: the reference's op order (up-sampling before `score`),
    pure fp32.  sim16=True: this implementation's op order (`score` at 1/8 resolution, then the x8 up-sampling) with every stored
    activation and weight rounded to bf16 where the kernels round it.  depth_blob [B,H,W,3]: the RGB-D graph.  Returns the
    parameters (with .grad) and loss_cls."""
    P = {k: v.detach().clone().requires_grad_(True) for k, v in net.params.items()}
    C = net.num_classes
    r16 = (lambda y: _ste(y, torch.bfloat16)) if sim16 else (lambda y: y)
    W = r16

    def trunk(x, sfx):
        x = r16(x)
        feats = {}
        for item in R.VGG_CFG:
            if isinstance(item, str):
                x = F.max_pool2d(x, 2)
            else:
                x = r16(R.conv(x, W(P[f"{item[0]}{sfx}/weights"]), P[f"{item[0]}{sfx}/biases"]))
                feats[item[0]] = x
        return feats
    f = trunk((data.float() - torch.tensor(MEANS, device=data.device)).permute(0, 3, 1, 2), "")
    h4, h5 = f["conv4_3"], f["conv5_3"]
    if depth_blob is not None:
        fp = trunk(depth_blob.permute(0, 3, 1, 2), "_p")
        h4, h5 = torch.cat([h4, fp["conv4_3"]], 1), torch.cat([h5, fp["conv5_3"]], 1)     # concat_conv4 / 5, colour first
    s5 = r16(R.conv(h5, W(P["score_conv5/weights"]), P["score_conv5/biases"]))
    s4 = r16(R.conv(h4, W(P["score_conv4/weights"]), P["score_conv4/biases"]))
    if sim16:
        add = r16(s4 + R.deconv(s5, 4, 2))
        lr = r16(R.conv(add, W(P["score/weights"]), torch.zeros(C, device=data.device), False))
        score = torch.relu(R.deconv(lr, 16, 8) + P["score/biases"][None, :, None, None])
    else:
        up = R.deconv(s4 + R.deconv(s5, 4, 2), 16, 8)
        score = R.conv(up, P["score/weights"], P["score/biases"])
    prob = F.softmax(score, 1)
    g = gt.long()
    pg = prob.detach().gather(1, g.clamp(min=0)[:, None])[:, 0]
    sel = (g >= 0) & ((g > 0) | (pg < net.threshold_label))
    logp = F.log_softmax(score, 1).gather(1, g.clamp(min=0)[:, None])[:, 0]
    loss_cls = -(logp * sel).sum() / (sel.sum() + 1e-10)
    loss_cls.backward()
    return P, loss_cls.item()
