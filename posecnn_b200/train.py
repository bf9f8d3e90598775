"""One SGD training step of the vgg16_convs network (BASELINE configs[4]) on the H100-native kernels.

Reference: the training graph lib/networks/vgg16_convs.py:79-212 driven by lib/fcn/train.py:206-260 —
    loss = loss_cls + VERTEX_W * loss_vertex + loss_pose + l2 regularisation (train.py:486-500),
    loss_cls    = Hardlabel-selected cross entropy of log_softmax(score)                 (train.py:455-465, hard_label_op_gpu.cu.cc:16-29)
    loss_vertex = smooth_l1_loss_vertex(vertex_pred, vertex_targets, vertex_weights)     (train.py:564-573)
    loss_pose   = Averagedistance(l2_normalize(poses_tanh * poses_weight), poses_target, poses_weight, points, symmetry)
    optimizer   = tf.train.MomentumOptimizer(lr, 0.9) (train.py:633), l2_regularizer(WEIGHT_REG) on every conv / fc weight AND bias.
This is the keep_prob = 1.0 graph (the reference trains with dropout 0.5; random masks cannot be compared, SURVEY App. A.7).
A network built with pose_reg=False (the linemod_{benchvise,camera,iron,lamp,phone}.yml models) trains
    loss = loss_cls + VERTEX_W * loss_vertex + l2 regularisation (train.py:517, vgg16_convs.py:128-163):
no Hough voting, RoiPool or fc6-fc8 in the step, and no fc6-fc8 parameters in it.
Every class count the kernels take trains: C = 2 (the single-object LINEMOD / YCB models), even C in 6..50, and C = 9 (the
multi-object LINEMOD model linemod_color_2d.yml, eight objects plus background, pose_reg=False).
A network built with vertex_reg_2d=False, vertex_reg_3d=True (the object-coordinate models linemod_*_3d.yml, lov_color_3d.yml) trains
its vertex head on 3-D targets (minibatch.py:595-600, 605-616): a labelled pixel of a listed class regresses its object coordinate
vertmap [B,H,W,3] scaled into [0, 1] by the class's extents.  Its graph has no pose head whatever pose_reg says (vgg16_convs.py:165-200
builds Hough voting, RoiPool and fc6-fc8 only under vertex_reg_2d), so it trains loss_cls + VERTEX_W * loss_vertex (+ l2).
A network built with vertex_reg_2d=False, vertex_reg_3d=False (the segmentation models rgbd_scene_single_*.yml, shapenet_*_single_*.yml,
lov_single_color_*.yml) has no vertex head (vgg16_convs.py:79-149) and trains loss = loss_cls + l2 regularisation (train.py:518-521):
its head tensor holds the C score channels only, its adjoint is the classification-only one (heads.up8_scores_bwd), and conv4_3 /
conv5_3 receive gradient through score_conv4 / score_conv5 alone.  pose_reg and adaptation do not apply to it.
input_format='RGBD' adds the depth trunk conv1_1_p .. conv5_3_p (vgg16_convs.py:99-126): score_conv4 / score_conv5 read the channel
concat [colour | depth] of conv4_3 / conv5_3 (c_i = 1024), the vertex heads, Hough voting and RoiPool read the colour trunk only.
A network built with adaptation=True adds the domain classifier (vgg16_convs.py:202-212) and
    loss_domain = adapt_weight * mean_rows sparse_softmax_cross_entropy(domain_score, label_domain)   (train.py:508-513)
on pool_score behind gradient_reversal(0.01): fc9's and domain_score's own gradients are the plain ones, and the gradient that
reaches pool_score (and through RoiPool the colour trunk) is multiplied by -0.01.  An "adapt" batch (real images without
annotation, lib/gt_synthesize_layer/minibatch.py:510-511) is given as gt_label_2d = -1 everywhere and gt_poses with 0 rows: Hough
then labels its rows domain 1, and the other losses and their gradients are exactly 0.

Everything heavy runs on this package's own kernels:
    forward   wgmma convolutions (bf16), un-fused heads (add + up2, 1x1 on the tensor cores, fused up8 / softmax / arg-max),
              Houghvotinggpu in train mode, RoiPool with arg-max, fp16 tensor-core fc6-fc8, fused losses
    backward  wgrad on wgmma with MN-major operands (csrc/wgrad_tc.cu), dgrad = the forward kernel on flipped weights,
              ReLU / max-pool routing with bias gradients, fused loss-gradient up-sampling adjoint (csrc/train_bwd.cu),
              RoiPoolGrad, fc input / weight gradients on wgmma
    update    fused SGD-with-momentum + weight decay + refresh of the 16-bit tensor-core weight copies
    multi-GPU images shard across ranks; loss normalisers use GLOBAL counts (one small all-reduce), gradients are summed with
              bucketed NCCL all-reduces issued on a communication stream while the backward pass continues (SURVEY.md §8(e))
PyTorch supplies device memory, streams, NCCL plumbing and a few tiny glue ops on [rows, 4C]-sized tensors.
"""
from __future__ import annotations

from typing import Callable, NamedTuple

import torch
import torch.distributed as dist

from . import backward as bw
from . import conv, heads, pose_head, train_ops
from ._lib import check, lib, ptr, stream
from .average_distance_loss import average_distance_loss_op
from .hough_voting_gpu_layer import hough_voting_gpu_op
from .networks.vgg16_convs import PIXEL_MEANS, VGG_CFG
from .roi_pooling_layer import roi_pooling_op

CONV_NAMES = [item[0] for item in VGG_CFG if isinstance(item, tuple)]
POOL_AFTER = {"conv1_2", "conv2_2", "conv3_3", "conv4_3"}          # pool1..pool4 (vgg16_convs.py:80-97)
GRL_LAMBDA = 0.01                                                  # gradient_reversal(0.01, name='greversal'), vgg16_convs.py:207
SCORE_HEADS = ("score_conv4", "score_conv5", "score_conv4_vertex", "score_conv5_vertex")


class Kind(NamedTuple):
    to_master: Callable            # (TF-layout tensor, master rows or None) -> fp32 master
    to_tf: Callable                # (master-layout tensor, TF shape) -> TF-layout tensor
    copy16: torch.dtype | None     # the 16-bit tensor-core copy kept beside the master, refreshed by every update


def _conv_master(w, rows=None):
    """conv.hwio_to_tc's [Cout][kh*kw*Cin] layout in fp32, the Cout rows zero-padded to `rows`."""
    t = conv.hwio_to_tc(w, torch.float32)
    if rows is None:
        return t
    out = t.new_zeros((rows, t.shape[1]))
    out[:t.shape[0]] = t
    return out


def _conv_to_tf(t, shape):
    kh, kw, ci, co = shape
    return t[:co].reshape(co, kh, kw, ci).permute(1, 2, 3, 0).contiguous()


# How the step keeps each kind of parameter: the fp32 master is the layout the kernels read, so the 16-bit copy is the master rounded.
KINDS = {
    # 3x3 trunk [Cout][9 Cin]; 1x1 score heads [Cout][Cin] (RGB-D score_conv4 / 5: Cin = 1024); score / vertex_pred padded
    "conv": Kind(_conv_master, _conv_to_tf, torch.bfloat16),
    # [64][27] (K = tap * 3 + c); its bf16 copy is the padded [64][64] tile Trainer.conv1_tc, refreshed in _refresh_derived
    "conv1_1": Kind(_conv_master, _conv_to_tf, None),
    # [out padded to a multiple of 128][in]
    "fc": Kind(lambda w, rows=None: pose_head.fc_weights_to_tc(w, torch.float32), lambda t, shape: t[:shape[1]].t().contiguous(),
               torch.float16),
    # [2][256], read in fp32 by the domain tail kernel
    "domain_score": Kind(lambda w, rows=None: w.t().contiguous(), lambda t, shape: t.t().contiguous(), None),
    "bias": Kind(lambda w, rows=None: w.clone(), lambda t, shape: t.clone(), None),
}


def trains_coords(net) -> bool:
    """True for the object-coordinate (VERTEX_REG_3D) training graph: 3-D vertex targets and no pose head."""
    return bool(net.vertex_reg_3d) and not bool(net.vertex_reg_2d)


def trains_segmentation(net) -> bool:
    """True for the segmentation training graph: no vertex head (built with vertex_reg_2d=False, vertex_reg_3d=False), loss_cls alone."""
    return not net.vertex_head


def head_names(net) -> tuple:
    """The 1x1 head layers of the training graph: score_conv4 / 5 and score, plus the vertex heads where the network has them."""
    if trains_segmentation(net):
        return ("score_conv4", "score_conv5", "score")
    return SCORE_HEADS + ("score", "vertex_pred")


def param_layout(net) -> dict:
    """{master name: (TF parameter name, kind, master rows)} for every parameter the training step updates.  score / vertex_pred
    keep C / 3C rows zero-padded to heads.SCORE_ROWS / heads.vertex_rows(C): the channel counts of their 1x1 GEMMs, which
    heads.pack_lowres and heads.up8_heads_bwd read.  A pose_reg=False network has no fc6-fc8: the reference creates those
    variables only under POSE_REG (vgg16_convs.py:175-200), so they are neither trained, decayed nor exported.  Neither has an object-coordinate network, whose
    pose head sits under vertex_reg_2d in the reference graph.  A segmentation network has the trunk(s), score_conv4 / 5 and score
    only."""
    trunks = ("", "_p") if net.input_format == "RGBD" else ("",)
    weights = [(layer + sfx, "conv1_1" if layer == "conv1_1" else "conv", None) for sfx in trunks for layer in CONV_NAMES]
    rows = {"score": heads.SCORE_ROWS, "vertex_pred": heads.vertex_rows(net.num_classes)}
    weights += [(name, "conv", rows.get(name)) for name in head_names(net)]
    pose = net.pose_reg and not trains_coords(net) and not trains_segmentation(net)
    fc = (("fc6", "fc7", "fc8") if pose else ()) + (("fc9",) if net.domain_branch else ())
    weights += [(name, "fc", None) for name in fc]
    if net.domain_branch:
        weights.append(("domain_score", "domain_score", None))
    layout = {}
    for name, kind, rows in weights:
        layout[name + "/w"] = (name + "/weights", kind, rows)
        layout[name + "/b"] = (name + "/biases", "bias", None)
    return layout


def _tc_dgrad(w_tc: torch.Tensor, k: int) -> torch.Tensor:
    """Tensor-core weights [Cout][k*k*Cin] -> the weights of the input-gradient convolution [Cin][k*k*Cout] (taps flipped,
    channels transposed; conv.hwio_to_tc_dgrad applied to the TC layout)."""
    co = w_tc.shape[0]
    ci = w_tc.shape[1] // (k * k)
    return w_tc.view(co, k, k, ci).flip(1, 2).permute(3, 1, 2, 0).reshape(ci, k * k * co).contiguous()


class Trainer:
    def __init__(self, net, lr=0.001, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=0.01, world=1,
                 adapt_weight=0.1):
        assert net.is_train and not net.fold_vertex_head and net.input_format in ("COLOR", "RGBD"), \
            "Trainer needs vgg16_convs(is_train=True, fold_vertex_head=False, input_format='COLOR' or 'RGBD')"
        self.rgbd = net.input_format == "RGBD"
        self.trunks = ("", "_p") if self.rgbd else ("",)           # conv*_p: the depth trunk (vgg16_convs.py:99-117)
        self.net, self.lr, self.mu, self.wd = net, float(lr), float(momentum), float(weight_decay)
        self.vertex_w, self.w_inside, self.margin, self.world = float(vertex_w), float(vertex_w_inside), float(margin), int(world)
        self.C = net.num_classes
        # POSE_REG: Hough voting, RoiPool, fc6-fc8 and loss_pose (vgg16_convs.py:165-200).  Without it the step is the dense heads'
        # loss_cls + VERTEX_W * loss_vertex (+ l2 regularisation) alone, as lib/fcn/train.py:517 trains it.  The object-coordinate
        # graph (3-D vertex targets) never has the pose head
        self.coord = trains_coords(net)
        self.seg = trains_segmentation(net)      # no vertex head: loss_cls alone
        self.pose_reg = bool(net.pose_reg) and not self.coord and not self.seg
        self.pose_loss_scale = 1.0               # last dynamic loss scale of the fp16 pose-head backward (see backward())
        self.adapt = net.domain_branch           # the domain classifier and loss_domain (ADAPT_WEIGHT, lib/fcn/config.py:95)
        self.adapt_weight = float(adapt_weight)
        self.domain_loss_scale = 1.0             # the same for the domain branch's fp16 backward
        self.fc_names = (("fc6", "fc7", "fc8") if self.pose_reg else ()) + (("fc9",) if self.adapt else ())
        self.comm = torch.cuda.Stream(device=net.device) if world > 1 else None
        P, dev = net.params, net.device
        self.layout = param_layout(net)
        self.master, self.accum, self.tc = {}, {}, {}
        for name, (tf, kind, rows) in self.layout.items():
            k = KINDS[kind]
            w = k.to_master(P[tf], rows)
            self.master[name] = w
            self.accum[name] = torch.zeros_like(w)
            self.tc[name] = w.to(k.copy16).contiguous() if k.copy16 else None
        self.conv1_tc = conv.conv1_1_weights_to_tc(P["conv1_1/weights"])
        self.conv1_tc_p = conv.conv1_1_weights_to_tc(P["conv1_1_p/weights"]) if self.rgbd else None
        self._refresh_derived()
        self.zero_bias = {n: torch.zeros(n, device=dev) for n in (64, 128, 256, 512, heads.vertex_rows(self.C))}

    # ------------------------------------------------------------------ derived weight copies
    def _refresh_derived(self):
        """Copies the backward GEMMs read: input-gradient (flipped / transposed) weights of every convolution, [in][out] fp16 copies of
        the fully connected weights, the padded conv1_1 tile (and conv1_1_p's)."""
        self.dg = {}
        for sfx in self.trunks:
            for name in CONV_NAMES[1:]:
                self.dg[name + sfx] = _tc_dgrad(self.tc[name + sfx + "/w"], 3)
        for name in head_names(self.net):
            self.dg[name] = _tc_dgrad(self.tc[name + "/w"], 1)
        if self.rgbd:
            # score_conv4/5 read the concat [colour 512 | depth 512]: their input-gradient weights [1024][U] split into two
            # contiguous [512][U] halves, one input-gradient convolution per trunk
            for name in ("score_conv4", "score_conv5"):
                d = self.dg[name]
                self.dg[name], self.dg[name + "_p"] = d[:512], d[512:]
        self.fc_t = {}
        for name in self.fc_names:
            self.fc_t[name] = pose_head.transpose16(self.tc[name + "/w"])
        self.conv1_tc.zero_()
        self.conv1_tc[:, :27] = self.master["conv1_1/w"].to(torch.bfloat16)
        if self.rgbd:
            self.conv1_tc_p.zero_()
            self.conv1_tc_p[:, :27] = self.master["conv1_1_p/w"].to(torch.bfloat16)

    def to_tf(self, name, t):
        """A master-layout tensor of parameter `name` (a master, a gradient) -> the TF layout of its net.params entry."""
        tf, kind, _ = self.layout[name]
        return KINDS[kind].to_tf(t, self.net.params[tf].shape)

    def export_params(self):
        """Write the fp32 master weights back into net.params (TF layouts) and re-derive the inference copies."""
        for name, (tf, _, _) in self.layout.items():
            self.net.params[tf] = self.to_tf(name, self.master[name])
        self.net.prepare()

    # ------------------------------------------------------------------ forward (training graph, activations kept)
    @staticmethod
    def _mean(data):
        return PIXEL_MEANS if data.dtype == torch.uint8 else None

    def _trunk_fwd(self, A, x, sfx=""):
        """conv1_2 .. conv5_3 of one trunk on its conv1_1 output x; every activation is kept in A (the backward pass reads them)."""
        M, T = self.master, self.tc
        A["conv1_1" + sfx] = x
        for layer in CONV_NAMES[1:]:
            name = layer + sfx
            x = conv.conv_bf16(x, T[name + "/w"], M[name + "/b"], 3, True)
            A[name] = x
            if layer in POOL_AFTER and layer != "conv5_3":
                x = conv.maxpool2x2(x)
                A[name + "/pool"] = x

    def _require_vertmap(self, vertmap, data):
        B, H, W = data.shape[:3]
        if vertmap is None:
            raise ValueError("an object-coordinate (vertex_reg_3d) network trains on 3-D targets: pass vertmap= [B,H,W,3] f32")
        if vertmap.dtype != torch.float32 or tuple(vertmap.shape) != (B, H, W, 3) or vertmap.device != data.device:
            raise ValueError(f"vertmap must be a [{B},{H},{W},3] float32 tensor on {data.device}")
        return vertmap.contiguous()

    def forward(self, data, gt_label_2d, centers=None, meta_data=None, extents=None, gt_poses=None, points=None, symmetry=None,
                batch_global=None, batch_offset=0, depth=None, data_p=None, vertmap=None):
        """RGBD: the depth trunk reads depth= (a raw [B,H,W] f32 depth image, sensor units; its blob is formed in conv1_1_p's loader)
        or data_p= (the pre-processed blob [B,H,W,3] f32), as vgg16_convs.forward does.  An object-coordinate network reads
        vertmap= [B,H,W,3] f32 (each pixel's object coordinate, metres in the model frame) and extents [C,3]; other networks ignore
        vertmap.  A segmentation network reads data, gt_label_2d and the depth input only."""
        net, C, M, T = self.net, self.C, self.master, self.tc
        B, H, W, _ = data.shape
        if self.coord:
            vertmap = self._require_vertmap(vertmap, data)
            extents = extents.contiguous()
        A = {}                                    # activations by layer name (bf16 NHWC), "<pool>" = pooled tensors
        # data: [B,H,W,3] u8 BGR (PIXEL_MEANS subtracted in conv1_1's loader) or the f32 blob of augment.augment_color (means
        # already subtracted), as vgg16_convs._trunk chooses
        self._trunk_fwd(A, conv.conv1_fused(data, self.conv1_tc, M["conv1_1/b"], self._mean(data), True))
        c4, c5 = A["conv4_3"], A["conv5_3"]
        h4, h5 = c4, c5
        if self.rgbd:
            assert (depth is None) != (data_p is None), "the RGB-D training step needs exactly one of depth= and data_p="
            if depth is not None:
                x = conv.conv1_depth_fused(depth, self.conv1_tc_p, M["conv1_1_p/b"], PIXEL_MEANS, True)
            else:
                x = conv.conv1_fused(data_p, self.conv1_tc_p, M["conv1_1_p/b"], None, True)
            self._trunk_fwd(A, x, "_p")
            # concat_conv4 / concat_conv5 (vgg16_convs.py:119-126): colour channels first; kept as score_conv4/5's wgrad input
            h4, h5 = torch.cat([c4, A["conv4_3_p"]], 3), torch.cat([c5, A["conv5_3_p"]], 3)
            A.update(concat_conv4=h4, concat_conv5=h5, depth_in=depth if depth is not None else data_p)
        s4 = conv.conv_bf16(h4, T["score_conv4/w"], M["score_conv4/b"], 1, True)
        s5 = conv.conv_bf16(h5, T["score_conv5/w"], M["score_conv5/b"], 1, True)
        if self.seg:
            # score heads only: add + up2, `score` at 1/8 resolution, the score-only head tensor, its x8 up-sampling and loss_cls
            add_s = heads.add_up2(s4, s5)
            lr_s = conv.conv_bf16(add_s, T["score/w"], self.zero_bias[heads.SCORE_ROWS], 1, False)
            lowres = heads.pack_scores(lr_s, C)
            label, prob, score = heads.up8_scores(lowres, M["score/b"], prob=True, score=True)
            A.update(s4=s4, s5=s5, add_s=add_s, label_2d=label, lowres=lowres, prob_normalized=prob, score=score, data=data)
            A["cls_out"] = train_ops.loss_cls(score, prob, gt_label_2d, net.threshold_label)
            return A
        v4 = conv.conv_bf16(c4, T["score_conv4_vertex/w"], M["score_conv4_vertex/b"], 1, False)
        v5 = conv.conv_bf16(c5, T["score_conv5_vertex/w"], M["score_conv5_vertex/b"], 1, False)
        add_s, add_v = heads.add_up2(s4, s5), heads.add_up2(v4, v5)
        lr_s = conv.conv_bf16(add_s, T["score/w"], self.zero_bias[heads.SCORE_ROWS], 1, False)   # bias added after the up-sampling
        lr_v = conv.conv_bf16(add_v, T["vertex_pred/w"], self.zero_bias[heads.vertex_rows(C)], 1, False)
        lowres = heads.pack_lowres(lr_s, lr_v, C)
        # The dense vertex_pred [B,H,W,3C] (81 MB / frame) is never written: its only consumers — the vertex loss, its gradient and the
        # Hough sampler — read three values per labelled / sampled pixel and form them on demand from `lowres` with k_up8_heads' own
        # operation sequence (heads_common.cuh: bit-identical).  dense_vertex_pred(A) materialises it for inspection.
        label, _, prob, score = heads.up8_heads(lowres, M["score/b"], M["vertex_pred/b"], prob=True, score=True)
        A.update(s4=s4, s5=s5, v4=v4, v5=v5, add_s=add_s, add_v=add_v, label_2d=label, lowres=lowres, prob_normalized=prob, score=score)
        # losses on the dense heads (fused kernels; the masks / targets are never materialised)
        cls_out = train_ops.loss_cls(score, prob, gt_label_2d, net.threshold_label)
        vtx_out = train_ops.loss_vertex(lowres, M["vertex_pred/b"], gt_label_2d, centers, self.w_inside, 1.0,
                                        vertmap if self.coord else None, extents if self.coord else None)
        if self.coord:
            A.update(extents=extents)
        A.update(cls_out=cls_out, vtx_out=vtx_out, data=data)
        if not self.pose_reg:
            return A
        # Hough voting in train mode (9 jittered ROIs per maximum, quaternion targets from the gt poses)
        Bg = B if batch_global is None else int(batch_global)
        box, pose, target, weight, domain, num_rois, status = hough_voting_gpu_op.hough_voting_gpu_capacity(
            label, None, extents, meta_data, gt_poses, 1, net.vote_threshold, net.vote_percentage, net.skip_pixels, lowres=lowres,
            bias_vertex=M["vertex_pred/b"], batch_global=Bg, batch_offset=batch_offset)
        # the op's output has a data-dependent number of rows (9 per kept maximum): one host read, like the reference's
        # copy_num_rois (hough_voting_gpu_op.cu.cc:591-594); Averagedistance then normalises by the true row count
        host = torch.cat([num_rois, status[:2]]).tolist()
        hough_voting_gpu_op.check_status(host[1], host[2])
        rows = max(1, min(host[0], (128 // Bg) * B * 9))
        rois = box[:rows].contiguous()
        rl = rois if not batch_offset else torch.cat([rois[:, :1] - float(batch_offset), rois[:, 1:]], 1).contiguous()
        p5, a5 = roi_pooling_op.roi_pool(c5, rl, 7, 7, 1.0 / 16.0, 0)
        p4, a4 = roi_pooling_op.roi_pool(c4, rl, 7, 7, 1.0 / 8.0, 0)
        pool = (p5 + p4).reshape(rows, -1).clamp(-65504.0, 65504.0).to(torch.float16)
        f6 = pose_head.fc(pool, T["fc6/w"], M["fc6/b"], "relu")
        f7 = pose_head.fc(f6, T["fc7/w"], M["fc7/b"], "relu")
        tanh = pose_head.fc(f7, T["fc8/w"], M["fc8/b"], "tanh", torch.float32)
        tw, wt = target[:rows].contiguous(), weight[:rows].contiguous()
        mul = tanh * wt                                                                         # vgg16_convs.py:195-196
        pred = (mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()).contiguous()     # tf.nn.l2_normalize(dim=1)
        loss_pose, pose_diff = average_distance_loss_op.average_distance_loss(pred, tw, wt, points, symmetry, self.margin)
        A.update(rois=rl, num_rois=num_rois, a5=a5, a4=a4, pool=pool, fc6=f6, fc7=f7, poses_tanh=tanh, poses_weight=wt, poses_target=tw,
                 pose_diff=pose_diff, loss_pose_raw=loss_pose, rows=rows)
        if self.adapt:
            # the domain classifier on the same fp16 pool_score (gradient_reversal is the identity forward); label_domain = Hough's
            # top_domain, decided by the whole batch's gt count (every rank is given the whole gt array)
            f9 = pose_head.fc(pool, T["fc9/w"], M["fc9/b"], "relu")
            A.update(fc9=f9, label_domain=domain[:rows].contiguous())
            A.update(pose_head.domain_tail(f9, M["domain_score/w"], M["domain_score/b"]))
        return A

    def dense_vertex_pred(self, A):
        """The dense vertex_pred [B,H,W,3C] of a forward pass (the training step itself never materialises it)."""
        return heads.up8_heads(A["lowres"], self.master["score/b"], self.master["vertex_pred/b"], vertex=True)[1]

    # ------------------------------------------------------------------ gradient plumbing
    def _emit(self, grads, name, g):
        """A finished gradient tensor: start its all-reduce (SUM over ranks) on the communication stream right away."""
        grads[name] = g
        if self.comm is not None:
            self.comm.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.comm):
                dist.all_reduce(g, op=dist.ReduceOp.SUM)

    def backward(self, A, gt_label_2d, centers=None, vertmap=None):
        """All parameter gradients of loss = loss_cls + vertex_w * loss_vertex + loss_pose (weight decay is applied in the update);
        without pose_reg, of loss_cls + vertex_w * loss_vertex.  Loss normalisers (selected-pixel count, vertex weight sum, ROI rows)
        are GLOBAL over the ranks.  An object-coordinate network needs the forward's vertmap= again (its extents are kept in A).  A
        segmentation network's loss is loss_cls alone, and centers is not read."""
        net, C, M, T = self.net, self.C, self.master, self.tc
        data = A["data"]
        dev = data.device
        grads = {}
        # ---- global loss normalisers: one all-reduce of [count_cls, sum_w_vertex(, rows)]
        rows = [torch.tensor(float(A["rows"]), device=dev)] if self.pose_reg else []
        norm = torch.stack([A["cls_out"][1]] + ([] if self.seg else [A["vtx_out"][1]]) + rows)
        if self.world > 1:
            local = norm.clone()
            dist.all_reduce(norm, op=dist.ReduceOp.SUM)
            A["cls_out"] = torch.stack([A["cls_out"][0] * local[0] / norm[0].clamp(min=1.0), norm[0]])     # this rank's share of the global mean
            if not self.seg:
                A["vtx_out"] = torch.stack([A["vtx_out"][0] * local[1] / norm[1].clamp(min=1e-10), norm[1]])
        g5_roi = g4_roi = None                    # the RoiPool gradients of the pose head (and the domain branch)
        if self.pose_reg:
            g5_roi, g4_roi = self._pose_bwd(grads, A, norm)
        # ---- FCN heads
        if self.seg:
            d_sc, dbias = heads.up8_scores_bwd(A["prob_normalized"], A["score"], gt_label_2d, A["cls_out"], 1.0, net.threshold_label)
            self._emit(grads, "score/b", dbias)
        else:
            vm, ext = (self._require_vertmap(vertmap, data), A["extents"]) if self.coord else (None, None)
            d_sc, d_vt, dbias = heads.up8_heads_bwd(A["prob_normalized"], A["score"], gt_label_2d, A["cls_out"], 1.0, net.threshold_label,
                                                    A["lowres"], M["vertex_pred/b"], centers, A["vtx_out"], self.vertex_w, self.w_inside, 1.0,
                                                    vertmap=vm, extents=ext)
            self._emit(grads, "score/b", dbias[:C].contiguous())
            self._emit(grads, "vertex_pred/b", dbias[C:].contiguous())
        self._emit(grads, "score/w", bw.conv_wgrad(A["add_s"], d_sc, 1))
        if not self.seg:
            self._emit(grads, "vertex_pred/w", bw.conv_wgrad(A["add_v"], d_vt, 1))
        d_add_s = conv.conv_bf16(d_sc, self.dg["score"], self.zero_bias[64], 1, False)
        if not self.seg:
            d_add_v = conv.conv_bf16(d_vt, self.dg["vertex_pred"], self.zero_bias[128], 1, False)
        d_s4, db = bw.relu_bwd(d_add_s, A["s4"], True, want_bias=True)
        self._emit(grads, "score_conv4/b", db)
        d_s5 = heads.up2_bwd(d_add_s, A["s5"])
        self._emit(grads, "score_conv5/b", bw.relu_bwd(d_s5, None, False, want_bias=True, want_dz=False)[1])
        if not self.seg:
            self._emit(grads, "score_conv4_vertex/b", bw.relu_bwd(d_add_v, None, False, want_bias=True, want_dz=False)[1])
            d_v5 = heads.up2_bwd(d_add_v)
            self._emit(grads, "score_conv5_vertex/b", bw.relu_bwd(d_v5, None, False, want_bias=True, want_dz=False)[1])
        c4, c5 = A["conv4_3"], A["conv5_3"]
        # RGB-D: score_conv4/5 read the 1024-channel concat, so their weight gradient is one wgrad on it
        self._emit(grads, "score_conv4/w", bw.conv_wgrad(A["concat_conv4"] if self.rgbd else c4, d_s4, 1))
        self._emit(grads, "score_conv5/w", bw.conv_wgrad(A["concat_conv5"] if self.rgbd else c5, d_s5, 1))
        z512 = self.zero_bias[512]
        if self.seg:
            # conv4_3 / conv5_3 receive gradient through score_conv4 / score_conv5 alone
            g4 = conv.conv_bf16(d_s4, self.dg["score_conv4"], z512, 1, False)
            g5 = conv.conv_bf16(d_s5, self.dg["score_conv5"], z512, 1, False)
        else:
            self._emit(grads, "score_conv4_vertex/w", bw.conv_wgrad(c4, d_add_v, 1))
            self._emit(grads, "score_conv5_vertex/w", bw.conv_wgrad(c5, d_v5, 1))
            g4 = bw.add_to_bf16(conv.conv_bf16(d_s4, self.dg["score_conv4"], z512, 1, False),
                                conv.conv_bf16(d_add_v, self.dg["score_conv4_vertex"], z512, 1, False), g4_roi)
            g5 = bw.add_to_bf16(conv.conv_bf16(d_s5, self.dg["score_conv5"], z512, 1, False),
                                conv.conv_bf16(d_v5, self.dg["score_conv5_vertex"], z512, 1, False), g5_roi)
        # ---- trunk, top down
        self._trunk_bwd(grads, A, g5, g4, "", lambda: conv.im2col_c3(data, self._mean(data)))
        if self.rgbd:
            # the depth trunk's gradient enters through the depth half of the concat only (the vertex heads and RoiPool read
            # the colour trunk, vgg16_convs.py:151-182)
            g4_p = conv.conv_bf16(d_s4, self.dg["score_conv4_p"], z512, 1, False)
            g5_p = conv.conv_bf16(d_s5, self.dg["score_conv5_p"], z512, 1, False)
            x_p = A["depth_in"]
            cols_p = (lambda: conv.im2col_depth(x_p, PIXEL_MEANS)) if x_p.dim() == 3 else (lambda: conv.im2col_c3(x_p, None))
            self._trunk_bwd(grads, A, g5_p, g4_p, "_p", cols_p)
        return grads

    def _pose_bwd(self, grads, A, norm):
        """Gradients of loss_pose (and loss_domain) through fc8 .. fc6 (and fc9) and RoiPool: emits the fc parameters' gradients and
        returns the dense fp32 RoiPool gradients (g5_roi, g4_roi) that enter conv5_3 / conv4_3."""
        C, M = self.C, self.master
        dev, rows = A["data"].device, A["rows"]
        # Averagedistance divides by the rows IT sees (capacity rows of this rank); the reference batch sees all of them
        if self.world > 1:
            pose_scale, rows_g = torch.stack([float(rows) / norm[2], norm[2]]).tolist()         # one host read
        else:
            pose_scale, rows_g = 1.0, float(rows)
        A["loss_pose"] = A["loss_pose_raw"] * pose_scale
        if self.adapt:
            # domain branch, un-scaled pass: its gradient maximum is read with the pose chain's below
            dom = pose_head.domain_tail(A["fc9"], M["domain_score/w"], M["domain_score/b"], A["label_domain"], self.adapt_weight / rows_g, 1.0)
        # ---- pose head
        # The head's backward GEMMs run on FP16 operands like its forward.  The pose-loss gradients are tiny (a mean over rows x points:
        # 1e-6 .. 1e-4 per element, below fp16's normal range), so the chain is LOSS-SCALED by a dynamic power of two S where it enters fp16 and un-scaled
        # where it leaves (weight gradients, bias sums, the RoiPool gradient); conversions saturate at +-65504.
        # dpre's row stride is fc8's output count padded to a multiple of 128 (its fp16 weight copy's rows): 128 up to C = 32, 256 above
        D, ld = 4 * C, self.tc["fc8/w"].shape[0]
        dpre = torch.empty((rows, ld), dtype=torch.float16, device=dev)
        pose_head.pose_chain_bwd(A["pose_diff"], A["poses_tanh"], A["poses_weight"], pose_scale, dpre)
        # dynamic loss scale: a power of two that puts the largest element of the chain's entry point at ~2^11 (one host read; the
        # un-scaled pass above is only used for its maximum, which fp16 represents well enough even when the small elements underflow)
        amax = torch.stack([dpre.float().abs().max()] + ([dom["amax"][0]] if self.adapt else []))
        if self.world > 1:
            dist.all_reduce(amax, op=dist.ReduceOp.MAX)
        amax = amax.tolist()
        S = self._loss_scale(amax[0])
        self.pose_loss_scale = S
        if self.adapt:
            # the same dynamic power of two for fc9's backward GEMMs (d fc9 is ~1e-5: below fp16's normal range)
            S_d = self._loss_scale(amax[1])
            self.domain_loss_scale = S_d
            dom = pose_head.domain_tail(A["fc9"], M["domain_score/w"], M["domain_score/b"], A["label_domain"], self.adapt_weight / rows_g, S_d)
            A["loss_domain"] = dom["loss"]
            self._emit(grads, "domain_score/w", dom["dw10"])
            self._emit(grads, "domain_score/b", dom["db10"])
            self._emit(grads, "fc9/w", pose_head.fc_wgrad(A["pool"], dom["dpre9"], 1.0 / S_d))
            self._emit(grads, "fc9/b", dom["db9"])
            d9 = pose_head.fc_dgrad(dom["dpre9"], self.fc_t["fc9"], None)                     # [rows, 25088], scaled by S_d
        pose_head.pose_chain_bwd(A["pose_diff"], A["poses_tanh"], A["poses_weight"], pose_scale * S, dpre)
        self._emit(grads, "fc8/w", pose_head.fc_wgrad(A["fc7"], dpre, 1.0 / S))
        self._emit(grads, "fc8/b", dpre[:, :D].float().sum(0) / S)
        d7 = pose_head.fc_dgrad(dpre, self.fc_t["fc8"], A["fc7"])
        self._emit(grads, "fc7/w", pose_head.fc_wgrad(A["fc6"], d7, 1.0 / S))
        self._emit(grads, "fc7/b", d7.float().sum(0) / S)
        d6 = pose_head.fc_dgrad(d7, self.fc_t["fc7"], A["fc6"])
        self._emit(grads, "fc6/w", pose_head.fc_wgrad(A["pool"], d6, 1.0 / S))
        self._emit(grads, "fc6/b", d6.float().sum(0) / S)
        dpool16 = pose_head.fc_dgrad(d6, self.fc_t["fc6"], None)                               # [rows, 25088]
        if self.adapt:
            # pool_score's gradient from both branches in one pass; gradient_reversal is the factor -lambda of the domain term
            dpool = pose_head.domain_grad_merge(dpool16, 1.0 / S, d9, -GRL_LAMBDA / S_d, (rows, 7, 7, 512))
        else:
            dpool = pose_head.half_to_float(dpool16, 1.0 / S).view(rows, 7, 7, 512)
        A["dpool"] = dpool                                                                      # d loss / d pool_score (kept for inspection)
        g5_roi = roi_pooling_op.roi_pool_grad(A["conv5_3"], A["rois"], A["a5"], dpool, 7, 7, 1.0 / 16.0, 0)       # fp32 dense
        g4_roi = roi_pooling_op.roi_pool_grad(A["conv4_3"], A["rois"], A["a4"], dpool, 7, 7, 1.0 / 8.0, 0)
        return g5_roi, g4_roi

    @staticmethod
    def _loss_scale(amax):
        """The power of two (1 .. 2^24) that puts a backward chain's largest fp16 entry at ~2^11."""
        return 2.0 ** max(0, min(24, int(torch.floor(torch.log2(torch.tensor(2048.0 / max(amax, 1e-30)))).item()))) if amax > 0 else 1.0

    def _trunk_bwd(self, grads, A, g5, g4, sfx, im2col):
        """conv5_3 .. conv1_1 of one trunk, top down.  g5 / g4: the gradients entering conv5_3 / conv4_3 from the heads (and
        RoiPool); im2col() builds the [B,H,W,64] view of the trunk's input that conv1_1's weight gradient reads."""
        g = g5                                    # gradient w.r.t. the (post-ReLU) output of the current layer
        for layer in reversed(CONV_NAMES):
            name = layer + sfx
            y = A[name]
            if layer == "conv4_3":
                # conv4_3 feeds pool4 (gradient routed to the window maxima) AND the heads / RoiPool (g4)
                dz = bw.add_to_bf16(bw.maxpool_relu_bwd(g, y), bw.relu_bwd(g4, y, True))
                db = bw.relu_bwd(dz, None, False, want_bias=True, want_dz=False)[1]
            elif layer in POOL_AFTER and layer != "conv5_3":
                dz, db = bw.maxpool_relu_bwd(g, y, want_bias=True)
            else:
                dz, db = bw.relu_bwd(g, y, True, want_bias=True)
            self._emit(grads, name + "/b", db)
            if layer == "conv1_1":
                # Cin = 3: the weight gradient is the 1x1 tensor-core wgrad on the im2col view of the input (K = tap * 3 + c, the same
                # bf16 (pixel - mean) values the forward MMA consumed)
                cols = im2col()                                                                 # [B,H,W,64] bf16, 27 columns used
                self._emit(grads, name + "/w", bw.conv_wgrad(cols, dz, 1)[:, :27].contiguous())
                break
            prev = CONV_NAMES[CONV_NAMES.index(layer) - 1] + sfx
            x_in = A.get(prev + "/pool", A[prev])
            self._emit(grads, name + "/w", bw.conv_wgrad(x_in, dz, 3))
            g = conv.conv_bf16(dz, self.dg[name], self.zero_bias[x_in.shape[3]], 3, False)      # gradient w.r.t. this layer's input

    def update(self, grads):
        """accum = mu * accum + (grad + wd * w); w -= lr * accum, on the fp32 masters; 16-bit tensor-core copies refreshed in the same
        kernel, derived copies (input-gradient weights, transposed fc weights) afterwards."""
        if self.comm is not None:
            torch.cuda.current_stream().wait_stream(self.comm)
        for name, g in grads.items():
            w = self.master[name]
            assert g.shape == w.shape, (name, tuple(g.shape), tuple(w.shape))
            c16 = self.tc[name]
            check(lib().pcnn_sgd_momentum(ptr(w), ptr(self.accum[name]), ptr(g), w.numel(), self.lr, self.mu, self.wd,
                                          1.0, ptr(c16), int(c16 is not None and c16.dtype == torch.float16), stream()))
        self._refresh_derived()

    def step(self, data, gt_label_2d, centers=None, meta_data=None, extents=None, gt_poses=None, points=None, symmetry=None,
             batch_global=None, batch_offset=0, depth=None, data_p=None, vertmap=None):
        """One forward, backward and update.  Returns loss_cls, loss_vertex, loss_pose, their sum `loss`, num_rois and the gradients
        `grads` (master layouts), plus loss_domain, label_domain and domain_label with the domain branch.  A pose_reg=False network
        returns no pose entries (loss_pose, num_rois): its loss is loss_cls + loss_vertex, and extents, gt_poses, points, symmetry,
        meta_data, batch_global and batch_offset are not read.  An object-coordinate (vertex_reg_3d) network steps the same way
        whatever its pose_reg, and reads vertmap= [B,H,W,3] f32 and extents [C,3].  A segmentation network (no vertex head) returns
        loss_cls, loss (= loss_cls) and grads, and reads neither centers nor any argument after it but the depth input."""
        A = self.forward(data, gt_label_2d, centers, meta_data, extents, gt_poses, points, symmetry, batch_global, batch_offset,
                         depth=depth, data_p=data_p, vertmap=vertmap)
        grads = self.backward(A, gt_label_2d, centers, vertmap=vertmap)
        self.update(grads)
        if self.seg:
            return dict(loss_cls=A["cls_out"][0:1], loss=A["cls_out"][0:1].clone(), grads=grads)
        if not self.pose_reg:
            loss_cls, loss_vertex = A["cls_out"][0:1], self.vertex_w * A["vtx_out"][0:1]
            return dict(loss_cls=loss_cls, loss_vertex=loss_vertex, loss=loss_cls + loss_vertex, grads=grads)
        loss_cls, loss_vertex, loss_pose = A["cls_out"][0:1], self.vertex_w * A["vtx_out"][0:1], A["loss_pose"]
        out = dict(loss_cls=loss_cls, loss_vertex=loss_vertex, loss_pose=loss_pose, loss=loss_cls + loss_vertex + loss_pose, num_rois=A["num_rois"],
                   grads=grads)
        if self.adapt:
            out.update(loss_domain=A["loss_domain"], loss=out["loss"] + A["loss_domain"], label_domain=A["label_domain"],
                       domain_label=A["domain_label"])
        return out
