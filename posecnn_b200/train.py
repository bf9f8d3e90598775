"""One SGD training step of the vgg16_convs network (BASELINE configs[4]) on the H100-native kernels.

Reference: the training graph lib/networks/vgg16_convs.py:79-212 driven by lib/fcn/train.py:206-260 —
    loss = loss_cls + VERTEX_W * loss_vertex + loss_pose + l2 regularisation (train.py:486-500),
    loss_cls    = Hardlabel-selected cross entropy of log_softmax(score)                 (train.py:455-465, hard_label_op_gpu.cu.cc:16-29)
    loss_vertex = smooth_l1_loss_vertex(vertex_pred, vertex_targets, vertex_weights)     (train.py:564-573)
    loss_pose   = Averagedistance(l2_normalize(poses_tanh * poses_weight), poses_target, poses_weight, points, symmetry)
    optimizer   = tf.train.MomentumOptimizer(lr, 0.9) (train.py:633), l2_regularizer(WEIGHT_REG) on every conv / fc weight AND bias.
This is the keep_prob = 1.0 graph (the reference trains with dropout 0.5; random masks cannot be compared, SURVEY App. A.7).

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

import ctypes

import torch
import torch.distributed as dist

from . import backward as bw
from . import conv, pose_head, train_ops
from ._lib import check, f32, lib, ptr, stream, workspace
from .average_distance_loss import average_distance_loss_op
from .hough_voting_gpu_layer import hough_voting_gpu_op
from .networks.vgg16_convs import PIXEL_MEANS, VGG_CFG
from .roi_pooling_layer import roi_pooling_op

CONV_NAMES = [item[0] for item in VGG_CFG if isinstance(item, tuple)]
POOL_AFTER = {"conv1_2", "conv2_2", "conv3_3", "conv4_3"}          # pool1..pool4 (vgg16_convs.py:80-97)


def _tc_dgrad(w_tc: torch.Tensor, k: int) -> torch.Tensor:
    """Tensor-core weights [Cout][k*k*Cin] -> the weights of the input-gradient convolution [Cin][k*k*Cout] (taps flipped,
    channels transposed; conv.hwio_to_tc_dgrad applied to the TC layout)."""
    co = w_tc.shape[0]
    ci = w_tc.shape[1] // (k * k)
    return w_tc.view(co, k, k, ci).flip(1, 2).permute(3, 1, 2, 0).reshape(ci, k * k * co).contiguous()


class Trainer:
    def __init__(self, net, lr=0.001, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=0.01, world=1):
        assert net.is_train and not net.fold_vertex_head and net.input_format == "COLOR", \
            "Trainer needs vgg16_convs(is_train=True, fold_vertex_head=False, input_format='COLOR')"
        self.net, self.lr, self.mu, self.wd = net, float(lr), float(momentum), float(weight_decay)
        self.vertex_w, self.w_inside, self.margin, self.world = float(vertex_w), float(vertex_w_inside), float(margin), int(world)
        self.C = net.num_classes
        self.pose_loss_scale = 1.0               # last dynamic loss scale of the fp16 pose-head backward (see backward())
        self.comm = torch.cuda.Stream(device=net.device) if world > 1 else None
        P, dev = net.params, net.device
        C = self.C
        self.master, self.accum, self.tc, self.kind = {}, {}, {}, {}

        def add(name, w32, copy16, kind):
            self.master[name] = w32.contiguous()
            self.accum[name] = torch.zeros_like(self.master[name])
            self.tc[name] = copy16
            self.kind[name] = kind

        for name in CONV_NAMES:
            w = P[f"{name}/weights"]
            if name == "conv1_1":
                add(name + "/w", w.reshape(27, 64).t().contiguous(), None, 0)                     # [64][27], refreshed into the padded [64][64] copy
            else:
                wt = w.permute(3, 0, 1, 2).reshape(w.shape[3], -1)
                add(name + "/w", wt, wt.to(torch.bfloat16).contiguous(), 0)
            add(name + "/b", P[f"{name}/biases"].clone(), None, 0)
        for name in ("score_conv4", "score_conv5", "score_conv4_vertex", "score_conv5_vertex"):
            wt = P[f"{name}/weights"].reshape(512, -1).t().contiguous()                           # [Cout][512]
            add(name + "/w", wt, wt.to(torch.bfloat16).contiguous(), 0)
            add(name + "/b", P[f"{name}/biases"].clone(), None, 0)
        ws = torch.zeros((64, net.num_units), device=dev)                                         # `score` 1x1: [C -> 64 rows][64]
        ws[:C] = P["score/weights"].reshape(net.num_units, C).t()
        add("score/w", ws, ws.to(torch.bfloat16).contiguous(), 0)
        add("score/b", P["score/biases"].clone(), None, 0)
        wv = torch.zeros((128, 128), device=dev)                                                  # `vertex_pred` 1x1: [3C -> 128 rows][128]
        wv[:3 * C] = P["vertex_pred/weights"].reshape(128, 3 * C).t()
        add("vertex_pred/w", wv, wv.to(torch.bfloat16).contiguous(), 0)
        add("vertex_pred/b", P["vertex_pred/biases"].clone(), None, 0)
        for name in ("fc6", "fc7", "fc8"):
            w = P[f"{name}/weights"]                                                              # [in, out]
            npad = (w.shape[1] + 127) // 128 * 128
            wt = torch.zeros((npad, w.shape[0]), device=dev)
            wt[:w.shape[1]] = w.t()
            add(name + "/w", wt, wt.to(torch.float16).contiguous(), 1)
            add(name + "/b", P[f"{name}/biases"].clone(), None, 0)
        self.conv1_tc = conv.conv1_1_weights_to_tc(P["conv1_1/weights"])
        self._refresh_derived()
        self.zero_bias = {n: torch.zeros(n, device=dev) for n in (64, 128, 256, 512)}

    # ------------------------------------------------------------------ derived weight copies
    def _refresh_derived(self):
        """Copies the backward GEMMs read: input-gradient (flipped / transposed) weights of every convolution, [in][out] fp16 copies of
        the fully connected weights, the padded conv1_1 tile."""
        self.dg = {}
        for name in CONV_NAMES[1:]:
            self.dg[name] = _tc_dgrad(self.tc[name + "/w"], 3)
        for name in ("score_conv4", "score_conv5", "score_conv4_vertex", "score_conv5_vertex", "score", "vertex_pred"):
            self.dg[name] = _tc_dgrad(self.tc[name + "/w"], 1)
        self.fc_t = {}
        for name in ("fc6", "fc7", "fc8"):
            w = self.tc[name + "/w"]
            t = torch.empty((w.shape[1], w.shape[0]), dtype=torch.float16, device=w.device)
            check(lib().pcnn_transpose16(ptr(w), w.shape[0], w.shape[1], ptr(t), stream()))
            self.fc_t[name] = t
        self.conv1_tc.zero_()
        self.conv1_tc[:, :27] = self.master["conv1_1/w"].to(torch.bfloat16)

    def export_params(self):
        """Write the fp32 master weights back into net.params (TF layouts) and re-derive the inference copies."""
        P, C = self.net.params, self.C
        for name in CONV_NAMES:
            shp = P[f"{name}/weights"].shape
            if name == "conv1_1":
                P[f"{name}/weights"] = self.master[name + "/w"].t().reshape(shp).contiguous()
            else:
                P[f"{name}/weights"] = self.master[name + "/w"].view(shp[3], shp[0], shp[1], shp[2]).permute(1, 2, 3, 0).contiguous()
            P[f"{name}/biases"] = self.master[name + "/b"].clone()
        for name in ("score_conv4", "score_conv5", "score_conv4_vertex", "score_conv5_vertex"):
            P[f"{name}/weights"] = self.master[name + "/w"].t().reshape(P[f"{name}/weights"].shape).contiguous()
            P[f"{name}/biases"] = self.master[name + "/b"].clone()
        P["score/weights"] = self.master["score/w"][:C].t().reshape(P["score/weights"].shape).contiguous()
        P["score/biases"] = self.master["score/b"].clone()
        P["vertex_pred/weights"] = self.master["vertex_pred/w"][:3 * C].t().reshape(P["vertex_pred/weights"].shape).contiguous()
        P["vertex_pred/biases"] = self.master["vertex_pred/b"].clone()
        for name in ("fc6", "fc7", "fc8"):
            n_out = P[f"{name}/weights"].shape[1]
            P[f"{name}/weights"] = self.master[name + "/w"][:n_out].t().contiguous()
            P[f"{name}/biases"] = self.master[name + "/b"].clone()
        self.net.prepare()

    # ------------------------------------------------------------------ forward (training graph, activations kept)
    def forward(self, data, gt_label_2d, centers, meta_data, extents, gt_poses, points, symmetry, batch_global=None, batch_offset=0):
        net, C, M, T = self.net, self.C, self.master, self.tc
        B, H, W, _ = data.shape
        A = {}                                    # activations by layer name (bf16 NHWC), "<pool>" = pooled tensors
        x = conv.conv1_fused(data, self.conv1_tc, M["conv1_1/b"], PIXEL_MEANS, True)
        A["conv1_1"] = x
        for name in CONV_NAMES[1:]:
            x = conv.conv_bf16(x, T[name + "/w"], M[name + "/b"], 3, True)
            A[name] = x
            if name in POOL_AFTER and name != "conv5_3":
                x = conv.maxpool2x2(x)
                A[name + "/pool"] = x
        c4, c5 = A["conv4_3"], A["conv5_3"]
        s4 = conv.conv_bf16(c4, T["score_conv4/w"], M["score_conv4/b"], 1, True)
        s5 = conv.conv_bf16(c5, T["score_conv5/w"], M["score_conv5/b"], 1, True)
        v4 = conv.conv_bf16(c4, T["score_conv4_vertex/w"], M["score_conv4_vertex/b"], 1, False)
        v5 = conv.conv_bf16(c5, T["score_conv5_vertex/w"], M["score_conv5_vertex/b"], 1, False)
        h, w = H // 8, W // 8
        add_s, add_v = torch.empty_like(s4), torch.empty_like(v4)
        check(lib().pcnn_add_up2_bf16(ptr(s4), ptr(s5), B, h, w, s4.shape[3], ptr(add_s), stream()))
        check(lib().pcnn_add_up2_bf16(ptr(v4), ptr(v5), B, h, w, v4.shape[3], ptr(add_v), stream()))
        lr_s = conv.conv_bf16(add_s, T["score/w"], self.zero_bias[64], 1, False)               # bias added after the up-sampling
        lr_v = conv.conv_bf16(add_v, T["vertex_pred/w"], self.zero_bias[128], 1, False)
        lowres = torch.empty((B, h, w, 4 * C), dtype=torch.float32, device=data.device)
        check(lib().pcnn_pack_lowres(ptr(lr_s), 64, ptr(lr_v), 128, B, h, w, C, ptr(lowres), stream()))
        label = torch.empty((B, H, W), dtype=torch.int32, device=data.device)
        prob = torch.empty((B, H, W, C), dtype=torch.float32, device=data.device)
        score = torch.empty((B, H, W, C), dtype=torch.float32, device=data.device)
        # The dense vertex_pred [B,H,W,3C] (81 MB / frame) is never written: its only consumers — the vertex loss, its gradient and the
        # Hough sampler — read three values per labelled / sampled pixel and form them on demand from `lowres` with k_up8_heads' own
        # operation sequence (heads_common.cuh: bit-identical).  dense_vertex_pred(A) materialises it for inspection.
        check(lib().pcnn_up8_heads(ptr(lowres), ptr(M["score/b"]), ptr(M["vertex_pred/b"]), B, h, w, C, ptr(label), ptr(None), ptr(prob),
                                   ptr(score), stream()))
        A.update(s4=s4, s5=s5, v4=v4, v5=v5, add_s=add_s, add_v=add_v, label_2d=label, lowres=lowres, prob_normalized=prob, score=score)
        # losses on the dense heads (fused kernels; the masks / targets are never materialised)
        ws = train_ops._workspace(data.device)
        cls_out = torch.empty((2,), dtype=torch.float32, device=data.device)
        check(lib().pcnn_loss_cls_hard_raw_fwd(ptr(score), ptr(prob), ptr(gt_label_2d), B, H, W, C, f32(net.threshold_label), ptr(cls_out), ptr(ws),
                                               ctypes.c_size_t(ws.numel()), stream()))
        vtx_out = torch.empty((2,), dtype=torch.float32, device=data.device)
        check(lib().pcnn_vertex_loss_fused_lowres_fwd(ptr(lowres), ptr(M["vertex_pred/b"]), ptr(gt_label_2d), ptr(centers), B, H, W, C,
                                                      f32(self.w_inside), f32(1.0), ptr(vtx_out), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
        A.update(cls_out=cls_out, vtx_out=vtx_out)
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
                 pose_diff=pose_diff, loss_pose_raw=loss_pose, rows=rows, data=data)
        return A

    def dense_vertex_pred(self, A):
        """The dense vertex_pred [B,H,W,3C] of a forward pass (the training step itself never materialises it)."""
        lowres = A["lowres"]
        B, h, w, _ = lowres.shape
        C, M = self.C, self.master
        label = torch.empty((B, 8 * h, 8 * w), dtype=torch.int32, device=lowres.device)
        vertex = torch.empty((B, 8 * h, 8 * w, 3 * C), dtype=torch.float32, device=lowres.device)
        check(lib().pcnn_up8_heads(ptr(lowres), ptr(M["score/b"]), ptr(M["vertex_pred/b"]), B, h, w, C, ptr(label), ptr(vertex), ptr(None),
                                   ptr(None), stream()))
        return vertex

    # ------------------------------------------------------------------ gradient plumbing
    def _emit(self, grads, name, g):
        """A finished gradient tensor: start its all-reduce (SUM over ranks) on the communication stream right away."""
        grads[name] = g
        if self.comm is not None:
            self.comm.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.comm):
                dist.all_reduce(g, op=dist.ReduceOp.SUM)

    def _fc_dgrad(self, dy, name, mask):
        wt = self.fc_t[name]                                    # [in][out_pad] fp16
        M_, K = dy.shape
        N = wt.shape[0]
        out = torch.empty((M_, N), dtype=torch.float16, device=dy.device)
        nbytes = ctypes.c_size_t(0)
        check(lib().pcnn_fc_workspace_bytes(M_, N, K, ctypes.byref(nbytes)))
        ws = workspace("fc", nbytes.value, dy.device)
        check(lib().pcnn_fc_dgrad_f16_tc(ptr(dy), ptr(wt), M_, N, K, ptr(mask), ptr(out), N, ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
        return out

    def _fc_wgrad(self, x, dy, scale=1.0):
        rows, Cin = x.shape
        Cout = dy.shape[1]
        out = torch.empty((Cout, Cin), dtype=torch.float32, device=x.device)
        nbytes = ctypes.c_size_t(0)
        check(lib().pcnn_conv_wgrad_workspace_bytes(1, 1, rows, Cin, Cout, 1, ctypes.byref(nbytes)))
        ws = workspace("wgrad", nbytes.value, x.device)
        check(lib().pcnn_fc_wgrad_f16_tc(ptr(x), ptr(dy), rows, Cin, Cout, f32(scale), ptr(None), f32(0.0), ptr(out), ptr(ws),
                                         ctypes.c_size_t(ws.numel()), stream()))
        return out

    def backward(self, A, gt_label_2d, centers):
        """All parameter gradients of loss = loss_cls + vertex_w * loss_vertex + loss_pose (weight decay is applied in the update).
        Loss normalisers (selected-pixel count, vertex weight sum, ROI rows) are GLOBAL over the ranks."""
        net, C, M, T = self.net, self.C, self.master, self.tc
        data = A["data"]
        B, H, W, _ = data.shape
        h, w = H // 8, W // 8
        dev = data.device
        grads = {}
        rows = A["rows"]
        # ---- global loss normalisers: one all-reduce of [count_cls, sum_w_vertex, rows]
        norm = torch.stack([A["cls_out"][1], A["vtx_out"][1], torch.tensor(float(rows), device=dev)])
        if self.world > 1:
            local = norm.clone()
            dist.all_reduce(norm, op=dist.ReduceOp.SUM)
            A["cls_out"] = torch.stack([A["cls_out"][0] * local[0] / norm[0].clamp(min=1.0), norm[0]])     # this rank's share of the global mean
            A["vtx_out"] = torch.stack([A["vtx_out"][0] * local[1] / norm[1].clamp(min=1e-10), norm[1]])
        rows_global = norm[2]
        # Averagedistance divides by the rows IT sees (capacity rows of this rank); the reference batch sees all of them
        pose_scale = (float(rows) / rows_global).item() if self.world > 1 else 1.0
        A["loss_pose"] = A["loss_pose_raw"] * pose_scale
        # ---- pose head
        # The head's backward GEMMs run on FP16 operands like its forward.  The pose-loss gradients are tiny (a mean over rows x points:
        # 1e-6 .. 1e-4 per element, below fp16's normal range), so the chain is LOSS-SCALED by a dynamic power of two S where it enters fp16 and un-scaled
        # where it leaves (weight gradients, bias sums, the RoiPool gradient); conversions saturate at +-65504.
        D = 4 * C
        dpre = torch.empty((rows, 128), dtype=torch.float16, device=dev)
        check(lib().pcnn_pose_chain_bwd(ptr(A["pose_diff"]), ptr(A["poses_tanh"]), ptr(A["poses_weight"]), rows, D, f32(pose_scale), ptr(dpre), 128,
                                        stream()))
        # dynamic loss scale: a power of two that puts the largest element of the chain's entry point at ~2^11 (one host read; the
        # un-scaled pass above is only used for its maximum, which fp16 represents well enough even when the small elements underflow)
        amax = float(dpre.float().abs().max().item())
        if self.world > 1:
            t = torch.tensor([amax], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX); amax = float(t.item())
        S = 2.0 ** max(0, min(24, int(torch.floor(torch.log2(torch.tensor(2048.0 / max(amax, 1e-30)))).item()))) if amax > 0 else 1.0
        self.pose_loss_scale = S
        check(lib().pcnn_pose_chain_bwd(ptr(A["pose_diff"]), ptr(A["poses_tanh"]), ptr(A["poses_weight"]), rows, D, f32(pose_scale * S), ptr(dpre), 128,
                                        stream()))
        self._emit(grads, "fc8/w", self._fc_wgrad(A["fc7"], dpre, 1.0 / S))
        self._emit(grads, "fc8/b", dpre[:, :D].float().sum(0) / S)
        d7 = self._fc_dgrad(dpre, "fc8", A["fc7"])
        self._emit(grads, "fc7/w", self._fc_wgrad(A["fc6"], d7, 1.0 / S))
        self._emit(grads, "fc7/b", d7.float().sum(0) / S)
        d6 = self._fc_dgrad(d7, "fc7", A["fc6"])
        self._emit(grads, "fc6/w", self._fc_wgrad(A["pool"], d6, 1.0 / S))
        self._emit(grads, "fc6/b", d6.float().sum(0) / S)
        dpool16 = self._fc_dgrad(d6, "fc6", None)                                              # [rows, 25088]
        dpool = torch.empty((rows, 7, 7, 512), dtype=torch.float32, device=dev)
        check(lib().pcnn_half_to_float(ptr(dpool16), ctypes.c_size_t(dpool16.numel()), f32(1.0 / S), ptr(dpool), stream()))
        g5_roi = roi_pooling_op.roi_pool_grad(A["conv5_3"], A["rois"], A["a5"], dpool, 7, 7, 1.0 / 16.0, 0)       # fp32 dense
        g4_roi = roi_pooling_op.roi_pool_grad(A["conv4_3"], A["rois"], A["a4"], dpool, 7, 7, 1.0 / 8.0, 0)
        # ---- FCN heads
        d_sc = torch.empty((B, h, w, 64), dtype=torch.bfloat16, device=dev)
        d_vt = torch.empty((B, h, w, 128), dtype=torch.bfloat16, device=dev)
        dbias = torch.empty((4 * C,), dtype=torch.float32, device=dev)
        ws = workspace("up8_bwd", 4 * B * max(h * ((w + 15) // 16), ((w + 3) // 4) * ((h + 15) // 16)) * 4 * C, dev)
        check(lib().pcnn_up8_heads_bwd_ex(ptr(A["prob_normalized"]), ptr(A["score"]), ptr(gt_label_2d), ptr(A["cls_out"]), f32(1.0),
                                          f32(net.threshold_label), ptr(None), ptr(A["lowres"]), ptr(M["vertex_pred/b"]), ptr(centers),
                                          ptr(A["vtx_out"]), f32(self.vertex_w), f32(self.w_inside), f32(1.0), B, h, w, C, 64, 128, ptr(d_sc),
                                          ptr(d_vt), ptr(dbias), ptr(ws), ctypes.c_size_t(ws.numel()), stream()))
        self._emit(grads, "score/b", dbias[:C].contiguous())
        self._emit(grads, "vertex_pred/b", dbias[C:].contiguous())
        self._emit(grads, "score/w", bw.conv_wgrad(A["add_s"], d_sc, 1))
        self._emit(grads, "vertex_pred/w", bw.conv_wgrad(A["add_v"], d_vt, 1))
        d_add_s = conv.conv_bf16(d_sc, self.dg["score"], self.zero_bias[64], 1, False)
        d_add_v = conv.conv_bf16(d_vt, self.dg["vertex_pred"], self.zero_bias[128], 1, False)
        d_s4, db = bw.relu_bwd(d_add_s, A["s4"], True, want_bias=True)
        self._emit(grads, "score_conv4/b", db)
        d_s5 = torch.empty_like(A["s5"])
        check(lib().pcnn_up2_bwd_bf16(ptr(d_add_s), ptr(A["s5"]), B, h, w, 64, ptr(d_s5), stream()))
        self._emit(grads, "score_conv5/b", bw.relu_bwd(d_s5, None, False, want_bias=True, want_dz=False)[1])
        self._emit(grads, "score_conv4_vertex/b", bw.relu_bwd(d_add_v, None, False, want_bias=True, want_dz=False)[1])
        d_v5 = torch.empty_like(A["v5"])
        check(lib().pcnn_up2_bwd_bf16(ptr(d_add_v), ptr(None), B, h, w, 128, ptr(d_v5), stream()))
        self._emit(grads, "score_conv5_vertex/b", bw.relu_bwd(d_v5, None, False, want_bias=True, want_dz=False)[1])
        c4, c5 = A["conv4_3"], A["conv5_3"]
        self._emit(grads, "score_conv4/w", bw.conv_wgrad(c4, d_s4, 1))
        self._emit(grads, "score_conv5/w", bw.conv_wgrad(c5, d_s5, 1))
        self._emit(grads, "score_conv4_vertex/w", bw.conv_wgrad(c4, d_add_v, 1))
        self._emit(grads, "score_conv5_vertex/w", bw.conv_wgrad(c5, d_v5, 1))
        z512 = self.zero_bias[512]
        g4 = bw.add_to_bf16(conv.conv_bf16(d_s4, self.dg["score_conv4"], z512, 1, False),
                            conv.conv_bf16(d_add_v, self.dg["score_conv4_vertex"], z512, 1, False), g4_roi)
        g5 = bw.add_to_bf16(conv.conv_bf16(d_s5, self.dg["score_conv5"], z512, 1, False),
                            conv.conv_bf16(d_v5, self.dg["score_conv5_vertex"], z512, 1, False), g5_roi)
        # ---- trunk, top down.  g = gradient w.r.t. the (post-ReLU) output of the current layer
        g = g5
        for name in reversed(CONV_NAMES):
            y = A[name]
            if name == "conv4_3":
                # conv4_3 feeds pool4 (gradient routed to the window maxima) AND the heads / RoiPool (g4)
                dz = bw.add_to_bf16(bw.maxpool_relu_bwd(g, y), bw.relu_bwd(g4, y, True))
                db = bw.relu_bwd(dz, None, False, want_bias=True, want_dz=False)[1]
            elif name in POOL_AFTER and name != "conv5_3":
                dz, db = bw.maxpool_relu_bwd(g, y, want_bias=True)
            else:
                dz, db = bw.relu_bwd(g, y, True, want_bias=True)
            self._emit(grads, name + "/b", db)
            if name == "conv1_1":
                # Cin = 3: the weight gradient is the 1x1 tensor-core wgrad on the im2col view of the image (K = tap * 3 + c, the same
                # bf16 (pixel - mean) values the forward MMA consumed); a CUDA-core kernel (pcnn_conv1_wgrad) took 2.6 ms at batch 16
                cols = conv.im2col_c3(data, PIXEL_MEANS)                                       # [B,H,W,64] bf16, 27 columns used
                self._emit(grads, name + "/w", bw.conv_wgrad(cols, dz, 1)[:, :27].contiguous())
                break
            prev = CONV_NAMES[CONV_NAMES.index(name) - 1]
            x_in = A.get(prev + "/pool", A[prev])
            self._emit(grads, name + "/w", bw.conv_wgrad(x_in, dz, 3))
            g = conv.conv_bf16(dz, self.dg[name], self.zero_bias[x_in.shape[3]], 3, False)      # gradient w.r.t. this layer's input
        return grads

    def update(self, grads):
        """accum = mu * accum + (grad + wd * w); w -= lr * accum, on the fp32 masters; 16-bit tensor-core copies refreshed in the same
        kernel, derived copies (input-gradient weights, transposed fc weights) afterwards."""
        if self.comm is not None:
            torch.cuda.current_stream().wait_stream(self.comm)
        for name, g in grads.items():
            w = self.master[name]
            assert g.shape == w.shape, (name, tuple(g.shape), tuple(w.shape))
            c16 = self.tc[name]
            check(lib().pcnn_sgd_momentum(ptr(w), ptr(self.accum[name]), ptr(g), ctypes.c_size_t(w.numel()), f32(self.lr), f32(self.mu), f32(self.wd),
                                          f32(1.0), ptr(c16), int(self.kind[name]), stream()))
        self._refresh_derived()

    def step(self, data, gt_label_2d, centers, meta_data, extents, gt_poses, points, symmetry, batch_global=None, batch_offset=0):
        A = self.forward(data, gt_label_2d, centers, meta_data, extents, gt_poses, points, symmetry, batch_global, batch_offset)
        grads = self.backward(A, gt_label_2d, centers)
        self.update(grads)
        loss_cls, loss_vertex, loss_pose = A["cls_out"][0:1], self.vertex_w * A["vtx_out"][0:1], A["loss_pose"]
        return dict(loss_cls=loss_cls, loss_vertex=loss_vertex, loss_pose=loss_pose, loss=loss_cls + loss_vertex + loss_pose, num_rois=A["num_rois"],
                    grads=grads)
