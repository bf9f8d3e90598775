"""vgg16_convs — the PoseCNN network of lib/networks/vgg16_convs.py on the H100-native kernels.

Mirrors the reference class (constructor arguments, layer names, parameter names `<layer>/weights`,
`<layer>/biases` in TF layouts: conv HWIO, fc [in, out]) so that a TF1 checkpoint / VGG16 .npy
dictionary (lib/networks/network.py:71-107) maps one to one.  The graph of
vgg16_convs.setup() (vgg16_convs.py:79-212) is executed eagerly on one CUDA stream:

    conv1_1 .. conv5_3 (+ _p trunk for RGBD)   wgmma implicit GEMM, bf16 x bf16 -> fp32   csrc/conv_tc.cu
    score / vertex heads                         1x1 on wgmma + fused bilinear/softmax     csrc/heads.cu
                                                 (score heads only on the segmentation network: vertex_reg_2d=False, vertex_reg_3d=False)
    hough_voting_gpu                             csrc/hough_vote.cu
    roi_pool x2 + add, fc6-fc8, tanh             csrc/fc_tc.cu (fused pooling, split-K wgmma GEMMs, fused epilogues)
    adaptation: fc9, domain_score / prob / label  fc9 on csrc/fc_tc.cu, the 256 -> 2 tail in one launch (csrc/domain.cu)

PyTorch supplies device memory and streams only.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import conv, heads, pose_head
from ..hough_voting_gpu_layer import hough_voting_gpu_op
from ..roi_pooling_layer import roi_pooling_op
from ..utils import nms as dev_nms
from .trunk import PIXEL_MEANS, VGG_CFG, conv_weights_to_tc, run_trunk, trunk_shapes  # noqa: F401


class vgg16_convs:
    def __init__(self, input_format="COLOR", num_classes=22, num_units=64, scales=(1.0,), threshold_label=1.0,
                 vote_threshold=-1.0, vertex_reg_2d=True, vertex_reg_3d=None, pose_reg=True, adaptation=False,
                 trainable=True, is_train=False, device="cuda", fold_vertex_head=True):
        self.input_format = input_format
        # fold_vertex_head: multiply the vertex_pred matrix (128 -> 3C) into score_conv4_vertex / score_conv5_vertex
        # (512 -> 128) once at prepare() time; exact algebra (no non-linearity between them, vgg16_convs.py:151-163),
        # removes 86 % of the 1/8-resolution matrix work.  False keeps the reference's intermediate layers.
        # vertex_head: False only for the segmentation network, built by giving vertex_reg_2d=False AND vertex_reg_3d=False
        # (vgg16_convs.py:79-149, the vertex block :151-212 skipped): score heads only, pose_reg and adaptation ignored, as the
        # reference ignores them outside vertex_reg_2d.  vertex_reg_3d left at its default (None, read as False) keeps the vertex
        # head, so a network built as vgg16_convs(vertex_reg_2d=False) has the parameter set and graph it always had.
        self.vertex_head = bool(vertex_reg_2d) or vertex_reg_3d is not False
        self.fold_vertex_head = bool(fold_vertex_head) and 3 * num_classes <= 128 and self.vertex_head
        self.num_classes = num_classes
        self.num_units = num_units
        self.threshold_label = threshold_label
        vertex_reg_3d = bool(vertex_reg_3d)
        self.vertex_reg = vertex_reg_2d or vertex_reg_3d
        self.vertex_reg_2d = vertex_reg_2d
        self.vertex_reg_3d = vertex_reg_3d
        self.scales = tuple(float(v) for v in scales)
        self.pose_reg = pose_reg
        # domain classifier on pool_score (vgg16_convs.py:202-212); built only where the reference builds it
        self.adaptation = bool(adaptation)
        self.domain_branch = self.adaptation and bool(vertex_reg_2d) and bool(pose_reg)
        # vgg16_convs.py:18-29
        self.is_train = 1 if is_train else 0
        self.skip_pixels = 10
        self.vote_threshold = vote_threshold
        self.vote_percentage = 0.02
        self.nms_thresh = 0.5                      # lib/fcn/test.py:198
        self.device = torch.device(device)
        self.params: dict[str, torch.Tensor] = {}
        self._tc: dict[str, torch.Tensor] = {}
        self.layers: dict[str, torch.Tensor] = {}

    # ------------------------------------------------------------------ parameters
    def param_shapes(self):
        C, U = self.num_classes, self.num_units
        shapes = {}
        trunks = [""] + (["_p"] if self.input_format == "RGBD" else [])
        for sfx in trunks:
            shapes.update(trunk_shapes(sfx))
        cin_head = 1024 if self.input_format == "RGBD" else 512
        vertex_heads = (("score_conv5_vertex", 128), ("score_conv4_vertex", 128)) if self.vertex_head else ()
        for name, co in (("score_conv5", U), ("score_conv4", U)) + vertex_heads:
            shapes[f"{name}/weights"] = (1, 1, cin_head if not name.endswith("vertex") else 512, co)
            shapes[f"{name}/biases"] = (co,)
        shapes["score/weights"] = (1, 1, U, C); shapes["score/biases"] = (C,)
        if not self.vertex_head:
            return shapes
        shapes["vertex_pred/weights"] = (1, 1, 128, 3 * C); shapes["vertex_pred/biases"] = (3 * C,)
        shapes["fc6/weights"] = (7 * 7 * 512, 4096); shapes["fc6/biases"] = (4096,)
        shapes["fc7/weights"] = (4096, 4096); shapes["fc7/biases"] = (4096,)
        shapes["fc8/weights"] = (4096, 4 * C); shapes["fc8/biases"] = (4 * C,)
        if self.domain_branch:   # after fc8: the seeded init of every other parameter is unchanged
            shapes["fc9/weights"] = (7 * 7 * 512, 256); shapes["fc9/biases"] = (256,)
            shapes["domain_score/weights"] = (256, 2); shapes["domain_score/biases"] = (2,)
        return shapes

    def init_random(self, seed=0, bias_std=0.0):
        """Seeded Kaiming-normal init (fan-in, gain sqrt 2), biases 0 — NOT the reference's
        truncated_normal(0.001), which makes the net output background only (SURVEY finding 10)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        for name, shp in self.param_shapes().items():
            if name.endswith("weights"):
                fan_in = int(np.prod(shp[:-1]))
                t = torch.randn(shp, generator=g) * math.sqrt(2.0 / fan_in)
            else:
                t = torch.randn(shp, generator=g) * bias_std if bias_std > 0 else torch.zeros(shp)
            self.params[name] = t.to(self.device)
        self.prepare()
        return self

    def calibrate_background(self, data, meta_data, extents, background_fraction=0.75, **forward_kwargs):
        """Benchmark-harness helper: a randomly initialised net labels (almost) every pixel as foreground, which is
        not what the Hough layer sees in use.  Shift `score/biases[0]` so that about `background_fraction` of the
        pixels of this batch are labelled background (YCB-like fill, SURVEY.md §8(d)).  Declared in bench.py's config."""
        self.forward(data, meta_data, extents, want_prob=False, sync_rois=False, **forward_kwargs)
        C = self.num_classes
        B, H, W, _ = data.shape
        label = torch.empty((B, H, W), dtype=torch.int32, device=data.device)
        if self.vertex_head:
            bufs = (label, torch.empty((B, H, W, 3 * C), dtype=torch.float32, device=data.device), None, None)
        lowres = self._last_lowres
        bias = self.params["score/biases"]
        base = float(bias[0])

        def fg_fraction(b0):
            bias[0] = b0
            if self.vertex_head:
                lab = heads.up8_heads(lowres, bias, self.params["vertex_pred/biases"], out=bufs)[0]
            else:
                lab = heads.up8_scores(lowres, bias, out=(label, None, None))[0]
            return float((lab > 0).float().mean())

        scale = float(lowres[..., :C].abs().max()) + 1.0
        lo, hi = base - scale, base + scale          # foreground fraction decreases as the background bias grows
        for _ in range(24):
            mid = 0.5 * (lo + hi)
            if fg_fraction(mid) > 1.0 - background_fraction:
                lo = mid
            else:
                hi = mid
        bias[0] = hi
        return hi - base

    def load(self, data_dict: dict):
        """TF-name dictionary {layer: {'weights': ..., 'biases': ...}} (VGG16 .npy, network.py:71-107) or flat
        {'layer/weights': ...}."""
        for k, v in data_dict.items():
            if isinstance(v, dict):
                for kk, vv in v.items():
                    self.params[f"{k}/{kk}"] = torch.as_tensor(np.asarray(vv), dtype=torch.float32, device=self.device)
                    if self.input_format == "RGBD" and k.startswith("conv") and "score" not in k:
                        self.params[f"{k}_p/{kk}"] = self.params[f"{k}/{kk}"].clone()  # '_p' duplicate scopes, network.py:88-95
            else:
                self.params[k] = torch.as_tensor(np.asarray(v), dtype=torch.float32, device=self.device)
        self.prepare()
        return self

    def prepare(self):
        """Derive the tensor-core weight layouts once ([Cout][k*k*Cin] bf16)."""
        P, T = self.params, self._tc
        T.clear()
        for name, shp in self.param_shapes().items():
            if not name.endswith("weights") or name.startswith("fc") or name in ("score/weights", "vertex_pred/weights", "domain_score/weights"):
                continue
            T[name] = conv_weights_to_tc(P[name])
        T["score/w"] = P["score/weights"].reshape(self.num_units, self.num_classes).contiguous()
        if not self.vertex_head:
            return
        for name in ("fc6", "fc7", "fc8"):
            T[f"{name}/weights"] = pose_head.fc_weights_to_tc(P[f"{name}/weights"])   # [out (padded to x128), in] fp16
        if self.domain_branch:
            T["fc9/weights"] = pose_head.fc_weights_to_tc(P["fc9/weights"])                # [256][25088] fp16
            T["domain_score/w"] = P["domain_score/weights"].t().contiguous()               # [2][256] f32
        T["vertex_pred/w"] = P["vertex_pred/weights"].reshape(128, 3 * self.num_classes).contiguous()
        if self.fold_vertex_head:
            Wp = T["vertex_pred/w"].double()
            for name in ("score_conv4_vertex", "score_conv5_vertex"):
                w = P[f"{name}/weights"].reshape(-1, 128).double() @ Wp              # [512, 3C]
                b = P[f"{name}/biases"].double() @ Wp                                # [3C]
                wpad = torch.zeros((1, 1, w.shape[0], 128), dtype=torch.float32, device=w.device)
                wpad[0, 0, :, :w.shape[1]] = w.float()
                bpad = torch.zeros((128,), dtype=torch.float32, device=w.device)
                bpad[:b.shape[0]] = b.float()
                T[f"{name}/folded_weights"], T[f"{name}/folded_biases"] = conv.hwio_to_tc(wpad), bpad

    # ------------------------------------------------------------------ graph pieces
    def _trunk(self, data, sfx=""):
        """13 x (conv3x3 + bias + ReLU), 4 x max-pool (vgg16_convs.py:80-97): trunk.run_trunk on this network's weights."""
        return run_trunk(self.params, self._tc, data, sfx)

    def forward(self, data, meta_data, extents, poses=None, data_p=None, want_prob=False, sync_rois=True, want_score=False,
                dense_vertex=None, batch_global=None, batch_offset=0, depth=None, refine_depth=None, refine_points=None,
                depth_factor=10000.0, estimate_depth=None, estimate_keys=None, estimate_rgb=False):
        """Inference / forward pass.  data [B,H,W,3] (u8 BGR or pre-processed f32), H, W multiples of 16
        (pad_im, lib/utils/blob.py:48-58).  Returns self.layers with the reference's layer names.

        dense_vertex=False: the pipeline mode — `vertex_pred` [B,H,W,3C] (81 MB / frame, only read back by the
        reference for visualisation, lib/fcn/test.py:587-599) is not materialised; Houghvotinggpu samples the vertex
        head on demand from the 1/8-resolution head tensor (bit-identical ROIs, pcnn_hough_vote_fwd_ex).  The default (None) is
        True where the network has a vertex head; a segmentation network (no vertex head) returns conv4_3, conv5_3,
        score_conv4, score_conv5, label_2d and prob_normalized / score when asked for, and refuses every vertex output.
        batch_global / batch_offset: this call is the image shard [batch_offset, batch_offset + B) of a batch of
        batch_global images (SURVEY.md §8(e)): ROI budget 128 // batch_global per image, global batch indices.
        refine_depth [B,H,W] f32 raw depth (sensor units, z = depth / depth_factor) + refine_points [C,P,3] (the model point
        table in this network's class numbering): at test time, refine the detections against the depth (pose_refine.py,
        TEST.POSE_REFINE) -> detections_poses_refined / detections_poses_icp / detections_icp_info, capacity-shaped like the
        other detections_* outputs.  Without refine_depth nothing else runs.
        estimate_depth [B,H,W] f32 raw depth at the network's resolution (+ estimate_keys [B] int64 Philox keys, default the global
        image indices): on a vertex_reg_3d network at test time, estimate the poses from the object coordinates of the
        1/8-resolution head and the depth (coord_pose.py, lib/fcn/test.py:1381-1399) -> estimate_poses [B,C,3,4], estimate_info
        [B,C,6] and the records detections_rois [B*(C-1),6] / detections_poses [B*(C-1),7] / num_detections [1] (im_scale =
        scales[0]).  Without estimate_depth nothing else runs.
        estimate_rgb=True: on the same networks, the colour-only estimate from the object coordinates alone (coord_pose.py
        estimate_poses_2d, lib/fcn/test.py:1362-1380, keys as for estimate_depth) -> estimate_poses_rgb, estimate_info_rgb,
        detections_rois_rgb, detections_poses_rgb, num_detections_rgb, shaped like the depth estimate's outputs.
        On a vertex_reg_3d network, refine_depth + refine_points refine the depth estimate's detections_* records (test.py:1403-1416;
        for C = 2 pass refine_points in the dataset's numbering and map the outputs with utils/results.py::to_dataset_classes)."""
        C = self.num_classes
        if dense_vertex is None:
            dense_vertex = self.vertex_head
        if not self.vertex_head and (dense_vertex or estimate_depth is not None or estimate_rgb or refine_depth is not None):
            raise ValueError("a segmentation network (vertex_reg_2d and vertex_reg_3d both False) has no vertex head: dense_vertex, "
                             "estimate_depth, estimate_rgb and refine_depth need one")
        coord_net = not self.is_train and self.vertex_reg_3d and not self.vertex_reg_2d
        if estimate_depth is not None and not coord_net:
            raise ValueError("estimate_depth estimates poses from object coordinates: it needs is_train=False and vertex_reg_3d "
                             "without vertex_reg_2d")
        if estimate_rgb and not coord_net:
            raise ValueError("estimate_rgb estimates poses from object coordinates: it needs is_train=False and vertex_reg_3d "
                             "without vertex_reg_2d")
        if refine_depth is not None and not (coord_net and estimate_depth is not None) and \
                (self.is_train or not (self.vertex_reg_2d and self.pose_reg)):
            raise ValueError("refine_depth refines the test-time detections: it needs is_train=False and vertex_reg_2d with pose_reg, "
                             "or vertex_reg_3d with estimate_depth")
        L = self.layers = {}
        P, T = self.params, self._tc
        B, H, W, _ = data.shape
        assert H % 16 == 0 and W % 16 == 0, "pad the image to a multiple of 16 (lib/utils/blob.py:48-58)"
        f = self._trunk(data)
        c4, c5 = f["conv4_3"], f["conv5_3"]
        L["conv4_3"], L["conv5_3"] = c4, c5
        if self.input_format == "RGBD":
            # data_p: the pre-processed depth blob [B,H,W,3] f32, or depth= the raw depth image [B,H,W] f32 (fused blob)
            fp = self._trunk(depth if depth is not None else data_p, "_p")
            h4, h5 = torch.cat([c4, fp["conv4_3"]], 3), torch.cat([c5, fp["conv5_3"]], 3)  # concat_conv4/5
        else:
            h4, h5 = c4, c5
        # 1x1 convolutions on the tensor cores (score_conv4/5 have a ReLU, the vertex ones do not)
        s5 = conv.conv_bf16(h5, T["score_conv5/weights"], P["score_conv5/biases"], 1, True)
        s4 = conv.conv_bf16(h4, T["score_conv4/weights"], P["score_conv4/biases"], 1, True)
        L["score_conv4"], L["score_conv5"] = s4, s5
        if not self.vertex_head:
            # the segmentation network's graph ends here (test fetch: label_2d, prob_normalized, lib/fcn/test.py:233-234); its head
            # tensor holds the C score channels only
            lowres = heads.lowres_scores(s4, s5, T["score/w"], C)
            self._last_lowres = lowres
            L["label_2d"], prob, score = heads.up8_scores(lowres, P["score/biases"], prob=want_prob, score=want_score)
            if want_prob:
                L["prob_normalized"] = prob
            if want_score:
                L["score"] = score
            return L
        if self.fold_vertex_head:
            v5 = conv.conv_bf16(c5, T["score_conv5_vertex/folded_weights"], T["score_conv5_vertex/folded_biases"], 1, False)
            v4 = conv.conv_bf16(c4, T["score_conv4_vertex/folded_weights"], T["score_conv4_vertex/folded_biases"], 1, False)
            w_vertex = None
        else:
            v5 = conv.conv_bf16(c5, T["score_conv5_vertex/weights"], P["score_conv5_vertex/biases"], 1, False)
            v4 = conv.conv_bf16(c4, T["score_conv4_vertex/weights"], P["score_conv4_vertex/biases"], 1, False)
            L["score_conv4_vertex"], L["score_conv5_vertex"] = v4, v5
            w_vertex = T["vertex_pred/w"]
        lowres = heads.lowres_heads(s4, s5, v4, v5, T["score/w"], w_vertex, C)
        self._last_lowres = lowres
        label, vertex, prob, score = heads.up8_heads(lowres, P["score/biases"], P["vertex_pred/biases"], vertex=dense_vertex,
                                                     prob=want_prob, score=want_score)
        L["label_2d"] = label
        if dense_vertex:
            L["vertex_pred"] = vertex
        if want_prob:
            L["prob_normalized"] = prob
        if want_score:
            L["score"] = score
        if not self.vertex_reg_2d:
            if not estimate_rgb and estimate_depth is None:
                return L
            from ..coord_pose import assemble_records, estimate_poses_2d, estimate_poses_3d
            keys = estimate_keys if estimate_keys is not None else \
                torch.arange(batch_offset, batch_offset + B, dtype=torch.int64, device=data.device)
            if estimate_rgb:
                est = estimate_poses_2d(label, meta_data, extents, keys, lowres=lowres, bias_vertex=P["vertex_pred/biases"])
                L["estimate_poses_rgb"], L["estimate_info_rgb"] = est["poses"], est["info"]
                L["detections_rois_rgb"], L["detections_poses_rgb"], L["num_detections_rgb"] = assemble_records(
                    est["poses"], extents, meta_data, self.scales[0], batch_offset)
            if estimate_depth is not None:
                est = estimate_poses_3d(label, estimate_depth, meta_data, extents, keys, lowres=lowres, bias_vertex=P["vertex_pred/biases"],
                                        factor_depth=depth_factor)
                L["estimate_poses"], L["estimate_info"] = est["poses"], est["info"]
                L["detections_rois"], L["detections_poses"], L["num_detections"] = assemble_records(
                    est["poses"], extents, meta_data, self.scales[0], batch_offset)
                if refine_depth is not None:
                    self._refine(L, label, refine_depth, meta_data, refine_points, depth_factor, batch_offset)
            return L
        Bg = B if batch_global is None else int(batch_global)
        box, pose, target, weight, domain, num_rois, status = hough_voting_gpu_op.hough_voting_gpu_capacity(
            label, vertex, extents, meta_data, poses, self.is_train, self.vote_threshold, self.vote_percentage, self.skip_pixels,
            lowres=lowres, bias_vertex=P["vertex_pred/biases"], batch_global=Bg, batch_offset=batch_offset)
        # fixed-shape pose head over the ROI capacity of this shard (rows beyond num_rois are all-zero ROIs)
        cap_rows = max(1, min(box.shape[0], (128 // Bg) * B * (9 if self.is_train else 1)))
        rois = box[:cap_rows]
        L["rois_capacity"], L["num_rois"] = rois, num_rois
        L["hough_status"] = status      # device status word (overflow bit, scan/recount mismatches); read in the sync path
        L["poses_init"], L["poses_target"], L["poses_weight"] = pose[:cap_rows], target[:cap_rows], weight[:cap_rows]
        if self.pose_reg:
            if self.is_train:
                # training graph: the reference ops with arg-max outputs for RoiPoolGrad (roi_pooling_op_grad.py:29-50)
                rl = rois if not batch_offset else torch.cat([rois[:, :1] - float(batch_offset), rois[:, 1:]], 1)
                p5, a5 = roi_pooling_op.roi_pool(c5, rl, 7, 7, 1.0 / 16.0, 0)
                p4, a4 = roi_pooling_op.roi_pool(c4, rl, 7, 7, 1.0 / 8.0, 0)
                L["pool5_argmax"], L["pool4_argmax"] = a5, a4
                x = (p5 + p4).reshape(cap_rows, -1).clamp(-65504.0, 65504.0).to(torch.float16)   # pool_score, flatten (h, w, c)
            else:
                x = pose_head.roi_pool_pair(c5, c4, rois, 7, 7, 1.0 / 16.0, 1.0 / 8.0, batch_offset)
            L["pool_score"] = x
            x = pose_head.fc(x, T["fc6/weights"], P["fc6/biases"], "relu")             # fc6 + ReLU (dropout keep_prob = 1)
            L["fc6"] = x
            x = pose_head.fc(x, T["fc7/weights"], P["fc7/biases"], "relu")
            L["fc7"] = x
            L["poses_tanh"] = pose_head.fc(x, T["fc8/weights"], P["fc8/biases"], "tanh", torch.float32)   # fc8 + tanh
            if self.domain_branch:
                # gradient_reversal is the identity forward; fc9 + ReLU (drop9 keep_prob = 1), domain_score + ReLU, softmax, argmax
                if self.is_train:
                    L["label_domain"] = domain[:cap_rows]
                h9 = pose_head.fc(L["pool_score"], T["fc9/weights"], P["fc9/biases"], "relu")
                L["fc9"] = h9
                L.update(pose_head.domain_tail(h9, T["domain_score/w"], P["domain_score/biases"]))
        if not self.is_train:
            # test-time post-processing on the device: per-class NMS + pose assembly (lib/utils/nms.py, test.py:197-211)
            keep, d_rois, d_poses, d_n = dev_nms.nms_pose_capacity(rois, L["poses_init"], L.get("poses_tanh"), num_rois,
                                                                   self.nms_thresh, per_image=True, num_classes=C)
            L["detections_keep"], L["detections_rois"], L["detections_poses"], L["num_detections"] = keep, d_rois, d_poses, d_n
            if refine_depth is not None:
                self._refine(L, label, refine_depth, meta_data, refine_points, depth_factor, batch_offset)
        if sync_rois:
            host = torch.cat([num_rois, status[:2]]).tolist()  # the one host read the op's data-dependent shape requires
            n = max(1, host[0])
            hough_voting_gpu_op.check_status(host[1], host[2])
            L["rois"] = rois[:n]
            for k in ("poses_init", "poses_target", "poses_weight"):
                L[k] = L[k][:n]
            if self.pose_reg:
                L["poses_tanh"] = L["poses_tanh"][:n]
            for k in ("label_domain", "fc9", "domain_score", "domain_prob", "domain_label"):
                if k in L:
                    L[k] = L[k][:n]
        return L


    def _refine(self, L, label, refine_depth, meta_data, refine_points, depth_factor, batch_offset):
        """TEST.POSE_REFINE on L's detections_* records -> detections_poses_refined / _icp / detections_icp_info."""
        if refine_points is None:
            raise ValueError("refine_depth needs refine_points (the [C,P,3] model point table)")
        from ..pose_refine import refine_poses
        rois = L["detections_rois"]
        if rois.shape[1] == 6:          # the object-coordinate records have no score column
            rois = torch.nn.functional.pad(rois, (0, 1))
        ref = refine_poses(label, refine_depth, meta_data, rois, L["detections_poses"], refine_points, num_rows=L["num_detections"],
                           factor_depth=depth_factor, batch_offset=batch_offset)
        L["detections_poses_refined"], L["detections_poses_icp"] = ref["poses_refined"], ref["poses_icp"]
        L["detections_icp_info"] = ref["icp_info"]


class GraphedForward:
    """The whole forward pass captured once into a CUDA graph (all shapes are static: Hough outputs are capacity
    buffers + a device row count).  Replays remove the ~60 per-launch host calls of the eager path."""

    def __init__(self, net: vgg16_convs, data: torch.Tensor, meta_data: torch.Tensor, extents: torch.Tensor, warmup: int = 2,
                 pack_records: bool = False, **forward_kwargs):
        """pack_records: also capture parallel.pack_detections (the fixed-size post-NMS records a rank all-gathers)
        into the graph -> self.layers["records"]; forward_kwargs go to net.forward (dense_vertex, batch_global, ...)."""
        self.net = net
        kw = dict(sync_rois=False)
        kw.update(forward_kwargs)

        def run():
            L = dict(net.forward(self.s_data, self.s_meta, self.s_ext, **kw))
            if pack_records:
                from .. import parallel
                L["records"] = parallel.pack_detections(L)
            return L
        # refine_depth / estimate_depth are static inputs like data: replays read the copies that __call__ makes
        self.s_depth = kw["refine_depth"].clone() if kw.get("refine_depth") is not None else None
        if self.s_depth is not None:
            kw["refine_depth"] = self.s_depth
        self.s_est_depth = kw["estimate_depth"].clone() if kw.get("estimate_depth") is not None else None
        if self.s_est_depth is not None:
            kw["estimate_depth"] = self.s_est_depth
        self.s_data = data.clone()
        self.s_meta = meta_data.clone()
        self.s_ext = extents.clone()
        side = torch.cuda.Stream(device=data.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.layers = run()

    def __call__(self, data: torch.Tensor, meta_data: torch.Tensor | None = None, refine_depth: torch.Tensor | None = None,
                 estimate_depth: torch.Tensor | None = None):
        self.s_data.copy_(data, non_blocking=True)
        if meta_data is not None:
            self.s_meta.copy_(meta_data, non_blocking=True)
        if refine_depth is not None:
            if self.s_depth is None:
                raise ValueError("this graph was captured without refine_depth")
            self.s_depth.copy_(refine_depth, non_blocking=True)
        if estimate_depth is not None:
            if self.s_est_depth is None:
                raise ValueError("this graph was captured without estimate_depth")
            self.s_est_depth.copy_(estimate_depth, non_blocking=True)
        self.graph.replay()
        return self.layers
