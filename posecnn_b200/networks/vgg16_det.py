"""vgg16_det — the detection network of lib/networks/vgg16_det.py (NETWORK: VGG16DET) at test time, on the H100-native kernels.

Parameter names and layouts are the reference's (`<layer>/weights`, `<layer>/biases`; conv HWIO, fc [in, out]), so a TF1
checkpoint maps one to one.  The graph of vgg16_det.setup() up to the five tensors lib/fcn/test.py:1727-1729 fetches:

    conv1_1 .. conv5_3, conv_rpn (3x3 + ReLU)      trunk.run_trunk / conv.conv_bf16          csrc/conv_tc.cu
    rpn_cls_score, rpn_bbox_pred (1x1 + ReLU),     one tensor-core kernel, fp32 outputs       csrc/det.cu
      pair softmax -> rpn_cls_prob
    anchors, proposals (TEST: 6000 -> NMS 0.7      rpn_layer/ (radix select, bitmask NMS)     csrc/det.cu
      -> 300 per image)
    crop_pool (crop_and_resize 14x14, max 2x2)     fp16 fc6 operand                           csrc/det.cu
    fc6, fc7 (ReLU), cls_score (ReLU) -> softmax,  split-K wgmma GEMMs                        csrc/fc_tc.cu, csrc/det.cu
      bbox_pred, poses_pred_unnormalized -> tanh
    with meta_data: the test loop's records        det_records.detection_records              csrc/det.cu
      (top box per class, box-fitted translation)

Dropout is the identity (keep_prob 1).  Proposals are per image (the reference runs one image; rois[:,0] is the image index
here), and every output is capacity-shaped with a device row count per image, so the whole forward needs no host
synchronisation and can be captured into a CUDA graph (GraphedForward).  COLOR input only.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import conv, pose_head
from ..det_records import detection_records
from ..rpn_layer.proposal_layer import proposal_layer, rpn_heads
from ..rpn_layer.snippets import generate_anchors_pre
from .trunk import conv_weights_to_tc, run_trunk, trunk_shapes


class vgg16_det:
    def __init__(self, input_format="COLOR", num_classes=22, feature_stride=16, anchor_scales=(4, 8, 16, 32),
                 anchor_ratios=(0.5, 0.75, 1, 1.5, 2), trainable=True, is_train=False, device="cuda"):
        if input_format != "COLOR":
            raise ValueError("vgg16_det runs on COLOR input only (every detection configuration is COLOR)")
        self.input_format = input_format
        self.num_classes = int(num_classes)
        self.feature_stride = int(feature_stride)
        self.anchor_scales = tuple(anchor_scales)
        self.anchor_ratios = tuple(anchor_ratios)
        self.num_anchors = len(self.anchor_scales) * len(self.anchor_ratios)
        self.trainable = trainable
        self.is_train = 1 if is_train else 0
        self.mode = "TRAIN" if is_train else "TEST"
        self.device = torch.device(device)
        self.params: dict[str, torch.Tensor] = {}
        self._tc: dict[str, torch.Tensor] = {}
        self._anchors: dict[tuple, torch.Tensor] = {}
        self.layers: dict[str, torch.Tensor] = {}
        self.points: torch.Tensor | None = None

    # ------------------------------------------------------------------ parameters
    def param_shapes(self):
        C, A = self.num_classes, self.num_anchors
        shapes = trunk_shapes()
        shapes["conv_rpn/weights"] = (3, 3, 512, 512); shapes["conv_rpn/biases"] = (512,)
        shapes["rpn_cls_score/weights"] = (1, 1, 512, 2 * A); shapes["rpn_cls_score/biases"] = (2 * A,)
        shapes["rpn_bbox_pred/weights"] = (1, 1, 512, 4 * A); shapes["rpn_bbox_pred/biases"] = (4 * A,)
        shapes["fc6/weights"] = (7 * 7 * 512, 4096); shapes["fc6/biases"] = (4096,)
        shapes["fc7/weights"] = (4096, 4096); shapes["fc7/biases"] = (4096,)
        shapes["cls_score/weights"] = (4096, C); shapes["cls_score/biases"] = (C,)
        shapes["bbox_pred/weights"] = (4096, 4 * C); shapes["bbox_pred/biases"] = (4 * C,)
        shapes["poses_pred_unnormalized/weights"] = (4096, 4 * C); shapes["poses_pred_unnormalized/biases"] = (4 * C,)
        return shapes

    def init_random(self, seed=0, bias_std=0.0):
        """Seeded Kaiming-normal init (fan-in, gain sqrt 2), biases 0 or N(0, bias_std) — as vgg16_convs.init_random."""
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

    def load(self, data_dict: dict):
        """TF-name dictionary {layer: {'weights': ..., 'biases': ...}} or flat {'layer/weights': ...}."""
        for k, v in data_dict.items():
            if isinstance(v, dict):
                for kk, vv in v.items():
                    self.params[f"{k}/{kk}"] = torch.as_tensor(np.asarray(vv), dtype=torch.float32, device=self.device)
            else:
                self.params[k] = torch.as_tensor(np.asarray(v), dtype=torch.float32, device=self.device)
        self.prepare()
        return self

    def prepare(self):
        """Derive the tensor-core weight layouts once: trunk and conv_rpn [Cout][k*k*Cin] bf16, the two RPN 1x1 layers stacked
        into one [6A][512] bf16 matrix (+ [6A] bias), the fc layers [out padded to x128][in] fp16."""
        P, T = self.params, self._tc
        T.clear()
        for name in trunk_shapes():
            if name.endswith("weights"):
                T[name] = conv_weights_to_tc(P[name])
        T["conv_rpn/weights"] = conv.hwio_to_tc(P["conv_rpn/weights"])
        T["rpn/weights"] = torch.cat([conv.hwio_to_tc(P["rpn_cls_score/weights"]), conv.hwio_to_tc(P["rpn_bbox_pred/weights"])]).contiguous()
        T["rpn/biases"] = torch.cat([P["rpn_cls_score/biases"], P["rpn_bbox_pred/biases"]]).float().contiguous()
        for name in ("fc6", "fc7", "cls_score", "bbox_pred", "poses_pred_unnormalized"):
            T[f"{name}/weights"] = pose_head.fc_weights_to_tc(P[f"{name}/weights"])

    def anchors(self, h, w):
        """generate_anchors_pre for an h x w feature map, on the device (cached per map size)."""
        key = (h, w)
        if key not in self._anchors:
            a, _ = generate_anchors_pre(h, w, self.feature_stride, self.anchor_scales, self.anchor_ratios)
            self._anchors[key] = torch.from_numpy(a).to(self.device)
        return self._anchors[key]

    def set_points(self, points):
        """The object-point table [C,P,3] compute_translations projects (the imdb's _points_all, lov.py:141-158: every class
        truncated to the smallest point count), P <= 4096."""
        pts = torch.as_tensor(points, dtype=torch.float32).to(self.device).contiguous()
        if pts.dim() != 3 or pts.shape[0] != self.num_classes or pts.shape[2] != 3:
            raise ValueError(f"points must be [C,P,3] with C = {self.num_classes}")
        self.points = pts
        return self

    # ------------------------------------------------------------------ forward
    def forward(self, data, sync_rois=True, meta_data=None):
        """Test-time forward.  data [B,H,W,3] u8 BGR (PIXEL_MEANS subtracted in conv1_1's loader) or pre-processed f32, H and W
        multiples of 16; im_info is (H, W) of this blob.  Returns self.layers: conv5_3, conv_rpn, rpn_cls_prob [B,h,w,2A],
        rpn_bbox_pred [B,h,w,4A], rois [B*N,5], rpn_scores [B*N,1], num_rois [B] int32, cls_prob [B*N,C], bbox_pred [B*N,4C],
        poses_tanh [B*N,4C] with N = 300 proposals per image (TEST.RPN_POST_NMS_TOP_N); rows past num_rois[b] are zero boxes
        carrying b, and their head outputs are those of that box.  sync_rois=True reads num_rois back and keeps only the
        proposals each image has (at B = 1: the reference's shapes).

        meta_data [B,>=9] f32 on the device (K = meta_data[b, 0:9]) adds the records of the reference's test loop
        (det_records.detection_records, points from set_points): dets [B*(C-1),7] (b, class, x1, y1, x2, y2, score), poses
        [B*(C-1),7] (quaternion, translation), num_dets [B] int32 and det_trace [B*(C-1),2] (Nelder-Mead iterations,
        evaluations), one slot per (image, class >= 1).  sync_rois=True drops the empty slots: the records of each image in
        ascending class order, whose columns 1: are the reference's `rois` [n,6] at B = 1."""
        if self.is_train:
            raise NotImplementedError("vgg16_det runs at test time only (is_train=False)")
        P, T = self.params, self._tc
        L = self.layers = {}
        B, H, W, _ = data.shape
        assert H % 16 == 0 and W % 16 == 0, "pad the image to a multiple of 16 (lib/utils/blob.py:48-58)"
        c5 = run_trunk(P, T, data)["conv5_3"]
        L["conv5_3"] = c5
        x = conv.conv_bf16(c5, T["conv_rpn/weights"], P["conv_rpn/biases"], 3, True)
        L["conv_rpn"] = x
        A = self.num_anchors
        L["rpn_cls_prob"], L["rpn_bbox_pred"] = rpn_heads(x, T["rpn/weights"], T["rpn/biases"], A)
        h, w = x.shape[1], x.shape[2]
        rois, scores, num = proposal_layer(L["rpn_cls_prob"], L["rpn_bbox_pred"], (H, W, 1.0), self.mode, self.feature_stride,
                                           self.anchors(h, w), A)
        L["rois"], L["rpn_scores"], L["num_rois"] = rois, scores, num
        x = pose_head.crop_pool(c5, rois, self.feature_stride)                   # pool5 [B*N, 7*7*512] fp16, (h, w, c)
        x = pose_head.fc(x, T["fc6/weights"], P["fc6/biases"], "relu")           # fc6 + ReLU (drop6: keep_prob 1)
        x = pose_head.fc(x, T["fc7/weights"], P["fc7/biases"], "relu")           # fc7 + ReLU (drop7: keep_prob 1)
        # The three heads run image by image: fc_tc's split-K plan depends on the row count, and one plan per image keeps every
        # image's outputs independent of the batch it runs in (fc6 / fc7 have one split at any N >= 1 image's rows).
        per_image = x.split(rois.shape[0] // B)
        heads = {"cls_score": "relu", "bbox_pred": "none", "poses_pred_unnormalized": "tanh"}
        out = {k: torch.cat([pose_head.fc(xi, T[f"{k}/weights"], P[f"{k}/biases"], act, torch.float32) for xi in per_image])
               for k, act in heads.items()}
        L["cls_score"] = out["cls_score"]
        L["cls_prob"] = pose_head.softmax_rows(out["cls_score"])
        L["bbox_pred"] = out["bbox_pred"]
        L["poses_tanh"] = out["poses_pred_unnormalized"]
        if meta_data is not None:
            if self.points is None:
                raise ValueError("the records need the object-point table: call set_points first")
            L["dets"], L["poses"], L["num_dets"], L["det_trace"] = detection_records(
                L["cls_prob"], L["bbox_pred"], L["poses_tanh"], rois, num, (H, W), meta_data, self.points)
        if sync_rois:
            counts = num.tolist()   # the one host read the reference's data-dependent shapes require
            per = rois.shape[0] // B
            idx = torch.cat([torch.arange(b * per, b * per + n, device=rois.device) for b, n in enumerate(counts)])
            for k in ("rois", "rpn_scores", "cls_score", "cls_prob", "bbox_pred", "poses_tanh"):
                L[k] = L[k].index_select(0, idx)
            if meta_data is not None:
                filled = (L["dets"][:, 1] > 0).nonzero().squeeze(1)
                for k in ("dets", "poses", "det_trace"):
                    L[k] = L[k].index_select(0, filled)
        return L


class GraphedForward:
    """vgg16_det.forward captured once into a CUDA graph (every shape is static: proposals are capacity buffers with a device
    count per image, records fixed slots per (image, class)).  With meta_data the graph includes the records stage.
    __call__(data, meta_data) copies the batch (and its meta data) into the captured inputs and replays."""

    def __init__(self, net: vgg16_det, data: torch.Tensor, warmup: int = 2, meta_data: torch.Tensor | None = None):
        self.net = net
        self.s_data = data.clone()
        self.s_meta = None if meta_data is None else meta_data.clone()
        side = torch.cuda.Stream(device=data.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                net.forward(self.s_data, sync_rois=False, meta_data=self.s_meta)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.layers = dict(net.forward(self.s_data, sync_rois=False, meta_data=self.s_meta))

    def __call__(self, data: torch.Tensor, meta_data: torch.Tensor | None = None):
        self.s_data.copy_(data, non_blocking=True)
        if meta_data is not None:
            if self.s_meta is None:
                raise ValueError("this graph was captured without meta_data")
            self.s_meta.copy_(meta_data, non_blocking=True)
        self.graph.replay()
        return self.layers
