"""Host-side bindings of the FCN-head kernels (include/posecnn_b200.h, csrc/heads.cu, csrc/train_bwd.cu): the 1x1 heads at 1/8
resolution, the fused x8 up-sampling / softmax / arg-max, and the training step's add + up2, 1/8-resolution pack and loss-gradient
adjoint (lib/networks/vgg16_convs.py:128-163, lib/fcn/train.py:455-465, 564-573).

Every function reads B, h, w and the channel counts from its tensors' shapes, allocates its outputs and launches on the current
stream.  Tensors are NHWC: bf16 for the 1x1-convolution outputs and their gradients, f32 for the head tensor and the dense heads."""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, stream, workspace

SCORE_ROWS = 64     # padded row count of the training step's `score` 1x1 conv (C <= 64), the row stride of its output


def vertex_rows(C: int) -> int:
    """Padded row count of the training step's `vertex_pred` 1x1 conv, the row stride of its output and its gradient: at least 3C
    and a multiple of 64 (the tensor-core conv and wgrad need Cout % 64 == 0); 128 for every C <= 42."""
    return max(128, -(-3 * C // 64) * 64)


def lowres_heads(s4, s5, v4, v5, w_score, w_vertex, num_classes):
    """pcnn_lowres_heads: the 1/8-resolution head tensor [B,h,w,4C] f32 = [score C | vertex 3C] of add = branch4 + up2(branch5).
    s4 / v4 [B,h,w,Cs|Cv] bf16, s5 / v5 [B,h/2,w/2,Cs|Cv]; w_score [Cs][C] f32, w_vertex [Cv][3C] f32, or None for the folded head
    (v4 / v5 already hold the 3C vertex channels, zero padded to Cv)."""
    B, h, w, Cs = s4.shape
    C = num_classes
    lowres = torch.empty((B, h, w, 4 * C), dtype=torch.float32, device=s4.device)
    check(lib().pcnn_lowres_heads(ptr(s4), ptr(s5), ptr(v4), ptr(v5), ptr(w_score), ptr(w_vertex), B, h, w, Cs, v4.shape[3], C,
                                  ptr(lowres), stream()))
    return lowres


def lowres_scores(s4, s5, w_score, num_classes):
    """pcnn_lowres_heads_nv at num_vertex = 0: the segmentation network's score-only head tensor [B,h,w,C] f32 of
    add = s4 + up2(s5); s4 [B,h,w,Cs] bf16, s5 [B,h/2,w/2,Cs], w_score [Cs][C] f32."""
    B, h, w, Cs = s4.shape
    C = num_classes
    lowres = torch.empty((B, h, w, C), dtype=torch.float32, device=s4.device)
    check(lib().pcnn_lowres_heads_nv(ptr(s4), ptr(s5), None, None, ptr(w_score), None, B, h, w, Cs, 0, C, 0, ptr(lowres), stream()))
    return lowres


def up8_scores(lowres, bias_score, prob=False, score=False, out=None):
    """pcnn_up8_heads_nv at num_vertex = 0 on the score-only head tensor lowres [B,h,w,C] f32: returns (label_2d [B,8h,8w] int32,
    prob_normalized [B,8h,8w,C], score [B,8h,8w,C]) f32, None for each of the last two not asked for (neither: the label-only
    call).  out: the three buffers to write instead (None where not wanted); prob / score are then ignored."""
    B, h, w, C = lowres.shape
    if out is None:
        dev, H, W = lowres.device, 8 * h, 8 * w
        f32 = lambda on: torch.empty((B, H, W, C), dtype=torch.float32, device=dev) if on else None
        out = (torch.empty((B, H, W), dtype=torch.int32, device=dev), f32(prob), f32(score))
    label, p, s = out
    check(lib().pcnn_up8_heads_nv(ptr(lowres), ptr(bias_score), None, B, h, w, C, 0, ptr(label), None, ptr(p), ptr(s), stream()))
    return out


def up8_heads(lowres, bias_score, bias_vertex, vertex=False, prob=False, score=False, out=None):
    """pcnn_up8_heads on lowres [B,h,w,4C] f32: returns (label_2d [B,8h,8w] int32, vertex_pred [B,8h,8w,3C], prob_normalized
    [B,8h,8w,C], score [B,8h,8w,C]) f32, None for each of the last three not asked for.  Asking for none of them is the
    label-only call.  out: the four buffers to write instead (None where not wanted); vertex / prob / score are then ignored."""
    B, h, w, C4 = lowres.shape
    C = C4 // 4
    if out is None:
        dev, H, W = lowres.device, 8 * h, 8 * w
        f32 = lambda on, c: torch.empty((B, H, W, c), dtype=torch.float32, device=dev) if on else None
        out = (torch.empty((B, H, W), dtype=torch.int32, device=dev), f32(vertex, 3 * C), f32(prob, C), f32(score, C))
    label, v, p, s = out
    check(lib().pcnn_up8_heads(ptr(lowres), ptr(bias_score), ptr(bias_vertex), B, h, w, C, ptr(label), ptr(v), ptr(p), ptr(s), stream()))
    return out


def add_up2(a4, a5):
    """pcnn_add_up2_bf16: a4 + up2(a5) [B,h,w,C] bf16 (the fixed bilinear conv2d_transpose 4x4 / 2); a5 [B,h/2,w/2,C]."""
    B, h, w, C = a4.shape
    out = torch.empty_like(a4)
    check(lib().pcnn_add_up2_bf16(ptr(a4), ptr(a5), B, h, w, C, ptr(out), stream()))
    return out


def up2_bwd(dadd, y5=None):
    """pcnn_up2_bwd_bf16: the adjoint of add_up2's up-sampling, d a5 [B,h/2,w/2,C] bf16 from dadd [B,h,w,C], masked by y5 > 0
    (the ReLU of a5) when y5 is given."""
    B, h, w, C = dadd.shape
    d5 = torch.empty((B, h // 2, w // 2, C), dtype=torch.bfloat16, device=dadd.device)
    check(lib().pcnn_up2_bwd_bf16(ptr(dadd), ptr(y5), B, h, w, C, ptr(d5), stream()))
    return d5


def pack_lowres(sc, vt, num_classes):
    """pcnn_pack_lowres: the head tensor [B,h,w,4C] f32 from the first C channels of sc [B,h,w,Cs] and the first 3C of
    vt [B,h,w,Cv] (bf16)."""
    B, h, w, Cs = sc.shape
    C = num_classes
    lowres = torch.empty((B, h, w, 4 * C), dtype=torch.float32, device=sc.device)
    check(lib().pcnn_pack_lowres(ptr(sc), Cs, ptr(vt), vt.shape[3], B, h, w, C, ptr(lowres), stream()))
    return lowres


def pack_scores(sc, num_classes):
    """pcnn_pack_lowres_nv at num_vertex = 0: the score-only head tensor [B,h,w,C] f32 from the first C channels of sc [B,h,w,Cs] bf16."""
    B, h, w, Cs = sc.shape
    C = num_classes
    lowres = torch.empty((B, h, w, C), dtype=torch.float32, device=sc.device)
    check(lib().pcnn_pack_lowres_nv(ptr(sc), Cs, None, 0, B, h, w, C, 0, ptr(lowres), stream()))
    return lowres


def up8_scores_bwd(prob, score, gt, cls_out, upstream_cls, threshold, out=None):
    """pcnn_up8_scores_bwd: the gradient of upstream_cls * loss_cls w.r.t. the score-only head tensor.  prob / score [B,8h,8w,C] f32,
    gt [B,8h,8w] int32, cls_out the loss's [value, normaliser].  Returns (d_sc [B,h,w,SCORE_ROWS] bf16, dbias [C] f32); channels past
    C are written as 0.  out: the two buffers to write instead (any channel stride >= C)."""
    B, H, W, C = prob.shape
    h, w, dev = H // 8, W // 8, prob.device
    if out is None:
        out = (torch.empty((B, h, w, SCORE_ROWS), dtype=torch.bfloat16, device=dev), torch.empty((C,), dtype=torch.float32, device=dev))
    d_sc, dbias = out
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_up8_scores_bwd_workspace_bytes(B, h, w, C, ctypes.byref(nbytes)))
    ws = workspace("up8_bwd", nbytes.value, dev)
    check(lib().pcnn_up8_scores_bwd(ptr(prob), ptr(score), ptr(gt), ptr(cls_out), upstream_cls, threshold, B, h, w, C, d_sc.shape[3],
                                    ptr(d_sc), ptr(dbias), ptr(ws), ws.numel(), stream()))
    return out


def up8_heads_bwd(prob, score, gt, cls_out, upstream_cls, threshold, lowres, bias_vertex, centers, vtx_out, upstream_vertex, w_inside,
                  sigma, vertmap=None, extents=None, out=None):
    """pcnn_up8_heads_bwd: the gradient of upstream_cls * loss_cls + upstream_vertex * loss_vertex w.r.t. the head tensor lowres
    [B,h,w,4C].  prob / score [B,8h,8w,C] f32, gt [B,8h,8w] int32, cls_out / vtx_out the losses' [value, normaliser], centers
    [B,C,3]; vertmap [B,8h,8w,3] with extents [C,3] select the 3-D target, neither the 2-D one.  Returns (d_sc [B,h,w,SCORE_ROWS]
    bf16, d_vt [B,h,w,vertex_rows(C)] bf16, dbias [4C] f32); channels past C / 3C are written as 0.  out: the three buffers to
    write instead (any channel strides >= C / 3C)."""
    B, h, w, C4 = lowres.shape
    C, dev = C4 // 4, lowres.device
    if out is None:
        out = (torch.empty((B, h, w, SCORE_ROWS), dtype=torch.bfloat16, device=dev),
               torch.empty((B, h, w, vertex_rows(C)), dtype=torch.bfloat16, device=dev), torch.empty((4 * C,), dtype=torch.float32, device=dev))
    d_sc, d_vt, dbias = out
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_up8_heads_bwd_workspace_bytes(B, h, w, C, ctypes.byref(nbytes)))
    ws = workspace("up8_bwd", nbytes.value, dev)
    check(lib().pcnn_up8_heads_bwd(ptr(prob), ptr(score), ptr(gt), ptr(cls_out), upstream_cls, threshold, ptr(lowres), ptr(bias_vertex),
                                   ptr(centers), ptr(vertmap), ptr(extents), ptr(vtx_out), upstream_vertex, w_inside, sigma, B, h, w, C,
                                   d_sc.shape[3], d_vt.shape[3], ptr(d_sc), ptr(d_vt), ptr(dbias), ptr(ws), ws.numel(), stream()))
    return out
