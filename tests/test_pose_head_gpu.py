"""Pose-regression head on own kernels (csrc/fc_tc.cu): fused RoiPool pair, split-K wgmma fully connected layers,
and the two pipeline extensions of Houghvotinggpu (vertex values sampled from the low-resolution head tensor; image
shards of a larger batch).  Reference: lib/networks/vgg16_convs.py:177-197, lib/networks/network.py:392-422,
lib/roi_pooling_layer/roi_pooling_op_gpu.cu.cc:19-101, lib/hough_voting_gpu_layer/hough_voting_gpu_op.cu.cc:733."""
import numpy as np
import pytest
import torch

from posecnn_b200 import synth

pytestmark = pytest.mark.gpu


def _rois(n, B, W, H, seed):
    g = np.random.default_rng(seed)
    r = np.zeros((n, 7), np.float32)
    r[:, 0] = g.integers(0, B, n)
    r[:, 1] = g.integers(1, 22, n)
    x1, y1 = g.uniform(-20, W - 40, n), g.uniform(-20, H - 40, n)
    r[:, 2], r[:, 3] = x1, y1
    r[:, 4], r[:, 5] = x1 + g.uniform(10, 300, n), y1 + g.uniform(10, 300, n)
    r[-1] = 0.0                                   # an all-zero row (the padding rows of the capacity buffer)
    r[-2, 2:6] = (0, 0, W - 1, H - 1)             # a whole-image ROI
    return r


def test_roi_pool_pair_equals_two_roi_pools(cuda):
    """k_roi_pool_pair == fp16(RoiPool(conv5_3, 1/16) + RoiPool(conv4_3, 1/8)) of the parity-tested RoiPool op: exact."""
    from posecnn_b200 import pose_head
    from posecnn_b200.roi_pooling_layer import roi_pooling_op as rop
    g = torch.Generator().manual_seed(0)
    B, C = 3, 512
    f5 = torch.randn(B, 30, 40, C, generator=g).to(torch.bfloat16).to(cuda)
    f4 = torch.randn(B, 60, 80, C, generator=g).to(torch.bfloat16).to(cuda)
    rois = torch.from_numpy(_rois(37, B, 640, 480, 1)).to(cuda)
    got = pose_head.roi_pool_pair(f5, f4, rois)
    p5, _ = rop.roi_pool(f5, rois, 7, 7, 1.0 / 16.0, 0)
    p4, _ = rop.roi_pool(f4, rois, 7, 7, 1.0 / 8.0, 0)
    want = (p5 + p4).reshape(rois.shape[0], -1).to(torch.float16)
    assert torch.equal(got, want)
    # image shard: global batch indices shifted by batch_offset select the same local images; foreign rows pool zeros
    shifted = rois.clone(); shifted[:, 0] += 5
    assert torch.equal(pose_head.roi_pool_pair(f5, f4, shifted, batch_offset=5), want)
    foreign = pose_head.roi_pool_pair(f5, f4, shifted, batch_offset=0)
    assert float(foreign.float().abs().max()) == 0.0


@pytest.mark.parametrize("M,K,N,act", [(128, 25088, 4096, "relu"), (128, 4096, 4096, "relu"), (128, 4096, 88, "tanh"),
                                        (37, 1024, 256, "none"), (300, 512, 128, "relu")])
def test_fc_tc_against_fp32_matmul(cuda, M, K, N, act):
    """Split-K wgmma GEMM + fused epilogue against an fp64 product of the SAME fp16-rounded operands (isolates the
    kernel from the operand rounding): |err| <= 1e-3 * (1 + |ref|) before the fp16 output rounding, fp16-exact after."""
    from posecnn_b200 import pose_head
    g = torch.Generator().manual_seed(K + N)
    a = (torch.randn(M, K, generator=g) * 0.5).to(torch.float16)
    w = (torch.randn(K, N, generator=g) / np.sqrt(K)).float()
    bias = torch.randn(N, generator=g) * 0.1
    w_tc = pose_head.fc_weights_to_tc(w.to(cuda))
    assert w_tc.shape == ((N + 127) // 128 * 128, K)
    ref = a.double() @ w.to(torch.float16).double() + bias.double()
    ref = {"relu": torch.relu, "tanh": torch.tanh, "none": lambda t: t}[act](ref)
    out32 = pose_head.fc(a.to(cuda), w_tc, bias.to(cuda), act, torch.float32).cpu().double()
    assert out32.shape == (M, N)
    assert torch.all((out32 - ref).abs() <= 1e-3 * (1 + ref.abs())), float((out32 - ref).abs().max())
    out16 = pose_head.fc(a.to(cuda), w_tc, bias.to(cuda), act, torch.float16).cpu()
    assert out16.shape == (M, w_tc.shape[0])
    assert torch.equal(out16[:, :N], out32.float().to(torch.float16))          # same accumulation, one rounding
    assert float(out16[:, N:].float().abs().max()) == 0.0 if w_tc.shape[0] > N else True
    again = pose_head.fc(a.to(cuda), w_tc, bias.to(cuda), act, torch.float32).cpu().double()
    assert torch.equal(again, out32)                                            # fixed-order split-K reduction


def _scene(B, H, W, C, seed):
    sc = synth.make_scene(batch=B, height=H, width=W, num_classes=C, objects_per_image=min(3, C - 1), seed=seed,
                          min_pixels=520 if H < 200 else 800)
    return sc


def test_hough_shards_concatenate_to_the_whole_batch(cuda):
    """SURVEY.md §8(e): rank r holds images [r B/G, (r+1) B/G) of ONE global batch, applies index_size = 128 / B_global
    (hough_voting_gpu_op.cu.cc:733) and writes global batch indices; the shards' rows in rank order == the single call."""
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as hop
    B, H, W, C = 8, 120, 160, 5
    sc = _scene(B, H, W, C, 11)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    for is_train in (0, 1):
        gt = T(sc["gt"]) if is_train else None
        whole = hop.hough_voting_gpu_capacity(T(sc["label"]), T(sc["vertex"]), T(sc["extents"]), T(sc["meta"]), gt, is_train,
                                              -1.0, 0.02, 10)
        n_whole = int(whole[5].item())
        assert n_whole >= B
        for shards in (2, 4):
            per = B // shards
            rows = [[] for _ in range(5)]
            for r in range(shards):
                sl = slice(r * per, (r + 1) * per)
                part = hop.hough_voting_gpu_capacity(T(sc["label"][sl]), T(sc["vertex"][sl]), T(sc["extents"]), T(sc["meta"][sl]),
                                                     gt, is_train, -1.0, 0.02, 10, batch_global=B, batch_offset=r * per)
                n = int(part[5].item())
                for k in range(5):
                    rows[k].append(part[k][:n])
            for k in range(5):
                assert torch.equal(torch.cat(rows[k]), whole[k][:n_whole]), (is_train, shards, k)


def test_hough_cap_uses_the_global_batch(cuda):
    """A single image of a global batch of 64 keeps at most 128 // 64 = 2 classes (first in ascending class order)."""
    from posecnn_b200.hough_voting_gpu_layer import hough_voting_gpu_op as hop
    sc = _scene(1, 240, 320, 8, 5)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    full = hop.hough_voting_gpu_capacity(T(sc["label"]), T(sc["vertex"]), T(sc["extents"]), T(sc["meta"]), None, 0, -1.0, 0.02, 10)
    n_full = int(full[5].item())
    assert n_full >= 3
    capped = hop.hough_voting_gpu_capacity(T(sc["label"]), T(sc["vertex"]), T(sc["extents"]), T(sc["meta"]), None, 0, -1.0, 0.02,
                                           10, batch_global=64, batch_offset=17)
    assert int(capped[5].item()) == 2
    want = full[0][:2].clone(); want[:, 0] = 17.0
    assert torch.equal(capped[0][:2], want) and torch.equal(capped[1][:2], full[1][:2])


@pytest.mark.parametrize("shape", [(2, 64, 96, 6), (2, 480, 640, 22)])
def test_pipeline_without_dense_vertex_is_bit_identical(cuda, shape):
    """dense_vertex=False (Hough samples the vertex head from `lowres` with k_up8_heads' operation sequence, the 2.6 GB
    vertex_pred is never written) must reproduce the dense pipeline bit for bit: labels, ROI rows, poses, detections."""
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    B, H, W, C = shape
    net = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0, bias_std=0.05 if H < 200 else 0.0)
    rgb, _ = synth.make_images(B, H, W, seed=3)
    data = torch.from_numpy(rgb).to(cuda)
    meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)).to(cuda)
    ext = torch.from_numpy(synth.extents_for(C)).to(cuda)
    if H >= 200:
        net.calibrate_background(data, meta, ext, 0.75)
    a = dict(net.forward(data, meta, ext, sync_rois=False, dense_vertex=True))
    b = dict(net.forward(data, meta, ext, sync_rois=False, dense_vertex=False))
    assert "vertex_pred" in a and "vertex_pred" not in b
    assert int(a["num_rois"].item()) >= 1
    for k in ("label_2d", "rois_capacity", "num_rois", "poses_init", "poses_tanh", "detections_rois", "detections_poses",
              "num_detections", "hough_status"):
        assert torch.equal(a[k], b[k]), k


def test_sharded_network_equals_whole_batch(cuda):
    """SURVEY.md §8(e) end to end on one GPU: the network run shard by shard (batch_global / batch_offset) emits, in
    shard order, exactly the post-NMS records of the whole-batch run (conv tiles never mix images, so even the bf16
    trunk is bit-identical)."""
    from posecnn_b200 import parallel
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    B, H, W, C = 4, 96, 128, 6
    net = vgg16_convs(num_classes=C, device=cuda).init_random(seed=0, bias_std=0.05)
    rgb, _ = synth.make_images(B, H, W, seed=9)
    data = torch.from_numpy(rgb).to(cuda)
    meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)).to(cuda)
    ext = torch.from_numpy(synth.extents_for(C)).to(cuda)
    whole = parallel.compact_records(parallel.pack_detections(net.forward(data, meta, ext, sync_rois=False, dense_vertex=False)))
    assert whole.shape[0] >= 2
    for world in (2, 4):
        parts = []
        for r in range(world):
            o, n = parallel.shard_range(B, r, world)
            L = net.forward(data[o:o + n], meta[o:o + n], ext, sync_rois=False, dense_vertex=False, batch_global=B, batch_offset=o)
            assert L["rois_capacity"].shape[0] == parallel.roi_capacity(B, n)
            parts.append(parallel.pack_detections(L))
        got = parallel.compact_records(torch.cat(parts))
        assert torch.equal(got, whole), world


# ---------------------------------------------------------------------------------------------------------------------
# Exact tests of the fully connected kernels at the head's shapes (tests/util.py): operands in {-1, 0, 1} and integer biases,
# so every sum is an integer <= 25,096 (below fp16's 65,504) and the fp32 output must equal the float64 reference exactly,
# the fp16 output that value rounded once.  M = 600 ROI rows = five M tiles.
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [128, 600])
@pytest.mark.parametrize("layer,K,N", [("fc6", 25088, 4096), ("fc7", 4096, 4096), ("fc8", 4096, 88)])
def test_fc_exact_at_head_shapes(cuda, layer, K, N, M):
    from posecnn_b200 import pose_head
    from tests.util import fc_plan, int_operands
    g = torch.Generator().manual_seed(K + N + M)
    a = int_operands((M, K), -1, 1, g).to(torch.float16).to(cuda)
    w = int_operands((K, N), -1, 1, g).to(cuda)
    bias = int_operands((N,), -8, 8, g).to(cuda)
    w_tc = pose_head.fc_weights_to_tc(w)
    plan = fc_plan(M, w_tc.shape[0], K)
    print(f"{layer} M={M}: {plan['m_tiles']} M tiles, {plan['splits']} splits x {plan['chunks_per_split']} K chunks "
          f"(fewest {plan['min_chunks']})")
    assert plan["min_chunks"] > 6 or plan["splits"] > 1      # the 6-stage ring is reused, or the split-K finish reduces
    lin = a.double() @ w.double() + bias.double()
    for act in ("none", "relu"):
        want = (lin.clamp(min=0) if act == "relu" else lin).float()
        out32 = pose_head.fc(a, w_tc, bias, act, torch.float32)
        out16 = pose_head.fc(a, w_tc, bias, act, torch.float16)
        torch.cuda.synchronize()
        assert torch.equal(out32, want), (act, int((out32 != want).sum()))
        assert torch.equal(out16[:, :N], want.to(torch.float16)), act
        assert not bool(out16[:, N:].any())


@pytest.mark.parametrize("M", [128, 600])
def test_fc_dgrad_exact_at_fc6(cuda, M):
    """pcnn_fc_dgrad_f16_tc at fc6 (N = 25,088 input features, K = 4096) with the ReLU mask of the stored pooled features:
    out = (dy @ W^T) * [mask > 0], exact against the float64 product."""
    import ctypes
    from posecnn_b200._lib import check, lib, ptr, stream, workspace
    from tests.util import fc_plan, int_operands
    N, K = 25088, 4096
    g = torch.Generator().manual_seed(M + 1)
    dy = int_operands((M, K), -1, 1, g).to(torch.float16).to(cuda)
    wt = int_operands((N, K), -1, 1, g).to(torch.float16).to(cuda)          # [in][out]: the transposed fc6 weights
    mask = int_operands((M, N), -1, 1, g).to(torch.float16).to(cuda)
    plan = fc_plan(M, N, K)
    print(f"fc6 dgrad M={M}: {plan['splits']} splits x {plan['chunks_per_split']} K chunks")
    out = torch.empty((M, N), dtype=torch.float16, device=cuda)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_fc_workspace_bytes(M, N, K, ctypes.byref(nbytes)))
    ws = workspace("fc", nbytes.value, cuda)
    check(lib().pcnn_fc_dgrad_f16_tc(ptr(dy), ptr(wt), M, N, K, ptr(mask), ptr(out), N, ptr(ws), ws.numel(), stream()))
    want = ((dy.double() @ wt.double().t()) * (mask > 0)).float().to(torch.float16)
    torch.cuda.synchronize()
    assert torch.equal(out, want), int((out != want).sum())
