"""Backward-pass kernels (csrc/wgrad_tc.cu) against torch autograd of the same layer in fp32 on the SAME bf16-rounded
operands: weight gradients on wgmma (MN-major operands, split-K), ReLU-mask / max-pool routing, bias gradients, and the
input gradient through the forward kernel on flipped weights.  Reference semantics: TensorFlow's gradients of
Network.conv / max_pool (lib/networks/network.py:159-188, 303-310) as driven by lib/fcn/train.py:206-260."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def rel_l2(a, b):
    return ((a - b).pow(2).sum() / b.pow(2).sum().clamp(min=1e-30)).sqrt().item()


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(2, 20, 36, 64, 64, 3), (1, 17, 50, 128, 128, 3), (2, 12, 16, 256, 512, 3),
                                              (3, 9, 7, 512, 128, 1), (2, 30, 40, 512, 64, 1), (1, 1, 128, 4096, 128, 1),
                                              (1, 1, 37, 1024, 256, 1)])
def test_conv_wgrad_against_autograd(cuda, B, H, W, Cin, Cout, k):
    from posecnn_b200 import backward
    g = torch.Generator().manual_seed(B * 1000 + Cin + Cout)
    x = torch.randn(B, H, W, Cin, generator=g).to(torch.bfloat16).to(cuda)
    dz = (torch.randn(B, H, W, Cout, generator=g) * 0.1).to(torch.bfloat16).to(cuda)
    w = torch.zeros(Cout, Cin, k, k, device=cuda, requires_grad=True)
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w, padding=k // 2)
    y.backward(dz.float().permute(0, 3, 1, 2))
    want = w.grad.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin)            # [Cout][tap * Cin + ci]
    got = backward.conv_wgrad(x, dz, k)
    assert got.shape == want.shape
    e = rel_l2(got, want)
    assert e < 1e-4, e                                                       # same bf16 operands, fp32 accumulation: order only
    again = backward.conv_wgrad(x, dz, k)
    assert torch.equal(again, got)                                           # fixed-order split-K reduction
    wm = torch.randn(Cout, k * k * Cin, generator=g).to(cuda)
    both = backward.conv_wgrad(x, dz, k, scale=0.5, w_master=wm, decay=1e-2)
    assert torch.allclose(both, 0.5 * got + 1e-2 * wm, rtol=1e-5, atol=1e-6)


def first_max_route(g, y):
    """Max-pool 2x2/2 backward fused with the ReLU mask, plainly: the window [..., 4] in raster order, its FIRST maximum
    (torch.argmax) takes g when that maximum is > 0; every other element gets 0.  g [B,H/2,W/2,C], y [B,H,W,C] -> [B,H,W,C]."""
    B, H, W, C = y.shape
    win = y.float().view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C, 4)
    first = win.argmax(-1, keepdim=True)
    take = (torch.arange(4, device=y.device) == first) & (win.amax(-1, keepdim=True) > 0)
    dz = torch.where(take, g.float()[..., None], torch.zeros((), device=y.device))
    return dz.view(B, H // 2, W // 2, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, C).to(torch.bfloat16)


def test_relu_and_maxpool_backward(cuda):
    from posecnn_b200 import backward
    g = torch.Generator().manual_seed(3)
    B, H, W, C = 2, 12, 20, 64
    y = torch.relu(torch.randn(B, H, W, C, generator=g)).to(torch.bfloat16).to(cuda)
    gr = torch.randn(B, H, W, C, generator=g).to(torch.bfloat16).to(cuda)
    dz, db = backward.relu_bwd(gr, y, True, want_bias=True)
    want = gr.float() * (y.float() > 0)
    assert torch.equal(dz.float(), want)
    assert torch.allclose(db, want.sum((0, 1, 2)), rtol=1e-5, atol=1e-4)
    dz2, db2 = backward.relu_bwd(gr, None, False, want_bias=True, scale=0.5, bias=torch.ones(C, device=cuda), decay=0.1)
    assert torch.equal(dz2, gr) and torch.allclose(db2, 0.5 * gr.float().sum((0, 1, 2)) + 0.1, rtol=1e-5, atol=1e-4)
    # max-pool routing: torch autograd of max_pool2d(relu(z)) on distinct values (ties are measure zero in fp32; the kernel's
    # first-maximum rule is checked separately on a crafted tie)
    z = torch.randn(B, C, H, W, generator=g).to(torch.bfloat16).float().to(cuda).requires_grad_(True)
    yp = torch.relu(z)
    pooled = F.max_pool2d(yp, 2)
    gp = torch.randn(pooled.shape, generator=g).to(torch.bfloat16).float().to(cuda)
    pooled.backward(gp)
    ynhwc = yp.detach().permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    got, dbp = backward.maxpool_relu_bwd(gp.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), ynhwc, want_bias=True)
    ties = (F.max_pool2d(yp.detach(), 2, return_indices=False).repeat_interleave(2, 2).repeat_interleave(2, 3) == yp.detach()).float()
    unique = F.avg_pool2d(ties, 2) * 4 <= 1.0                                # windows with a unique maximum (zeros tie after ReLU)
    mask = unique.repeat_interleave(2, 2).repeat_interleave(2, 3).permute(0, 2, 3, 1)
    assert torch.equal(got.float()[mask], z.grad.permute(0, 2, 3, 1)[mask])
    assert torch.equal(got, first_max_route(gp.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), ynhwc))   # every window, ties included
    assert torch.allclose(dbp, got.float().sum((0, 1, 2)), rtol=1e-5, atol=1e-4)
    tie = torch.zeros(1, 2, 2, 8, dtype=torch.bfloat16, device=cuda); tie[0, :, :, :] = 1.5
    gt = torch.ones(1, 1, 1, 8, dtype=torch.bfloat16, device=cuda)
    rt = backward.maxpool_relu_bwd(gt, tie)
    assert rt[0, 0, 0].float().sum() == 8 and rt.float().sum() == 8          # all four equal: the first (top-left) takes the gradient
    s = backward.add_to_bf16(gr, dz, want)
    assert torch.equal(s, (gr.float() + dz.float() + want).to(torch.bfloat16))


@pytest.mark.parametrize("Cin,Cout,k", [(64, 128, 3), (512, 512, 3), (512, 64, 1)])
def test_conv_dgrad_through_forward_kernel(cuda, Cin, Cout, k):
    """dx = conv(dz, W flipped / transposed): the forward wgmma kernel on conv.hwio_to_tc_dgrad weights, zero bias, no ReLU."""
    from posecnn_b200 import conv
    g = torch.Generator().manual_seed(Cin + Cout + k)
    B, H, W = 2, 16, 24
    w = (torch.randn(k, k, Cin, Cout, generator=g) / (k * k * Cin) ** 0.5).to(cuda)
    dz = torch.randn(B, H, W, Cout, generator=g).to(torch.bfloat16).to(cuda)
    x = torch.zeros(B, Cin, H, W, device=cuda, requires_grad=True)
    wq = w.to(torch.bfloat16).float()
    y = F.conv2d(x, wq.permute(3, 2, 0, 1), padding=k // 2)
    y.backward(dz.float().permute(0, 3, 1, 2))
    got = conv.conv_bf16(dz, conv.hwio_to_tc_dgrad(w), torch.zeros(Cin, device=cuda), k, False)
    e = rel_l2(got.float(), x.grad.permute(0, 2, 3, 1))
    assert e < 5e-3, e                                                        # one bf16 rounding of the output


def test_fc_dgrad_wgrad_and_pose_chain(cuda):
    """Fully connected backward GEMMs (fp16 operands) and the pose-loss chain against torch on the same operands."""
    from posecnn_b200 import pose_head
    g = torch.Generator().manual_seed(11)
    rows, Kin, Nout = 45, 4096, 256
    x = torch.relu(torch.randn(rows, Kin, generator=g)).to(torch.float16).to(cuda)          # stored output of the layer below (ReLU)
    w = (torch.randn(Kin, Nout, generator=g) / Kin ** 0.5).to(cuda)                           # TF layout [in, out]
    dy = (torch.randn(rows, Nout, generator=g) * 0.3).to(torch.float16).to(cuda)
    w_tc = pose_head.fc_weights_to_tc(w)                                                       # [out][in] fp16
    w_t = pose_head.transpose16(w_tc)
    assert torch.equal(w_t, w_tc.t().contiguous())
    # input gradient with the ReLU mask of the layer below
    out = pose_head.fc_dgrad(dy, w_t, x)
    want = (dy.float() @ w_tc.float()) * (x.float() > 0)
    assert rel_l2(out.float(), want) < 2e-3
    # weight gradient [out][in] with a scale
    dw = pose_head.fc_wgrad(x, dy, 0.25)
    assert rel_l2(dw, 0.25 * dy.float().t() @ x.float()) < 1e-4
    # pose chain: d pre-activation of fc8 from d loss / d poses_pred, poses_pred = l2_normalize(tanh(pre) * weight)
    N, D = 19, 24
    pre = torch.randn(N, D, generator=g).to(cuda).requires_grad_(True)
    wt = torch.zeros(N, D); wt[:, 4:8] = 1.0; wt[3] = 0.0; wt = wt.to(cuda)                   # one class active; one all-zero row (clamped norm)
    gup = torch.randn(N, D, generator=g).to(cuda)
    th = torch.tanh(pre)
    mul = th * wt
    pred = mul / mul.pow(2).sum(1, keepdim=True).clamp(min=1e-12).sqrt()
    (pred * gup).sum().backward()
    dpre = pose_head.pose_chain_bwd(gup, th.detach().contiguous(), wt, 1.0, torch.empty((N, 128), dtype=torch.float16, device=cuda))
    assert rel_l2(dpre[:, :D].float(), pre.grad) < 2e-3 and float(dpre[:, D:].float().abs().max()) == 0.0


def _up8_problem(cuda, B, h, w, C, seed):
    """A low-resolution head tensor, its dense up-sampling (pcnn_up8_heads), ground-truth labels with ignore / background /
    foreground pixels, centres with one listed and one unlisted class."""
    from posecnn_b200 import heads
    g = torch.Generator().manual_seed(seed)
    H, W = 8 * h, 8 * w
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(cuda)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(cuda), (torch.randn(3 * C, generator=g) * 0.1).to(cuda)
    _, vertex, prob, score = heads.up8_heads(lowres, bs, bv, vertex=True, prob=True, score=True)
    gt = torch.randint(-1, C, (B, H, W), generator=g).to(torch.int32)
    gt[:, : H // 3] = 0                                                      # a background region (Hardlabel: selected only if uncertain)
    gt[:, H // 3: H // 2, : W // 2] = 3                                      # a coherent object
    gt = gt.to(cuda)
    centers = torch.zeros(B, C, 3)
    for c in range(1, C):
        if c != 2:                                                           # class 2 is labelled but not listed (z = 0)
            centers[:, c] = torch.tensor([W * 0.3 + 3 * c, H * 0.6 - 2 * c, 0.5 + 0.05 * c])
    return dict(lowres=lowres, bs=bs, bv=bv, vertex=vertex, prob=prob, score=score, gt=gt, centers=centers.to(cuda), B=B, h=h, w=w, C=C)


def _up8_bwd(P, thr=0.7, up_cls=1.0, up_vtx=2.0, w_in=10.0, sigma=1.0, count=937.0, sumw=411.0):
    from posecnn_b200 import heads
    B, h, w, C = P["B"], P["h"], P["w"], P["C"]
    dev = P["lowres"].device
    out = (torch.full((B, h, w, 64), 7.0, dtype=torch.bfloat16, device=dev), torch.full((B, h, w, 128), 7.0, dtype=torch.bfloat16, device=dev),
           torch.empty((4 * C,), device=dev))
    cls_out, vtx_out = torch.tensor([0.5, count], device=dev), torch.tensor([0.25, sumw], device=dev)
    return heads.up8_heads_bwd(P["prob"], P["score"], P["gt"], cls_out, up_cls, thr, P["lowres"], P["bv"], P["centers"], vtx_out, up_vtx, w_in,
                               sigma, out=out)


@pytest.mark.parametrize("C,h,w", [(22, 8, 12), (6, 18, 10), (22, 60, 80)])
def test_up8_heads_backward_against_torch(cuda, C, h, w):
    """Gradient of the Hardlabel cross entropy and of the vertex smooth-L1 w.r.t. the low-resolution head tensor
    (k_up8_bwd_strip) against the formulas of lib/fcn/train.py:455-465, 564-573 written in torch and the adjoint of the fixed
    bilinear x8 transposed convolution (network.py:141-157, 207-222) = a stride-8 depthwise convolution with the same filter.
    The vertex values come from the low-resolution head tensor; the torch formulas read the dense vertex_pred of pcnn_up8_heads."""
    B = 2
    P = _up8_problem(cuda, B, h, w, C, seed=C + h)
    thr, up_cls, up_vtx, w_in, sigma, count, sumw = 0.7, 1.0, 2.0, 10.0, 1.0, 937.0, 411.0
    d_sc, d_vt, dbias = _up8_bwd(P)
    H, W = 8 * h, 8 * w
    gt = P["gt"].long()
    prob, score, vertex = P["prob"], P["score"], P["vertex"]
    valid = gt >= 0
    g0 = gt.clamp(min=0)
    pg = prob.gather(3, g0[..., None])[..., 0]
    sel = valid & ((gt > 0) | (pg < thr))
    onehot = F.one_hot(g0, C).float()
    d_up_s = (up_cls / (count + 1e-10)) * sel[..., None] * (prob - onehot) * (score > 0)
    cen = P["centers"]
    ys, xs = torch.meshgrid(torch.arange(H, device=cuda), torch.arange(W, device=cuda), indexing="ij")
    cpix = cen[torch.arange(B, device=cuda)[:, None, None], g0]                                  # [B,H,W,3]
    listed = (gt > 0) & (cpix[..., 2] > 0)
    dx, dy = cpix[..., 0].double() - xs, cpix[..., 1].double() - ys
    nrm = (dx * dx + dy * dy).sqrt() + 1e-10
    tg = torch.stack([(dx / nrm).float(), (dy / nrm).float(), cpix[..., 2].clamp(min=1e-30).double().log().float()], -1)
    own = vertex.view(B, H, W, C, 3).gather(3, g0[..., None, None].expand(B, H, W, 1, 3))[..., 0, :]
    diff = w_in * (own - tg)
    dt = torch.where(diff.abs() < 1.0 / sigma ** 2, diff * sigma ** 2, diff.sign())
    d_own = (up_vtx / (sumw + 1e-10)) * w_in * dt * listed[..., None]
    d_up_v = torch.zeros(B, H, W, C, 3, device=cuda).scatter_(3, g0[..., None, None].expand(B, H, W, 1, 3), d_own[..., None, :]).view(B, H, W, 3 * C)
    d_up = torch.cat([d_up_s, d_up_v], 3).permute(0, 3, 1, 2).contiguous()
    k1 = torch.tensor([1.0 - abs(i / 8.0 - 0.9375) for i in range(16)], device=cuda)
    filt = (k1[:, None] * k1[None, :])[None, None].expand(4 * C, 1, 16, 16).contiguous()
    want = F.conv2d(d_up, filt, stride=8, padding=4, groups=4 * C).permute(0, 2, 3, 1)             # [B,h,w,4C]
    assert rel_l2(d_sc[..., :C].float(), want[..., :C]) < 4e-3                                     # bf16 output rounding
    assert rel_l2(d_vt[..., :3 * C].float(), want[..., C:]) < 4e-3
    assert (d_vt[..., 3 * C:].float() == 0).all()                                                  # GEMM padding channels
    assert torch.allclose(dbias, d_up.sum((0, 2, 3)), rtol=2e-4, atol=1e-7)
    assert (d_sc[..., C:].float() == 0).all()


def test_add_up2_and_adjoint(cuda):
    """add = a4 + up2(a5) (fixed bilinear conv2d_transpose 4x4 / 2, vgg16_convs.py:134-138) and the adjoint with the ReLU mask."""
    from posecnn_b200 import heads
    g = torch.Generator().manual_seed(5)
    B, h, w, C = 2, 12, 16, 64
    a4 = torch.randn(B, h, w, C, generator=g).to(torch.bfloat16).to(cuda)
    a5 = torch.randn(B, h // 2, w // 2, C, generator=g).to(torch.bfloat16).to(cuda)
    out = heads.add_up2(a4, a5)
    k1 = torch.tensor([1.0 - abs(i / 2.0 - 0.75) for i in range(4)], device=cuda)
    filt = (k1[:, None] * k1[None, :])[None, None].expand(C, 1, 4, 4).contiguous()
    up = F.conv_transpose2d(a5.float().permute(0, 3, 1, 2), filt, stride=2, padding=1, groups=C).permute(0, 2, 3, 1)
    assert rel_l2(out.float(), a4.float() + up) < 3e-3
    dadd = torch.randn(B, h, w, C, generator=g).to(torch.bfloat16).to(cuda)
    d5 = heads.up2_bwd(dadd, a5)
    want = F.conv2d(dadd.float().permute(0, 3, 1, 2), filt, stride=2, padding=1, groups=C).permute(0, 2, 3, 1) * (a5.float() > 0)
    assert rel_l2(d5.float(), want) < 3e-3
    d5 = heads.up2_bwd(dadd)
    assert rel_l2(d5.float(), F.conv2d(dadd.float().permute(0, 3, 1, 2), filt, stride=2, padding=1, groups=C).permute(0, 2, 3, 1)) < 3e-3


def test_relu_and_maxpool_backward_at_conv1_2(cuda):
    """ReLU-mask / max-pool routing and the bias gradients at conv1_2's pre-pool shape (2 x 480 x 640 x 64).  Small integer
    activations make ReLU zeros and equal window values common, so the first-maximum rule is checked on many ties; integer
    gradients make the bias sums exact (every fp32 partial is an integer < 2^24), so they must equal the fp64 sum.  With
    random gradients two runs must give bit-identical bias gradients (fixed-order per-CTA and cross-CTA reductions)."""
    from posecnn_b200 import backward
    from tests.util import int_operands
    g = torch.Generator().manual_seed(12)
    B, H, W, C = 2, 480, 640, 64
    y = torch.relu(int_operands((B, H, W, C), -3, 3, g)).to(torch.bfloat16).to(cuda)
    gp = int_operands((B, H // 2, W // 2, C), -2, 2, g).to(torch.bfloat16).to(cuda)
    gf = int_operands((B, H, W, C), -2, 2, g).to(torch.bfloat16).to(cuda)
    dz, db = backward.maxpool_relu_bwd(gp, y, want_bias=True)
    want = first_max_route(gp, y)
    assert torch.equal(dz, want)
    assert torch.equal(db, want.double().sum((0, 1, 2)).float())
    dz2, db2 = backward.relu_bwd(gf, y, True, want_bias=True)
    want2 = gf.float() * (y.float() > 0)
    assert torch.equal(dz2.float(), want2)
    assert torch.equal(db2, want2.double().sum((0, 1, 2)).float())
    gr = torch.randn((B, H // 2, W // 2, C), generator=g).to(torch.bfloat16).to(cuda)
    grf = torch.randn((B, H, W, C), generator=g).to(torch.bfloat16).to(cuda)
    a = backward.maxpool_relu_bwd(gr, y, want_bias=True)[1].clone()
    b = backward.maxpool_relu_bwd(gr, y, want_bias=True)[1]
    assert torch.equal(a, b)
    a = backward.relu_bwd(grf, y, True, want_bias=True)[1].clone()
    b = backward.relu_bwd(grf, y, True, want_bias=True)[1]
    assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# Weight gradients at training shapes with exact integer operands ({-1, 0, 1}: every sum is an integer <= the pixel count,
# far below 2^24), so the fp32 gradient must equal the float64 reference exactly.  The batch of every case is the smallest
# whose every work item runs at least eight K tiles (twice k_wgrad_tc's four-stage ring): stages are reused, the
# release-previous-stage path runs, and direct mode (splits == 1) reduces over many tiles.
# ---------------------------------------------------------------------------------------------------------------------
def _wgrad_cases(H=480, W=640):
    """(id, H, W, Cin, Cout, k) of every convolution weight gradient of the training step (train.py: backward)."""
    from posecnn_b200.networks.vgg16_convs import VGG_CFG
    cases, h, w = [], H, W
    for item in VGG_CFG:
        if isinstance(item, str):
            h, w = h // 2, w // 2
            continue
        name, ci, co = item
        # conv1_1: the 1x1 weight gradient on the im2col view of the image (K = tap * 3 + c in 64 columns)
        cases.append((name, h, w, 64, co, 1) if name == "conv1_1" else (name, h, w, ci, co, 3))
    h4, w4 = H // 8, W // 8
    cases += [("score_conv4", h4, w4, 512, 64, 1), ("score_conv5", h4 // 2, w4 // 2, 512, 64, 1),
              ("score_conv4_vertex", h4, w4, 512, 128, 1), ("score_conv5_vertex", h4 // 2, w4 // 2, 512, 128, 1),
              ("score", h4, w4, 64, 64, 1), ("vertex_pred", h4, w4, 128, 128, 1)]
    return cases


_WG = _wgrad_cases()


@pytest.mark.parametrize("name,H,W,Cin,Cout,k", _WG, ids=[c[0] for c in _WG])
def test_conv_wgrad_exact_at_training_shapes(cuda, name, H, W, Cin, Cout, k):
    from posecnn_b200 import backward, conv
    from tests.util import int_operands, ref_wgrad_exact, wgrad_batch_for_coverage
    B, plan = wgrad_batch_for_coverage(H, W, Cin, Cout, k)
    print(f"{name}: B={B} splits={plan['splits']} ktiles={plan['ktiles']} -> {plan['min_ktiles']}..{plan['ktiles_per_split']} "
          f"K tiles per item")
    assert plan["min_ktiles"] >= 8
    g = torch.Generator().manual_seed(H + Cin + 5 * Cout + k)
    if name == "conv1_1":
        mean = (103.0, 116.0, 123.0)                  # integer means: the im2col values are the bytes' offsets {-1, 0, 1}
        img = (int_operands((B, H, W, 3), -1, 1, g) + torch.tensor(mean)).to(torch.uint8).to(cuda)
        x = conv.im2col_c3(img, mean)
    else:
        x = int_operands((B, H, W, Cin), -1, 1, g).to(torch.bfloat16).to(cuda)
    dz = int_operands((B, H, W, Cout), -1, 1, g).to(torch.bfloat16).to(cuda)
    want = ref_wgrad_exact(x, dz, k).float()
    got = backward.conv_wgrad(x, dz, k, scale=0.5)
    torch.cuda.synchronize()
    bad = got != 0.5 * want
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} gradients differ; first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("name,Cin,Cout,rows", [("fc6", 25088, 4096, 600), ("fc7", 4096, 4096, 600),
                                                ("cin192", 192, 4096, 0), ("cin384", 384, 4096, 0)])
def test_fc_wgrad_exact(cuda, name, Cin, Cout, rows):
    """pcnn_fc_wgrad_f16_tc at the fc6 / fc7 shapes with 600 ROI rows (direct mode, ten 64-row K tiles, the last ragged) and
    at Cin = 192 / 384 (one / two 64-channel B blocks), with a power-of-two scale: exact against the float64 product."""
    from posecnn_b200 import pose_head
    from tests.util import int_operands, wgrad_batch_for_coverage, wgrad_plan
    if rows == 0:
        rows, plan = wgrad_batch_for_coverage(1, 1, Cin, Cout, 1)
    else:
        plan = wgrad_plan(1, 1, rows, Cin, Cout, 1)
    print(f"{name}: rows={rows} splits={plan['splits']} direct={plan['direct']} -> {plan['min_ktiles']}..{plan['ktiles_per_split']} "
          f"K tiles per item")
    assert plan["min_ktiles"] >= 8
    g = torch.Generator().manual_seed(Cin + rows)
    x = int_operands((rows, Cin), -1, 1, g).to(torch.float16).to(cuda)
    dy = int_operands((rows, Cout), -1, 1, g).to(torch.float16).to(cuda)
    dw = pose_head.fc_wgrad(x, dy, 0.25)
    want = (dy.double().t() @ x.double()).float() * 0.25
    torch.cuda.synchronize()
    bad = dw != want
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} gradients differ; first at {bad.nonzero()[0].tolist()}"
