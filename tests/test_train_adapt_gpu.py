"""The domain-adaptation branch of vgg16_convs (lib/networks/vgg16_convs.py:202-212) and loss_domain (lib/fcn/train.py:508-513):
the fused tail kernel, fc9's GEMMs at their shapes, the merge that applies the gradient reversal, the training step against torch
fp32 autograd with the reversal restated as an autograd Function (identity forward, -lambda backward), invariants against the
step without the branch, the dummy Hough row, inference and CUDA-graph capture, and two ranks."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.train_ref import (LAMBDA, bits, compare_grads, grads_of, limits_adapt, make_inputs, make_net, reference_grads, rel_l2,
                             run_two_ranks, synthetic_pose_targets, train_worker)

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


# ---------------------------------------------------------------------------------------------------------------------
# 1. the tail kernel against float64
# ---------------------------------------------------------------------------------------------------------------------
def tail_ref64(h9, w10, b10, lab, loss_scale, grad_scale):
    h, w, b = h9.double(), w10.double(), b10.double()
    z = (h @ w.t() + b).clamp(min=0)
    q = torch.softmax(z, 1)
    oh = F.one_hot(lab.long(), 2).double()
    ce = torch.logsumexp(z, 1) - (z * oh).sum(1)
    gz = loss_scale * (q - oh) * (z > 0)
    d = (gz @ w) * (h > 0)
    return dict(score=z, prob=q, loss=loss_scale * ce.sum(), dw10=gz.t() @ h, db10=gz.sum(0), db9=d.sum(0), d=d, amax=d.abs().max(),
                dpre9=(grad_scale * d).to(torch.float16))


@pytest.mark.parametrize("rows", [1, 9, 127, 1152])
def test_domain_tail_against_float64(cuda, rows):
    """Every output of pcnn_domain_tail against float64 on the same fp16 fc9 values.  The input has exact zeros (fc9's ReLU
    mask), rows whose two logits are both <= 0 (label 0, no gradient) and mixed labels; two launches are bit-identical."""
    from posecnn_b200 import pose_head
    g = torch.Generator().manual_seed(rows)
    h9 = (torch.randn((rows, 256), generator=g) * 0.5).clamp(min=0)          # about half the units exactly 0
    h9[::5] = 0.0                                                             # both logits = relu(b10) = 0
    w10 = torch.randn((2, 256), generator=g) * 0.1
    b10 = torch.tensor([-0.3, -0.2])
    lab = torch.randint(0, 2, (rows,), generator=g, dtype=torch.int32)
    h9, w10, b10, lab = h9.to(torch.float16).to(cuda), w10.to(cuda), b10.to(cuda), lab.to(cuda)
    ls, gs = 0.1 / rows, 2.0 ** 12
    a = pose_head.domain_tail(h9, w10, b10, lab, ls, gs)
    b = pose_head.domain_tail(h9, w10, b10, lab, ls, gs)
    inf = pose_head.domain_tail(h9, w10, b10)
    torch.cuda.synchronize()
    want = tail_ref64(h9, w10, b10, lab, ls, gs)
    z = want["score"]
    dead = (z <= 0).all(1)
    print(f"rows={rows}: {int(dead.sum())} rows with both logits <= 0, {int((lab == 1).sum())} labelled 1, "
          f"{float((h9 == 0).float().mean()):.2f} of fc9 zero")
    if rows > 1:
        assert bool(dead.any()) and bool((~dead).any())
    for k in a:
        assert torch.equal(bits(a[k]), bits(b[k])), k                     # run-to-run bit-identical
    for k in ("domain_score", "domain_prob", "domain_label"):
        assert torch.equal(a[k], inf[k]), k
    assert torch.allclose(a["domain_score"].double(), z, rtol=1e-5, atol=1e-6)
    assert torch.allclose(a["domain_prob"].double(), want["prob"], rtol=1e-5, atol=1e-6)
    margin = (z[:, 0] - z[:, 1]).abs()
    lab_want = (z[:, 1] > z[:, 0]).int()
    sure = margin > 1e-5
    assert torch.equal(a["domain_label"][sure], lab_want[sure])
    assert bool((a["domain_label"][dead] == 0).all())                       # first maximum on the tie 0 == 0
    assert abs(a["loss"].item() - want["loss"].item()) <= 1e-5 * abs(want["loss"].item())
    for k in ("dw10", "db10", "db9"):
        e = rel_l2(a[k].double(), want[k])
        print(f"  {k}: rel-L2 {e:.2e}")
        assert e < 1e-5, (k, e)
    assert abs(a["amax"].item() - want["amax"].item()) <= 1e-5 * want["amax"].item()
    # the fp16 operand: the fp32 value rounded once; it may sit one fp16 step from the float64 value rounded once
    got, ref = a["dpre9"].double(), want["dpre9"].double()
    assert bool(((got - ref).abs() <= 2.0 ** -10 * ref.abs() + 2.0 ** -24).all())
    assert float((got == ref).double().mean()) > 0.99
    assert not bool(a["dpre9"][dead].any())                                   # rows without a gradient
    assert not bool(a["dpre9"][h9 == 0].any())                                # fc9's ReLU mask


def test_domain_tail_padded_rows(cuda):
    """ld > 256: the padding columns of the gradient operand are written as zeros, the values match ld = 256."""
    from posecnn_b200 import pose_head
    g = torch.Generator().manual_seed(3)
    h = (torch.randn((40, 256), generator=g) * 0.5).clamp(min=0).to(torch.float16).to(cuda)
    hp = torch.full((40, 320), 7.0, dtype=torch.float16, device=cuda)
    hp[:, :256] = h
    w10, b10 = (torch.randn((2, 256), generator=g) * 0.1).to(cuda), torch.tensor([0.1, -0.1], device=cuda)
    lab = (torch.arange(40, device=cuda) % 2).to(torch.int32)
    a = pose_head.domain_tail(h, w10, b10, lab, 0.01, 1024.0)
    b = pose_head.domain_tail(hp, w10, b10, lab, 0.01, 1024.0)
    torch.cuda.synchronize()
    assert torch.equal(b["dpre9"][:, :256], a["dpre9"]) and not bool(b["dpre9"][:, 256:].any())
    for k in ("domain_score", "loss", "dw10", "db9"):
        assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# 2. fc9 exact at its shapes (tests/util.py integer operands: every sum is an integer below 2^24)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [128, 600, 1152])
def test_fc9_exact(cuda, M):
    """fc9 forward (N = 256, K = 25088), input gradient ([M,256] -> [M,25088], K = 256) and weight gradient (25088 x 256): the
    fp16 outputs equal the float64 result rounded once, the fp32 weight gradient equals it.  The forward's work items run >= 8
    K chunks; the input gradient's K = 256 is four 64-wide chunks, all of which every item runs; the weight gradient's items
    run >= 8 of its 64-row K tiles where the rows hold that many (M = 128 has 2)."""
    from posecnn_b200 import pose_head
    from posecnn_b200._lib import check, lib, ptr, stream, workspace
    from tests.util import fc_plan, int_operands, wgrad_plan
    K, N = 25088, 256
    g = torch.Generator().manual_seed(M + 9)
    pool = int_operands((M, K), -1, 1, g).to(torch.float16).to(cuda)
    w9 = int_operands((K, N), -1, 1, g).to(cuda)
    b9 = int_operands((N,), -8, 8, g).to(cuda)
    w_tc = pose_head.fc_weights_to_tc(w9)
    assert w_tc.shape == (N, K)
    pf = fc_plan(M, N, K)
    pd = fc_plan(M, K, N)
    pw = wgrad_plan(1, 1, M, K, N, 1)
    print(f"fc9 M={M}: forward {pf['splits']} splits x {pf['chunks_per_split']} chunks (fewest {pf['min_chunks']}); dgrad "
          f"{pd['splits']} split x {pd['chunks_per_split']} chunks; wgrad {pw['splits']} split, {pw['min_ktiles']}..{pw['ktiles_per_split']} K tiles")
    assert pf["min_chunks"] >= 8
    assert pd["splits"] == 1 and pd["min_chunks"] == N // 64
    assert pw["min_ktiles"] >= 8 or pw["ktiles"] == pw["min_ktiles"] == (M + 63) // 64
    lin = pool.double() @ w9.double() + b9.double()
    out = pose_head.fc(pool, w_tc, b9, "relu")
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(lin.clamp(min=0).float().to(torch.float16)))
    # input gradient: dy [M,256] against the [25088][256] transposed copy, no mask (pool_score has none)
    dy = int_operands((M, N), -1, 1, g).to(torch.float16).to(cuda)
    wt = w_tc.t().contiguous()
    dx = torch.empty((M, K), dtype=torch.float16, device=cuda)
    nbytes = ctypes.c_size_t(0)
    check(lib().pcnn_fc_workspace_bytes(M, K, N, ctypes.byref(nbytes)))
    ws = workspace("fc", nbytes.value, cuda)
    check(lib().pcnn_fc_dgrad_f16_tc(ptr(dy), ptr(wt), M, K, N, ptr(None), ptr(dx), K, ptr(ws), ws.numel(), stream()))
    torch.cuda.synchronize()
    assert torch.equal(bits(dx), bits((dy.double() @ wt.double().t()).float().to(torch.float16)))
    # weight gradient [256][25088] with a power-of-two scale
    dw = torch.empty((N, K), dtype=torch.float32, device=cuda)
    check(lib().pcnn_conv_wgrad_workspace_bytes(1, 1, M, K, N, 1, ctypes.byref(nbytes)))
    ws = workspace("wgrad", nbytes.value, cuda)
    check(lib().pcnn_fc_wgrad_f16_tc(ptr(pool), ptr(dy), M, K, N, 0.25, ptr(None), 0.0, ptr(dw), ptr(ws), ws.numel(), stream()))
    torch.cuda.synchronize()
    want = (dy.double().t() @ pool.double()).float() * 0.25
    bad = dw != want
    assert not bool(bad.any()), f"{int(bad.sum())} of {bad.numel()} gradients differ"


# ---------------------------------------------------------------------------------------------------------------------
# 3. the merge
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 37, 1152])
def test_domain_grad_merge_bit_exact(cuda, rows):
    """dst = (s_a * a) + (s_b * b) in float32, each product rounded: bit-exact against numpy; with b = 0 it is
    pcnn_half_to_float(a, s_a) bit for bit (signed zeros included)."""
    from posecnn_b200 import pose_head
    from posecnn_b200._lib import check, lib, ptr, stream
    g = torch.Generator().manual_seed(rows)
    n = rows * 25088
    a = (torch.randn(n, generator=g) * torch.exp2(torch.randint(-20, 12, (n,), generator=g).float())).to(torch.float16)
    b = (torch.randn(n, generator=g) * 300.0).to(torch.float16)
    a[::7] = 0.0
    a[3::11] = -0.0
    b[::5] = 0.0
    sa, sb = 2.0 ** -13, -LAMBDA / 2.0 ** 9
    got = pose_head.domain_grad_merge(a.to(cuda), sa, b.to(cuda), sb, (rows, 7, 7, 512))
    an, bn = a.numpy().astype(np.float32), b.numpy().astype(np.float32)
    want = np.float32(sa) * an + np.float32(sb) * bn
    torch.cuda.synchronize()
    assert np.array_equal(got.cpu().numpy().reshape(-1).view(np.int32), want.view(np.int32))
    ad = a.to(cuda)
    zero = pose_head.domain_grad_merge(ad, sa, torch.zeros_like(ad), sb, (rows, 7, 7, 512))
    h2f = torch.empty(n, dtype=torch.float32, device=cuda)
    check(lib().pcnn_half_to_float(ptr(ad), n, sa, ptr(h2f), stream()))
    torch.cuda.synchronize()
    assert torch.equal(bits(zero.reshape(-1)), bits(h2f))


# ---------------------------------------------------------------------------------------------------------------------
# 4-7. the training step
# ---------------------------------------------------------------------------------------------------------------------
def test_labelled_batch_matches_fp32_autograd(cuda):
    """Domain 0 (the batch has gt poses), ADAPT_WEIGHT = 1.0 as the shipped adaptation config: every gradient, the new ones
    included, against the 16-bit-rounded and the pure fp32 autograd graph.  The reversal itself is checked on pool_score's
    gradient: the step's with the branch minus the step's at adapt_weight = 0 is the reversed domain term alone, held against
    autograd of loss_domain alone — a wrong sign or lambda would be off by 2x or more."""
    from posecnn_b200.train import Trainer
    C, aw, margin = 6, 1.0, 0.01
    net = make_net(cuda, adaptation=True, C=C)
    args, _, _ = make_inputs(cuda, C=C)
    data, gt, centers, meta, ext, gtp, pts, sym = args
    tr = Trainer(net, lr=0.01, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=margin, adapt_weight=aw)
    assert tr.master["fc9/w"].shape == (256, 25088) and tr.master["domain_score/w"].shape == (2, 256)
    assert tr.fc_t["fc9"].shape == (25088, 256)
    A = tr.forward(*args)
    assert A["rows"] >= 9
    assert not bool(A["label_domain"].any())
    tw, wt = synthetic_pose_targets(A, pts, sym, margin)
    tr.adapt_weight = 0.0
    tr.backward(A, gt, centers)
    dpool0 = A["dpool"].clone()
    tr.adapt_weight = aw
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    assert set(grads) == set(tr.master)
    P, ref = reference_grads(net, A, args, tw, wt, True, 1.0, 10.0, margin, adapt_weight=aw)
    Pf, reff = reference_grads(net, A, args, tw, wt, False, 1.0, 10.0, margin, adapt_weight=aw)
    for r_ in (ref, reff):
        assert abs(A["loss_domain"].item() - r_["loss_domain"]) < 3e-2 * abs(r_["loss_domain"]), (A["loss_domain"].item(), r_["loss_domain"])
        assert abs(A["loss_pose"].item() - r_["loss_pose"]) < 3e-2 * max(1e-3, abs(r_["loss_pose"]))
    print(f"loss_domain {A['loss_domain'].item():.6f} (16-bit graph {ref['loss_domain']:.6f}, fp32 {reff['loss_domain']:.6f}); "
          f"domain loss scale {tr.domain_loss_scale:g}")
    compare_grads(tr, grads, P, Pf, sorted(grads))
    # the reversed domain gradient of pool_score
    _, dref = reference_grads(net, A, args, tw, wt, True, 1.0, 10.0, margin, adapt_weight=aw, domain_only=True)
    _, dreff = reference_grads(net, A, args, tw, wt, False, 1.0, 10.0, margin, adapt_weight=aw, domain_only=True)
    ours = (A["dpool"] - dpool0).reshape(A["rows"], -1)
    e16, e32 = rel_l2(ours, dref["dpool"]), rel_l2(ours, dreff["dpool"])
    flipped = rel_l2(ours, -dref["dpool"])
    print(f"reversed pool_score gradient: rel-L2 {e16:.3e} / {e32:.3e}, against the un-reversed sign {flipped:.3e}, "
          f"|ref| {dref['dpool'].norm().item():.3e}")
    assert dref["dpool"].norm() > 0
    assert e16 < 0.15 and e32 < 0.15 and flipped > 1.5
    # update and export cover the new parameters
    before = {k: v.clone() for k, v in tr.master.items()}
    tr.update(grads)
    for name in ("fc9/w", "fc9/b", "domain_score/w", "domain_score/b"):
        want = before[name] - 0.01 * (grads[name] + 1e-4 * before[name])
        assert torch.allclose(tr.master[name], want, rtol=1e-5, atol=1e-8), name
    assert torch.equal(tr.tc["fc9/w"], tr.master["fc9/w"].to(torch.float16))
    assert torch.equal(tr.fc_t["fc9"], tr.tc["fc9/w"].t().contiguous())
    out = tr.step(*args)
    assert torch.isfinite(out["loss"]).all()
    assert torch.allclose(out["loss"], out["loss_cls"] + out["loss_vertex"] + out["loss_pose"] + out["loss_domain"])
    assert out["label_domain"].shape == out["domain_label"].shape == (max(1, int(out["num_rois"].item())),)
    tr.export_params()
    assert torch.equal(net.params["fc9/weights"], tr.master["fc9/w"].t())
    assert torch.equal(net.params["domain_score/weights"], tr.master["domain_score/w"].t())


def test_adapt_batch_isolates_the_reversal(cuda):
    """Labels -1 everywhere and no gt poses (an adapt batch): Hough labels every row domain 1, loss_cls / loss_vertex / loss_pose
    and the head gradients are exactly 0, and the trunk's gradients — whose only source is now the reversed domain branch —
    match autograd."""
    from posecnn_b200.train import Trainer
    C = 6
    net = make_net(cuda, adaptation=True, C=C)
    _, args, _ = make_inputs(cuda, C=C)
    gt, centers = args[1], args[2]
    tr = Trainer(net, lr=0.01, adapt_weight=1.0)
    A = tr.forward(*args)
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    rows = A["rows"]
    assert rows >= 9 and A["num_rois"].item() == rows
    assert bool((A["label_domain"] == 1).all())
    assert A["cls_out"][0].item() == 0.0 and A["vtx_out"][0].item() == 0.0 and A["loss_pose"].item() == 0.0
    zero = [k for k in grads if k.split("/")[0] in ("score", "vertex_pred", "score_conv4", "score_conv5", "score_conv4_vertex",
                                                     "score_conv5_vertex", "fc6", "fc7", "fc8")]
    assert len(zero) == 18
    for k in zero:
        assert not bool(grads[k].any()), k
    P, ref = reference_grads(net, A, args, A["poses_target"], A["poses_weight"], True, adapt_weight=1.0)
    Pf, reff = reference_grads(net, A, args, A["poses_target"], A["poses_weight"], False, adapt_weight=1.0)
    for r_ in (ref, reff):
        assert abs(A["loss_domain"].item() - r_["loss_domain"]) < 3e-2 * abs(r_["loss_domain"])
    trunk = sorted(k for k in grads if k.startswith("conv"))
    compare_grads(tr, grads, P, Pf, trunk, limits_adapt)
    compare_grads(tr, grads, P, Pf, sorted(k for k in grads if k not in zero and k not in trunk))
    # the same comparison against a graph whose reversal has the wrong sign fails by far
    Pw, _ = reference_grads(net, A, args, A["poses_target"], A["poses_weight"], True, adapt_weight=1.0, lam=-LAMBDA)
    e = rel_l2(tr.to_tf("conv5_3/w", grads["conv5_3/w"]), Pw["conv5_3/weights"].grad)
    print(f"conv5_3/w against the un-reversed graph: {e:.3e}")
    assert e > 1.5


def _same(a, b, k, unfixed):
    """Byte-identical, except the score / vertex_pred bias gradients when two runs of one input already differ in them
    (tests/test_train_rgbd_gpu.py)."""
    if k in unfixed:
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-9), k
    else:
        assert torch.equal(bits(a), bits(b)), k


def test_adapt_weight_zero_leaves_shared_gradients_unchanged(cuda):
    from posecnn_b200.train import Trainer
    args, _, _ = make_inputs(cuda)
    base = Trainer(make_net(cuda), lr=0.01)
    a, a2 = grads_of(base, args), grads_of(base, args)
    unfixed = {k for k in a if not torch.equal(a[k], a2[k])}
    assert unfixed <= {"score/b", "vertex_pred/b"}
    tr = Trainer(make_net(cuda, adaptation=True), lr=0.01, adapt_weight=0.0)
    b = grads_of(tr, args)
    assert set(b) == set(a) | {"fc9/w", "fc9/b", "domain_score/w", "domain_score/b"}
    for k in a:
        _same(a[k], b[k], k, unfixed)
    for k in ("fc9/w", "fc9/b", "domain_score/w", "domain_score/b"):
        assert not bool(b[k].any()), k


def test_rgbd_depth_trunk_gradients_unchanged(cuda):
    """RGB-D with the branch at adapt_weight = 1: the reversed gradient enters the colour trunk only, so every `_p` gradient is
    byte-identical to the step without the branch."""
    from posecnn_b200.train import Trainer
    args, _, dm = make_inputs(cuda)
    a = grads_of(Trainer(make_net(cuda, "RGBD"), lr=0.01), args, depth=dm)
    tr = Trainer(make_net(cuda, "RGBD", adaptation=True), lr=0.01, adapt_weight=1.0)
    b = grads_of(tr, args, depth=dm)
    assert "fc9/w" in b and tr.domain_loss_scale > 1
    p = [k for k in a if k.split("/")[0].endswith("_p")]
    assert len(p) == 26
    for k in p:
        assert torch.equal(bits(a[k]), bits(b[k])), k
    assert not torch.equal(a["conv5_3/w"], b["conv5_3/w"])


def test_dummy_row(cuda):
    """An all-background label map: Hough finds nothing, the pose head and the domain branch see the one all-zero dummy row,
    label_domain = 0 (also on an adapt batch), and the loss is finite and equals the restatement."""
    from posecnn_b200.train import Trainer
    net = make_net(cuda, adaptation=True)
    net.params["score/biases"][0] += 1000.0
    net.prepare()
    _, args, _ = make_inputs(cuda)
    tr = Trainer(net, lr=0.01, adapt_weight=0.1)
    A = tr.forward(*args)
    assert A["rows"] == 1 and A["num_rois"].item() == 0
    tr.backward(A, args[1], args[2])
    torch.cuda.synchronize()
    assert A["label_domain"].tolist() == [0]
    z = A["domain_score"].double()[0]
    want = 0.1 * (torch.logsumexp(z, 0) - z[0]).item()
    got = A["loss_domain"].item()
    print(f"dummy row: domain_score {z.tolist()}, loss_domain {got} (restated {want})")
    assert np.isfinite(got) and abs(got - want) <= 1e-6 * max(1.0, abs(want))


# ---------------------------------------------------------------------------------------------------------------------
# 8. inference
# ---------------------------------------------------------------------------------------------------------------------
def test_inference_domain_outputs_and_graph(cuda):
    from posecnn_b200.networks.vgg16_convs import GraphedForward
    args, _, _ = make_inputs(cuda)
    data, meta, ext = args[0], args[3], args[4]
    net = make_net(cuda, adaptation=True, is_train=False)
    L = dict(net.forward(data, meta, ext))
    P = net.params
    n = L["rois"].shape[0]
    pre = torch.relu(L["pool_score"][:n].float() @ P["fc9/weights"] + P["fc9/biases"]) @ P["domain_score/weights"]
    P["domain_score/biases"] = 1.0 - pre.min(0).values                               # both logits above the ReLU's kink
    net.prepare()
    L = dict(net.forward(data, meta, ext))
    torch.cuda.synchronize()
    assert "label_domain" not in L
    for k in ("fc9", "domain_score", "domain_prob", "domain_label"):
        assert L[k].shape[0] == n, k
    h9 = torch.relu(L["pool_score"][:n].float() @ P["fc9/weights"] + P["fc9/biases"])
    z = torch.relu(h9 @ P["domain_score/weights"] + P["domain_score/biases"])
    prob = torch.softmax(z, 1)
    e = (L["domain_prob"] - prob).abs().max().item()
    sure = (z[:, 0] - z[:, 1]).abs() > 1e-2
    print(f"{n} rows: max |prob - fp32| {e:.2e}; {int(sure.sum())} rows with margin > 1e-2")
    assert e < 2e-3 and bool(sure.any())
    assert torch.equal(L["domain_label"][sure], z.argmax(1).int()[sure])
    eager = dict(net.forward(data, meta, ext, sync_rois=False))
    g = GraphedForward(net, data, meta, ext)
    out = g(data)
    torch.cuda.synchronize()
    for k in ("fc9", "domain_score", "domain_prob", "domain_label"):
        assert torch.equal(out[k], eager[k]), k
    assert torch.equal(eager["domain_label"][:n], L["domain_label"])
    plain = make_net(cuda, is_train=False)
    Lp = plain.forward(data, meta, ext)
    assert not any(k in Lp for k in ("fc9", "domain_score", "domain_prob", "domain_label", "label_domain"))
    assert "fc9/weights" not in plain.params


def test_training_losses_adds_loss_domain(cuda):
    """training_losses() on an is_train network's forward: loss_domain = adapt_weight * mean cross entropy of the rows."""
    from posecnn_b200.networks.vgg16_convs import training_losses
    args, _, _ = make_inputs(cuda)
    data, gt, centers, meta, ext, gtp, pts, sym = args
    net = make_net(cuda, adaptation=True)
    L = net.forward(data, meta, ext, poses=gtp, want_prob=True, want_score=True)
    out = training_losses(net, L, gt, None, None, pts, sym, centers=centers, adapt_weight=0.5)
    torch.cuda.synchronize()
    z, lab = L["domain_score"].double(), L["label_domain"].long()
    want = 0.5 * (torch.logsumexp(z, 1) - z.gather(1, lab[:, None])[:, 0]).mean().item()
    assert not bool(lab.any())
    assert abs(out["loss_domain"].item() - want) < 1e-5 * max(1.0, want)
    assert torch.allclose(out["loss"], out["loss_cls"] + out["loss_vertex"] + out["loss_pose"] + out["loss_domain"])


# ---------------------------------------------------------------------------------------------------------------------
# 9. two ranks
# ---------------------------------------------------------------------------------------------------------------------
def test_two_rank_adaptation_step_equals_single_gpu(tmp_path):
    """One adaptation step on image shards over 2 ranks == the step on the whole batch on one GPU; the second shard holds no gt
    pose of its own and still gets label_domain 0."""
    run_two_ranks(tmp_path, train_worker(adaptation=True))
