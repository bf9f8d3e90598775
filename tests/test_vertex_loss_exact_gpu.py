"""The training step's vertex loss and the targets it is built from, bit for bit against the float64 references of
tests/vertex_loss_ref.py at training shapes.

- loss_vertex (pcnn_vertex_loss_fwd) at 2 x 480 x 640, C = 22 and 2, sigma 1 and 2.5, both
  target modes: out[0] is the fp32 rounding of the exact term sum over the weight sum (an order-independent check that
  raises Straddle where the kernel's double accumulation could round either way), out[1] the exact weight sum.  Checked on
  a fresh workspace, after loss_cls on the same workspace and on a repeated call (both read the ticket the previous launch
  re-armed), through train_ops, and under CUDA-graph replay (each replay zero-fills its captured workspace, so replay
  checks the captured launch, not the re-arm); on the boundary-only and tiny-band-only label maps; and against the loss
  of the materialised targets of the same inputs.  One case runs at the Trainer's batch of 64 frames.
- The materialised 2-D, 3-D and multi-instance targets at 4 x 480 x 640 x 22: every channel bit for bit.  The 3-D operands
  (YCB-sized extents, float32 object coordinates) make coord_scale / coord_target round, so a fused or reordered formula
  shows.
- pack_pose_meta at 1024 instance slots (its shared offset table full), 256 threads looping: rows, counts and meta exact.
Each case prints its foreground count, boundary pixels and the accumulation bound."""
import numpy as np
import pytest
import torch

from tests import vertex_loss_ref as V

pytestmark = pytest.mark.gpu


def _fresh_ws(dev):
    import ctypes
    from posecnn_b200._lib import check, lib
    n = ctypes.c_size_t(0)
    check(lib().pcnn_train_loss_workspace_bytes(ctypes.byref(n)))
    return torch.zeros(int(n.value), dtype=torch.uint8, device=dev)


def _on(P, dev):
    T = lambda a: a.contiguous().to(dev) if isinstance(a, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(a)).to(dev)
    D = dict(lowres=T(P["lowres"]), bias_v=T(P["bias_v"]), label=T(P["label"]), centers=T(P["centers"]))
    if P["coord"]:
        D.update(vertmap=T(P["vertmap"]), extents=T(P["extents"]))
    return D


def _loss_abi(P, D, ws, label=None):
    """One launch of the entry point on workspace ws into a NaN-filled [2] buffer (an unwritten output cannot pass)."""
    from posecnn_b200._lib import check, lib, ptr, stream
    lab = D["label"] if label is None else label
    out = torch.full((2,), float("nan"), device=ws.device)
    B, H, W, C = P["B"], P["H"], P["W"], P["C"]
    check(lib().pcnn_vertex_loss_fwd(ptr(D["lowres"]), ptr(D["bias_v"]), ptr(lab), ptr(D["centers"]), ptr(D.get("vertmap")),
                                     ptr(D.get("extents")), B, H, W, C, P["w_inside"], P["sigma"], ptr(out), ptr(ws), ws.numel(), stream()))
    return out


def _train_ops_loss(P, D, label=None):
    from posecnn_b200 import train_ops
    lab = D["label"] if label is None else label
    kw = dict(vertmap=D["vertmap"], extents=D["extents"]) if P["coord"] else {}
    return train_ops.loss_vertex(D["lowres"], D["bias_v"], lab, D["centers"], P["w_inside"], P["sigma"], **kw)


def _assert_loss(out, ref, what):
    got = out.cpu().numpy()
    assert got[1] == ref["out1"], f"{what}: weight sum {got[1]!r} != {ref['out1']!r}"
    assert got[0] == ref["out0"], f"{what}: loss {got[0]!r} != {ref['out0']!r} (exact sum / weights, bound {ref['bound']:.3e})"


def _report(tag, P, ref):
    plan = V.loss_plan(P["B"] * P["H"] * P["W"])
    print(f"{tag}: {plan['npix']} pixels = {plan['sweeps']:.2f} sweeps of {plan['sweep']} threads (tail {plan['tail']}); "
          f"foreground {ref['count']}, {ref['n_terms']} terms, {ref['boundary']} at |diff| == 1/sigma^2, {ref['tiny']} below "
          f"2^-30; bit budget {ref['budget']:.0f} of 2^24; accumulation bound {ref['bound']:.3e} on sum {float(ref['S']):.6e}; "
          f"loss {ref['out0']!r}, sum w {ref['out1']!r}")


def _check_label_contents(P, ref):
    lab, C, z = P["label"], P["C"], P["centers"][..., 2]
    assert (lab == -1).any() and (lab == 0).any() and (lab == C).any() and (lab > C).any()
    inr = (lab > 0) & (lab < C)
    b_idx = np.broadcast_to(np.arange(P["B"])[:, None, None], lab.shape)
    zl = z[b_idx[inr], lab[inr]]
    assert (zl == 0).any(), "a labelled class with z = 0"
    if C > 2:
        assert np.isnan(zl).any() and (zl < 0).any(), "labelled classes with NaN and negative z"
    assert ref["listed"][-1, -1, -1] and ref["terms"][-3:].max() > 1e-3, "the last pixel carries a sizable term"


_CASES = [(coord, C, s) for coord in (False, True) for C in (22, 2) for s in (1.0, 2.5)]


@pytest.mark.parametrize("coord,C,sigma", _CASES, ids=[f"{'3d' if c else '2d'}-C{C}-sigma{s}" for c, C, s in _CASES])
def test_loss_vertex_exact(cuda, coord, C, sigma):
    from posecnn_b200 import train_ops
    from posecnn_b200._lib import check, lib, ptr, stream
    B, H, W = 2, 480, 640
    g = torch.Generator().manual_seed(4000 + 10 * C + 2 * int(sigma) + coord)
    P = V.loss_problem(B, H, W, C, coord, sigma, g)
    ref = V.reference(P)
    _report(f"{'3-D' if coord else '2-D'} C={C} sigma={sigma}", P, ref)
    plan = V.loss_plan(B * H * W)
    assert plan["sweeps"] > 4 and plan["tail"] > 0
    _check_label_contents(P, ref)
    assert ref["boundary"] > 0 and ref["tiny"] > 0
    D = _on(P, cuda)
    # fresh workspace; then loss_cls on the same workspace; then twice more
    ws = _fresh_ws(cuda)
    first = _loss_abi(P, D, ws)
    score = V.R.dyadic((B, H, W, C), -2, 2, 0.25, g).to(cuda)
    prob = V.R.dyadic((B, H, W, C), 0, 1, 0.125, g).to(cuda)
    cls_out = torch.full((2,), float("nan"), device=cuda)
    check(lib().pcnn_loss_cls_hard_raw_fwd(ptr(score), ptr(prob), ptr(D["label"]), B, H, W, C, 0.5, ptr(cls_out), ptr(ws), ws.numel(),
                                           stream()))
    after_cls = _loss_abi(P, D, ws)
    again = _loss_abi(P, D, ws)
    lab = D["label"].long()
    sel = (lab >= 0) & (lab < C) & ((lab > 0) | (prob[..., 0] < 0.5))
    assert cls_out[1].item() == int(sel.sum())
    for out, what in ((first, "fresh workspace"), (after_cls, "after loss_cls"), (again, "repeated call")):
        _assert_loss(out, ref, what)
    # the library's own entry: train_ops.loss_cls and loss_vertex on their shared workspace, then a CUDA graph
    train_ops.loss_cls(score, prob, D["label"], 0.5)
    _assert_loss(_train_ops_loss(P, D), ref, "train_ops after loss_cls")
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _train_ops_loss(P, D)                                           # warm-up on the capture stream
        with torch.cuda.graph(graph, stream=s):
            captured = _train_ops_loss(P, D)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        captured.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _assert_loss(captured, ref, "graph replay")
    # label maps reduced to the planted boundary pixels and to the tiny band, where a dropped small term moves the loss
    bnd = np.zeros(P["label"].shape, bool)
    for (i, j) in P["blocks"]:
        bnd[:, 8 * i + 4:8 * i + 20, 8 * j + 4:8 * j + 20] = True
    band = np.zeros(P["label"].shape, bool)
    band[:, :28] = True
    # 3-D, C = 22: without the planted classes (their axis 1 has target 0 and a predicted +-1/sigma^2) every term of the
    # band is tiny, so the loss moves with a 1-ulp change of the targets (a fused or reordered coord_target)
    only_tiny = coord and C > 2
    if only_tiny:
        band &= ~np.isin(P["label"], P["planted"])
    for name, keep in (("boundary blocks", bnd), ("tiny band", band)):
        sub = np.where(keep, P["label"], -1).astype(np.int32)
        r2 = V.reference(P, sub)
        print(f"  {name}: foreground {r2['count']}, {r2['boundary']} boundary terms, {r2['tiny']} tiny terms, loss {r2['out0']!r}")
        if name == "tiny band" and only_tiny:
            assert r2["count"] > 0 and r2["tiny"] == r2["n_terms"]
        _assert_loss(_loss_abi(P, D, ws, torch.as_tensor(sub).to(cuda)), r2, name)
    # the loss of the materialised targets of the same inputs (vertex_target<kCoord> of both paths)
    if coord:
        tg, wt = train_ops.generate_vertex_targets_3d(D["label"], D["vertmap"], D["centers"], D["extents"], P["w_inside"])
    else:
        tg, wt = train_ops.generate_vertex_targets(D["label"], D["centers"], P["w_inside"])
    wt5 = wt.view(B, H, W, C, 3)
    listed = (wt5 > 0).any(-1).any(-1)
    cls_m = (wt5[..., 0] > 0).int().argmax(-1)
    assert torch.equal(listed.cpu(), torch.as_tensor(ref["listed"])) and torch.equal(cls_m.cpu().long(), torch.as_tensor(ref["cls"]))
    t_m = tg.view(B, H, W, C, 3).gather(3, cls_m.long()[..., None, None].expand(B, H, W, 1, 3))[..., 0, :].cpu().numpy()
    w_m = wt5.gather(3, cls_m.long()[..., None, None].expand(B, H, W, 1, 3))[..., 0, :].cpu().numpy()
    assert np.all(w_m[ref["listed"]] == np.float32(P["w_inside"]))
    mat = V.loss_vertex(ref["pv"], t_m, ref["listed"], P["w_inside"], sigma)
    assert mat["out0"] == first.cpu().numpy()[0] and mat["out1"] == first.cpu().numpy()[1], "fused loss != loss of the materialised targets"


def test_loss_vertex_trainer_batch(cuda):
    """The Trainer's batch (64 frames of 640 x 480 on one GPU, bench.py's training workload), C = 22, its w_inside of 10 and
    sigma 1, 2-D targets: 32.4 sweeps of the loss grid."""
    B, H, W, C = 64, 480, 640, 22
    g = torch.Generator().manual_seed(64)
    P = V.loss_problem(B, H, W, C, False, 1.0, g, w_inside=10.0)
    P["lowres"] = P["lowres"].to(cuda)                                   # the float64 up-sampling runs on the device
    ref = V.reference(P)
    _report("Trainer batch 2-D C=22 sigma=1 w_inside=10", P, ref)
    assert ref["tiny"] > 0 and ref["listed"][-1, -1, -1]
    D = _on(P, cuda)
    ws = _fresh_ws(cuda)
    _assert_loss(_loss_abi(P, D, ws), ref, "batch 64")
    _assert_loss(_loss_abi(P, D, ws), ref, "batch 64, repeated")


# ---------------------------------------------------------------------------------------------------------------------
# materialised targets
# ---------------------------------------------------------------------------------------------------------------------
def _assert_targets(tg, wt, listed, cls, t, w_inside, what):
    """Own-class channels equal the reference targets and w_inside, every other channel is 0, bit for bit."""
    B, H, W, C3 = tg.shape
    C = C3 // 3
    cls_d = torch.as_tensor(cls).to(tg.device).long()[..., None, None].expand(B, H, W, 1, 3)
    lst = torch.as_tensor(listed).to(tg.device)
    tg5, wt5 = tg.view(B, H, W, C, 3).clone(), wt.view(B, H, W, C, 3).clone()
    own_t, own_w = tg5.gather(3, cls_d)[..., 0, :], wt5.gather(3, cls_d)[..., 0, :]
    want_t = torch.as_tensor(t).to(tg.device)
    bad = lst[..., None] & (own_t.view(torch.int32) != want_t.view(torch.int32))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} target values differ; first at {bad.nonzero()[0].tolist()}"
    assert bool((own_w[lst] == np.float32(w_inside)).all()), f"{what}: weights"
    zero = torch.zeros_like(own_t)
    tg5.scatter_(3, cls_d, torch.where(lst[..., None], zero, own_t)[..., None, :])
    wt5.scatter_(3, cls_d, torch.where(lst[..., None], zero, own_w)[..., None, :])
    assert not bool(tg5.ne(0).any()) and not bool(wt5.ne(0).any()), f"{what}: a channel outside the own class is written"


def test_vertex_targets_exact(cuda):
    """pcnn_vertex_targets_fwd and _3d_fwd at 4 x 480 x 640 x 22 on the loss problem's labels (ignore, >= C, unlisted
    classes with z 0 / NaN / negative, centres on and off the image), every channel bit for bit, log z included (z values
    checked against fp32 midpoints).  The 3-D extents lie in [0.03, 0.3] and the object coordinates are float32 values, so
    a, b, a v and a v + b all round."""
    from posecnn_b200 import train_ops
    B, H, W, C = 4, 480, 640, 22
    for coord in (False, True):
        g = torch.Generator().manual_seed(500 + coord)
        P = V.loss_problem(B, H, W, C, coord, 1.0, g)
        D = _on(P, cuda)
        if coord:
            listed, cls, t = V.targets_3d(P["label"], P["vertmap"], P["centers"], P["extents"])
            tg, wt = train_ops.generate_vertex_targets_3d(D["label"], D["vertmap"], D["centers"], D["extents"], 10.0)
        else:
            listed, cls, t = V.targets_2d(P["label"], P["centers"])
            tg, wt = train_ops.generate_vertex_targets(D["label"], D["centers"], 10.0)
        print(f"{'3-D' if coord else '2-D'}: {int(listed.sum())} listed pixels of {listed.size}, "
              f"{len(np.unique(P['centers'][..., 2][P['centers'][..., 2] > 0]))} distinct z")
        _assert_targets(tg, wt, listed, cls, t, 10.0, "3-D targets" if coord else "2-D targets")
        del tg, wt


def test_vertex_targets_instances_exact(cuda):
    """pcnn_vertex_targets_instances_fwd at 4 x 480 x 640 x 22, I = 8: two rows of the same (class, mask id) with different
    centres (the last must win), an unused slot (z = 0) in the middle of the list that matches pixels, one with z < 0 and
    one with NaN z; direction and log-z channels bit for bit."""
    from posecnn_b200 import train_ops
    B, H, W, C, I = 4, 480, 640, 22, 8
    rng = np.random.default_rng(11)
    label = rng.choice(np.array([-1, 0, 1, 2, 3, C, C + 1]), size=(B, H, W), p=[.05, .15, .3, .25, .15, .05, .05]).astype(np.int32)
    mask = rng.integers(0, 3, (B, H, W)).astype(np.int32)
    inst = np.zeros((B, I, 5), np.float32)
    pairs = [(1, 1), (2, 1), (1, 2), (2, 2), (3, 1), (1, 1), (3, 2), (2, 1)]
    for b in range(B):
        for i, (c, m) in enumerate(pairs):
            inst[b, i] = (c, m, rng.integers(-64 * 4096, (W + 64) * 4096) / 4096, rng.integers(-64 * 4096, (H + 64) * 4096) / 4096,
                          V.LOGZ_TABLE[rng.integers(0, V.LOGZ_TABLE.size)])
    inst[:, 3, 4] = 0.0                                                     # unused slot in the middle, (2, 2) matches pixels
    inst[:, 6, 4] = -1.0
    inst[1, 7, 4] = np.nan
    listed, cls, t = V.targets_instances(label, mask, inst, C)
    first_wins = V.targets_instances(label, mask, np.concatenate([inst[:, 5:6], inst[:, :5], inst[:, 6:]], 1), C)[2]
    n_dup = int((listed & (label == 1) & (mask == 1)).sum())
    print(f"instances: {int(listed.sum())} listed pixels; {n_dup} owned by the repeated (1, 1) instance")
    assert n_dup > 0 and not np.array_equal(first_wins, t) and not ((label == 2) & (mask == 2) & listed).any()
    T = lambda a: torch.as_tensor(a).to(cuda)
    tg, wt = train_ops.generate_vertex_targets_instances(T(label), T(mask), T(inst), C, 10.0)
    _assert_targets(tg, wt, listed, cls, t, 10.0, "instance targets")


# ---------------------------------------------------------------------------------------------------------------------
# pose blob and meta packing
# ---------------------------------------------------------------------------------------------------------------------
def test_pack_pose_meta_exact(cuda):
    """pcnn_pack_pose_meta_fwd at B x I = 4 x 256 = 1024 slots (s_off[1025] full; 256 threads loop four times), a third of
    the slots unused, im_scale 1 and 0.5, with and without flip_x: row count, image / class / box / translation columns and
    meta_data exact, quaternions within 2e-6 of float64; rows past the count zero.  1025 slots are refused."""
    from scipy.spatial.transform import Rotation
    from posecnn_b200 import train_ops
    B, I = 4, 256
    rng = np.random.default_rng(5)
    cls = np.where(rng.random((B, I)) < 1 / 3, -1, rng.integers(1, 22, (B, I))).astype(np.int32)
    cls[B - 1, I - 1] = 7                                                   # the last slot is listed
    poses = np.zeros((B, I, 3, 4), np.float32)
    poses[..., :3] = Rotation.random(B * I, random_state=5).as_matrix().reshape(B, I, 3, 3)
    poses[..., 3] = rng.uniform(-0.3, 1.2, (B, I, 3))
    K = np.zeros((B, 3, 3), np.float32)
    K[:, 0, 0] = rng.integers(2000, 4400, B) / 4
    K[:, 1, 1] = rng.integers(2000, 4400, B) / 4
    K[:, 0, 2] = rng.integers(280 * 128, 360 * 128, B) / 128
    K[:, 1, 2] = rng.integers(200 * 128, 280 * 128, B) / 128
    K[:, 2, 2] = 1
    T = lambda a: torch.as_tensor(a).to(cuda)
    for scale, flip in ((1.0, False), (0.5, True)):
        blob, nrows, meta = train_ops.pack_pose_meta(T(poses), T(cls), T(K), scale, flip)
        wb, n, wm = V.pack_pose_meta(poses, cls, K, scale, flip)
        got = blob.cpu().numpy()
        print(f"scale {scale} flip {flip}: {n} rows of {B * I} slots")
        assert int(nrows.item()) == n == int((cls >= 0).sum())
        np.testing.assert_array_equal(got[:, :6], wb[:, :6])
        np.testing.assert_array_equal(got[:, 10:], wb[:, 10:])
        q = got[:n, 6:10] * np.where(np.abs(wb[:n, 6:7]) < 1e-6, np.sign((got[:n, 6:10] * wb[:n, 6:10]).sum(1, keepdims=True)), 1)
        np.testing.assert_allclose(q, wb[:n, 6:10], rtol=0, atol=2e-6)
        assert not got[n:].any()
        np.testing.assert_array_equal(meta.cpu().numpy().reshape(B, 48), wm)
    with pytest.raises(RuntimeError, match="at most 1024 instance slots"):
        train_ops.pack_pose_meta(T(np.zeros((5, 205, 3, 4), np.float32)), T(np.zeros((5, 205), np.int32)), T(np.zeros((5, 3, 3), np.float32)))
