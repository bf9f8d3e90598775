"""The training image blobs on the device (csrc/augment.cu) against the numpy oracle (tests/augment_ref.py), which equals the
reference's chromatic_transform / add_noise on the golden vectors and cv2's HLS conversions on every input (test_augment_cpu.py)."""
import numpy as np
import pytest
import torch

from tests import augment_ref as ref

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def row(bg=-1, chroma=0, dh=0.0, dl=0.0, ds=0.0, noise=0, sigma=0.0, size=0, axis=0):
    return [bg, chroma, dh, dl, ds, noise, sigma, size, axis]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def same(a, b):
    """Bit for bit, except that NaNs match any NaN: IEEE leaves the payload of 0 / 0 open (the device gives 0x7fffffff, x86
    numpy 0xffc00000)."""
    return bool(((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))).all())


def test_every_colour_through_the_chromatic_transform(cuda):
    """All 2^24 BGR colours as one 4096 x 4096 image, at shift triples that wrap the hue both ways and clip L / S at both ends."""
    from posecnn_b200 import augment
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], 1).astype(np.uint8).reshape(1, 4096, 4096, 3)
    shifts = [(0.0, 0.0, 0.0), (-1.7999, 25.6, -25.6), (1.75, -25.6, 25.6), (-1e-17, 3.3, -7.9), (0.4, -300.0, 300.0),
              (179.5, 300.0, -300.0)]
    x = T(img, cuda)
    keys = torch.zeros(1, dtype=torch.int64, device=cuda)
    for dh, dl, ds in shifts:
        params = T(np.array([row(chroma=1, dh=dh, dl=dl, ds=ds)]), cuda)
        got = augment.augment_color(x, None, params, keys).cpu().numpy()
        want = ref.color_blob(img, None, np.array([row(chroma=1, dh=dh, dl=dl, ds=ds)]), [0])
        assert (bits(got) != bits(want)).sum() == 0, (dh, dl, ds)


def _batch(H=480, W=640, seed=5):
    """Fifteen frames covering composites with and without a background, an out-of-range background index, and every noise
    mode, blur size and orientation."""
    g = np.random.default_rng(seed)
    B = 15
    rgba = g.integers(0, 256, (B, H, W, 4), dtype=np.uint8)
    rgba[..., 3] = np.where(g.random((B, H, W)) < 0.3, 0, rgba[..., 3] | 1)
    rgba[:, :H // 5, :, 3] = 0
    bgs = g.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    rows = [row(0, 1, -1.3, 12.0, -20.0, 1, 8.1), row(-1, 1, 1.7, -25.0, 25.0, 1, 0.5), row(7, 1, 0.2, 0.0, 3.0, 0)]
    rows += [row(i % 3, 1, 0.9 - 0.2 * i, 4.0 * i - 20, 10.0 - 3 * i, 2, 0.0, z, a)
             for i, (z, a) in enumerate((z, a) for z in ref.BLUR_SIZES for a in (0, 1))]
    table = np.array(rows, np.float64)
    field = g.standard_normal((B, H, W))
    return rgba, bgs, table, field


def test_batch_with_injected_field_equals_oracle(cuda):
    from posecnn_b200 import augment
    rgba, bgs, table, field = _batch()
    B = len(table)
    keys = np.arange(B, dtype=np.int64) + 11
    got = augment.augment_color(T(rgba, cuda), T(bgs, cuda), T(table, cuda), T(keys, cuda), T(field, cuda)).cpu().numpy()
    want = ref.color_blob(rgba, bgs, table, keys, field)
    for b in range(B):
        assert (bits(got[b]) != bits(want[b])).sum() == 0, (b, table[b])
    # a 3-channel frame (no alpha, no compositing), odd sizes that cut every tile
    rgb = np.ascontiguousarray(rgba[:4, :37, :101, :3])
    got = augment.augment_color(T(rgb, cuda), None, T(table[[0, 5, 11, 12]], cuda), T(keys[:4], cuda),
                                T(field[:4, :37, :101], cuda)).cpu().numpy()
    want = ref.color_blob(rgb, None, table[[0, 5, 11, 12]], keys[:4], field[:4, :37, :101])
    assert (bits(got) != bits(want)).sum() == 0


def test_philox_field(cuda):
    """The kernel's own field.  It is observed through the f32 blob: a mid-grey frame with sigma = 1 gives f32(128 + g) - mean.
    The oracle's Philox + Box-Muller gives the same blob bit for bit except where a change of 1e-12 relative in g (the device's
    log / cos against libm's) moves f32(128 + g) across a rounding boundary: at most 1 ulp, on at most 8 of 2.4 M pixels.
    The field has a normal's moments; two launches are identical; images [4, 8) launched alone equal rows 4-7 of the batch."""
    from posecnn_b200 import augment
    B, H, W = 8, 480, 640
    rgba = np.full((B, H, W, 4), 255, np.uint8)
    rgba[..., :3] = 128
    table = np.array([row(noise=1, sigma=1.0)] * B, np.float64)
    keys = np.array([(0x9E3779B97F4A7C15 * (b + 1)) & (2 ** 63 - 1) for b in range(B)], np.int64)
    a = augment.augment_color(T(rgba, cuda), None, T(table, cuda), T(keys, cuda))
    assert torch.equal(a, augment.augment_color(T(rgba, cuda), None, T(table, cuda), T(keys, cuda)))
    assert torch.equal(augment.augment_color(T(rgba[4:8], cuda), None, T(table[4:8], cuda), T(keys[4:8], cuda)), a[4:8])
    got = a.cpu().numpy()
    g_np = np.stack([ref.philox_normal(int(k), H, W) for k in keys])
    want = ref.color_blob(rgba, None, table, keys, g_np)
    diff = bits(got).astype(np.int64) - bits(want).astype(np.int64)
    assert np.abs(diff).max() <= 1 and (diff != 0).sum() <= 8, int((diff != 0).sum())
    n = g_np.size
    assert abs(g_np.mean()) < 5 / np.sqrt(n) and abs(g_np.var() - 1) < 5 * np.sqrt(2 / n)
    g_dev = got[..., 0].astype(np.float64) + ref.PIXEL_MEANS[0] - 128.0
    assert abs(g_dev.mean()) < 5 / np.sqrt(n) and abs(g_dev.var() - 1) < 5 * np.sqrt(2 / n) + 1e-6


def test_depth_blob_equals_oracle(cuda):
    from posecnn_b200 import augment
    g = np.random.default_rng(3)
    B, H, W = 8, 480, 640
    depth = g.integers(0, 6000, (B, H, W), dtype=np.uint16)
    depth[3] = 0                                                                     # all-zero: 0 / 0 = NaN, as numpy
    rows = [row(noise=1, sigma=3.3), row(noise=2, size=15, axis=0), row(noise=2, size=15, axis=1), row(noise=1, sigma=2.0),
            row(noise=2, size=3, axis=1), row(noise=0), row(noise=2, size=7, axis=0), row(noise=2, size=11, axis=1)]
    table = np.array(rows, np.float64)
    field = g.standard_normal((B, H, W))
    keys = np.arange(B, dtype=np.int64)
    for d in (depth, depth.astype(np.float32) * np.float32(0.25)):
        dt = T(d.view(np.int16), cuda).view(torch.uint16) if d.dtype == np.uint16 else T(d, cuda)
        got, mx = augment.depth_blob_train(dt, T(table, cuda), T(keys, cuda), T(field, cuda), return_max=True)
        want, wmx = ref.depth_blob(d, table, keys, field)
        assert np.array_equal(mx.cpu().numpy(), wmx)
        got = got.cpu().numpy()
        assert np.isnan(got[3]).all()
        if d.dtype == np.uint16:
            got_u16 = got
        for b in range(B):
            assert same(got[b], want[b]), (b, d.dtype)
    # against cv2's float filter2D (DFT at 15 taps) on the same float image
    cv2 = pytest.importorskip("cv2")
    for b in (1, 2, 4, 6, 7):
        v = (depth[b].astype(np.float32) / np.float32(depth[b].max())) * np.float32(255)
        z, a = int(table[b, 7]), int(table[b, 8])
        k = np.zeros((z, z))
        if a == 0:
            k[(z - 1) // 2, :] = 1
        else:
            k[:, (z - 1) // 2] = 1
        cvb = (cv2.filter2D(np.tile(v[..., None], (1, 1, 3)), -1, k / z).astype(np.float64) - ref.PIXEL_MEANS).astype(np.float32)
        assert np.abs(got_u16[b] - cvb).max() < 2e-4, b


def test_graph_capture_replays_the_same_blob(cuda):
    from posecnn_b200 import augment
    rgba, bgs, table, _ = _batch(H=120, W=160)
    args = (T(rgba, cuda), T(bgs, cuda), T(table, cuda), T(np.arange(len(table), dtype=np.int64), cuda))
    eager = augment.augment_color(*args)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        augment.augment_color(*args)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = augment.augment_color(*args)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_training_step_on_augmented_blob(cuda):
    """Trainer.step on the f32 blob (no means subtracted again) matches fp32 autograd within the limits of the uint8 step."""
    from posecnn_b200 import augment
    from posecnn_b200.networks.vgg16_convs import PIXEL_MEANS
    from posecnn_b200.train import Trainer
    from tests.train_ref import compare_grads, make_inputs, make_net, reference_grads, synthetic_pose_targets
    net = make_net(cuda)
    args, _, _ = make_inputs(cuda)
    data, gt, centers, meta, ext, gtp, pts, sym = args
    B, H, W, _ = data.shape
    rgba = torch.cat([data, torch.full((B, H, W, 1), 255, dtype=torch.uint8, device=cuda)], 3).contiguous()
    params, keys = augment.draw_params(np.random.RandomState(4), B, 0, device=cuda)
    blob = augment.augment_color(rgba, None, params, keys)
    tr = Trainer(net, lr=0.01)
    A = tr.forward(blob, gt, centers, meta, ext, gtp, pts, sym)
    tw, wt = synthetic_pose_targets(A, pts, sym, 0.01)
    grads = tr.backward(A, gt, centers)
    torch.cuda.synchronize()
    # the autograd reference subtracts the means from its input: give it blob + means (equal to the blob to an ulp after it)
    ref_args = (blob + torch.tensor(PIXEL_MEANS, device=cuda),) + tuple(args[1:])
    P, r16 = reference_grads(net, A, ref_args, tw, wt, True)
    Pf, r32 = reference_grads(net, A, ref_args, tw, wt, False)
    compare_grads(tr, grads, P, Pf, list(grads))
