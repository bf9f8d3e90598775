"""Backproject, Project, BackprojectGrad and ProjectGrad (csrc/pixel_ops.cu) bit for bit against the C oracle, at the shape of
`bench.py --workload project` (480 x 640, G = 128, Cf = 64, C = 22, kernel_size 3, threshold 0.02) and on every kernel the
dispatchers can choose.

The oracle (oracle/posecnn_oracle.c, built with -ffp-contract=off) spells out the device's fmaf sequence and sums each window
in the kernels' order (x outer, y inner), so every output equals it bit for bit except where the oracle marks an entry
ambiguous (a pre-round coordinate within 1e-3 of a half integer, a depth difference within 1e-5 of the threshold).  The
ambiguous fraction of every case is printed and bounded.  The device variants (aligned tensors, tensors offset by one float,
the unfused passes) run the same arithmetic and must agree with each other on every entry, ambiguous ones included.

Two depth maps: the benchmark's i.i.d. depth (synth.make_projection_case), where hit voxels are isolated, and a smooth scene
(a tilted plane at 0.8 to 1.6 m, spheres in front of it, a band of zero-depth holes) where surface voxels have full windows,
windows are clipped at the image border and consecutive slabs of the fused kernel both hold hits.

The dispatch rule is restated below (like tests/util.py::conv_plan restates the conv dispatcher); each case asserts which
kernels and branches it ran and the last test asserts that the cases together reach every one."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import oracle
from posecnn_b200 import synth
from tests.util import to_np

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMIT32 = 0x7FFFFFFF      # the launchers' per-image element limit
KBPVOX = 64               # voxels per CTA slab of k_backproject_fused

# ---------------------------------------------------------------------------------------------------------------------
# dispatch restatement (pcnn_backproject_fwd, launch_average, launch_gather)
# ---------------------------------------------------------------------------------------------------------------------
FUSED = "k_backproject_fused"
TABLE = {
    (FUSED, "label float4"), (FUSED, "label scalar"), (FUSED, "partial slab"), (FUSED, "C = 1"),
    ("k_voxel_average_wide<32,true>", "flag"), ("k_voxel_average_wide<32,true>", "fallback"),
    ("k_voxel_average_wide<16,false>", "plain"), ("k_voxel_average_wide<16,false>", "flag"),
    ("k_voxel_average_wide<16,false>", "fallback"),
    ("k_voxel_average<4>", "plain"), ("k_voxel_average<4>", "flag"), ("k_voxel_average<4>", "fallback"),
    ("k_voxel_average<1>", "plain"), ("k_voxel_average<1>", "flag"), ("k_voxel_average<1>", "fallback"),
    ("k_pixel_gather<4>", ""), ("k_pixel_gather<1>", ""),
    ("offsets past 2^31 elements", "B = 17"),
}
REACHED = set()
RAN = set()


def _a16(*ptrs):
    return all(p % 16 == 0 for p in ptrs if p is not None)


def average_row(nch, src, dst, fallback=None, flag=None):
    """launch_average: (kernel, role) for one window-average pass; arguments are data pointers."""
    v4 = nch % 4 == 0 and _a16(src, dst, fallback, flag)
    role = "flag" if flag is not None else ("fallback" if fallback is not None else "plain")
    if v4 and nch % 16 == 0:
        return ("k_voxel_average_wide<16,false>", role)
    if not v4 and nch <= 32:
        return ("k_voxel_average_wide<32,true>", role)
    return ("k_voxel_average<4>" if v4 else "k_voxel_average<1>", role)


def gather_row(Cf, vox, out):
    return ("k_pixel_gather<4>" if Cf % 4 == 0 and _a16(vox, out) else "k_pixel_gather<1>", "")


def backproject_rows(B, G, Cf, C, data, label_3d, top_data, top_label, top_flag, fused_on=True):
    """pcnn_backproject_fwd: the fused kernel (and which top_label branches its slabs take) or the two unfused passes."""
    G3 = G ** 3
    if fused_on and Cf % 4 == 0 and _a16(data, top_data, top_flag) and B <= 65535 and G3 * max(Cf, C) < LIMIT32:
        rows = set()
        v0 = np.arange(-(-G3 // KBPVOX), dtype=np.int64) * KBPVOX
        nvox = np.minimum(KBPVOX, G3 - v0)
        if G3 % KBPVOX:
            rows.add((FUSED, "partial slab"))
        if C == 1:
            rows.add((FUSED, "C = 1"))
        for n in range(B):
            off = (n * G3 + v0) * C * 4
            f4 = (C > 1) & ((nvox * C) % 4 == 0) & ((((top_label + off) | (label_3d + off)) % 16) == 0)
            if f4.any():
                rows.add((FUSED, "label float4"))
            if not f4.all():
                rows.add((FUSED, "label scalar"))
        return rows
    return None


def bp_rows(B, G, Cf, C, t, outs, fused_on=True):
    """The rows one pcnn_backproject_fwd call on tensors t (dict) with outputs outs runs: fused, or the data pass with
    top_flag and the label pass with the label_3d fallback."""
    p = {k: v.data_ptr() for k, v in t.items()}
    td, tl, tf = (o.data_ptr() for o in outs)
    rows = backproject_rows(B, G, Cf, C, p["data"], p["label_3d"], td, tl, tf, fused_on)
    if rows is None:
        rows = {average_row(Cf, p["data"], td, flag=tf), average_row(C, p["label"], tl, fallback=p["label_3d"])}
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# scenes and cases
# ---------------------------------------------------------------------------------------------------------------------
def smooth_depth(B, H, W, seed):
    """A tilted plane (inverse depth linear in the pixel: a plane) from 0.8 to 1.6 m, two spheres in front of it, a near
    sphere off the optical axis whose front reaches 0.445 m, and sensor holes (depth 0): a vertical band and a speckled block.
    The near sphere puts hits below z = 0.465 m, i.e. (at G = 128) in the first 64-voxel slab of a voxel row, next to rows
    whose second slab holds the plane's hits."""
    rng = np.random.default_rng(seed)
    K = synth.intrinsics(H, W)
    Ki = np.linalg.inv(K)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    rays = np.einsum("ij,jhw->ihw", Ki, np.stack([u, v, np.ones_like(u)]))        # z component 1: t = depth
    out = np.zeros((B, H, W, 1), np.float32)
    for b in range(B):
        a = rng.uniform(0.3, 0.7)
        z = 1.0 / (1 / 0.8 + (1 / 1.6 - 1 / 0.8) * (a * u / (W - 1) + (1 - a) * v / (H - 1)))
        spheres = [(rng.uniform(0.88, 0.92) * W, rng.uniform(0.4, 0.6) * H, 0.49, 0.045)]
        spheres += [(rng.uniform(0.15, 0.85) * W, rng.uniform(0.15, 0.85) * H, rng.uniform(0.9, 1.2), rng.uniform(0.08, 0.12))
                    for _ in range(2)]
        for cu, cv, cz, r in spheres:
            c = cz * (Ki @ np.array([cu, cv, 1.0]))
            dc = np.einsum("ihw,i->hw", rays, c)
            dd = np.einsum("ihw,ihw->hw", rays, rays)
            disc = dc * dc - dd * (c @ c - r * r)
            hit = disc > 0
            t = np.where(hit, (dc - np.sqrt(np.maximum(disc, 0))) / dd, np.inf)
            z = np.minimum(z, t)
        c0 = int(rng.uniform(0.2, 0.3) * W)
        z[:, c0:c0 + max(2, W // 20)] = 0                                            # shadow band
        r0, q0 = int(0.7 * H), int(0.6 * W)
        blk = z[r0:r0 + H // 8, q0:q0 + W // 8]
        blk[rng.random(blk.shape) < 0.5] = 0                                         # speckled dropouts
        out[b, ..., 0] = z
    return out


def make_case(scene, B, H, W, Cf, C, G, seed):
    c = synth.make_projection_case(B, H, W, Cf, C, G, seed=seed)
    if scene == "smooth":
        c["depth"] = smooth_depth(B, H, W, seed + 1000)
    rng = np.random.default_rng(seed + 2000)
    c["grad2"] = rng.standard_normal((B, H, W, Cf), dtype=np.float32)       # ProjectGrad's top_diff
    return c


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def T_offset(a, dev):
    """The same values in a contiguous view one float past a 16-byte boundary (require_cuda keeps the view)."""
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.empty(a.size + 4, dtype=torch.float32, device=dev)
    v = buf[1:1 + a.size].view(a.shape)
    v.copy_(torch.from_numpy(a))
    assert v.data_ptr() % 16 == 4 and v.is_contiguous()
    return v


def bits(a):
    return a.view(torch.int32) if isinstance(a, torch.Tensor) else np.ascontiguousarray(a).view(np.int32)


def assert_device_equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(bits(a), bits(b)):
        n = int((bits(a) != bits(b)).sum())
        raise AssertionError(f"{what}: {n} of {a.numel()} entries differ between device variants")


def assert_oracle_equal(got, want, amb, what):
    """Bitwise on every entry whose voxel / pixel the oracle does not mark ambiguous; returns how many ambiguous entries
    differ (printed: the marks are conservative)."""
    got = np.ascontiguousarray(got); want = np.ascontiguousarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    diff = bits(got) != bits(want)
    ok = ~amb[..., None]
    bad = diff & ok
    if bad.any():
        idx = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} non-ambiguous entries differ from the oracle; first at {idx}: "
                             f"got {got[idx]!r} want {want[idx]!r}")
    return int((diff & ~ok).sum())


def coverage(scene, depth, meta, G, ks, thr, tf_w, label):
    """Hit fraction, the largest window count, clipped windows with hits and consecutive fused slabs that both hold hits."""
    cnt, clip = oracle.voxel_window(depth, meta, G, ks, thr)
    hit = cnt > 0
    assert np.array_equal(hit, tf_w[..., 0] > 0)                   # the oracle's own flag agrees with its window counts
    B = cnt.shape[0]
    flat = hit.reshape(B, -1)
    nslab = -(-flat.shape[1] // KBPVOX)
    pad = np.zeros((B, nslab * KBPVOX), bool)
    pad[:, :flat.shape[1]] = flat
    slab = pad.reshape(B, nslab, KBPVOX).any(-1)
    facts = dict(hit=float(hit.mean()), max_count=int(cnt.max()), full=(2 * ks + 1) ** 2, clipped=int((hit & clip).sum()),
                 slab_pairs=int((slab[:, 1:] & slab[:, :-1]).sum()))
    print(f"  {label}: voxels hit {facts['hit']:.4%}, max count {facts['max_count']} of {facts['full']}, clipped windows with "
          f"hits {facts['clipped']}, consecutive slabs both hit {facts['slab_pairs']}")
    if thr > 0:
        assert hit.sum() > 0, facts
    # at 480 x 640 the smooth scene must reach every fact (a 48 x 64 image at these grids holds too few surface voxels)
    if scene == "smooth" and thr > 0 and depth.shape[2] >= 640:
        assert facts["max_count"] == facts["full"], facts
        assert facts["slab_pairs"] > 0, facts
        if ks > 0:
            assert facts["clipped"] > 0, facts
    return facts


# Ambiguous fractions measured on these cases (printed per case; largest 0.48 % for Backproject, 0.70 % for Project), with
# a margin of about 2x: Backproject's
# marks are voxels with a pre-round pixel coordinate within 1e-3 of a half integer (~0.4 %) or a window depth difference within
# 1e-5 of the threshold; Project's are pixels with a voxel coordinate within 1e-3 of a half integer (~0.6 %).
# Project's bound applies to pixels with depth: every hole pixel (depth 0) lands on the camera centre, one grid point (G / 2 in
# x and y when the camera's offset is ~0, a half integer for odd G), so the hole pixels of an image are all ambiguous or none.
AMBIG_MAX = {"backproject": 0.01, "project": 0.013}


def check_ambig(kind, amb, label, depth=None):
    valid = np.ones(amb.shape, bool) if depth is None else depth.reshape(amb.shape) > 0
    frac = float(amb[valid].mean())
    print(f"  {label}: ambiguous {kind} fraction {frac:.4%} (bound {AMBIG_MAX[kind]:.2%})"
          + ("" if depth is None else f", {float(amb[~valid].mean()) if (~valid).any() else 0:.2%} of the hole pixels"))
    assert frac <= AMBIG_MAX[kind], (kind, frac)


# (id, scene, B, H, W, Cf, C, G, kernel_size, threshold, project on Backproject's output)
CASES = []
for _scene in ("iid", "smooth"):
    CASES += [
        (f"bench-{_scene}", _scene, 2, 480, 640, 64, 22, 128, 3, 0.02, True),
        (f"64-22-32-{_scene}", _scene, 2, 48, 64, 64, 22, 32, 3, 0.02, False),          # the earlier test's three shapes
        (f"6-3-16-{_scene}", _scene, 2, 48, 64, 6, 3, 16, 3, 0.02, False),
        (f"8-3-128-{_scene}", _scene, 2, 48, 64, 8, 3, 128, 3, 0.02, False),
        (f"4-1-16-{_scene}", _scene, 2, 48, 64, 4, 1, 16, 3, 0.02, False),               # C = 1
        (f"4-1-128-{_scene}", _scene, 2, 48, 64, 4, 1, 128, 5, 0.02, False),
        (f"8-2-128-{_scene}", _scene, 2, 48, 64, 8, 2, 128, 0, 0.02, False),
        (f"4-3-37-{_scene}", _scene, 2, 48, 64, 4, 3, 37, 3, 0.02, False),               # odd C, odd G: scalar label branch
        (f"36-40-37-{_scene}", _scene, 2, 48, 64, 36, 40, 37, 5, 0.02, False),           # partial slab, float4 labels
        (f"33-41-16-{_scene}", _scene, 2, 48, 64, 33, 41, 16, 3, 0.02, False),           # unfused: <1> passes
        (f"6-22-37-{_scene}", _scene, 2, 48, 64, 6, 22, 37, 5, 0.02, False),
    ]
CASES.append(("thr0-8-22-16-smooth", "smooth", 2, 48, 64, 8, 22, 16, 3, 0.0, False))      # nothing hits


def _seed(cid):
    return 11 + sum(ord(ch) for ch in cid)


@pytest.mark.parametrize("cid,scene,B,H,W,Cf,C,G,ks,thr,feed", CASES, ids=[c[0] for c in CASES])
def test_project_backproject_exact(cuda, cid, scene, B, H, W, Cf, C, G, ks, thr, feed):
    from posecnn_b200.backprojecting_layer import backprojecting_op as bop
    from posecnn_b200.projecting_layer import projecting_op as pop
    c = make_case(scene, B, H, W, Cf, C, G, _seed(cid))
    print(f"\n{cid}: B={B} {H}x{W} Cf={Cf} C={C} G={G} k={ks} thr={thr}")
    keys = ("data", "label", "depth", "meta", "label_3d")
    al = {k: T(c[k], cuda) for k in keys}
    off = {k: T_offset(c[k], cuda) for k in keys}
    l3off = dict(al, label_3d=off["label_3d"])
    rows = set()

    # ---- Backproject forward: oracle, three device variants
    td_w, tl_w, tf_w, amb3 = oracle.backproject(c["data"], c["label"], c["depth"], c["meta"], c["label_3d"], G, ks, thr,
                                                return_ambig=True)
    coverage(scene, c["depth"], c["meta"], G, ks, thr, tf_w, "windows")
    check_ambig("backproject", amb3, "Backproject")
    outs = {}
    for name, t in (("aligned", al), ("offset", off), ("label_3d offset", l3off)):
        o = bop.backproject(t["data"], t["label"], t["depth"], t["meta"], t["label_3d"], G, ks, thr)
        r = bp_rows(B, G, Cf, C, t, o)
        print(f"  Backproject {name}: {sorted(r)}")
        rows |= r
        outs[name] = o
    for name in ("offset", "label_3d offset"):
        for i, what in enumerate(("top_data", "top_label", "top_flag")):
            assert_device_equal(outs[name][i], outs["aligned"][i], f"{what} {name}")
    td, tl, tf = outs.pop("aligned")
    outs.clear()
    nd = assert_oracle_equal(to_np(tf), tf_w, amb3, "top_flag")
    nd += assert_oracle_equal(to_np(td), td_w, amb3, "top_data")
    nd += assert_oracle_equal(to_np(tl), tl_w, amb3, "top_label")
    print(f"  Backproject: {nd} ambiguous entries differ from the oracle")
    if thr == 0:
        assert not tf.any() and not bits(td).any()
        assert torch.equal(bits(tl), bits(al["label_3d"]))
    if C == 1:                           # the one-channel labels: every hit voxel is an average, not the label_3d copy
        hitv = (tf_w[..., 0] > 0) & ~amb3
        assert hitv.sum() > 0
        np.testing.assert_array_equal(to_np(tl)[hitv], tl_w[hitv])
    del td_w, tl_w, tf_w, tl, tf

    # ---- Project forward (on Backproject's output, as the benchmark does, or on a random grid)
    vox = td if feed else al["data"].new_tensor(c["vox"])
    vox_np = to_np(vox)
    want, amb = oracle.project(vox_np, c["depth"], c["meta"], return_ambig=True)
    check_ambig("project", amb, "Project", c["depth"])
    got = pop.project(vox, al["depth"], al["meta"], ks, thr)
    rows.add(gather_row(Cf, vox.data_ptr(), got.data_ptr()))
    vox_off = T_offset(vox_np, cuda)
    got_off = pop.project(vox_off, off["depth"], off["meta"], ks, thr)
    rows.add(gather_row(Cf, vox_off.data_ptr(), got_off.data_ptr()))
    assert_device_equal(got_off, got, "Project offset")
    nd = assert_oracle_equal(to_np(got), want, amb, "Project")
    if feed or scene == "smooth":
        assert (np.abs(want).sum(-1) > 0).mean() > 0.3
    del vox, vox_off, got, got_off, td

    # ---- BackprojectGrad: the gather of top_diff [B,G,G,G,Cf]
    g3 = al["data"].new_tensor(c["vox"])
    want, amb = oracle.backproject_grad(c["vox"], c["depth"], c["meta"], return_ambig=True)
    got = bop.backproject_grad(al["data"], al["depth"], al["meta"], g3, G)
    rows.add(gather_row(Cf, g3.data_ptr(), got.data_ptr()))
    g3o = T_offset(c["vox"], cuda)
    got_off = bop.backproject_grad(off["data"], off["depth"], off["meta"], g3o, G)
    rows.add(gather_row(Cf, g3o.data_ptr(), got_off.data_ptr()))
    assert_device_equal(got_off, got, "BackprojectGrad offset")
    nd += assert_oracle_equal(to_np(got), want, amb, "BackprojectGrad")
    del g3, g3o, got, got_off

    # ---- ProjectGrad: the window average of top_diff [B,H,W,Cf]
    want, amb = oracle.project_grad(c["grad2"], c["depth"], c["meta"], G, ks, thr, return_ambig=True)
    grid = torch.empty((B, G, G, G, Cf), device=cuda)                  # bottom_data: only its shape is read
    g2, g2o = T(c["grad2"], cuda), T_offset(c["grad2"], cuda)
    got = pop.project_grad(grid, al["depth"], al["meta"], g2, ks, thr)
    rows.add(average_row(Cf, g2.data_ptr(), got.data_ptr()))
    got_off = pop.project_grad(grid, off["depth"], off["meta"], g2o, ks, thr)
    rows.add(average_row(Cf, g2o.data_ptr(), got_off.data_ptr()))
    assert_device_equal(got_off, got, "ProjectGrad offset")
    nd += assert_oracle_equal(to_np(got), want, amb, "ProjectGrad")
    if thr == 0:
        assert not bits(got).any()
    print(f"  Project / BackprojectGrad / ProjectGrad: {nd} ambiguous entries differ from the oracle; kernels {sorted(rows)}")
    REACHED.update(rows)
    RAN.add(cid)


# ---------------------------------------------------------------------------------------------------------------------
# voxels on the camera plane facing depth holes
# ---------------------------------------------------------------------------------------------------------------------
def test_camera_plane_voxels_facing_depth_holes(cuda):
    """A grid with 0.25 m voxels whose plane w = 4 lies exactly on the camera plane (Z1 = 0, so x3 = 0): those voxels project
    to +-inf, and voxel (8, 8, 4) at the camera centre to 0 / 0 = NaN.  The left half of the image is a depth hole (0 m), so
    a NaN converted to pixel 0 would find |0 - Z1| = 0 < threshold in its window: the clamp before the conversion must keep
    every such voxel out of the image (no hit, the label_3d copy).  Hole pixels project to that same voxel (8, 8, 4)."""
    from posecnn_b200.backprojecting_layer import backprojecting_op as bop
    from posecnn_b200.projecting_layer import projecting_op as pop
    B, H, W, Cf, C, G, ks, thr = 1, 48, 64, 8, 3, 16, 3, 0.02
    rng = np.random.default_rng(41)
    meta = synth.make_meta(synth.intrinsics(H, W), G).reshape(1, 1, 1, 48)
    meta[..., 42:45] = 0.25
    meta[..., 45:48] = (-2.0, -2.0, -1.0)
    depth = np.full((B, H, W, 1), 1.25, np.float32)                      # the right half: on the voxel plane w = 9
    depth[:, :, :W // 2] = 0
    data = rng.standard_normal((B, H, W, Cf), dtype=np.float32)
    label = rng.random((B, H, W, C), dtype=np.float32)
    l3 = rng.random((B, G, G, G, C), dtype=np.float32)
    vox = rng.standard_normal((B, G, G, G, Cf), dtype=np.float32)
    d = {k: T(v, cuda) for k, v in dict(data=data, label=label, depth=depth, meta=meta, l3=l3, vox=vox).items()}
    td, tl, tf = bop.backproject(d["data"], d["label"], d["depth"], d["meta"], d["l3"], G, ks, thr)
    td, tl, tf = to_np(td), to_np(tl), to_np(tf)
    assert not tf[:, :, :, 4].any() and not td[:, :, :, 4].any()
    np.testing.assert_array_equal(bits(tl[:, :, :, 4]), bits(l3[:, :, :, 4]))
    td_w, tl_w, tf_w, amb = oracle.backproject(data, label, depth, meta, l3, G, ks, thr, return_ambig=True)
    assert amb[:, :, :, 4].all()                                       # the oracle cannot speak for them: checked above
    assert tf_w[:, :, :, 9].any()
    for got, want in ((tf, tf_w), (td, td_w), (tl, tl_w)):
        assert_oracle_equal(got, want, amb, "camera-plane Backproject")
    gp = to_np(pop.project_grad(d["vox"], d["depth"], d["meta"], T(data, cuda), ks, thr))
    assert not bits(gp[:, :, :, 4]).any()
    gp_w, amb2 = oracle.project_grad(data, depth, meta, G, ks, thr, return_ambig=True)
    assert_oracle_equal(gp, gp_w, amb2, "camera-plane ProjectGrad")
    pf = to_np(pop.project(d["vox"], d["depth"], d["meta"], ks, thr))
    np.testing.assert_array_equal(bits(pf[0, :, :W // 2]), bits(np.broadcast_to(vox[0, 8, 8, 4], (H, W // 2, Cf))))
    pf_w, amb3 = oracle.project(vox, depth, meta, return_ambig=True)
    assert_oracle_equal(pf, pf_w, amb3, "camera-plane Project")


# ---------------------------------------------------------------------------------------------------------------------
# the unfused passes: PCNN_BACKPROJECT_FUSED=0 is read once per process, so they run in a child process
# ---------------------------------------------------------------------------------------------------------------------
# (scene, B, H, W, Cf, C, G, kernel_size, threshold, seed)
UNFUSED = [
    ("iid", 2, 48, 64, 64, 16, 16, 3, 0.02, 51),        # wide<16> with flag and with fallback
    ("smooth", 2, 48, 64, 36, 40, 37, 3, 0.02, 52),     # <4> with flag and with fallback
    ("iid", 2, 48, 64, 4, 41, 16, 5, 0.02, 53),         # <4> with flag, <1> with fallback
    ("iid", 2, 48, 64, 64, 22, 16, 3, 0.02, 54),        # wide<16> with flag, wide<32> with fallback
]


def _unfused_child(path):
    """Runs in a child process with PCNN_BACKPROJECT_FUSED=0: Backproject of every UNFUSED case, saved to `path`."""
    from posecnn_b200.backprojecting_layer import backprojecting_op as bop
    assert os.environ.get("PCNN_BACKPROJECT_FUSED") == "0"
    dev = torch.device("cuda:0")
    res = {}
    for i, (scene, B, H, W, Cf, C, G, ks, thr, seed) in enumerate(UNFUSED):
        c = make_case(scene, B, H, W, Cf, C, G, seed)
        t = {k: T(c[k], dev) for k in ("data", "label", "depth", "meta", "label_3d")}
        o = bop.backproject(t["data"], t["label"], t["depth"], t["meta"], t["label_3d"], G, ks, thr)
        for name, x in zip(("td", "tl", "tf"), o):
            res[f"{i}_{name}"] = to_np(x)
    torch.cuda.synchronize()
    np.savez(path, **res)


def test_unfused_passes_equal_the_fused_kernel(cuda, tmp_path):
    from posecnn_b200.backprojecting_layer import backprojecting_op as bop
    path = str(tmp_path / "unfused.npz")
    env = dict(os.environ, PCNN_BACKPROJECT_FUSED="0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import sys; from tests.test_project_exact_gpu import _unfused_child; _unfused_child(sys.argv[1])", path]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = np.load(path)
    rows = set()
    for i, (scene, B, H, W, Cf, C, G, ks, thr, seed) in enumerate(UNFUSED):
        c = make_case(scene, B, H, W, Cf, C, G, seed)
        t = {k: T(c[k], cuda) for k in ("data", "label", "depth", "meta", "label_3d")}
        o = bop.backproject(t["data"], t["label"], t["depth"], t["meta"], t["label_3d"], G, ks, thr)
        fused = bp_rows(B, G, Cf, C, t, o)
        # the child's tensors are fresh allocations like these: the same pointer alignment, with the fused kernel off
        child = bp_rows(B, G, Cf, C, t, o, fused_on=False)
        print(f"\nunfused case {i} ({scene}, Cf={Cf} C={C} G={G} k={ks}): parent {sorted(fused)}, child {sorted(child)}")
        assert all(k != FUSED for k, _ in child)
        rows |= fused | child
        td_w, tl_w, tf_w, amb = oracle.backproject(c["data"], c["label"], c["depth"], c["meta"], c["label_3d"], G, ks, thr,
                                                   return_ambig=True)
        coverage(scene, c["depth"], c["meta"], G, ks, thr, tf_w, "windows")
        check_ambig("backproject", amb, "Backproject")
        for name, x, w in zip(("td", "tl", "tf"), o, (td_w, tl_w, tf_w)):
            np.testing.assert_array_equal(bits(got[f"{i}_{name}"]), bits(to_np(x)), err_msg=f"unfused {name} case {i}")
            assert_oracle_equal(got[f"{i}_{name}"], w, amb, f"unfused {name} case {i}")
    REACHED.update(rows)
    RAN.add("unfused")


# ---------------------------------------------------------------------------------------------------------------------
# offsets past 2^31 elements: B = 17 at the benchmark's shape (run once)
# ---------------------------------------------------------------------------------------------------------------------
def test_offsets_past_2_31_elements(cuda):
    """Image 16's top_data starts at element 16 * 128^3 * 64 = 2^31.  Images 0 and 16 of all four ops equal the op run on that
    image alone (compared on the device), and image 16 equals the oracle.  The ops run in sequence and free what the next
    does not need: peak device memory ~28 GB (top_data + top_flag 18.3 GB, top_label + label_3d 6.3 GB, inputs 1.8 GB, one
    single-image call 1.4 GB)."""
    from posecnn_b200.backprojecting_layer import backprojecting_op as bop
    from posecnn_b200.projecting_layer import projecting_op as pop
    B, H, W, Cf, C, G, ks, thr = 17, 480, 640, 64, 22, 128, 3, 0.02
    assert 16 * G ** 3 * Cf == 2 ** 31
    geo = synth.make_projection_case(B, H, W, 1, 1, G, seed=71)              # the benchmark's depth and meta
    depth = geo["depth"]
    depth[::2] = smooth_depth(B, H, W, 72)[::2]                              # images 0, 2, ..., 16: the smooth scene
    meta = geo["meta"]
    del geo
    g = torch.Generator(device=cuda).manual_seed(73)
    data = torch.randn((B, H, W, Cf), device=cuda, generator=g)
    label = torch.rand((B, H, W, C), device=cuda, generator=g)
    l3 = torch.rand((B, G, G, G, C), device=cuda, generator=g)
    dep, met = T(depth, cuda), T(meta, cuda)
    rows = set()
    one = lambda x, i: x[i:i + 1]

    td, tl, tf = bop.backproject(data, label, dep, met, l3, G, ks, thr)
    rows |= backproject_rows(B, G, Cf, C, data.data_ptr(), l3.data_ptr(), td.data_ptr(), tl.data_ptr(), tf.data_ptr())
    for i in (0, 16):
        s = bop.backproject(one(data, i), one(label, i), one(dep, i), one(met, i), one(l3, i), G, ks, thr)
        for what, a, b in zip(("top_data", "top_label", "top_flag"), (td, tl, tf), s):
            assert_device_equal(one(a, i), b, f"{what} image {i}")
        del s
    td16 = to_np(td[16])[None]
    td_w, tl_w, tf_w, amb = oracle.backproject(to_np(data[16])[None], to_np(label[16])[None], depth[16:17], meta[16:17],
                                               to_np(l3[16])[None], G, ks, thr, return_ambig=True)
    facts = coverage("smooth", depth[16:17], meta[16:17], G, ks, thr, tf_w, "image 16 windows")
    check_ambig("backproject", amb, "image 16 Backproject")
    assert_oracle_equal(td16, td_w, amb, "top_data image 16")
    del td_w
    assert_oracle_equal(to_np(tf[16])[None], tf_w, amb, "top_flag image 16")
    del tf_w
    assert_oracle_equal(to_np(tl[16])[None], tl_w, amb, "top_label image 16")
    del tl_w

    # Project on top_data, then BackprojectGrad with top_data as its top_diff
    for name, fn in (("Project", lambda v, i=None: pop.project(v, dep if i is None else one(dep, i),
                                                               met if i is None else one(met, i), ks, thr)),
                     ("BackprojectGrad", lambda v, i=None: bop.backproject_grad(data if i is None else one(data, i),
                                                                                dep if i is None else one(dep, i),
                                                                                met if i is None else one(met, i), v, G))):
        out = fn(td)
        rows.add(gather_row(Cf, td.data_ptr(), out.data_ptr()))
        for i in (0, 16):
            assert_device_equal(one(out, i), fn(one(td, i), i), f"{name} image {i}")
        want, amb = oracle.project(td16, depth[16:17], meta[16:17], return_ambig=True)
        check_ambig("project", amb, f"image 16 {name}", depth[16:17])
        assert_oracle_equal(to_np(out[16])[None], want, amb, f"{name} image 16")
        del out

    # ProjectGrad of data: its 9.1 GB grid takes the place of top_flag, top_label and label_3d
    del tf, tl, l3
    torch.cuda.empty_cache()
    pg = pop.project_grad(td, dep, met, data, ks, thr)
    rows.add(average_row(Cf, data.data_ptr(), pg.data_ptr()))
    for i in (0, 16):
        assert_device_equal(one(pg, i), pop.project_grad(one(td, i), one(dep, i), one(met, i), one(data, i), ks, thr),
                            f"ProjectGrad image {i}")
    del td
    want, amb = oracle.project_grad(to_np(data[16])[None], depth[16:17], meta[16:17], G, ks, thr, return_ambig=True)
    check_ambig("backproject", amb, "image 16 ProjectGrad")
    assert_oracle_equal(to_np(pg[16])[None], want, amb, "ProjectGrad image 16")
    print(f"\nB = 17: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB; kernels {sorted(rows)}; {facts}")
    del pg
    torch.cuda.empty_cache()
    rows.add(("offsets past 2^31 elements", "B = 17"))
    REACHED.update(rows)
    RAN.add("B17")


def test_every_dispatch_row_is_reached():
    """The union of the cases above reaches every kernel and branch of the dispatch table."""
    expected = {c[0] for c in CASES} | {"unfused", "B17"}
    if RAN != expected:
        pytest.skip(f"only part of the module ran ({len(RAN)} of {len(expected)} producers)")
    for row in sorted(TABLE):
        print(f"{row[0]:34s} {row[1]:12s} {'reached' if row in REACHED else 'MISSING'}")
    assert TABLE <= REACHED, sorted(TABLE - REACHED)
