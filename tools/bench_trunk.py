"""Per-launch timing of the convolution trunk (net._trunk) at batch 32, 640x480 uint8 input, launch by launch as the trunk
issues it: conv1_1 fused from uint8, the row-mode layer, the pooled conv1_2 / conv2_2 / conv3_3, pool4 and every
tile-kernel layer with the pixel tile and N tile (BN) the dispatcher picks.  Layers with Cout >= 256 are also timed at the
other BN (128 / 256), and the Cout = 128 layers (256-pixel tile) on the 128-pixel tile at BN = 128 (explicit block_n).
CUDA events around each launch, L2 flushed (256 MB write) before each one; median of --reps.

For the wgmma layers the table gives the operand bytes the CTAs request from L2 and their rate (bytes / time):
  tile kernel:  work items x K steps x (A box 16 KB + B box BN x 128 B)
  256-px tile:  work items x K steps x (A box 32 KB + B box BN x 128 B)
  row mode:     work items x 64-channel chunks x (A patch 65 KB + 9 weight slices of BN x 128 B unless they stay resident)
If a kernel were bound by L2 -> SM operand delivery, its layers would show the same rate at BN = 128 and BN = 256.

    python tools/bench_trunk.py [--batch 32] [--reps 10] [--json FILE]
"""
import argparse, json, math, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import conv
from posecnn_b200.build import build_native
from posecnn_b200.networks.vgg16_convs import PIXEL_MEANS, VGG_CFG, vgg16_convs

KC = 64                       # channels per K step
A_BYTES = 128 * KC * 2        # one 128-pixel A box
PATCH_BYTES = 130 * 4 * 128   # row mode: one {64 ch, 130 px, 4 rows} patch


def plan(B, H, W, Cin, Cout, block_n, pool):
    """Kernel, BN and L2 operand bytes of one pcnn_conv_bf16_tc / pcnn_conv_pool_bf16_tc call (the dispatcher's rule)."""
    if block_n == 0 and Cin <= 128 and Cout == 128:
        items = B * math.ceil(H / 16) * math.ceil(W / 16)
        return "tile256", 128, items * (9 * Cin // KC) * (2 * A_BYTES + 128 * 128)
    if block_n == 0 and Cin <= 128 and Cout == 64 and H % 2 == 0 and W >= 128:
        resb = Cin == 64
        items = B * (H // 2) * math.ceil(W / 128) * (Cout // 64)
        per_chunk = PATCH_BYTES + (0 if resb else 9 * 64 * 128)
        return ("row_resb" if resb else "row"), 64, items * (Cin // KC) * per_chunk
    bn = block_n or (256 if Cout % 256 == 0 and 9 * Cin >= 2304 else (128 if Cout % 128 == 0 else 64))
    th, tw = 8, 16
    if not pool and math.ceil(H / 16) * math.ceil(W / 8) < math.ceil(H / 8) * math.ceil(W / 16):
        th, tw = 16, 8
    pix = B * math.ceil(H / th) * math.ceil(W / tw)
    ksteps = 9 * Cin // KC
    return "tile", bn, pix * (Cout // bn) * ksteps * (A_BYTES + bn * 128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json")
    args = ap.parse_args()
    build_native()
    dev = torch.device("cuda:0")
    B, H, W = args.batch, 480, 640
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    net = vgg16_convs(num_classes=22, device=dev).init_random(seed=0)
    P, T = net.params, net._tc
    img = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device=dev, generator=torch.Generator(device=dev).manual_seed(21))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(3):
            out = fn()
        ts = []
        for _ in range(args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); out = fn(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2], out

    rows = []
    ms, x = timed(lambda: conv.conv1_fused(img, T["conv1_1/weights"], P["conv1_1/biases"], PIXEL_MEANS, True))
    rows.append(dict(layer="conv1_1", kernel="conv1_fused", bn=64, ms=ms, flop=2.0 * B * H * W * 27 * 64, operand_bytes=None, in_trunk=True))
    h, w = H, W
    cfg = VGG_CFG[1:]
    i = 0
    while i < len(cfg):
        item = cfg[i]
        if isinstance(item, str):
            ms, x = timed(lambda x=x: conv.maxpool2x2(x))
            rows.append(dict(layer=item, kernel="maxpool", bn=None, ms=ms, flop=0.0, operand_bytes=None, in_trunk=True))
            h, w = h // 2, w // 2
            i += 1
            continue
        name, ci, co = item
        pool = i + 1 < len(cfg) and isinstance(cfg[i + 1], str) and name not in ("conv4_3", "conv5_3")
        wt, bias = T[f"{name}/weights"], P[f"{name}/biases"]
        fl = 2.0 * B * h * w * 9 * ci * co
        kern, bn, nbytes = plan(B, h, w, ci, co, 0, pool)
        call = (lambda bn_, x=x: conv.conv_pool_bf16(x, wt, bias, 3, True, bn_)) if pool else (lambda bn_, x=x: conv.conv_bf16(x, wt, bias, 3, True, bn_))
        ms, y = timed(lambda: call(0))
        label = name + ("+" + cfg[i + 1] if pool else "")
        rows.append(dict(layer=label, kernel=kern, bn=bn, ms=ms, flop=fl, operand_bytes=nbytes, in_trunk=True))
        if co >= 256 or kern == "tile256":
            alt = 128 if bn == 256 or kern == "tile256" else 256
            _, _, nb_alt = plan(B, h, w, ci, co, alt, pool)
            ms_alt, _ = timed(lambda: call(alt))
            rows.append(dict(layer=label, kernel="tile", bn=alt, ms=ms_alt, flop=fl, operand_bytes=nb_alt, in_trunk=False))
        x = y
        if pool:
            h, w = h // 2, w // 2
            i += 2
        else:
            i += 1
    trunk_ms, _ = timed(lambda: net._trunk(img))

    print(f"GPU: {gpu}; batch {B} x {H}x{W}")
    print(f"{'layer':<16}{'kernel':<10}{'BN':>5}{'ms':>9}{'TFLOP/s':>9}{'L2->SM GB':>11}{'TB/s':>7}")
    for r in rows:
        tf = r["flop"] / r["ms"] / 1e9 if r["flop"] else None
        tbs = r["operand_bytes"] / r["ms"] / 1e9 if r["operand_bytes"] else None
        r["tflops"], r["operand_tbs"] = tf, tbs
        print(f"{r['layer'] if r['in_trunk'] else '  (other tile)':<16}{r['kernel']:<10}{r['bn'] or '-':>5}{r['ms']:>9.3f}"
              f"{(f'{tf:.0f}' if tf else '-'):>9}{(f'{r['operand_bytes'] / 1e9:.2f}' if r['operand_bytes'] else '-'):>11}{(f'{tbs:.2f}' if tbs else '-'):>7}")
    sum_ms = sum(r["ms"] for r in rows if r["in_trunk"])
    tile_ms = sum(r["ms"] for r in rows if r["in_trunk"] and r["kernel"].startswith("tile"))
    tile_fl = sum(r["flop"] for r in rows if r["in_trunk"] and r["kernel"].startswith("tile"))
    print(f"sum of the trunk's launches: {sum_ms:.3f} ms; tile-kernel layers {tile_ms:.3f} ms at {tile_fl / tile_ms / 1e9:.0f} TFLOP/s; "
          f"net._trunk as one call: {trunk_ms:.3f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=gpu, batch=B, rows=rows, sum_ms=sum_ms, tile_ms=tile_ms,
                           trunk_ms=trunk_ms), f, indent=1)


if __name__ == "__main__":
    main()
