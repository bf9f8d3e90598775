"""Per-layer timing of the VGG16 conv stack (batch 32, 640x480): TFLOP/s and fraction of the bf16 peak
(MEASURED_PEAKS.json if present, else the H100 SXM data-sheet figure)."""
import json, os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from posecnn_b200 import conv
from posecnn_b200.build import build_native
build_native()
B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
dev = torch.device("cuda:0")
peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"bf16_tflops": 989.0}
layers = [("conv1_2", 480, 640, 64, 64), ("conv2_1", 240, 320, 64, 128), ("conv2_2", 240, 320, 128, 128),
          ("conv3_1", 120, 160, 128, 256), ("conv3_2", 120, 160, 256, 256), ("conv4_1", 60, 80, 256, 512),
          ("conv4_2", 60, 80, 512, 512), ("conv5_1", 30, 40, 512, 512)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
tot_t = tot_f = 0
for name, H, W, Cin, Cout in layers:
    x = torch.randn((B, H, W, Cin), device=dev).to(torch.bfloat16)
    w = conv.hwio_to_tc(torch.randn((3, 3, Cin, Cout), device=dev) * 0.05)
    b = torch.zeros((Cout,), device=dev)
    out = torch.empty((B, H, W, Cout), dtype=torch.bfloat16, device=dev)
    res = {}
    for bn in ([64, 0] if Cout == 64 else [128, 0] if Cout == 128 else [128, 256]):
        for _ in range(3):
            conv.conv_bf16(x, w, b, 3, True, bn, out)
        ts = []
        for _ in range(5):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); conv.conv_bf16(x, w, b, 3, True, bn, out); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]
        fl = 2.0 * B * H * W * 9 * Cin * Cout
        res[bn] = (ms, fl / ms / 1e9)
    best = min(res.items(), key=lambda kv: kv[1][0])
    mult = {"conv1_2": 1, "conv2_1": 1, "conv2_2": 1, "conv3_1": 1, "conv3_2": 2, "conv4_1": 1, "conv4_2": 2, "conv5_1": 3}[name]
    tot_t += best[1][0] * mult; tot_f += 2.0 * B * H * W * 9 * Cin * Cout * mult
    print(name, f"M={B*H*W} K={9*Cin} N={Cout}", " ".join(f"{('row-mode' if Cout == 64 else 'tile256') if bn == 0 else 'bn%d' % bn}: {ms:.3f} ms {tf:.0f} TFLOP/s ({tf/peaks['bf16_tflops']*100:.0f}%)" for bn, (ms, tf) in res.items()))
print(f"stack (12 tensor-core layers, best tile each): {tot_t:.2f} ms, {tot_f/tot_t/1e9:.0f} TFLOP/s = {tot_f/tot_t/1e9/peaks['bf16_tflops']*100:.0f}% of measured bf16 peak {peaks['bf16_tflops']}")
x = torch.randn((B, 480, 640, 3), device=dev); w = torch.randn((3, 3, 3, 64), device=dev) * 0.1; b = torch.zeros(64, device=dev)
for _ in range(2): y = conv.conv3x3_small_cin(x, w, b)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); y = conv.conv3x3_small_cin(x, w, b); e1.record(); torch.cuda.synchronize(); print("conv1_1 (CUDA cores)", e0.elapsed_time(e1), "ms")
e0.record(); p = conv.maxpool2x2(y); e1.record(); torch.cuda.synchronize(); print("pool1", e0.elapsed_time(e1), "ms")
