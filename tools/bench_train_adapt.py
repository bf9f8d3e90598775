"""Training-step time of the domain-adaptation network against the colour network, in one process on one GPU.

Both steps run on the seeded synthetic 640x480 scene of `bench.py --workload train` (22 classes, labels / centres / poses from
synth.make_scene(seed=4234), images from synth.make_images(seed=21)), through tools/bench_train_rgbd.py's make_inputs.  The
adaptation step alternates a labelled batch with an "adapt" batch (the same images, labels -1 everywhere, no gt poses, no
centres), as the reference's data layer does at ADAPT_RATIO = 1 (lib/gt_synthesize_layer/layer.py:92-99), with ADAPT_WEIGHT = 1.0
of experiments/cfgs/lov_color_sugar_box_adapt.yml.  The two networks alternate, three runs each: every run is --warmup untimed
steps and --steps steps timed with CUDA events.  A third trainer runs the adaptation network on labelled batches only.  The
adaptation step adds fc9's three GEMMs (2 x rows x 25088 x 256 FLOP each)
and the pool_score gradient merge.  The card name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/bench_train_adapt.py [--batch 64] [--steps 20] [--warmup 4] [--runs 3]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_train_rgbd import C, H, W, gpu_info, make_inputs        # noqa: E402
from posecnn_b200.networks.vgg16_convs import vgg16_convs         # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402


def make_trainer(dev, adaptation):
    net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False, adaptation=adaptation).init_random(seed=0)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02; net.params["fc8/weights"] *= 0.01
    net.prepare()
    return Trainer(net, lr=1e-4, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0, margin=0.01, adapt_weight=1.0)


def timed_run(tr, batches, steps, warmup):
    """steps over the batches in turn (one batch: the colour step; two: labelled / adapt)."""
    torch.cuda.reset_peak_memory_stats()
    for i in range(warmup):
        out = tr.step(*batches[i % len(batches)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    outs = []
    for i in range(steps):
        out = tr.step(*batches[i % len(batches)])
        if i >= steps - len(batches):
            outs.append(out)
    e1.record()
    torch.cuda.synchronize()
    keys = ("loss_cls", "loss_vertex", "loss_pose") + (("loss_domain",) if "loss_domain" in outs[0] else ())
    losses = [{k: float(o[k].item()) for k in keys} for o in outs]
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated(), losses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    B = a.batch
    labelled, _ = make_inputs(dev, B)
    adapt = (labelled[0], torch.full_like(labelled[1], -1), torch.zeros_like(labelled[2]), labelled[3], labelled[4],
             torch.zeros((0, 13), device=dev), labelled[6], labelled[7])
    # "adapt_labelled": the adaptation network on labelled batches only, which isolates the branch's own cost (an adapt batch has no
    # labelled pixel, so its head-loss gradient is cheaper than a labelled batch's)
    runs = {"color": (make_trainer(dev, False), [labelled]), "adapt": (make_trainer(dev, True), [labelled, adapt]),
            "adapt_labelled": (make_trainer(dev, True), [labelled])}
    res = {k: dict(ms=[], mem=0, losses=None) for k in runs}
    for _ in range(a.runs):
        for k, (tr, batches) in runs.items():
            ms, mem, losses = timed_run(tr, batches, a.steps, a.warmup)
            res[k]["ms"].append(ms)
            res[k]["mem"] = max(res[k]["mem"], mem)
            res[k]["losses"] = losses
            assert all(np.isfinite(v) for d in losses for v in d.values()), (k, losses)
    out = dict(metric="training step, domain adaptation (labelled / adapt batches alternating) vs colour network", batch=B,
               steps=a.steps, warmup=a.warmup, runs=a.runs, image=f"{W}x{H}", gpu=info["name"], power_limit=info["power_limit"])
    for k in runs:
        ms = statistics.median(res[k]["ms"])
        out[k] = dict(ms_per_step=ms, ms_per_step_runs=res[k]["ms"], frames_per_s=B / (ms * 1e-3),
                      max_memory_allocated_gib=res[k]["mem"] / 2**30, last_losses=res[k]["losses"])
    out["ratio_adapt_over_color"] = out["adapt"]["ms_per_step"] / out["color"]["ms_per_step"]
    out["ratio_adapt_labelled_over_color"] = out["adapt_labelled"]["ms_per_step"] / out["color"]["ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
