"""Object-coordinate (VERTEX_REG_3D) training against the 2-D pose_reg=False step, in one process on one GPU, arms alternating.

Inputs: the seeded synthetic 640x480 scene of `bench.py --workload train` (tools/bench_train_rgbd.py make_inputs: 22 classes), at C = 2
its single-class view (tools/bench_single_class.py two_class_inputs), and a seeded object-coordinate map vertmap [B,H,W,3] (uniform
in +-0.1 m; the cost does not depend on the values).  Both arms of a class count train the same labels and presence table; the 2-D
arm is vgg16_convs(pose_reg=False), the 3-D arm vgg16_convs(vertex_reg_2d=False, vertex_reg_3d=True).  Reported per C in (2, 22):
  train    ms per step at --batch (64), --runs runs of --warmup + --steps steps, the two arms in turn, CUDA events
  up8_bwd  ms per launch of the up-sampling adjoint alone, pcnn_up8_heads_bwd with the 2-D and with the 3-D target (vertmap and
           extents given) on the same heads, labels and presence table, alternating
The card name and power limit are read in the same run with a read-only nvidia-smi query.

    python tools/bench_train_coord.py [--batch 64] [--steps 10] [--warmup 3] [--runs 3]
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
from bench_single_class import timed, timed_steps, two_class_inputs   # noqa: E402
from bench_train_rgbd import H, W, gpu_info, make_inputs           # noqa: E402
from posecnn_b200 import heads                                     # noqa: E402
from posecnn_b200.networks.vgg16_convs import vgg16_convs         # noqa: E402
from posecnn_b200.train import Trainer                             # noqa: E402


class CoordStep:
    """Trainer.step with the object-coordinate map bound (timed_steps calls tr.step(*args))."""
    def __init__(self, tr, vertmap):
        self.tr, self.vertmap = tr, vertmap

    def step(self, *args):
        return self.tr.step(*args, vertmap=self.vertmap)


def make_trainer(dev, C, coord):
    kw = dict(vertex_reg_2d=False, vertex_reg_3d=True) if coord else {}
    net = vgg16_convs(num_classes=C, device=dev, is_train=True, fold_vertex_head=False, pose_reg=False, **kw).init_random(seed=0)
    net.params["score/weights"] *= 0.02; net.params["vertex_pred/weights"] *= 0.02
    net.prepare()
    return Trainer(net, lr=1e-4, momentum=0.9, weight_decay=1e-4, vertex_w=1.0, vertex_w_inside=10.0)


def up8_problem(dev, B, C, gt, centers, vertmap, ext):
    """Heads of a random low-resolution tensor (pcnn_up8_heads) and the two launches of the adjoint on the step's labels."""
    h, w = H // 8, W // 8
    g = torch.Generator().manual_seed(C)
    lowres = (torch.randn(B, h, w, 4 * C, generator=g) * 0.7).to(dev)
    bs, bv = (torch.randn(C, generator=g) * 0.1).to(dev), (torch.randn(3 * C, generator=g) * 0.1).to(dev)
    _, _, prob, score = heads.up8_heads(lowres, bs, bv, prob=True, score=True)
    cls_out, vtx_out = torch.tensor([0.5, 1e5], device=dev), torch.tensor([0.5, 1e5], device=dev)
    out = heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0)

    def run(vm, ex):                                   # vertmap / extents None: the 2-D target
        heads.up8_heads_bwd(prob, score, gt, cls_out, 1.0, 0.7, lowres, bv, centers, vtx_out, 1.0, 10.0, 1.0, vertmap=vm, extents=ex, out=out)
    return (lambda: run(None, None)), (lambda: run(vertmap, ext))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = gpu_info()
    B = a.batch
    args22, _ = make_inputs(dev, B)
    _, args2 = two_class_inputs(args22)
    vertmap = ((torch.rand((B, H, W, 3), generator=torch.Generator().manual_seed(7)) - 0.5) * 0.2).to(dev)
    out = dict(metric="object-coordinate (VERTEX_REG_3D) training step vs the 2-D pose_reg=False step", batch=B, image=f"{W}x{H}",
               steps=a.steps, warmup=a.warmup, runs=a.runs, gpu=info["name"], power_limit=info["power_limit"])
    for C, args in ((2, args2), (22, args22)):
        arms = {f"train_2d_c{C}": make_trainer(dev, C, False), f"train_3d_c{C}": CoordStep(make_trainer(dev, C, True), vertmap)}
        res = {k: [] for k in arms}
        losses = {}
        for _ in range(a.runs):
            for k, tr in arms.items():
                ms, losses[k] = timed_steps(tr, args, a.steps, a.warmup)
                assert all(np.isfinite(v) for v in losses[k].values()), (k, losses[k])
                res[k].append(ms)
        for k in arms:
            out[k] = dict(ms_per_step=statistics.median(res[k]), ms_per_step_runs=res[k], frames_per_s=B / (statistics.median(res[k]) * 1e-3),
                          last_losses=losses[k])
        out[f"ratio_train_3d_over_2d_c{C}"] = out[f"train_3d_c{C}"]["ms_per_step"] / out[f"train_2d_c{C}"]["ms_per_step"]
        del arms
        torch.cuda.empty_cache()
        run_2d, run_3d = up8_problem(dev, B, C, args[1], args[2], vertmap, args[4])
        kres = {"2d": [], "3d": []}
        for _ in range(a.runs):
            kres["2d"].append(timed(run_2d, 20))
            kres["3d"].append(timed(run_3d, 20))
        for k, v in kres.items():
            out[f"up8_bwd_{k}_c{C}"] = dict(ms_per_launch=statistics.median(v), ms_runs=v)
        out[f"ratio_up8_bwd_3d_over_2d_c{C}"] = statistics.median(kres["3d"]) / statistics.median(kres["2d"])
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
