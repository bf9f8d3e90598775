"""N = 2 over NCCL (needs two GPUs: `python -m pytest tests/test_multigpu_nccl_gpu.py -m gpu` on a two-GPU machine):
the gathered post-NMS records of two image shards of ONE global batch equal the single-GPU records (SURVEY.md §8(e))."""
import pytest

from tests.train_ref import ROOT, run_two_ranks, train_worker

pytestmark = pytest.mark.gpu

WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %r)
from posecnn_b200 import parallel, synth
from posecnn_b200.networks.vgg16_convs import vgg16_convs, GraphedForward
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
B, H, W, C = 8, 96, 128, 6
net = vgg16_convs(num_classes=C, device=dev).init_random(seed=0, bias_std=0.05)
rgb, _ = synth.make_images(B, H, W, seed=9)
data = torch.from_numpy(rgb).to(dev)
meta = torch.from_numpy(np.stack([synth.make_meta(synth.intrinsics(H, W))] * B)).to(dev)
ext = torch.from_numpy(synth.extents_for(C)).to(dev)
whole = parallel.compact_records(parallel.pack_detections(net.forward(data, meta, ext, sync_rois=False, dense_vertex=False)))
o, n = parallel.shard_range(B, rank, world)
fwd = GraphedForward(net, data[o:o + n], meta[o:o + n], ext, pack_records=True, dense_vertex=False, batch_global=B, batch_offset=o)
pipe = parallel.GatherPipeline(world, fwd.layers["records"])
ok = True
for step in range(4):                      # the double-buffered pipeline, several steps in flight
    pipe.before_step()
    L = fwd(data[o:o + n])
    i = pipe.submit(L["records"])
    got = parallel.compact_records(pipe.results(i))
    ok = ok and torch.equal(got, whole)
pipe.drain()
torch.cuda.synchronize()
assert whole.shape[0] >= 2 and ok, (rank, whole.shape)
dist.barrier()
dist.destroy_process_group()
print("RANK_OK", rank, whole.shape[0])
''' % ROOT


def test_two_rank_gather_equals_single_gpu(tmp_path):
    run_two_ranks(tmp_path, WORKER, "RANK_OK", timeout=600)


def test_two_rank_training_step_equals_single_gpu(tmp_path):
    """configs[4] contract: one SGD step on image shards over 2 ranks (global loss normalisers, NCCL all-reduce of the gradients)
    == the step on the whole batch on one GPU (gradients to 2e-3 relative: only the fp32 summation order differs)."""
    run_two_ranks(tmp_path, train_worker())
