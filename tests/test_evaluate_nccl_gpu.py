"""N = 2 over NCCL (needs two GPUs): evaluators on two image shards of one batch, summed by Evaluator.all_reduce, hold the state
of one evaluator over the whole batch (DESIGN.md §14)."""
import pytest

from tests.train_ref import ROOT, run_two_ranks

pytestmark = pytest.mark.gpu

WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, %r)
from posecnn_b200 import synth
from posecnn_b200.evaluate import Evaluator
from tests import eval_ref
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
c = eval_ref.make_case("lov")
C = c["C"]
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
sets = ("poses", "poses_refined", "poses_icp")
new = lambda: Evaluator(C, synth.make_model_points(C, 2620), c["extents"], c["symmetric"], pose_sets=sets, device=dev)
def score(ev, b0, b1):
    sel = (c["gt_rows"][:, 0] >= b0) & (c["gt_rows"][:, 0] < b1)
    ev.add_poses(T(c["gt_rows"][sel]), T(c["rois"]), {s: T(c["poses"][i]) for i, s in enumerate(sets)},
                 torch.tensor([c["num_rows"]], dtype=torch.int32, device=dev), T(c["meta"][b0:b1]), batch_offset=b0)
    ev.add_labels(T(c["gt_label"][b0:b1]), T(c["label"][b0:b1]))
whole = new()
score(whole, 0, 2)
shard = new()
score(shard, rank, rank + 1)
shard.all_reduce()
torch.cuda.synchronize()
assert torch.equal(shard.state, whole.state), rank
dist.barrier()
dist.destroy_process_group()
print("EVAL_RANK_OK", rank)
''' % ROOT


def test_two_rank_all_reduce_equals_single_evaluator(tmp_path):
    run_two_ranks(tmp_path, WORKER, "EVAL_RANK_OK", timeout=600)
