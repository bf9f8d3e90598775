"""Generate tests/golden/eval.npz by running the REFERENCE'S OWN lib/utils/pose_error.py (re, te, add, adi, reproj) and
lib/utils/se3.py (se3_mul) on the seeded cases of tests/eval_ref.make_case.  pose_error.py imports quat2mat / mat2quat from
transforms3d, which is not installed: a stub `transforms3d.quaternions` module carrying eval_ref.quat2mat (the published
function on float64) is placed in sys.modules first.  The Python 2 dataset code cannot be imported; fast_hist (imdb.py:123-125)
and the pairing loops of lov.py:576-628 / linemod.py:700-760 are the restatements of tests/eval_ref.py, which cite their lines.

    python tests/golden/make_golden_eval.py          # needs /root/reference; the .npz is committed
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from posecnn_b200 import synth  # noqa: E402
from tests import eval_ref  # noqa: E402

REF = "/root/reference/lib/utils"


def _load(name):
    spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(REF, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    t3d, quat = types.ModuleType("transforms3d"), types.ModuleType("transforms3d.quaternions")
    quat.quat2mat = eval_ref.quat2mat
    quat.mat2quat = None                                  # imported by pose_error.py, never called by the scorer
    t3d.quaternions = quat
    sys.modules.update({"transforms3d": t3d, "transforms3d.quaternions": quat})
    pe, se3 = _load("pose_error"), _load("se3")
    fns = dict(re=pe.re, te=pe.te, add=pe.add, adi=pe.adi, reproj=pe.reproj, se3_mul=se3.se3_mul)
    out = {}
    for tag in eval_ref.CASES:
        c = eval_ref.make_case(tag)
        C = c["C"]
        pts = synth.make_model_points(C, 2620)
        hist = eval_ref.fast_hist(c["gt_label"].reshape(-1), c["label"].reshape(-1), C)
        pairs, errors, flags, counts = eval_ref.score(c["gt_rows"], c["rois"], list(c["poses"]), c["num_rows"], c["meta"], pts,
                                                      c["symmetric"], c["threshold"], c["flip_z"], C, fns=fns)
        for k, v in c.items():
            out[f"{tag}_{k}"] = np.asarray(v)
        out.update({f"{tag}_hist": hist, f"{tag}_pairs": pairs, f"{tag}_errors": errors, f"{tag}_flags": flags,
                    f"{tag}_counts": counts})
        print(tag, "pairs", pairs.shape[0], "flips", int((flags & 4).astype(bool).sum()), "correct", counts[:, 1].sum(1).tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "eval.npz"), **out)


if __name__ == "__main__":
    main()
