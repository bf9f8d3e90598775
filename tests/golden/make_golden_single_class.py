"""Generate tests/golden/single_class.npz by EXECUTING THE REFERENCE'S OWN two-class rewrite of a frame's annotation
(lib/gt_synthesize_layer/minibatch.py:355-367) and its inverse before ICP (lib/fcn/test.py:1409-1414).  Both modules are
Python 2 and cannot be imported, so the blocks are cut out of the files unmodified (only de-indented) and exec'd with the
names they read.

    python tests/golden/make_golden_single_class.py        # needs /root/reference; the .npz is committed
"""
import os
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference/lib"
CLS_INDEX = 4                          # the object of the two-class model (e.g. LINEMOD 'camera')
NUM_CLASSES_ALL, B, H, W = 9, 4, 24, 32


def cut(path, first, last):
    """The lines from the first one starting with `first` to the next one starting with `last`, both stripped of indentation."""
    src = open(path).read().splitlines()
    s = next(i for i, l in enumerate(src) if l.strip().startswith(first))
    e = next(i for i in range(s, len(src)) if src[i].strip().startswith(last))
    return textwrap.dedent("\n".join(src[s:e + 1]))


def inputs():
    """B frames of a multi-object dataset: label images with up to 4 objects (image 2 does not contain CLS_INDEX) and their meta
    data (cls_indexes, poses [3,4,n], center [n,2], box [n,4]); ROI rows and labels of a two-class network's output."""
    rng = np.random.default_rng(17)
    frames = []
    for b in range(B):
        others = [c for c in range(1, NUM_CLASSES_ALL) if c != CLS_INDEX]
        cls = list(rng.choice(others, size=3, replace=False)) + ([] if b == 2 else [CLS_INDEX])
        rng.shuffle(cls)
        label = np.zeros((H, W), np.uint8)
        n = len(cls)
        box = np.zeros((n, 4), np.float32)
        for k, c in enumerate(cls):
            x1, y1 = rng.integers(0, W - 8), rng.integers(0, H - 6)
            x2, y2 = x1 + rng.integers(4, 9), y1 + rng.integers(3, 7)
            label[y1:y2, x1:x2] = c
            box[k] = (x1, y1, x2, y2)
        poses = rng.standard_normal((3, 4, n)).astype(np.float32)
        poses[2, 3, :] = rng.uniform(0.5, 1.5, n)
        frames.append(dict(label=label, cls_indexes=np.asarray(cls, np.float64).reshape(-1, 1), poses=poses,
                           center=rng.uniform(0, W, (n, 2)).astype(np.float64), box=box))
    labels2 = rng.integers(0, 2, (B, H, W)).astype(np.int32)
    rois2 = np.concatenate([rng.integers(0, B, (6, 1)), np.ones((6, 1)), rng.uniform(0, W, (6, 4)), rng.uniform(0, 1, (6, 1))], 1)
    return frames, labels2, rois2.astype(np.float32)


def main():
    fwd = cut(os.path.join(REF, "gt_synthesize_layer", "minibatch.py"), "if num_classes == 2 and roidb[i]['cls_index'] > 0:",
              "meta_data['box'] = meta_data['box'][ind,:]")
    inv = cut(os.path.join(REF, "fcn", "test.py"), "labels_icp = labels.copy();", "rois_icp[:, 1] = imdb._cls_index")
    frames, labels2, rois2 = inputs()
    out = {}
    for b, f in enumerate(frames):
        meta = dict(cls_indexes=f["cls_indexes"].flatten(), poses=f["poses"].copy(), center=f["center"].copy(), box=f["box"].copy())
        ns = dict(np=np, num_classes=2, roidb=[{"cls_index": CLS_INDEX}], i=0, im=f["label"].copy(), meta_data=meta)
        exec(fwd, ns)
        for k in ("label", "cls_indexes", "poses", "center", "box"):
            out[f"in{b}_{k}"] = f[k]
        out[f"out{b}_label"] = ns["im"]
        out[f"out{b}_ind"] = np.asarray(ns["cls_indexes_old"], np.int64)
        for k in ("cls_indexes", "poses", "center", "box"):
            out[f"out{b}_{k}"] = np.asarray(ns["meta_data"][k])
    labels_out, rois_out = [], []
    for b in range(B):
        ns = dict(np=np, imdb=types.SimpleNamespace(num_classes=2, _cls_index=CLS_INDEX), labels=labels2[b], rois=rois2)
        exec(inv, ns)
        labels_out.append(ns["labels_icp"])
        rois_out.append(ns["rois_icp"])
    assert all((r == rois_out[0]).all() for r in rois_out)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "single_class.npz"), cls_index=CLS_INDEX, num_classes_all=NUM_CLASSES_ALL,
                        batch=B, icp_labels_in=labels2, icp_rois_in=rois2, icp_labels_out=np.stack(labels_out), icp_rois_out=rois_out[0],
                        **out)
    print("kept rows per image:", [len(out[f"out{b}_ind"]) for b in range(B)])


if __name__ == "__main__":
    main()
