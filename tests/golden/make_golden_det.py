"""Generate tests/golden/det.npz by running the REFERENCE'S OWN region-proposal code (plain numpy, imports under Python 3):
lib/rpn_layer/snippets.py::generate_anchors_pre and lib/rpn_layer/proposal_layer.py with the TEST settings of
lib/fcn/config.py:224-231.  Two modules of that chain need what is not here, and are bound as the reference binds them:
`fcn.config.cfg` becomes a stub holding the three RPN settings, and `utils.nms_wrapper.nms` becomes the reference's
lib/nms/py_cpu_nms.py (whose suppression predicate, IoU > thresh with +1 areas, is nms_kernel.cu's).

The inputs are tie-free (every foreground probability of an image is distinct), so the reference's unstable argsort orders
them exactly as the canonical order does.

    python tests/golden/make_golden_det.py          # needs /root/reference; the .npz is committed
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF_LIB = "/root/reference/lib"

# (tag, map h, map w, anchor scales): lov_det.yml (A = 20), linemod_*_det.yml (A = 30), a map with fewer than 6,000 anchors,
# and one whose NMS keeps fewer than 300 boxes
CASES = (("lov", 30, 40, (4, 8, 16, 32)), ("linemod", 30, 40, (3, 4, 5, 6, 7, 8)), ("small", 5, 7, (4, 8, 16, 32)),
         ("few", 4, 5, (4, 8, 16, 32)))
RATIOS = (0.5, 0.75, 1, 1.5, 2)


def inputs(seed, h, w, A):
    """rpn_cls_prob [1,h,w,2A] with distinct foreground probabilities (a shuffled grid of (0, 1)), rpn_bbox_pred [1,h,w,4A]."""
    rng = np.random.default_rng(seed)
    n = h * w * A
    fg = ((rng.permutation(n) + 1.0) / (n + 1.0)).astype(np.float32).reshape(1, h, w, A)
    prob = np.concatenate([np.float32(1) - fg, fg], axis=-1)
    deltas = rng.normal(0.0, 0.25, size=(1, h, w, 4 * A)).astype(np.float16).astype(np.float32)   # stored as fp16, exactly
    return prob, deltas


def load_reference():
    class Settings:
        RPN_PRE_NMS_TOP_N, RPN_POST_NMS_TOP_N, RPN_NMS_THRESH = 6000, 300, 0.7     # config.py:224-231

    config = types.ModuleType("fcn.config")
    config.cfg = {"TEST": Settings}
    fcn = types.ModuleType("fcn")
    fcn.config = config
    sys.modules["fcn"], sys.modules["fcn.config"] = fcn, config
    sys.path.insert(0, REF_LIB)
    from nms.py_cpu_nms import py_cpu_nms
    wrapper = types.ModuleType("utils.nms_wrapper")
    wrapper.nms = lambda dets, thresh: py_cpu_nms(dets, thresh)
    import utils  # noqa: F401  (the reference's lib/utils package)
    sys.modules["utils.nms_wrapper"] = wrapper
    from rpn_layer.proposal_layer import proposal_layer
    from rpn_layer.snippets import generate_anchors_pre
    return generate_anchors_pre, proposal_layer


def main():
    generate_anchors_pre, proposal_layer = load_reference()
    out = {}
    for k, (tag, h, w, scales) in enumerate(CASES):
        A = len(scales) * len(RATIOS)
        anchors, length = generate_anchors_pre(h, w, 16, scales, RATIOS)
        prob, deltas = inputs(100 + k, h, w, A)
        im_info = np.array([16 * h, 16 * w, 1.0], dtype=np.float32)
        rois, scores = proposal_layer(prob, deltas, im_info, "TEST", 16, anchors, A)
        out[f"{tag}_anchors"] = anchors
        out[f"{tag}_fg"], out[f"{tag}_deltas"] = prob[..., A:], deltas.astype(np.float16)   # rpn_cls_prob = [1 - fg, fg]
        out[f"{tag}_im"] = im_info[:2].copy()
        out[f"{tag}_rois"], out[f"{tag}_scores"] = rois.astype(np.float32), scores.astype(np.float32)
        print(tag, "A", A, "anchors", int(length), "proposals", rois.shape[0])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "det.npz"), **out)


if __name__ == "__main__":
    main()
