"""Generate tests/golden/coord_pose_records.npz by EXECUTING THE REFERENCE'S OWN record assembly of the VERTEX_REG_3D test path
(lib/fcn/test.py:1383-1399, after SYN.estimate_poses_3d) and its `_get_bb2D` (test.py:1115-1148).  The module is Python 2 and
cannot be imported, so the function and the block are cut out of the file unmodified and exec'd with the names they need:
`np`, `xrange = range`, `imdb` (num_classes, _extents), `meta_data['intrinsic_matrix']`, `im_scale`, `poses_tmp`, and transforms3d's
`mat2quat` / `quat2mat` (absent here: oracle.mat2quat and the published quat2mat formula stand in).

    python tests/golden/make_golden_coord_pose.py        # needs /root/reference; the .npz is committed
"""
import os
import sys
import textwrap
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle  # noqa: E402
from posecnn_b200 import synth  # noqa: E402


def quat2mat(q):
    """transforms3d.quaternions.quat2mat (published formula), on the dtype it is given."""
    w, x, y, z = q
    Nq = w * w + x * x + y * y + z * z
    if Nq < np.finfo(np.float64).eps * 4:
        return np.eye(3)
    s = 2.0 / Nq
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ = w * X, w * Y, w * Z
    xX, xY, xZ = x * X, x * Y, x * Z
    yY, yZ, zZ = y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY], [xY + wZ, 1.0 - (xX + zZ), yZ - wX], [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def reference_code():
    src = open("/root/reference/lib/fcn/test.py").read().splitlines()
    a = next(i for i, l in enumerate(src) if l.startswith("def _get_bb2D"))
    b = next(i for i in range(a + 1, len(src)) if src[i].startswith("def "))
    s = next(i for i, l in enumerate(src) if "SYN.estimate_poses_3d(" in l)
    e = [i for i in range(s, len(src)) if src[i].strip() == "count += 1"][0]
    return "\n".join(src[a:b]), textwrap.dedent("\n".join(src[s + 1:e + 1]))


def cases():
    """(C, im_scale, poses_tmp [3,4,C]) with objects in front of the camera, one behind it, one absent."""
    out = []
    for C, scale, seed in ((22, 1.0, 1), (22, 1.5, 2), (2, 1.5, 3), (2, 1.0, 4)):
        rng = np.random.default_rng(seed)
        P = np.zeros((3, 4, C), np.float32)
        for j in range(1, C):
            if rng.random() < 0.25:
                continue                      # no pose
            P[:3, :3, j] = synth.quat_to_rot(synth._rand_quat(rng))
            P[:, 3, j] = (rng.uniform(-0.2, 0.2), rng.uniform(-0.15, 0.15), rng.uniform(0.5, 1.5))
            if rng.random() < 0.15:
                P[2, 3, j] = -P[2, 3, j]      # behind the camera: no record
        out.append((C, scale, P))
    return out


def main():
    fn_src, block = reference_code()
    K = synth.intrinsics(480, 640)
    data = {}
    for n, (C, scale, P) in enumerate(cases()):
        ns = dict(np=np, xrange=range, mat2quat=oracle.mat2quat, quat2mat=quat2mat, poses_tmp=P, im_scale=scale,
                  imdb=types.SimpleNamespace(num_classes=C, _extents=synth.extents_for(C)), meta_data={"intrinsic_matrix": K})
        exec(fn_src, ns)
        exec(block, ns)
        data[f"poses_tmp_{n}"] = P
        data[f"im_scale_{n}"] = np.float32(scale)
        data[f"rois_{n}"] = ns["rois"]
        data[f"poses_{n}"] = ns["poses"]
    data["K"] = K
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "coord_pose_records.npz"), **data)
    print({k: v.shape for k, v in data.items()})


if __name__ == "__main__":
    main()
