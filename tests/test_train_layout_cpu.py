"""The training step's parameter-layout table (posecnn_b200/train.py param_layout / KINDS) on the CPU: every parameter of the
colour, RGB-D and adaptation networks is trained exactly once, its fp32 master is the layout the step's kernels read (restated
below as explicit expressions), its 16-bit copy is the inference network's copy, and the inverse gives the TF tensor back bit for
bit."""
import pytest
import torch

from posecnn_b200 import conv, pose_head


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _explicit_master(name, w, C, U):
    """The master layouts, restated: [Cout][kh*kw*Cin] convolutions (conv1_1 [64][27]), score / vertex_pred zero-padded to 64 /
    max(128, 3C rounded up to a multiple of 64) rows, fc [out padded to x128][in], domain_score [2][256], biases as they are."""
    layer, kind = name.split("/")
    if kind == "b":
        return w
    if layer in ("conv1_1", "conv1_1_p"):
        return w.reshape(27, 64).t()
    if layer.startswith("conv"):
        return w.permute(3, 0, 1, 2).reshape(w.shape[3], -1)
    if layer in ("score_conv4", "score_conv5", "score_conv4_vertex", "score_conv5_vertex"):
        return w.reshape(w.shape[2], w.shape[3]).t()
    if layer in ("score", "vertex_pred"):
        rows, n = (64, C) if layer == "score" else (max(128, -(-3 * C // 64) * 64), 3 * C)
        out = torch.zeros((rows, w.shape[2]))
        out[:n] = w.reshape(w.shape[2], n).t()
        return out
    if layer == "domain_score":
        return w.t()
    out = torch.zeros(((w.shape[1] + 127) // 128 * 128, w.shape[0]))
    out[:w.shape[1]] = w.t()
    return out


@pytest.mark.parametrize("num_classes", [6, 44, 50])
@pytest.mark.parametrize("fmt,adaptation", [("COLOR", False), ("RGBD", False), ("COLOR", True)])
def test_param_layout_round_trips_bit_for_bit(fmt, adaptation, num_classes):
    from posecnn_b200.networks.vgg16_convs import vgg16_convs
    from posecnn_b200.train import KINDS, param_layout
    net = vgg16_convs(input_format=fmt, num_classes=num_classes, device="cpu", is_train=True, fold_vertex_head=False, adaptation=adaptation)
    shapes = net.param_shapes()
    layout = param_layout(net)
    assert sorted(tf for tf, _, _ in layout.values()) == sorted(shapes)
    g = torch.Generator().manual_seed(7)
    for name, (tf, kind, rows) in layout.items():
        k = KINDS[kind]
        w = torch.randn(shapes[tf], generator=g)
        master = k.to_master(w, rows)
        assert master.dtype == torch.float32 and master.is_contiguous(), name
        assert torch.equal(_bits(master), _bits(_explicit_master(name, w, net.num_classes, net.num_units))), name
        assert torch.equal(_bits(k.to_tf(master, w.shape)), _bits(w)), name
        if k.copy16 is not None and rows is None:
            want = pose_head.fc_weights_to_tc(w) if kind == "fc" else conv.hwio_to_tc(w)
            assert torch.equal(_bits(master.to(k.copy16)), _bits(want)), name
