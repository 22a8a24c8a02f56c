"""The "tf32x3" backbone mode (convolutions on the tensor cores in 3xTF32), the parts that need no GPU:
the switch and its environment preset, the errors it shares with "kernels", the autograd path on CPU
tensors and in eval mode, and the entry points the bindings pick."""
import copy

import pytest
import torch

from oracle import make_train_backbone_golden as mtb
from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, _lib, ops, train_backbone, train_path


def _model():
    return OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG)).train()


def test_mode_is_accepted_and_preset_by_the_environment(monkeypatch):
    assert "tf32x3" in train_backbone.MODES
    assert _model().backbone_train_mode == "autograd"
    monkeypatch.setenv("OPP_B200_BACKBONE_TRAIN", "tf32x3")
    m = _model()
    assert m.backbone_train_mode == "tf32x3"
    img = torch.zeros(1, 1, 64, 64)
    assert not train_backbone.use_kernels(m, {"query_image": img})               # CPU tensors: autograd path
    assert not train_backbone.use_kernels(m.eval(), {"query_image": img})       # eval mode: autograd path
    for bad in ("cudnn", "TF32x3", "tf32", ""):
        m.backbone_train_mode = bad
        with pytest.raises(ValueError, match="backbone_train_mode"):
            train_backbone.use_kernels(m, {"query_image": img})
    with pytest.raises(ValueError, match="device mode"):
        train_backbone.backbone(m.backbone, img, "autograd")


def test_cpu_forward_in_tf32x3_mode_is_the_autograd_path():
    """On CPU tensors a model.train() backbone in "tf32x3" mode is train_path.backbone, bit for bit."""
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    ref = mtb.run(mtb.backbone_module(sd, torch.float32), train_path.backbone, case, torch.float32)
    m = _model()
    m.backbone_train_mode = "tf32x3"
    bb = mtb.backbone_module(sd, torch.float32)
    assert not train_backbone.use_kernels(m, {"query_image": case["img"].float()})
    got = mtb.run(bb, train_path.backbone, case, torch.float32)
    for a, b in zip([ref[0], ref[1]] + ref[2], [got[0], got[1]] + got[2]):
        assert torch.equal(a, b)


def test_bindings_pick_the_tensor_core_entry_points():
    for name in ("opp_backbone_train_conv", "opp_backbone_train_conv_dgrad", "opp_backbone_train_conv_wgrad"):
        assert ops._tc(name, False) == name
        tc = ops._tc(name, True)
        assert tc == name + "_tf32x3"
        assert _lib.SIGNATURES[tc] == _lib.SIGNATURES[name]
    assert _lib.KERNELS_PER_CALL["opp_backbone_train_conv_wgrad_tf32x3"] == 2


def test_tf32x3_shares_the_kernels_mode_checks():
    m = _model()
    m.backbone_train_mode = "tf32x3"
    img = torch.zeros(1, 1, 64, 64)
    with pytest.raises(NotImplementedError, match="query_image"):
        train_backbone.check(m, {"query_image": img.clone().requires_grad_(True)})
    with pytest.raises(ValueError, match="multiples of 8"):
        train_backbone.check(m, {"query_image": torch.zeros(1, 1, 64, 60)})
    with pytest.raises(ValueError, match="more than 1 value"):
        train_backbone.check(m, {"query_image": torch.zeros(1, 1, 8, 8)})
