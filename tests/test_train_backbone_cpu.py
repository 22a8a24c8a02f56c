"""Backbone of training on the device (model.backbone_train_mode), the parts that need no GPU: the
switch and its errors, the reference fixture pinned to train_path.backbone in fp64, the fp64
restatements of the kernels' index arithmetic against autograd, and the running-statistics update
against nn.BatchNorm2d."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import make_train_backbone_golden as mtb
from oracle import oracle, workload
from oracle import train_backbone as otb
from onepose_plus_plus_b200 import OnePosePlus_model, train_backbone, train_path

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_backbone.npz")


def _model():
    return OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG)).train()


def test_switch_defaults_and_errors(monkeypatch):
    m = _model()
    assert m.backbone_train_mode == "autograd"
    monkeypatch.setenv("OPP_B200_BACKBONE_TRAIN", "kernels")
    assert _model().backbone_train_mode == "kernels"
    img = torch.zeros(1, 1, 64, 64)
    for bad in ("cudnn", "tf32x3", "TF32x3", "tf32", ""):
        m.backbone_train_mode = bad
        with pytest.raises(ValueError, match="backbone_train_mode"):
            train_backbone.use_kernels(m, {"query_image": img})
    monkeypatch.setenv("OPP_B200_BACKBONE_TRAIN", "tf32x3")
    with pytest.raises(ValueError, match="backbone_train_mode"):
        train_backbone.use_kernels(_model(), {"query_image": img})
    m.backbone_train_mode = "kernels"
    assert not train_backbone.use_kernels(m, {"query_image": img})               # CPU tensors: unchanged path
    assert not train_backbone.use_kernels(m.eval(), {"query_image": img})
    m.train()
    with pytest.raises(NotImplementedError, match="query_image"):
        train_backbone.check(m, {"query_image": img.clone().requires_grad_(True)})
    with pytest.raises(ValueError, match="multiples of 8"):
        train_backbone.check(m, {"query_image": torch.zeros(1, 1, 64, 60)})
    with pytest.raises(ValueError, match="more than 1 value"):
        train_backbone.check(m, {"query_image": torch.zeros(1, 1, 8, 8)})
    train_backbone.check(m, {"query_image": torch.zeros(2, 1, 8, 8)})
    m.backbone.eval()
    with pytest.raises(NotImplementedError, match="frozen"):
        train_backbone.check(m, {"query_image": torch.zeros(2, 1, 8, 8)})
    for p in m.backbone.parameters():
        p.requires_grad_(False)
    train_backbone.check(m, {"query_image": torch.zeros(1, 1, 8, 8)})           # pretrained_fix: forward only


def test_parameter_order_covers_the_backbone():
    bb = _model().backbone
    assert len(train_backbone.CONVS) == 22 and len(train_backbone.BNS) == 17
    got = {id(p) for p in train_backbone.params(bb)}
    assert got == {id(p) for p in bb.parameters()} and len(got) == len(train_backbone.params(bb))


@pytest.mark.parametrize("case_name", mtb.CASES)
def test_fixture_pinned_to_train_path_backbone_fp64(case_name):
    z = np.load(GOLDEN)
    sd = workload.synthetic_state_dict(0)
    bb = mtb.backbone_module(sd, train=case_name == "train")
    feat_c, feat_f, grads, bufs = mtb.run(bb, train_path.backbone, mtb.make_case())
    named = {"feat_c": feat_c, "feat_f": feat_f}
    named.update({f"d_{n}": g for n, g in zip(mtb.param_names(bb), grads)})
    for key, t in named.items():
        k = f"{case_name}_{key}"
        amax = float(z[k + "_absmax"])
        got = t.flatten()[torch.from_numpy(z[k + "_idx"])].numpy()
        assert np.abs(got - z[k]).max() <= 1e-10 * max(amax, 1.0), key
        assert abs(float(t.abs().max()) - amax) <= 1e-10 * max(amax, 1.0), key
    for n, b in bufs.items():
        np.testing.assert_allclose(b.numpy(), z[f"{case_name}_buf_{n}"], rtol=0, atol=1e-10, err_msg=n)
    if case_name == "eval":
        for n, b in sd.items():
            if n.startswith("backbone.") and ("running" in n or "num_batches" in n):
                assert torch.equal(bufs[n[len("backbone."):]].to(b.dtype), b), n


@pytest.mark.parametrize("k,stride,hw", [(3, 2, (7, 9)), (3, 2, (8, 8)), (1, 2, (6, 5)), (7, 2, (9, 12)),
                                         (3, 1, (5, 6))])
def test_dgrad_tap_selection_against_autograd(k, stride, hw):
    g = torch.Generator().manual_seed(k * 10 + stride)
    x = torch.randn(2, 3, *hw, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(4, 3, k, k, generator=g, dtype=torch.float64)
    y = F.conv2d(x, w, stride=stride, padding=k // 2)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, x, dy)
    torch.testing.assert_close(otb.conv_dgrad(dy, w, stride, hw), ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("hw", [(1, 1), (1, 3), (2, 2), (3, 5), (12, 16), (64, 48)])
def test_upsample_backward_ranges_against_autograd(hw):
    g = torch.Generator().manual_seed(hw[0] * 100 + hw[1])
    # fp32 input: autograd then uses the fp32 source index the kernels restate
    x = torch.randn(2, 3, *hw, generator=g).requires_grad_(True)
    y = F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=True)
    dy = torch.randint(-8, 9, y.shape, generator=g).float() / 16       # 2^-4 grid: every sum exact in fp64
    (ref,) = torch.autograd.grad(y, x, dy)
    got = otb.up2x_bwd(dy, hw)
    torch.testing.assert_close(got, ref.double(), rtol=0, atol=1e-5)
    for n in hw:
        for i in range(n):                     # the bound the kernel's scan window relies on
            assert all(2 * i - 2 <= d <= 2 * i + 3 for d in otb.up2x_taps(i, n)), (i, n)


@pytest.mark.parametrize("momentum", [0.1, None])
def test_running_statistics_update_against_batchnorm2d(momentum):
    g = torch.Generator().manual_seed(2)
    bn = torch.nn.BatchNorm2d(5, momentum=momentum).double().train()
    bn.running_mean.copy_(torch.randn(5, generator=g, dtype=torch.float64))
    bn.running_var.copy_(torch.rand(5, generator=g, dtype=torch.float64) + 0.5)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    x = torch.randn(3, 5, 4, 7, generator=g, dtype=torch.float64) * 2 + 1
    bn(x)
    assert int(bn.num_batches_tracked) == 1
    m = 1.0 if momentum is None else momentum                 # cumulative average after one batch: 1 / 1
    em, ev = otb.bn_running_update(x, rm, rv, m)
    torch.testing.assert_close(bn.running_mean, em, rtol=0, atol=1e-12)
    torch.testing.assert_close(bn.running_var, ev, rtol=0, atol=1e-12)
