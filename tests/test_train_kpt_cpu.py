"""Keypoint encoder of training on the device (model.kpt_encoder_train_mode), the parts that need no
GPU: the switch and its errors, the reference fixture pinned to train_path.keypoint_encoding in fp64,
and the fp64 restatement of the manual backward (oracle/kpt_enc.py) against autograd."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import kpt_enc
from oracle import make_train_kpt_golden as mtk
from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, train_kpt, train_path

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_kpt.npz")


def _model(config=None):
    return OnePosePlus_model(copy.deepcopy(config or oracle.DEFAULT_CONFIG)).train()


def _data(B=1, N=4):
    return {"keypoints3d": torch.rand(B, N, 3), "descriptors3d_db": torch.randn(B, 256, N),
            "descriptors3d_coarse_db": torch.randn(B, 256, N)}


def test_switch_defaults_and_environment_preset(monkeypatch):
    m = _model()
    assert m.kpt_encoder_train_mode == "autograd"
    monkeypatch.setenv("OPP_B200_KPT_TRAIN", "kernels")
    assert _model().kpt_encoder_train_mode == "kernels"
    data = _data()
    assert not train_kpt.use_kernels(m, data)                      # default: unchanged path
    m.kpt_encoder_train_mode = "cublas"
    with pytest.raises(ValueError, match="kpt_encoder_train_mode"):
        train_kpt.use_kernels(m, data)
    m.kpt_encoder_train_mode = "kernels"
    assert not train_kpt.use_kernels(m, data)                      # CPU tensors: unchanged path
    assert not train_kpt.use_kernels(m.eval(), data)
    m.train()
    train_kpt.check(m, data)


def test_errors():
    m = _model()
    data = _data()
    with pytest.raises(NotImplementedError, match="keypoints3d"):
        train_kpt.check(m, dict(data, keypoints3d=data["keypoints3d"].clone().requires_grad_(True)))
    with pytest.raises(NotImplementedError, match="descriptors"):
        coarse = data["descriptors3d_coarse_db"].clone().requires_grad_(True)
        train_kpt.check(m, dict(data, descriptors3d_coarse_db=coarse))
    plain = {k: v for k, v in _data().items() if k != "descriptors3d_coarse_db"}
    with pytest.raises(NotImplementedError, match="descriptors"):         # the selected tensor is checked
        train_kpt.check(m, dict(plain, descriptors3d_db=plain["descriptors3d_db"].requires_grad_(True)))
    train_kpt.check(m, dict(_data(), descriptors3d_db=torch.zeros(1, 256, 4, requires_grad=True)))
    for enc, dim in (([32, 64, 64], 256), ([32, 64, 128], 128), ([64, 128], 256)):
        cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
        cfg["keypoints_encoding"]["keypoints_encoder"] = enc
        cfg["keypoints_encoding"]["descriptor_dim"] = dim
        if dim != 256:
            cfg["loftr_coarse"]["d_model"] = dim
        try:
            other = _model(cfg)
        except (NotImplementedError, ValueError):
            continue                                               # refused by the constructor already
        with pytest.raises(NotImplementedError, match="channels"):
            train_kpt.check(other, data)
    m.precision = "fp16"
    with pytest.raises(ValueError, match="fp16x3"):
        train_kpt.check(m, data)


def test_parameter_order_covers_the_encoder():
    enc = _model().kpt_3d_pos_encoding
    got = train_kpt.params(enc)
    assert [tuple(p.shape) for p in got] == [(32, 3), (32,), (64, 32), (64,), (128, 64), (128,), (256, 128), (256,)]
    assert {id(p) for p in got} == {id(p) for p in enc.parameters()}
    assert tuple(n for n, _ in enc.named_parameters()) == mtk.PARAMS


def _encoder64(sd):
    m = _model()
    m.load_state_dict(sd, strict=True)
    return m.kpt_3d_pos_encoding.double()


def test_fixture_pinned_to_train_path_keypoint_encoding_fp64():
    z = np.load(GOLDEN)
    enc = _encoder64(workload.synthetic_state_dict(0))
    case = mtk.make_case()
    out = train_path.keypoint_encoding(enc, train_path.normalize_3d_keypoints(case["kpts"]), case["desc"])
    params = [dict(enc.named_parameters())[n] for n in mtk.PARAMS]
    grads = torch.autograd.grad(mtk.objective(out, case), params)
    named = {"out": out.detach()}
    named.update({f"d_{n}": g for n, g in zip(mtk.PARAMS, grads)})
    for key, t in named.items():
        amax = float(z[key + "_absmax"])
        got = t.flatten()[torch.from_numpy(z[key + "_idx"])].numpy()
        assert np.abs(got - z[key]).max() <= 1e-10 * max(amax, 1.0), key
        assert abs(float(t.abs().max()) - amax) <= 1e-10 * max(amax, 1.0), key


def _oracle_case(name):
    g = torch.Generator().manual_seed(5)
    f64 = torch.float64
    B, N = (1, 1) if name == "n1" else (2, 37)
    params = [p.detach().clone() for p in train_kpt.params(_encoder64(workload.synthetic_state_dict(0)))]
    x0 = torch.randn(B, N, 3, generator=g, dtype=f64)
    if name == "const_row":           # a1 = b1 constant on every 7th point: var = 0, y = 0
        x0[:, ::7] = 0
        params[1] = torch.full_like(params[1], 0.25)
    if name == "zero_preact":         # point 0: a1 = b1 = (0, 0, ±1 .. ±15), mean 0: y is exactly 0 twice
        x0[0, 0] = 0
        params[1] = torch.tensor([0.0, 0.0] + [s * k for k in range(1, 16) for s in (1, -1)], dtype=f64)
    desc = torch.randn(B, 256, N, generator=g, dtype=f64)
    up = torch.randn(B, 256, N, generator=g, dtype=f64)
    return params, x0, desc, up


@pytest.mark.parametrize("name", ["random", "const_row", "zero_preact", "n1"])
def test_oracle_backward_against_autograd(name):
    params, x0, desc, up = _oracle_case(name)
    enc = _encoder64(workload.synthetic_state_dict(0))
    with torch.no_grad():
        for p, v in zip(train_kpt.params(enc), params):
            p.copy_(v)
    ref = train_path.keypoint_encoding(enc, x0, desc)
    ref_grads = torch.autograd.grad(ref, train_kpt.params(enc), up)
    out, (cache, _) = kpt_enc.forward(params, x0, desc)
    torch.testing.assert_close(out, ref.detach(), rtol=0, atol=1e-10)
    if name == "const_row":
        assert torch.equal(cache[0][1][:, ::7], torch.zeros_like(cache[0][1][:, ::7]))
    if name == "zero_preact":
        assert int((cache[0][1][0, 0] == 0).sum()) == 2
    for i, (got, want) in enumerate(zip(kpt_enc.backward(params, x0, up), ref_grads)):
        torch.testing.assert_close(got, want, rtol=0, atol=1e-10, msg=lambda m: f"param {i}: {m}")
