"""CPU checks of the coarse transformer of training on the device: the coarse_transformer_train_mode
switch and its errors, the fp64 restatement of the manual linear-attention backward (oracle/coarse_tf.py,
what the opp_coarse_tf_* kernels compute) against autograd through train_path._linear_attention, and
the reference fixture against an fp64 autograd run of train_path.transformer (which pins the oracle
the GPU tests use to the reference)."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import coarse_tf
from oracle import make_train_coarse_tf_golden as mct
from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, train_coarse_tf, train_path

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_coarse_tf.npz")


def _model(attention="linear"):
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    cfg["loftr_coarse"]["attention"] = attention
    return OnePosePlus_model(cfg)


def test_default_and_environment_preset(monkeypatch):
    monkeypatch.delenv("OPP_B200_COARSE_TF_TRAIN", raising=False)
    assert _model().coarse_transformer_train_mode == "autograd"
    monkeypatch.setenv("OPP_B200_COARSE_TF_TRAIN", "kernels")
    assert _model().coarse_transformer_train_mode == "kernels"


def test_cpu_eval_and_default_do_not_use_the_kernels():
    m = _model().train()
    data = {"query_image": torch.zeros(1, 1, 8, 8)}
    assert not train_coarse_tf.use_kernels(m, data)                 # default
    m.coarse_transformer_train_mode = "kernels"
    assert not train_coarse_tf.use_kernels(m, data)                 # CPU tensors
    m.eval()
    assert not train_coarse_tf.use_kernels(m, data)
    m.coarse_transformer_train_mode = "fast"
    with pytest.raises(ValueError, match="coarse_transformer_train_mode"):
        train_coarse_tf.use_kernels(m, data)


def test_errors():
    train_coarse_tf.check(_model(), {})
    train_coarse_tf.check(_model(), {"query_image_mask": workload.pad_mask(2, 6, 8)})
    train_coarse_tf.check(_model(), {"query_image_mask": workload.pad_mask(2, 6, 8).float()})
    with pytest.raises(NotImplementedError, match="full"):
        train_coarse_tf.check(_model("full"), {})
    m = _model()
    m.loftr_coarse.d_model = 128
    with pytest.raises(NotImplementedError, match="d_model 256"):
        train_coarse_tf.check(m, {})
    m = _model()
    m.loftr_coarse.nhead = 4
    with pytest.raises(NotImplementedError, match="8 heads"):
        train_coarse_tf.check(m, {})
    m = _model()
    m.loftr_coarse.layer_names[3] = "global"
    with pytest.raises(NotImplementedError, match="global"):
        train_coarse_tf.check(m, {})
    mask = torch.ones(2, 6, 8)
    mask[1, :, 5:] = 0.5
    with pytest.raises(ValueError, match="0/1"):
        train_coarse_tf.check(_model(), {"query_image_mask": mask})


def _masks(B, n, kind, g):
    if kind == "none":
        return None
    m = torch.ones(B, n, dtype=torch.float64)
    if kind == "partial":
        m[:, n - n // 3:] = 0
        m[0, :: 5] = 0
    if kind == "empty_element":                                       # ksum = 0, Z = 1 / eps
        m[B - 1] = 0
    return m


@pytest.mark.parametrize("q_kind,kv_kind", [("partial", "partial"), ("none", "partial"), ("partial", "none"),
                                            ("empty_element", "empty_element"), ("none", "empty_element"),
                                            ("none", "none")])
@pytest.mark.parametrize("L,S", [(40, 40), (23, 57)])               # self (L = S) and cross shapes
def test_manual_backward_against_autograd(q_kind, kv_kind, L, S):
    g = torch.Generator().manual_seed(L * 100 + S)
    B, H, Dh = 3, 8, 32
    q = torch.randn(B, L, H, Dh, generator=g, dtype=torch.float64).requires_grad_(True)
    k = torch.randn(B, S, H, Dh, generator=g, dtype=torch.float64).requires_grad_(True)
    v = torch.randn(B, S, H, Dh, generator=g, dtype=torch.float64).requires_grad_(True)
    dout = torch.randn(B, L, H, Dh, generator=g, dtype=torch.float64)
    qm, km = _masks(B, L, q_kind, g), _masks(B, S, kv_kind, g)
    out = train_path._linear_attention(q, k, v, qm, km)
    ref = torch.autograd.grad(out, [q, k, v], dout)
    out = out.detach()
    got_out = coarse_tf.forward(q.detach(), k.detach(), v.detach(), qm, km)
    assert (got_out - out).abs().max() <= 1e-10 * max(1.0, float(out.abs().max()))
    got = coarse_tf.backward(q.detach(), k.detach(), v.detach(), dout, qm, km)
    for name, a, b in zip("qkv", got, ref):
        assert (a - b).abs().max() <= 1e-10 * max(1.0, float(b.abs().max())), name
    if kv_kind == "empty_element":
        KV, ksum = coarse_tf.state(k.detach(), v.detach(), km)
        assert float(ksum[B - 1].abs().max()) == 0.0 and float(KV[B - 1].abs().max()) == 0.0


@pytest.mark.parametrize("case_name", mct.CASES)
def test_fixture_against_train_path_fp64(case_name):
    z = np.load(GOLDEN)
    case = mct.make_case(masked=case_name == "masked")
    if case["mask"] is not None:
        assert not bool(case["mask"][1].all()) and bool(case["mask"][0].all())
    got = mct.flat_results(mct.train_path_coarse(mct.coarse_module(workload.synthetic_state_dict(0)), case))
    assert len(got) == 64
    for name, t in zip(mct.tensor_names(), got):
        key = f"{case_name}_{name}"
        amax = float(z[key + "_absmax"])
        assert amax > 0, name
        assert abs(float(t.abs().max()) - amax) <= 1e-10 * amax, name
        assert np.abs(t.flatten().numpy()[z[key + "_idx"]] - z[key]).max() <= 1e-10 * amax, name
