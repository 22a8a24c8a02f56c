"""CPU checks of the fine level of training on the device: the fine_train_mode switch and its
errors, a numpy restatement of the gather-backward index against F.fold, and the reference fixture
against an fp64 autograd run of train_path's fine functions (which pins the oracle the GPU tests use
to the reference)."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import make_train_fine_golden as mtf
from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, train_fine

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_fine.npz")


def _model(precision=None, off=None):
    cfg = copy.deepcopy(oracle.DEFAULT_CONFIG)
    if off is not None:
        cfg[off]["enable"] = False
    return OnePosePlus_model(cfg, precision=precision)


def test_default_and_environment_preset(monkeypatch):
    monkeypatch.delenv("OPP_B200_FINE_TRAIN", raising=False)
    assert _model().fine_train_mode == "autograd"
    monkeypatch.setenv("OPP_B200_FINE_TRAIN", "kernels")
    assert _model().fine_train_mode == "kernels"


def test_cpu_eval_and_default_do_not_use_the_kernels():
    m = _model().train()
    data = {"query_image": torch.zeros(1, 1, 8, 8), "descriptors3d_db": torch.zeros(1, 128, 4)}
    assert not train_fine.use_kernels(m, data)                       # default
    m.fine_train_mode = "kernels"
    assert not train_fine.use_kernels(m, data)                       # CPU tensors
    m.eval()
    assert not train_fine.use_kernels(m, data)
    m.fine_train_mode = "fast"
    with pytest.raises(ValueError, match="fine_train_mode"):
        train_fine.use_kernels(m, data)


def test_errors():
    data = {"descriptors3d_db": torch.zeros(1, 128, 4)}
    train_fine.check(_model(), data)
    with pytest.raises(ValueError, match="fp16x3"):
        train_fine.check(_model("fp16"), data)
    with pytest.raises(NotImplementedError, match="enable"):
        train_fine.check(_model(off="loftr_fine"), data)
    with pytest.raises(NotImplementedError, match="enable"):
        train_fine.check(_model(off="fine_matching"), data)
    m = _model()
    m.fine_preprocess.W = 7
    with pytest.raises(NotImplementedError, match="window size"):
        train_fine.check(m, data)
    with pytest.raises(NotImplementedError, match="descriptors3d_db"):
        train_fine.check(_model(), {"descriptors3d_db": torch.zeros(1, 128, 4, requires_grad=True)})


def gather_backward_numpy(dx, b_ids, j_ids, B, hc, wc, stride, hf, wf):
    """d feat as the kernel forms it: per pixel, the covering cells in raster order, each cell's matches
    (bucket of (b, j), ascending match index)."""
    M = len(b_ids)
    buckets = {}
    for m in range(M):
        buckets.setdefault((int(b_ids[m]), int(j_ids[m])), []).append(m)
    out = np.zeros((B, dx.shape[2], hf, wf))
    worst = 0
    for b in range(B):
        for y in range(hf):
            for x in range(wf):
                cells = [(cy, cx) for cy in range(hc) for cx in range(wc)
                         if abs(y - cy * stride) <= 2 and abs(x - cx * stride) <= 2]
                worst = max(worst, len(cells))
                for cy, cx in cells:
                    t = (y - cy * stride + 2) * 5 + (x - cx * stride + 2)
                    for m in buckets.get((b, cy * wc + cx), []):
                        out[b, :, y, x] += dx[m, t]
    return out, worst


@pytest.mark.parametrize("stride", [4, 2])
def test_gather_backward_index_against_fold(stride):
    case = mtf.make_case(seed=2, hc=4, wc=5, stride=stride, M=60)
    B, _, hf, wf = case["feat_f"].shape
    hc, wc = case["q_hw_c"]
    g = torch.Generator().manual_seed(5)
    dx = torch.randn(60, 25, 128, generator=g, dtype=torch.float64)
    b, j = case["b_ids"], case["j_ids"]
    dunf = torch.zeros(B, hc * wc, 25, 128, dtype=torch.float64)
    dunf.index_put_((b, j), dx, accumulate=True)
    ref = F.fold(dunf.permute(0, 3, 2, 1).reshape(B, 128 * 25, hc * wc), (hf, wf), kernel_size=5, stride=stride,
                 padding=2)
    got, worst = gather_backward_numpy(dx.numpy(), b.numpy(), j.numpy(), B, hc, wc, stride, hf, wf)
    assert np.abs(got - ref.numpy()).max() <= 1e-12
    assert worst == (4 if stride == 4 else 9)                       # 2 x 2 cells at the training stride


@pytest.mark.parametrize("stride", [2, 4, 8])
def test_fold_reference_against_fine_preprocess_autograd(stride):
    """The gather-backward reference of test_train_fine_kernels_gpu (index_put_ + F.fold) is the
    fp64 autograd backward of train_path.fine_preprocess's window rows."""
    from tests.test_train_fine_kernels_gpu import fold_reference
    from onepose_plus_plus_b200 import train_path
    case = mtf.make_case(seed=7, B=3, hc=5, wc=7, stride=stride, n3d=4, M=60)
    B, _, hf, wf = case["feat_f"].shape
    feat = case["feat_f"].clone().requires_grad_(True)
    _, f2d = train_path.fine_preprocess(5, 128, mtf.fine_data(case), case["desc3d"], feat)
    dx = torch.randn(f2d.shape, generator=torch.Generator().manual_seed(stride), dtype=torch.float64)
    (ref,) = torch.autograd.grad(f2d, feat, dx)
    got = fold_reference(dx, case["b_ids"], case["j_ids"], B, 5, 7, stride, hf, wf)
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)


def test_attention_reference_against_train_path_transformer(monkeypatch):
    """The attention reference of test_train_fine_kernels_gpu (train_path._linear_attention on the
    26-row [q | k | v] layout, self and cross) gives the messages train_path.transformer computes
    in the two fine layers, from the q, k, v those calls receive."""
    from tests.test_train_fine_kernels_gpu import attention_reference
    from onepose_plus_plus_b200 import train_path
    calls = []
    orig = train_path._linear_attention

    def record(q, k, v, q_mask=None, kv_mask=None, eps=1e-6):
        out = orig(q, k, v, q_mask, kv_mask, eps)
        calls.append([t.reshape(t.shape[0], t.shape[1], 128) for t in (q, k, v, out)])
        return out

    monkeypatch.setattr(train_path, "_linear_attention", record)
    g = torch.Generator().manual_seed(6)
    f3d = torch.randn(7, 128, 1, generator=g, dtype=torch.float64)
    f2d = torch.randn(7, 25, 128, generator=g, dtype=torch.float64)
    with torch.no_grad():
        train_path.transformer(mtf.fine_module(workload.synthetic_state_dict(0)), f3d, f2d)
    (qa, ka, va, oa), (qb, kb, vb, ob), (qc, kc, vc, oc), (qd, kd, vd, od) = calls   # self 2D, 3D; cross 2D, 3D
    self_qkv = torch.cat([torch.cat([qa, ka, va], 2), torch.cat([qb, kb, vb], 2)], 1)
    cross_qkv = torch.cat([torch.cat([qc, kd, vd], 2), torch.cat([qd, kc, vc], 2)], 1)
    for qkv, cross, outs in ((self_qkv, 0, (oa, ob)), (cross_qkv, 1, (oc, od))):
        assert torch.allclose(attention_reference(qkv, cross), torch.cat(outs, 1), rtol=1e-12, atol=1e-14)


def test_fixture_against_train_path_fp64():
    z = np.load(GOLDEN)
    case = mtf.make_case()
    expec, loss, dfeat, dparams = mtf.train_path_fine(mtf.fine_module(workload.synthetic_state_dict(0)), case)
    assert np.abs(expec.numpy() - z["expec_f"]).max() <= 1e-12
    assert abs(loss.item() - float(z["loss"])) <= 1e-12 * abs(float(z["loss"]))
    for name, t in zip(["feat_f"] + list(mtf.FINE_PARAMS), [dfeat] + dparams):
        key = "d_" + name
        got = t.flatten().numpy()[z[key + "_idx"]]
        assert float(z[key + "_absmax"]) > 0, name
        assert np.abs(got - z[key]).max() <= 1e-10 * float(z[key + "_absmax"]), name
