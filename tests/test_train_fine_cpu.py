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
