"""Coarse transformer of training on the device (model.coarse_transformer_train_mode "kernels"):
train_coarse_tf.CoarseTransformerStage against the reference fixture and fp64 autograd of
train_path.transformer on the small case and at the training shape, determinism, the memory of the
stage, ctx.needs_input_grad, and one model.train() step against the autograd coarse transformer."""
import os

import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_coarse_tf_golden as mct
from oracle import make_train_fine_golden as mtf
from oracle import train_gt as otg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, losses, train_coarse_tf, train_fine, train_gt
from tests.test_train_gt_gpu import planted_gt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_coarse_tf.npz")
pytestmark = pytest.mark.gpu


def kernels_coarse(tf32, case, need=(True, True, True)):
    """CoarseTransformerStage on the device: (d3, d2, d desc3d, d desc2d, [d param]); need = which of
    (desc3d, desc2d, the parameters) take a gradient."""
    desc3d = case["desc3d"].to("cuda", torch.float32).requires_grad_(need[0])
    desc2d = case["desc2d"].to("cuda", torch.float32).requires_grad_(need[1])
    mask = None if case["mask"] is None else case["mask"].cuda()
    params = [p for layer in tf32.layers for p in train_fine.layer_params(layer)]
    d3, d2 = train_coarse_tf.coarse_transformer(tf32, desc3d, desc2d, mask)
    wrt = ([desc3d] if need[0] else []) + ([desc2d] if need[1] else []) + (params if need[2] else [])
    grads = list(torch.autograd.grad(mct.objective(d3, d2, case), wrt))
    gx3 = grads.pop(0) if need[0] else None
    gx2 = grads.pop(0) if need[1] else None
    return d3.detach(), d2.detach(), gx3, gx2, grads


def _runs(case):
    sd = workload.synthetic_state_dict(0)
    r64 = mct.train_path_coarse(mct.coarse_module(sd, torch.float64, "cuda"), case, torch.float64, "cuda")
    r32 = mct.train_path_coarse(mct.coarse_module(sd, torch.float32, "cuda"), case, torch.float32, "cuda")
    rk = kernels_coarse(mct.coarse_module(sd, torch.float32, "cuda"), case)
    return r64, r32, rk


def _assert_fp64_distance(r64, r32, rk, report=None, check=True, factor=1.0):
    """Outputs within the fp32 path's own distance from fp64 (times factor) + 1e-5 absmax; gradients
    within its distance (times factor) + 2e-4 absmax + 1e-6."""
    for name, a64, a32, ak in zip(mct.tensor_names(), *(mct.flat_results(r) for r in (r64, r32, rk))):
        amax = float(a64.abs().max())
        ek, et = float((ak.double() - a64).abs().max()), float((a32.double() - a64).abs().max())
        if report is not None:
            report.append(f"{name}: kernels {ek / max(amax, 1e-30):.2e}, torch fp32 {et / max(amax, 1e-30):.2e}")
        tol = 1e-5 * amax if name in ("d3", "d2") else 2e-4 * amax + 1e-6
        assert not check or ek <= factor * et + tol, (name, ek, et, amax)


@pytest.mark.parametrize("case_name", mct.CASES)
def test_small_case_against_the_reference_fixture_and_fp64(case_name):
    case = mct.make_case(masked=case_name == "masked")
    r64, r32, rk = _runs(case)
    report = []
    _assert_fp64_distance(r64, r32, rk, report, check=False)
    print("\n".join(report))
    # Without the mask, one mlp pre-activation lies so close to 0 that fp32 and fp64 take different
    # sides of the ReLU: the two fp32 paths are equally far from fp64 (5.0e-3 of absmax in d desc3d
    # on an H100), so the fixture check allows the fp32 autograd path's own distance, as the fp64 one does.
    z = np.load(GOLDEN)
    for name, t, t32 in zip(mct.tensor_names(), mct.flat_results(rk), mct.flat_results(r32)):
        key = f"{case_name}_{name}"
        amax = float(z[key + "_absmax"])
        idx = z[key + "_idx"]
        got = t.flatten().cpu().double().numpy()[idx]
        e32 = np.abs(t32.flatten().cpu().double().numpy()[idx] - z[key]).max()
        tol = 1e-5 * amax if name in ("d3", "d2") else 2e-4 * amax + 1e-6
        assert np.abs(got - z[key]).max() <= e32 + tol, name
    _assert_fp64_distance(r64, r32, rk)


def training_case(masked):
    """The reference training shape: batch 4, 512 x 512 images (a 64 x 64 coarse grid), 7000 points."""
    case = mct.make_case(seed=1, B=4, hc=64, wc=64, N=7000, masked=False)
    if masked:
        m = workload.pad_mask(4, 64, 64).reshape(4, 64 * 64)
        assert not bool(m.all())
        case["mask"] = m
    return case


@pytest.mark.parametrize("masked", [False, True])
def test_training_shape_accuracy(masked):
    """At 44,384 rows per layer many mlp pre-activations sit at the ReLU's kink, and which of them flip
    sides against fp64 depends on the summation order: both fp32 paths are 1e-3 to 3e-2 of absmax from
    fp64 in the gradients, and the kernels' distance ranges from 0.3 to 1.8 times the autograd path's
    (H100, both masks).  The gradients are therefore held to twice the autograd path's distance + 2e-4
    absmax + 1e-6; the outputs to its distance + 1e-5 absmax as well (they are within 1e-6 of absmax)."""
    case = training_case(masked)
    r64, r32, rk = _runs(case)
    report = []
    _assert_fp64_distance(r64, r32, rk, report, check=False)
    print("\n".join(report))
    _assert_fp64_distance(r64, r32, rk, factor=2.0)
    for a64, a32, ak in zip(r64[:2], r32[:2], rk[:2]):
        amax = float(a64.abs().max())
        assert float((ak.double() - a64).abs().max()) <= float((a32.double() - a64).abs().max()) + 1e-5 * amax


def _stage(tf, d3, d2, mask, w3, w2):
    params = [p for layer in tf.layers for p in train_fine.layer_params(layer)]
    o3, o2 = train_coarse_tf.coarse_transformer(tf, d3, d2, mask)
    return torch.autograd.grad((o3 * w3).sum() + (o2 * w2).sum(), [d3, d2] + params)


def _autograd(tf, d3, d2, mask, w3, w2):
    from onepose_plus_plus_b200 import train_path
    params = [p for layer in tf.layers for p in train_fine.layer_params(layer)]
    o3, o2 = train_path.transformer(tf, d3, d2, mask)
    return torch.autograd.grad((o3 * w3).sum() + (o2 * w2).sum(), [d3, d2] + params)


def test_training_shape_determinism_and_memory():
    case = training_case(True)
    tf = mct.coarse_module(workload.synthetic_state_dict(0), torch.float32, "cuda")
    d3 = case["desc3d"].cuda().float().requires_grad_(True)
    d2 = case["desc2d"].cuda().float().requires_grad_(True)
    mask, w3, w2 = case["mask"].cuda(), case["w3"].cuda().float(), case["w2"].cuda().float()
    a = _stage(tf, d3, d2, mask, w3, w2)
    b = _stage(tf, d3, d2, mask, w3, w2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    o = [train_coarse_tf.coarse_transformer(tf, d3, d2, mask) for _ in range(2)]
    assert torch.equal(o[0][0], o[1][0]) and torch.equal(o[0][1], o[1][1])
    del a, b, o
    peaks = {}
    for name, fn in (("kernels", _stage), ("autograd", _autograd)):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(tf, d3, d2, mask, w3, w2)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    print(f"coarse transformer peak above its inputs: kernels {peaks['kernels'] / 2**20:.1f} MiB, "
          f"autograd {peaks['autograd'] / 2**20:.1f} MiB")
    assert peaks["kernels"] <= 1536 * 2 ** 20
    assert peaks["kernels"] < 0.4 * peaks["autograd"]


def test_needs_input_grad():
    """Frozen coarse parameters (no weight gradient runs) and 3D tokens without a gradient: the
    gradients that are formed equal the full call's."""
    case = mct.make_case(seed=4, masked=True)
    tf = mct.coarse_module(workload.synthetic_state_dict(0), torch.float32, "cuda")
    full = kernels_coarse(tf, case)
    frozen = kernels_coarse(tf, case, need=(True, True, False))
    assert torch.equal(frozen[2], full[2]) and torch.equal(frozen[3], full[3]) and frozen[4] == []
    no3d = kernels_coarse(tf, case, need=(False, True, True))
    assert torch.equal(no3d[3], full[3])
    assert all(torch.equal(x, y) for x, y in zip(no3d[4], full[4]))
    params_only = kernels_coarse(tf, case, need=(False, False, True))
    assert all(torch.equal(x, y) for x, y in zip(params_only[4], full[4]))


def test_training_with_a_bank_set_still_raises():
    sd = workload.synthetic_state_dict(0)
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    m.coarse_transformer_train_mode = "kernels"
    g = torch.Generator().manual_seed(0)
    m.set_banks([(torch.randn(1, 20, 3, generator=g), torch.randn(1, 128, 20, generator=g),
                  torch.randn(1, 256, 20, generator=g))])
    with pytest.raises(NotImplementedError, match="bank set"):
        m.train()


STEP_PARAMS = ("backbone.conv1.weight", "kpt_3d_pos_encoding.encoder.0.weight", "loftr_coarse.layers.0.q_proj.weight",
               "loftr_coarse.layers.5.mlp.2.weight", "loftr_coarse.layers.3.norm1.bias")


def _step(sd, masked, mode, gt, dtype=torch.float32):
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().to(dtype).train()
    m.conf_matrix_mode = "lazy"
    m.fine_train_mode = "kernels" if dtype == torch.float32 else "autograd"
    m.coarse_transformer_train_mode = mode
    data = mrg.train_batch(sd, masked)
    del data["conf_matrix_gt"]
    data = {k: (v.to("cuda", dtype) if torch.is_tensor(v) and v.is_floating_point() else
                v.to("cuda") if torch.is_tensor(v) else v) for k, v in data.items()}
    data["gt_sparse"] = gt.to("cuda")
    torch.manual_seed(11)
    with mtf.default_dtype(dtype):                 # train_path.fine_matching's grid
        m(data)
    train_gt.fine_supervision(data, otg.config())
    losses.Loss(cl.LOSS_CONFIG).train()(data)
    m.zero_grad()
    data["loss"].backward()
    return m, data


@pytest.mark.parametrize("masked", [False, True])
def test_training_step_kernels_against_autograd(masked):
    """One model.train() step on the planted train batch with lazy coarse matching, the fine kernels and
    gt_sparse; only the coarse-transformer mode differs.  The matches are identical, the loss within 1e-5
    relative, and five gradients across the model within the autograd fp32 run's distance from an fp64
    run + 2e-4 absmax + 1e-6, plus the autograd path's own run-to-run spread (a second autograd run:
    cuDNN's convolution backward is not bit-reproducible, and conv1's gradient is 15 % of absmax from
    fp64 in both fp32 runs)."""
    sd = workload.synthetic_state_dict(0)
    gt = planted_gt(mrg.train_batch(sd, masked)["conf_matrix_gt"])
    ma, da = _step(sd, masked, "autograd", gt)
    ma2, _ = _step(sd, masked, "autograd", gt)
    mk, dk = _step(sd, masked, "kernels", gt)
    m64, d64 = _step(sd, masked, "autograd", gt, torch.float64)
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask"):
        assert torch.equal(da[k], dk[k]), k
        assert torch.equal(da[k], d64[k]), k                           # the fp64 run is comparable
    assert abs(da["loss"].item() - dk["loss"].item()) <= 1e-5 * abs(da["loss"].item())
    pa, pa2 = dict(ma.named_parameters()), dict(ma2.named_parameters())
    pk, p64 = dict(mk.named_parameters()), dict(m64.named_parameters())
    for n in STEP_PARAMS:
        g64 = p64[n].grad
        amax = float(g64.abs().max())
        ek = float((pk[n].grad.double() - g64).abs().max())
        ea = float((pa[n].grad.double() - g64).abs().max())
        spread = float((pa[n].grad - pa2[n].grad).abs().max())
        print(f"{n}: kernels {ek / amax:.2e}, autograd fp32 {ea / amax:.2e}, its spread {spread / amax:.2e} of absmax")
        assert ek <= ea + spread + 2e-4 * amax + 1e-6, (n, ek, ea, spread, amax)
