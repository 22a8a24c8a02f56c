"""Keypoint encoder of training on the device (model.kpt_encoder_train_mode "kernels"):
train_kpt.KeypointEncoderStage against the reference fixture and fp64 autograd of
train_path.keypoint_encoding on the small case and at the training shape, determinism, the memory of
the stage, ctx.needs_input_grad, and whole model.train() steps with every device stage on: the same
matches and loss as with the encoder on autograd, every parameter gradient within its stage's rule,
and two steps from the same state bit-equal."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_fine_golden as mtf
from oracle import make_train_kpt_golden as mtk
from oracle import oracle
from oracle import train_gt as otg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, losses, ops, train_gt, train_kpt, train_path
from tests.test_train_gt_gpu import planted_gt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_kpt.npz")
pytestmark = pytest.mark.gpu

# workspace of the stage beyond its output rows: one slice of weight-gradient partials, the flat
# gradient, two weight packs and the statistics, plus allocator rounding
WORKSPACE_MIB = train_kpt.WGRAD_SLICE_GROUPS * 43584 * 4 / 2 ** 20 + 2.0


def _encoder(dtype):
    m = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    m.load_state_dict(workload.synthetic_state_dict(0), strict=True)
    return m.kpt_3d_pos_encoding.to(device="cuda", dtype=dtype).train()


def _autograd(enc, kpts, desc):
    return train_path.keypoint_encoding(enc, train_path.normalize_3d_keypoints(kpts), desc)


def _run(enc, fwd, case, dtype):
    """(output [B, 256, N], the eight gradients) of fwd under the fixture's objective."""
    kpts, desc = case["kpts"].to("cuda", dtype), case["desc"].to("cuda", dtype)
    out = fwd(enc, kpts, desc)
    params = train_kpt.params(enc)
    grads = torch.autograd.grad(mtk.objective(out, {"g": case["g"].cuda()}), params)
    return out.detach(), list(grads)


def _check(rk, r32, r64, label):
    """Output within 1e-6 absmax of fp64; each gradient within the fp32 autograd path's distance from
    fp64 + 2e-4 absmax + 1e-6."""
    amax = float(r64[0].abs().max())
    eo = float((rk[0].double() - r64[0]).abs().max())
    assert eo <= 1e-6 * amax, (label, eo, amax)
    for name, gk, g32, g64 in zip(mtk.PARAMS, rk[1], r32[1], r64[1]):
        amax = float(g64.abs().max())
        ek, et = float((gk.double() - g64).abs().max()), float((g32.double() - g64).abs().max())
        print(f"{label} {name}: kernels {ek / amax:.2e}, autograd fp32 {et / amax:.2e} of absmax")
        assert ek <= et + 2e-4 * amax + 1e-6, (label, name, ek, et, amax)


def test_small_case_against_the_reference_fixture_and_fp64():
    z = np.load(GOLDEN)
    case = mtk.make_case()
    rk = _run(_encoder(torch.float32), train_kpt.keypoint_encoding, case, torch.float32)
    r32 = _run(_encoder(torch.float32), _autograd, case, torch.float32)
    r64 = _run(_encoder(torch.float64), _autograd, case, torch.float64)
    _check(rk, r32, r64, "B=2 N=301")
    for key, t, t32 in zip(["out"] + [f"d_{n}" for n in mtk.PARAMS], [rk[0]] + rk[1], [r32[0]] + r32[1]):
        amax = float(z[key + "_absmax"])
        idx = torch.from_numpy(z[key + "_idx"])
        got = t.flatten().cpu()[idx].double().numpy()
        if key == "out":
            assert np.abs(got - z[key]).max() <= 1e-6 * amax, key
        else:
            d32 = np.abs(t32.flatten().cpu()[idx].double().numpy() - z[key]).max()
            assert np.abs(got - z[key]).max() <= d32 + 2e-4 * amax + 1e-6, key


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def test_training_shape_accuracy_determinism_and_memory():
    """B = 4, N = 7000: accuracy as on the small case, two calls bit-equal, and the stage's peak above its
    inputs below autograd's and within the output rows + WORKSPACE_MIB."""
    B, N = 4, 7000
    case = {k: v.cuda() for k, v in mtk.make_case(seed=1, B=B, N=N).items()}
    enc = _encoder(torch.float32)
    kpts, desc = case["kpts"].float(), case["desc"].float()
    up = case["g"].float().transpose(1, 2).contiguous()        # the rows' gradient, as the transformers give it
    params = train_kpt.params(enc)

    def stage(fwd):
        def go():
            out = fwd(enc, kpts, desc)
            return out.detach(), list(torch.autograd.grad(out, params, up.transpose(1, 2)))
        return go

    rk, peak_k = _peak(stage(train_kpt.keypoint_encoding))
    rk2 = stage(train_kpt.keypoint_encoding)()
    assert torch.equal(rk[0], rk2[0])
    for name, a, b in zip(mtk.PARAMS, rk[1], rk2[1]):
        assert torch.equal(a, b), name
    r32, peak_a = _peak(stage(_autograd))
    r64 = _run(_encoder(torch.float64), _autograd, case, torch.float64)
    _check(rk, r32, r64, "B=4 N=7000")
    rows_mib = B * N * 256 * 4 / 2 ** 20
    grads_mib = 43584 * 4 / 2 ** 20
    print(f"peak above inputs: kernels {peak_k:.1f} MiB (rows {rows_mib:.1f} + workspace {WORKSPACE_MIB:.1f}), "
          f"autograd {peak_a:.1f} MiB")
    assert peak_k < peak_a, (peak_k, peak_a)
    assert peak_k <= rows_mib + grads_mib + WORKSPACE_MIB, (peak_k, rows_mib, WORKSPACE_MIB)


def test_frozen_encoder_runs_no_wgrad_and_partial_freeze_follows_needs_input_grad():
    case = mtk.make_case()
    kpts, desc = case["kpts"].float().cuda(), case["desc"].float().cuda()
    calls = []
    real = ops.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)

    enc = _encoder(torch.float32)
    ops.call = spy
    try:
        for p in enc.parameters():
            p.requires_grad_(False)
        out = train_kpt.keypoint_encoding(enc, kpts, desc)
        assert not out.requires_grad
        assert "opp_kpt_train_fwd" in calls and "opp_kpt_train_bwd" not in calls
        trainable = {"encoder.9.weight", "encoder.9.bias"}
        for n, p in enc.named_parameters():
            p.requires_grad_(n in trainable)
        desc_leaf = desc.clone().requires_grad_(False)
        out = train_kpt.keypoint_encoding(enc, kpts, desc_leaf)
        (out * case["g"].float().cuda()).sum().backward()
    finally:
        ops.call = real
    assert calls.count("opp_kpt_train_bwd") == 1
    for n, p in enc.named_parameters():
        assert (p.grad is not None) == (n in trainable), n
    r64 = _run(_encoder(torch.float64), _autograd, case, torch.float64)
    for n, g64 in zip(mtk.PARAMS, r64[1]):
        if n in trainable:
            p = dict(enc.named_parameters())[n]
            assert float((p.grad.double() - g64).abs().max()) <= 1e-5 * float(g64.abs().max()), n


# the rule of each stage's own test for a gradient of the whole step: (factor on the fp32 autograd
# path's distance from fp64, share of absmax); the backbone's and the coarse transformer's are their
# training-shape rules (DESIGN §7 f4)
RULES = (("backbone.", 5.0, 4e-3), ("loftr_coarse.", 2.0, 2e-4), ("", 1.0, 2e-4))


def _rule(name):
    return next((f, rel) for prefix, f, rel in RULES if name.startswith(prefix))


def _step(sd, gt, masked, kpt_mode, dtype=torch.float32):
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().to(dtype).train()
    m.conf_matrix_mode = "lazy"
    kernels = "kernels" if dtype == torch.float32 else "autograd"
    m.fine_train_mode = m.coarse_transformer_train_mode = m.backbone_train_mode = kernels
    m.kpt_encoder_train_mode = kpt_mode
    data = mrg.train_batch(sd, masked)
    del data["conf_matrix_gt"]
    data = {k: (v.to("cuda", dtype) if torch.is_tensor(v) and v.is_floating_point() else
                v.to("cuda") if torch.is_tensor(v) else v) for k, v in data.items()}
    data["gt_sparse"] = gt.to("cuda")
    torch.manual_seed(11)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with mtf.default_dtype(dtype):
            m(data)
            train_gt.fine_supervision(data, otg.config())
            losses.Loss(cl.LOSS_CONFIG).train()(data)
            m.zero_grad()
            data["loss"].backward()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    return m, data


@pytest.mark.parametrize("masked", [False, True])
def test_whole_training_step_on_the_kernels(masked):
    """model.train() on the planted train batch with lazy, gt_sparse and all four *_train_mode switches
    on "kernels", against the same step with the encoder on autograd and against fp64 autograd."""
    sd = workload.synthetic_state_dict(0)
    gt = planted_gt(mrg.train_batch(sd, masked)["conf_matrix_gt"])
    ma, da = _step(sd, gt, masked, "autograd")
    ma2, _ = _step(sd, gt, masked, "autograd")
    mk, dk = _step(sd, gt, masked, "kernels")
    mk2, dk2 = _step(sd, gt, masked, "kernels")
    m64, _ = _step(sd, gt, masked, "autograd", torch.float64)
    # 1. the same matches, the loss within 1e-5 relative
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask"):
        assert torch.equal(da[k], dk[k]), k
    assert abs(da["loss"].item() - dk["loss"].item()) <= 1e-5 * abs(da["loss"].item())
    # 2. every trainable parameter's gradient within its stage's rule
    pa, pa2, pk = dict(ma.named_parameters()), dict(ma2.named_parameters()), dict(mk.named_parameters())
    p64 = dict(m64.named_parameters())
    worst = []
    for n, p in pk.items():
        if not p.requires_grad:
            continue
        g64 = p64[n].grad
        if g64 is None:
            assert p.grad is None or not bool(p.grad.any()), n
            continue
        amax = float(g64.abs().max())
        ek = float((p.grad.double() - g64).abs().max())
        ea = float((pa[n].grad.double() - g64).abs().max())
        spread = float((pa[n].grad - pa2[n].grad).abs().max())
        factor, rel = _rule(n)
        if n.startswith("kpt_3d_pos_encoding."):
            print(f"{n}: kernels {ek / amax:.2e}, autograd fp32 {ea / amax:.2e}, its spread {spread / amax:.2e} "
                  f"of absmax")
        worst.append((ek / max(amax, 1e-30), n))
        assert ek <= factor * ea + spread + rel * amax + 1e-6, (n, ek, ea, spread, amax)
    worst.sort(reverse=True)
    print("largest kernel-step distances from fp64 (of absmax):", worst[:5])
    # 3. two steps from the same state and seed: bit-equal loss, gradients and BatchNorm buffers
    assert torch.equal(dk["loss"], dk2["loss"])
    pk2 = dict(mk2.named_parameters())
    differ = [n for n, p in pk.items() if p.requires_grad and not (
        (p.grad is None and pk2[n].grad is None) or torch.equal(p.grad, pk2[n].grad))]
    assert not differ, differ
    bk, bk2 = dict(mk.named_buffers()), dict(mk2.named_buffers())
    differ = [n for n, b in bk.items() if ("running" in n or "num_batches" in n) and not torch.equal(b, bk2[n])]
    assert not differ, differ
