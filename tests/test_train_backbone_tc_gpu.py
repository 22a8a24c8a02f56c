"""Backbone of training on the device with the convolutions on the tensor cores (model.backbone_train_mode
"tf32x3"): train_backbone.BackboneStage against the reference fixture and fp64 autograd on the small case
and at the training shape (each tensor's distance printed beside the "kernels" mode's), determinism, the
memory of the stage against "kernels", eval-mode BatchNorm, a partial freeze, feat_f without gradient,
and whole model.train() steps against the autograd backbone."""
import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_backbone_golden as mtb
from oracle import make_train_fine_golden as mtf
from oracle import train_gt as otg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, losses, ops, train_backbone, train_gt, train_path
from tests.test_train_backbone_gpu import GOLDEN, STEP_PARAMS, _flat, _names, _NoTF32, _run, _stage_peak
from tests.test_train_gt_gpu import planted_gt

pytestmark = pytest.mark.gpu


def tc(bb, img):
    return train_backbone.backbone(bb, img, "tf32x3")


def _assert_fp64_distance(sd, r64, r32, rt, rk, label, factor=2.0):
    """Each tensor of the tf32x3 run within factor x the fp32 autograd path's (cudnn TF32 off) distance
    from fp64 + 4e-3 absmax + 1e-6 (outputs and running statistics: + 2e-4 absmax), the rule of the
    "kernels" mode's tests; the "kernels" mode's distance is printed beside it."""
    rows = []
    for name, a64, a32, at, ak in zip(_names(sd), _flat(r64), _flat(r32), _flat(rt), _flat(rk)):
        amax = max(float(a64.abs().max()), 1e-30)
        et, e32 = float((at.double() - a64).abs().max()), float((a32.double() - a64).abs().max())
        ek = float((ak.double() - a64).abs().max())
        rows.append((et / amax, ek / amax, e32 / amax, name))
        rel = 4e-3 if name.startswith("d_") else 2e-4
        assert et <= factor * e32 + rel * amax + 1e-6, (label, name, et, e32, amax)
    print(f"{label}: distance from fp64 of absmax (tf32x3, kernels, torch fp32)")
    for et, ek, e32, name in rows:
        print(f"  {name:40s} {et:.2e} {ek:.2e} {e32:.2e}")


def test_small_case_against_the_reference_fixture_and_fp64():
    z = np.load(GOLDEN)
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    rt = _run(sd, case, tc)
    rk = _run(sd, case, train_backbone.backbone)
    r64 = _run(sd, case, train_path.backbone, torch.float64)
    with _NoTF32():
        r32 = _run(sd, case, train_path.backbone)
    _assert_fp64_distance(sd, r64, r32, rt, rk, "train")
    bb = mtb.backbone_module(sd)
    names = ["feat_c", "feat_f"] + [f"d_{n}" for n in mtb.param_names(bb)]
    for key, t, t32 in zip(names, [rt[0], rt[1]] + rt[2], [r32[0], r32[1]] + r32[2]):
        k = f"train_{key}"
        amax = float(z[k + "_absmax"])
        idx = torch.from_numpy(z[k + "_idx"])
        got = t.flatten().cpu()[idx].double().numpy()
        d32 = np.abs(t32.flatten().cpu()[idx].double().numpy() - z[k]).max()
        assert np.abs(got - z[k]).max() <= 2 * d32 + (4e-3 if key.startswith("d_") else 2e-4) * amax + 1e-6, key
    for n, b in rt[3].items():
        ref = z[f"train_buf_{n}"]
        assert np.abs(b.double().cpu().numpy() - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1.0), n


def test_training_shape_accuracy_determinism_and_memory():
    """B = 4, 512 x 512: outputs, the 56 parameter gradients and the running statistics under the rule of
    the "kernels" mode's test (five times the fp32 autograd distance + 4e-3 / 2e-4 absmax); two calls
    bit-equal; the stage's peak above its inputs within the "kernels" mode's + 64 MiB."""
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case(seed=1, B=4, H=512, W=512)
    case = {k: v.cuda() for k, v in case.items()}
    rt, peak_t = _stage_peak(lambda: _run(sd, case, tc))
    rt2 = _run(sd, case, tc)
    for name, a, b in zip(_names(sd), _flat(rt), _flat(rt2)):
        assert torch.equal(a, b), name
    del rt2
    rk, peak_k = _stage_peak(lambda: _run(sd, case, train_backbone.backbone))
    with _NoTF32():
        r32 = _run(sd, case, train_path.backbone)
    r64 = _run(sd, case, train_path.backbone, torch.float64)
    assert len(_names(sd)) == 2 + 56 + 34
    _assert_fp64_distance(sd, r64, r32, rt, rk, "B=4 512x512", factor=5.0)
    print(f"peak above inputs: tf32x3 {peak_t:.0f} MiB, kernels {peak_k:.0f} MiB")
    assert peak_t <= peak_k + 64, (peak_t, peak_k)


def test_eval_mode_batchnorm_frozen():
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    bb = mtb.backbone_module(sd, torch.float32, "cuda", train=False)
    for p in bb.parameters():
        p.requires_grad_(False)
    before = {n: b.clone() for n, b in bb.named_buffers()}
    img = case["img"].float().cuda()
    fc, ff = tc(bb, img)
    assert not fc.requires_grad and not ff.requires_grad
    with _NoTF32(), torch.no_grad():
        rc, rf = train_path.backbone(bb, img)
    for a, b in ((fc, rc), (ff, rf)):
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max())
    for n, b in bb.named_buffers():
        assert torch.equal(b, before[n]), n
    z = np.load(GOLDEN)
    for key, t in (("feat_c", fc), ("feat_f", ff)):
        k = f"eval_{key}"
        got = t.flatten().cpu()[torch.from_numpy(z[k + "_idx"])].double().numpy()
        assert np.abs(got - z[k]).max() <= 2e-4 * float(z[k + "_absmax"]), key


def test_partial_freeze_runs_no_wgrad_for_frozen_convolutions():
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    bb = mtb.backbone_module(sd, torch.float32, "cuda")
    trainable = {"layer3.1.conv2.weight", "layer3.1.bn2.weight", "layer1_outconv2.3.weight"}
    for n, p in bb.named_parameters():
        p.requires_grad_(n in trainable)
    img = case["img"].float().cuda()
    calls = []
    real = ops.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)

    ops.call = spy
    try:
        fc, ff = tc(bb, img)
        mtb.objective(fc, ff, {k: v.cuda() for k, v in case.items()}).backward()
    finally:
        ops.call = real
    assert calls.count("opp_backbone_train_conv_wgrad_tf32x3") == 2      # one slice each at this size
    convs = [c for c in calls if c.startswith("opp_backbone_train_conv")]
    assert convs and all(c.endswith("_tf32x3") for c in convs), set(convs)
    for n, p in bb.named_parameters():
        assert (p.grad is not None) == (n in trainable), n
    ref = mtb.backbone_module(sd, torch.float64, "cuda")
    r64 = mtb.run(ref, train_path.backbone, case, torch.float64, "cuda")
    names = mtb.param_names(ref)
    for n, p in bb.named_parameters():
        if n in trainable:
            g64 = r64[2][names.index(n)]
            assert float((p.grad.double() - g64).abs().max()) <= 5e-3 * float(g64.abs().max()), n


def test_feat_f_without_gradient_skips_the_fpn_backward():
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    bb = mtb.backbone_module(sd, torch.float32, "cuda")
    fc, _ = tc(bb, case["img"].float().cuda())
    (fc * case["g_c"].float().cuda()).sum().backward()
    grads = dict((n, p.grad) for n, p in bb.named_parameters())
    assert all(grads[n] is None for n in grads if n.startswith(("layer1_outconv", "layer2_outconv")))
    ref = mtb.backbone_module(sd, torch.float64, "cuda")
    c64, _ = train_path.backbone(ref, case["img"].double().cuda())
    (c64 * case["g_c"].cuda()).sum().backward()
    for n, p in ref.named_parameters():
        if p.grad is not None:
            assert float((grads[n].double() - p.grad).abs().max()) <= 5e-3 * float(p.grad.abs().max()) + 1e-6, n


def _step(sd, gt, backbone_mode, dtype=torch.float32):
    """One model.train() step; in fp32 every other device mode is on (lazy coarse loss, gt_sparse, fine,
    coarse transformer, keypoint encoder), in fp64 every mode is autograd."""
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().to(dtype).train()
    m.conf_matrix_mode = "lazy"
    kernels = "kernels" if dtype == torch.float32 else "autograd"
    m.fine_train_mode = m.coarse_transformer_train_mode = m.kpt_encoder_train_mode = kernels
    m.backbone_train_mode = backbone_mode
    data = mrg.train_batch(sd, False)
    del data["conf_matrix_gt"]
    data = {k: (v.to("cuda", dtype) if torch.is_tensor(v) and v.is_floating_point() else
                v.to("cuda") if torch.is_tensor(v) else v) for k, v in data.items()}
    data["gt_sparse"] = gt.to("cuda")
    torch.manual_seed(11)
    with mtf.default_dtype(dtype), _NoTF32():
        m(data)
        train_gt.fine_supervision(data, otg.config())
        losses.Loss(cl.LOSS_CONFIG).train()(data)
        m.zero_grad()
        data["loss"].backward()
    return m, data


def test_training_step_tf32x3_against_autograd():
    """One model.train() step with every other device mode on and the backbone in "tf32x3", against the same step with the backbone on autograd (cudnn TF32 off): same
    matches, loss within 1e-5 relative, backbone gradients within autograd's distance + its spread +
    2e-4 absmax; two tf32x3 steps bit-identical."""
    sd = workload.synthetic_state_dict(0)
    gt = planted_gt(mrg.train_batch(sd, False)["conf_matrix_gt"])
    ma, da = _step(sd, gt, "autograd")
    ma2, _ = _step(sd, gt, "autograd")
    mt, dt = _step(sd, gt, "tf32x3")
    mt2, dt2 = _step(sd, gt, "tf32x3")
    m64, _ = _step(sd, gt, "autograd", torch.float64)
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask"):
        assert torch.equal(da[k], dt[k]), k
    assert abs(da["loss"].item() - dt["loss"].item()) <= 1e-5 * abs(da["loss"].item())
    assert torch.equal(dt["loss"], dt2["loss"])
    for (n, p), (_, p2) in zip(mt.named_parameters(), mt2.named_parameters()):
        assert (p.grad is None) == (p2.grad is None) and (p.grad is None or torch.equal(p.grad, p2.grad)), n
    for (n, b), (_, b2) in zip(mt.named_buffers(), mt2.named_buffers()):
        assert torch.equal(b, b2), n
    pa, pa2 = dict(ma.named_parameters()), dict(ma2.named_parameters())
    pt, p64 = dict(mt.named_parameters()), dict(m64.named_parameters())
    for n in STEP_PARAMS:
        g64 = p64[n].grad
        amax = float(g64.abs().max())
        et = float((pt[n].grad.double() - g64).abs().max())
        ea = float((pa[n].grad.double() - g64).abs().max())
        spread = float((pa[n].grad - pa2[n].grad).abs().max())
        print(f"{n}: tf32x3 {et / amax:.2e}, autograd fp32 {ea / amax:.2e}, its spread {spread / amax:.2e} of absmax")
        assert et <= ea + spread + 2e-4 * amax + 1e-6, (n, et, ea, spread, amax)
