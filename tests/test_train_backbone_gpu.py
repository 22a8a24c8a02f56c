"""Backbone of training on the device (model.backbone_train_mode "kernels"): train_backbone.BackboneStage
against the reference fixture and fp64 autograd of train_path.backbone on the small case and at the
training shape, eval-mode BatchNorm, a partial freeze, determinism, the memory of the stage, and one
model.train() step against the autograd backbone."""
import os

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
from tests.test_train_gt_gpu import planted_gt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_backbone.npz")
pytestmark = pytest.mark.gpu


class _NoTF32:
    def __enter__(self):
        self.old = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32 = self.old


def _run(sd, case, fwd, dtype=torch.float32, train=True):
    bb = mtb.backbone_module(sd, dtype, "cuda", train)
    return mtb.run(bb, fwd, case, dtype, "cuda")


def _flat(r):
    return [r[0], r[1]] + list(r[2]) + [v for k, v in sorted(r[3].items()) if "running" in k]


def _names(sd):
    bb = mtb.backbone_module(sd)
    return ["feat_c", "feat_f"] + ["d_" + n for n in mtb.param_names(bb)] + \
        sorted(n for n in mtb.buffer_names(bb) if "running" in n)


def _assert_fp64_distance(sd, r64, r32, rk, label, factor=2.0):
    """Each tensor within twice the fp32 autograd path's (cudnn TF32 off) distance from fp64 + 4e-3 absmax
    + 1e-6 (outputs and running statistics: + 2e-4 absmax).  The rule is relative to the autograd path
    with an absmax margin because at B = 4, 512 x 512 both fp32-grade paths are up to ~2e-2 of absmax
    from fp64 in the deep-layer weight gradients (layer3.1.conv1: kernels 1.8e-2, autograd 1.9e-2) and
    which one is closer differs per tensor; running statistics reach 3.5x the autograd distance, at
    3.4e-7 of absmax (DESIGN §7 f4)."""
    worst = []
    for name, a64, a32, ak in zip(_names(sd), _flat(r64), _flat(r32), _flat(rk)):
        amax = float(a64.abs().max())
        ek, et = float((ak.double() - a64).abs().max()), float((a32.double() - a64).abs().max())
        worst.append((ek / max(amax, 1e-30), et / max(amax, 1e-30), name))
        rel = 4e-3 if name.startswith("d_") else 2e-4
        assert ek <= factor * et + rel * amax + 1e-6, (label, name, ek, et, amax)
    worst.sort(reverse=True)
    print(label, "largest kernel distances (kernels, torch fp32, of absmax):", worst[:5])


@pytest.mark.parametrize("case_name", ["train"])
def test_small_case_against_the_reference_fixture_and_fp64(case_name):
    z = np.load(GOLDEN)
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    train = case_name == "train"
    rk = _run(sd, case, train_backbone.backbone, train=train)
    r64 = _run(sd, case, train_path.backbone, torch.float64, train)
    with _NoTF32():
        r32 = _run(sd, case, train_path.backbone, train=train)
    _assert_fp64_distance(sd, r64, r32, rk, case_name)
    bb = mtb.backbone_module(sd)
    names = ["feat_c", "feat_f"] + [f"d_{n}" for n in mtb.param_names(bb)]
    for key, t, t32 in zip(names, [rk[0], rk[1]] + rk[2], [r32[0], r32[1]] + r32[2]):
        k = f"{case_name}_{key}"
        amax = float(z[k + "_absmax"])
        idx = torch.from_numpy(z[k + "_idx"])
        got = t.flatten().cpu()[idx].double().numpy()
        d32 = np.abs(t32.flatten().cpu()[idx].double().numpy() - z[k]).max()
        assert np.abs(got - z[k]).max() <= 2 * d32 + (4e-3 if key.startswith("d_") else 2e-4) * amax + 1e-6, key
    for n, b in rk[3].items():
        ref = z[f"{case_name}_buf_{n}"]
        assert np.abs(b.double().cpu().numpy() - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1.0), n


def _stage_peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def test_training_shape_accuracy_determinism_and_memory():
    """B = 4, 512 x 512: outputs, every parameter gradient and the running statistics within the fp32
    autograd path's distance from fp64 (cudnn TF32 off) + 2e-4 absmax + 1e-6; two kernel calls bit-equal;
    the stage's peak above its inputs under 60 % of autograd's (default cudnn TF32)."""
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case(seed=1, B=4, H=512, W=512)
    case = {k: v.cuda() for k, v in case.items()}
    rk, peak_k = _stage_peak(lambda: _run(sd, case, train_backbone.backbone))
    rk2 = _run(sd, case, train_backbone.backbone)
    for name, a, b in zip(_names(sd), _flat(rk), _flat(rk2)):
        assert torch.equal(a, b), name
    # the default TF32 path: its peak is the memory yardstick (with TF32 off cuDNN picks workspace-heavy
    # fp32 algorithms, ~28 GiB), its distance from fp64 is printed for the record
    rt, peak_a = _stage_peak(lambda: _run(sd, case, train_path.backbone))
    with _NoTF32():
        r32 = _run(sd, case, train_path.backbone)
    r64 = _run(sd, case, train_path.backbone, torch.float64)
    for name, a64, at in zip(_names(sd), _flat(r64), _flat(rt)):
        if name in ("feat_c", "feat_f", "d_conv1.weight"):
            print(f"TF32 default: {name} {float((at.double() - a64).abs().max() / a64.abs().max()):.2e} of absmax")
    del rt
    # five times the fp32 path's distance: at this shape the two paths' distances from fp64 differ per
    # tensor with the summation order (DESIGN §7 f4)
    _assert_fp64_distance(sd, r64, r32, rk, "B=4 512x512", factor=5.0)
    print(f"peak above inputs: kernels {peak_k:.0f} MiB, autograd (default TF32) {peak_a:.0f} MiB")
    assert peak_k < 0.6 * peak_a, (peak_k, peak_a)


def test_eval_mode_batchnorm_frozen():
    """pretrained_fix: the backbone in eval mode with frozen parameters: outputs match autograd and the
    reference fixture's eval case, the running statistics stay untouched, and nothing needs a backward."""
    sd = workload.synthetic_state_dict(0)
    case = mtb.make_case()
    bb = mtb.backbone_module(sd, torch.float32, "cuda", train=False)
    for p in bb.parameters():
        p.requires_grad_(False)
    before = {n: b.clone() for n, b in bb.named_buffers()}
    img = case["img"].float().cuda()
    fc, ff = train_backbone.backbone(bb, img)
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
        fc, ff = train_backbone.backbone(bb, img)
        mtb.objective(fc, ff, {k: v.cuda() for k, v in case.items()}).backward()
    finally:
        ops.call = real
    assert calls.count("opp_backbone_train_conv_wgrad") == 2       # one slice each at this size
    assert not [c for c in calls if c.endswith("_tf32x3")], set(calls)
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
    fc, _ = train_backbone.backbone(bb, case["img"].float().cuda())
    (fc * case["g_c"].float().cuda()).sum().backward()
    grads = dict((n, p.grad) for n, p in bb.named_parameters())
    assert all(grads[n] is None for n in grads if n.startswith(("layer1_outconv", "layer2_outconv"))), \
        [n for n in grads if grads[n] is not None and "outconv" in n and "layer3" not in n]
    ref = mtb.backbone_module(sd, torch.float64, "cuda")
    c64, _ = train_path.backbone(ref, case["img"].double().cuda())
    (c64 * case["g_c"].cuda()).sum().backward()
    for n, p in ref.named_parameters():
        if p.grad is not None:
            # fp32 level of this gradient: both fp32 paths are ~1e-3 of absmax from fp64 here
            assert float((grads[n].double() - p.grad).abs().max()) <= 5e-3 * float(p.grad.abs().max()) + 1e-6, n


STEP_PARAMS = ("backbone.conv1.weight", "backbone.layer2.0.bn1.weight", "backbone.layer1_outconv2.3.weight",
               "kpt_3d_pos_encoding.encoder.0.weight", "loftr_coarse.layers.0.q_proj.weight")


def _step(sd, gt, backbone_mode, dtype=torch.float32):
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().to(dtype).train()
    m.conf_matrix_mode = "lazy"
    kernels = "kernels" if dtype == torch.float32 else "autograd"
    m.fine_train_mode = m.coarse_transformer_train_mode = kernels
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


def test_training_step_kernels_against_autograd():
    """One model.train() step on the planted train batch with lazy, gt_sparse, fine and coarse-transformer
    kernels; only the backbone mode differs (autograd with cudnn TF32 off).  Two kernel steps are
    bit-identical in the loss, every gradient and every buffer."""
    sd = workload.synthetic_state_dict(0)
    gt = planted_gt(mrg.train_batch(sd, False)["conf_matrix_gt"])
    ma, da = _step(sd, gt, "autograd")
    ma2, _ = _step(sd, gt, "autograd")
    mk, dk = _step(sd, gt, "kernels")
    mk2, dk2 = _step(sd, gt, "kernels")
    m64, d64 = _step(sd, gt, "autograd", torch.float64)
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask"):
        assert torch.equal(da[k], dk[k]), k
    assert abs(da["loss"].item() - dk["loss"].item()) <= 1e-5 * abs(da["loss"].item())
    assert torch.equal(dk["loss"], dk2["loss"])
    for (n, p), (_, p2) in zip(mk.named_parameters(), mk2.named_parameters()):
        assert (p.grad is None) == (p2.grad is None) and (p.grad is None or torch.equal(p.grad, p2.grad)), n
    for (n, b), (_, b2) in zip(mk.named_buffers(), mk2.named_buffers()):
        assert torch.equal(b, b2), n
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
