"""Fine level of training on the device (model.fine_train_mode "kernels"): the opp_fine_train_* kernels
against the reference fixture and an fp64 autograd run of train_path's fine functions, on the small
case and at the training shape; the clamp of the variance; determinism; the memory of the stage; and
one training step against the autograd fine level."""
import os

import numpy as np
import pytest
import torch

from oracle import make_reference_golden as mrg
from oracle import make_train_fine_golden as mtf
from oracle import train_gt as otg
from oracle import coarse_loss as cl
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, losses, ops, train_fine, train_gt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_fine.npz")
pytestmark = pytest.mark.gpu
UNFOLD_BYTES = 4 * 3200 * 4096 * 4      # F.unfold's [B, 128*25, L] fp32 tensor at the training shape


def kernels_fine(fine32, case, weights=None):
    """FineStage on the device: (expec_f, loss, d feat_f, [d param])."""
    dev = "cuda"
    feat = case["feat_f"].to(dev, torch.float32).requires_grad_(True)
    desc = case["desc3d"].to(dev, torch.float32).contiguous()
    ids = [case[k].to(dev) for k in ("b_ids", "i_ids", "j_ids")]
    (hc, wc), (hf, _) = case["q_hw_c"], case["q_hw_f"]
    params = [p for layer in fine32.layers for p in train_fine.layer_params(layer)]
    expec = train_fine.FineStage.apply(feat, desc, *ids, (hc, wc, hf // hc), *params)
    loss = mtf.objective(expec, {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in case.items()},
                         None if weights is None else weights.to(dev, torch.float32))
    grads = torch.autograd.grad(loss, [feat] + params)
    return expec.detach(), loss.detach(), grads[0], list(grads[1:])


def _runs(case, weights=None):
    sd = workload.synthetic_state_dict(0)
    r64 = mtf.train_path_fine(mtf.fine_module(sd, torch.float64, "cuda"), case, torch.float64, "cuda",
                              None if weights is None else weights.cuda().double())
    r32 = mtf.train_path_fine(mtf.fine_module(sd, torch.float32, "cuda"), case, torch.float32, "cuda",
                              None if weights is None else weights.cuda().float())
    rk = kernels_fine(mtf.fine_module(sd, torch.float32, "cuda"), case, weights)
    return r64, r32, rk


def _assert_fp64_distance(r64, r32, rk, report=None):
    """expec_f within 1e-5 of fp64; each gradient's max |err| within the fp32 path's own + 2e-4 absmax + 1e-6."""
    assert (rk[0].double() - r64[0]).abs().max() <= 1e-5
    names = ["feat_f"] + list(mtf.FINE_PARAMS)
    for name, g64, g32, gk in zip(names, [r64[2]] + r64[3], [r32[2]] + r32[3], [rk[2]] + rk[3]):
        amax = float(g64.abs().max())
        ek, et = float((gk.double() - g64).abs().max()), float((g32.double() - g64).abs().max())
        if report is not None:
            report.append(f"{name}: kernels {ek / max(amax, 1e-30):.2e}, torch fp32 {et / max(amax, 1e-30):.2e} of absmax")
        assert ek <= et + 2e-4 * amax + 1e-6, (name, ek, et, amax)


def test_small_case_against_the_reference_fixture_and_fp64():
    case = mtf.make_case()
    dup = case["b_ids"] * 1000 + case["j_ids"]
    assert len(torch.unique(dup)) < len(dup)                      # a repeated (b, j) cell
    r64, r32, rk = _runs(case)
    z = np.load(GOLDEN)
    assert np.abs(rk[0].cpu().numpy() - z["expec_f"]).max() <= 1e-5
    assert abs(rk[1].item() - float(z["loss"])) <= 1e-5 * abs(float(z["loss"])) + 1e-7
    for name, g in zip(["feat_f"] + list(mtf.FINE_PARAMS), [rk[2]] + rk[3]):
        key = "d_" + name
        got = g.detach().flatten().cpu().double().numpy()[z[key + "_idx"]]
        assert np.abs(got - z[key]).max() <= 2e-4 * float(z[key + "_absmax"]) + 1e-6, name
    _assert_fp64_distance(r64, r32, rk)
    # the std column as well (the fine loss passes it no gradient)
    w = torch.randn(len(case["b_ids"]), 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    _assert_fp64_distance(*_runs(case, w))


def test_clamp_of_the_variance_passes_no_gradient():
    """x rows whose heatmap is one-hot (var = 0 < 1e-10: the clamp is active) and ordinary rows: the
    kernels' expectation and its backward against autograd through train_path.fine_matching in fp64."""
    from onepose_plus_plus_b200 import train_path
    g = torch.Generator().manual_seed(3)
    M = 8
    x = torch.randn(M, 26, 128, generator=g, dtype=torch.float64)
    x[:3, 7] = x[:3, 25] * 40.0                                   # token 7 dominates: heat one-hot
    x[3, 0:25] = x[3, 25] * 0.0                                   # uniform heat
    xr = x.clone().requires_grad_(True)
    data = {"q_hw_i": (64, 64), "q_hw_f": (32, 32), "mkpts_query_c": torch.zeros(M, 2, dtype=torch.float64),
            "b_ids": torch.zeros(M, dtype=torch.long)}
    with mtf.default_dtype(torch.float64):
        train_path.fine_matching(xr[:, 25:26], xr[:, :25], data, True)
    w = torch.randn(M, 3, generator=g, dtype=torch.float64)
    (data["expec_f"] * w).sum().backward()
    assert torch.allclose(data["expec_f"][:3, 2].detach(), torch.full((3,), 2e-5, dtype=torch.float64))  # clamp active
    xd = x.float().reshape(M * 26, 128).cuda().contiguous()
    expec = torch.empty(M, 3, device="cuda")
    ops.fine_train_match(xd, M, expec)
    dx = torch.empty_like(xd)
    ops.fine_train_match_bwd(xd, w.float().cuda().contiguous(), M, dx)
    assert (expec.double().cpu() - data["expec_f"].detach()).abs().max() <= 1e-5
    ref = xr.grad.reshape(M * 26, 128)
    amax = float(ref.abs().max())
    assert (dx.double().cpu() - ref).abs().max() <= 2e-4 * amax + 1e-6


def training_case(seed=0, B=4, hc=64, wc=64, stride=4, n3d=7000, M=4915):
    """The reference training shape: 512 x 512 images, L = 7000, M = int(B min(L, S) 0.3) (the
    prediction subset plus the GT paddings always add up to it)."""
    return mtf.make_case(seed, B, hc, wc, stride, n3d, M)


def test_training_shape_accuracy_determinism_and_memory():
    case = training_case()
    w = torch.randn(len(case["b_ids"]), 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    report = []
    r64, r32, rk = _runs(case, w)
    _assert_fp64_distance(r64, r32, rk, report)
    print("\n".join(report))
    del r64, r32
    # determinism: a second call gives the same bits
    sd = workload.synthetic_state_dict(0)
    fine = mtf.fine_module(sd, torch.float32, "cuda")
    rk2 = kernels_fine(fine, case, w)
    for a, b in zip([rk[0], rk[2]] + rk[3], [rk2[0], rk2[2]] + rk2[3]):
        assert torch.equal(a, b)
    del rk, rk2
    # memory: the stage's peak, forward and backward, above its inputs
    feat = case["feat_f"].cuda().float().requires_grad_(True)
    desc = case["desc3d"].cuda().float().contiguous()
    ids = [case[k].cuda() for k in ("b_ids", "i_ids", "j_ids")]
    wd = w.cuda().float()
    params = [p for layer in fine.layers for p in train_fine.layer_params(layer)]
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    expec = train_fine.FineStage.apply(feat, desc, *ids, (64, 64, 4), *params)
    torch.autograd.grad((expec * wd).sum(), [feat] + params)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"fine stage peak above its inputs: {peak / 2**20:.1f} MiB (unfold tensor {UNFOLD_BYTES / 2**20:.1f} MiB)")
    assert peak < UNFOLD_BYTES


def test_feat_gradient_only_and_parameters_only():
    """ctx.needs_input_grad: with frozen parameters only d feat_f is formed, with a frozen map only the
    parameter gradients; both equal the full call's."""
    case = mtf.make_case(seed=4)
    sd = workload.synthetic_state_dict(0)
    fine = mtf.fine_module(sd, torch.float32, "cuda")
    full = kernels_fine(fine, case)
    params = [p for layer in fine.layers for p in train_fine.layer_params(layer)]
    feat = case["feat_f"].cuda().float()
    desc = case["desc3d"].cuda().float().contiguous()
    ids = [case[k].cuda() for k in ("b_ids", "i_ids", "j_ids")]
    cg = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in case.items()}
    f = feat.clone().requires_grad_(True)
    loss = mtf.objective(train_fine.FineStage.apply(f, desc, *ids, (4, 5, 4), *[p.detach() for p in params]), cg)
    (d_feat,) = torch.autograd.grad(loss, [f])
    assert torch.equal(d_feat, full[2])
    loss = mtf.objective(train_fine.FineStage.apply(feat, desc, *ids, (4, 5, 4), *params), cg)
    gp = torch.autograd.grad(loss, params)
    for a, b in zip(gp, full[3]):
        assert torch.equal(a, b)


def test_training_step_kernels_against_autograd():
    """One model.train() step on the planted train batch, lazy coarse matching, the fine level by
    autograd and by the kernels under one seed: identical matches, gt_mask and expec_f_gt; expec_f,
    mkpts_query_f and the loss within the fp64 tolerances; the fine parameters' gradients within 2e-4
    of absmax plus what the PyTorch fp32 path's run-to-run spread allows."""
    sd = workload.synthetic_state_dict(0)
    cfg = otg.config()
    runs = {}
    for mode in ("autograd", "kernels"):
        m = OnePosePlus_model(mrg.train_config())
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
        m.conf_matrix_mode = "lazy"
        m.fine_train_mode = mode
        data = mrg.train_batch(sd, True)
        data["fine_location_matrix_gt"] = torch.zeros(*data["conf_matrix_gt"].shape, 2)
        data = {k: (v.to("cuda") if torch.is_tensor(v) else v) for k, v in data.items()}
        torch.manual_seed(11)
        m(data)
        train_gt.fine_supervision(data, cfg)
        losses.Loss(cl.LOSS_CONFIG).train()(data)
        m.zero_grad()
        data["loss"].backward()
        runs[mode] = (m, data)
    (ma, da), (mk, dk) = runs["autograd"], runs["kernels"]
    assert dk["expec_f"].grad_fn is not None and type(dk["expec_f"].grad_fn).__name__.startswith("FineStage")
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "expec_f_gt"):
        assert torch.equal(da[k], dk[k]), k
    # (x, y): each fp32 path is within 1e-5 of fp64, so the two are within 2e-5 of each other.  std =
    # sqrt(E[g^2] - c^2) cancels in fp32 for sharp heatmaps (two fp32 evaluations differ by ~1e-4
    # there); the loss reads it only as a detached weight
    assert (da["expec_f"][:, :2] - dk["expec_f"][:, :2]).abs().max() <= 2e-5
    assert (da["mkpts_query_f"] - dk["mkpts_query_f"]).abs().max() <= 1e-5 * float(da["mkpts_query_f"].abs().max())
    assert abs(da["loss"].item() - dk["loss"].item()) <= 1e-3 * abs(da["loss"].item())
    pa, pk = dict(ma.named_parameters()), dict(mk.named_parameters())
    for n in mtf.FINE_PARAMS:
        a, b = pa[n].grad, pk[n].grad
        assert torch.allclose(a, b, rtol=0, atol=1e-3 * float(a.abs().max()) + 1e-9), n
