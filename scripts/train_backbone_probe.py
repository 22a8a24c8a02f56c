"""Time and memory of the backbone of a training step, forward + backward, at the reference training
shape (B = 4, 512 x 512), alternating in one process: train_path.backbone by autograd with PyTorch's
default cudnn TF32, the same with TF32 off, and train_backbone.BackboneStage (the opp_backbone_train_*
kernels, convolutions in 3xTF32 on the tensor cores).  Two torch.profiler runs time the convolutions:
the stage's launches summed per pass kind (forward / dgrad / wgrad, k), and the dominant convolution
(layer1_outconv2.0, 196 -> 196 3 x 3 at 256 x 256) on its own.  A second JSON line times one whole
model.train() forward + Loss + backward (B = 4, 512 x 512, N = 7000, planted) with every device mode on
and with all of them off.  Card name, power limit and SM clock are read in the same call.

    python scripts/train_backbone_probe.py [--reps 10]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import coarse_loss as cl  # noqa: E402
from oracle import make_reference_golden as mrg  # noqa: E402
from oracle import make_train_backbone_golden as mtb  # noqa: E402
from oracle import train_gt as otg  # noqa: E402
from oracle import workload  # noqa: E402
from onepose_plus_plus_b200 import OnePosePlus_model, losses, ops, train_backbone, train_gt, train_path  # noqa: E402
from tests.test_train_gt_gpu import planted_gt  # noqa: E402

PASS = {"0": "fwd", "1": "dgrad", "2": "wgrad"}


def _smi():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def _timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def _by_pass(prof, n):
    """{pass_k: ms per run} from bb_conv_kernel<MODE, KS>, and the wgrad's bb_reduce_kernel."""
    out = {}
    for ev in prof.key_averages():
        m = re.search(r"bb_conv_kernel<(\d), (\d)>", ev.key)
        if m:
            key = f"{PASS[m.group(1)]}_k{m.group(2)}"
        elif "bb_reduce" in ev.key:
            key = "wgrad_reduce"
        else:
            continue
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        out[key] = round(out.get(key, 0.0) + t / 1e3 / n, 3)
    return out


def stage(reps):
    sd = workload.synthetic_state_dict(0)
    case = {k: v.cuda().float() for k, v in mtb.make_case(seed=1, B=4, H=512, W=512).items()}
    bb = mtb.backbone_module(sd, torch.float32, "cuda")
    params = list(bb.parameters())

    def run(fn, tf32):
        torch.backends.cudnn.allow_tf32 = tf32
        fc, ff = fn(bb, case["img"])
        torch.autograd.grad(mtb.objective(fc, ff, case), params)

    runs = {"autograd_tf32": lambda: run(train_path.backbone, True),
            "autograd_fp32": lambda: run(train_path.backbone, False),
            "kernels": lambda: run(train_backbone.backbone, True)}
    peaks = {}
    for name, fn in runs.items():
        fn()
        peaks[name] = _peak(fn)
    times = {k: [] for k in runs}
    smi_during = None
    for r in range(reps):
        for name, fn in runs.items():
            times[name].append(_timed(fn))
            if r == reps // 2 and name == "kernels":
                smi_during = _smi()
    torch.backends.cudnn.allow_tf32 = True
    out = {"device": smi_during, "B": 4, "H": 512, "W": 512, "reps": reps}
    for name in runs:
        t = sorted(times[name])
        out[name] = {"median_ms": round(t[len(t) // 2], 2), "min_ms": round(t[0], 2), "max_ms": round(t[-1], 2),
                     "peak_mib": peaks[name]}
    # every convolution launch of the stage, per pass kind, under the profiler
    runs["kernels"]()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            runs["kernels"]()
        torch.cuda.synchronize()
    out["stage_conv_ms_by_pass"] = _by_pass(prof, 3)
    # the dominant convolution on its own, under the profiler
    x = torch.randn(4, 196, 256, 256, device="cuda")
    w = bb.layer1_outconv2[0].weight.detach().contiguous()
    y, dx, dw = torch.empty_like(x), torch.empty_like(x), torch.zeros_like(w)
    group = ops.backbone_wgrad_group()
    part = torch.empty(train_backbone.WGRAD_SLICE_GROUPS * w.numel(), device="cuda")
    pixels = 4 * 256 * 256
    step = train_backbone.WGRAD_SLICE_GROUPS * group

    def conv_passes():
        ops.backbone_conv(x, w, 1, y)
        ops.backbone_conv_dgrad(y, w, 1, dx, False)
        for p0 in range(0, pixels, step):
            ops.backbone_conv_wgrad(x, y, 1, dw, part, p0, step, True)

    conv_passes()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            conv_passes()
        torch.cuda.synchronize()
    smi_conv = _smi()
    flop = 2.0 * pixels * 196 * 196 * 9
    d = _by_pass(prof, 5)
    kt = {"fwd": d.get("fwd_k3", 0.0), "dgrad": d.get("dgrad_k3", 0.0),
          "wgrad": d.get("wgrad_k3", 0.0) + d.get("wgrad_reduce", 0.0)}
    # fp32-equivalent algorithmic FLOPs (the 3xTF32 MMAs issue three times as many)
    out["layer1_outconv2.0"] = {"device": smi_conv, "flop_per_pass": flop, **{
        m: {"ms": round(t, 3), "tflops_fp32_equiv": round(flop / (t * 1e-3) / 1e12, 2)} for m, t in kt.items()}}
    return out


def _step(sd, gt, on):
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.conf_matrix_mode = "lazy" if on else "eager"
    m.fine_train_mode = m.coarse_transformer_train_mode = m.backbone_train_mode = m.kpt_encoder_train_mode = \
        "kernels" if on else "autograd"
    return m


def whole_step(reps):
    sd = workload.synthetic_state_dict(0)
    data, _ = workload.planted_workload(sd, 512, 512, 7000, 3000, batch=4, seed=5)
    S = 64 * 64
    g = torch.Generator().manual_seed(3)
    cm = torch.zeros(4, 7000, S, dtype=torch.bool)
    cm[torch.randint(0, 4, (2000,), generator=g), torch.randint(0, 7000, (2000,), generator=g),
       torch.randint(0, S, (2000,), generator=g)] = True
    gt = planted_gt(cm)
    out = {"device": None, "B": 4, "H": 512, "W": 512, "N": 7000, "reps": reps}
    models = {"all_kernels": _step(sd, gt, True), "all_autograd": _step(sd, gt, False)}

    def run(name):
        m = models[name]
        d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
        if name == "all_kernels":
            d["gt_sparse"] = gt.to("cuda")
        else:
            d["conf_matrix_gt"] = cm.cuda()
            fl = torch.full((4, 7000, S, 2), train_gt.FINE_FILL, device="cuda")
            fl[gt.b_ids.cuda(), gt.i_ids.cuda(), gt.j_ids.cuda()] = gt.fine_xy.cuda()
            d["fine_location_matrix_gt"] = fl
        torch.manual_seed(11)
        m(d)
        train_gt.fine_supervision(d, otg.config())
        losses.Loss(cl.LOSS_CONFIG).train()(d)
        m.zero_grad(set_to_none=True)
        d["loss"].backward()

    peaks, times = {}, {k: [] for k in models}
    for name in models:
        run(name)
        peaks[name] = _peak(lambda: run(name))
    for r in range(reps):
        for name in models:
            times[name].append(_timed(lambda: run(name)))
    out["device"] = _smi()
    for name in models:
        t = sorted(times[name])
        out[name] = {"median_ms": round(t[len(t) // 2], 1), "min_ms": round(t[0], 1), "max_ms": round(t[-1], 1),
                     "peak_mib": peaks[name]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--step-reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps(stage(args.reps)), flush=True)
    print(json.dumps(whole_step(args.step_reps)), flush=True)


if __name__ == "__main__":
    main()
