"""Time and memory of the backbone of a training step, forward + backward, at the reference training
shape (B = 4, 512 x 512), alternating in one process: train_path.backbone by autograd with PyTorch's
default cudnn TF32, train_backbone.BackboneStage in mode "kernels" (fp32 CUDA cores) and in mode
"tf32x3" (3xTF32 tensor cores).  A torch.profiler run times the dominant convolution
(layer1_outconv2.0, 196 -> 196 3 x 3 at 256 x 256) forward, dgrad and wgrad in both device modes, and a
second one sums the stage's convolution time per pass kind (MODE, k) in both modes.  A last JSON line
times one whole model.train() forward + Loss + backward (B = 4, 512 x 512, N = 7000, planted) with every
device mode on, the backbone in "kernels" and in "tf32x3".  Card name, power limit and SM clock are read
in the same call.

    python scripts/train_backbone_tc_probe.py [--reps 10] [--step-reps 3]
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


def _dev_ms(ev, n):
    t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return t / 1e3 / n


def _by_pass(prof, n):
    """{family: {pass_k: ms}} from bb_conv_kernel<MODE, KS> / bb_tc_conv_kernel<MODE, KS> (+ their reduces)."""
    out = {}
    for ev in prof.key_averages():
        m = re.search(r"(bb_tc_conv_kernel|bb_conv_kernel)<(\d), (\d)>", ev.key)
        if m:
            fam = "tf32x3" if m.group(1) == "bb_tc_conv_kernel" else "kernels"
            key = f"{PASS[m.group(2)]}_k{m.group(3)}"
        elif "bb_tc_reduce" in ev.key or "bb_reduce" in ev.key:
            fam = "tf32x3" if "bb_tc_reduce" in ev.key else "kernels"
            key = "wgrad_reduce"
        else:
            continue
        out.setdefault(fam, {})
        out[fam][key] = round(out[fam].get(key, 0.0) + _dev_ms(ev, n), 3)
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
            "kernels": lambda: run(train_backbone.backbone, True),
            "tf32x3": lambda: run(lambda b, i: train_backbone.backbone(b, i, "tf32x3"), True)}
    peaks = {}
    for name, fn in runs.items():
        fn()
        peaks[name] = _peak(fn)
    times = {k: [] for k in runs}
    smi_during = None
    for r in range(reps):
        for name, fn in runs.items():
            times[name].append(_timed(fn))
            if r == reps // 2 and name == "tf32x3":
                smi_during = _smi()
    out = {"device": smi_during, "B": 4, "H": 512, "W": 512, "reps": reps}
    for name in runs:
        t = sorted(times[name])
        out[name] = {"median_ms": round(t[len(t) // 2], 2), "min_ms": round(t[0], 2), "max_ms": round(t[-1], 2),
                     "peak_mib": peaks[name]}
    out["speedup_tf32x3_over_kernels"] = round(out["kernels"]["median_ms"] / out["tf32x3"]["median_ms"], 2)
    # every convolution launch of the stage, per pass kind, under the profiler
    for name in ("kernels", "tf32x3"):
        runs[name]()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            runs["kernels"]()
            runs["tf32x3"]()
        torch.cuda.synchronize()
    out["stage_conv_ms_by_pass"] = _by_pass(prof, 3)
    torch.backends.cudnn.allow_tf32 = True
    # the dominant convolution on its own, under the profiler
    x = torch.randn(4, 196, 256, 256, device="cuda")
    w = bb.layer1_outconv2[0].weight.detach().contiguous()
    y, dx, dw = torch.empty_like(x), torch.empty_like(x), torch.zeros_like(w)
    group = ops.backbone_wgrad_group()
    part = torch.empty(train_backbone.WGRAD_SLICE_GROUPS * w.numel(), device="cuda")
    pixels = 4 * 256 * 256
    step = train_backbone.WGRAD_SLICE_GROUPS * group

    def conv_passes(tc):
        ops.backbone_conv(x, w, 1, y, tf32x3=tc)
        ops.backbone_conv_dgrad(y, w, 1, dx, False, tf32x3=tc)
        for p0 in range(0, pixels, step):
            ops.backbone_conv_wgrad(x, y, 1, dw, part, p0, step, True, tf32x3=tc)

    for tc in (False, True):
        conv_passes(tc)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            conv_passes(False)
            conv_passes(True)
        torch.cuda.synchronize()
    smi_conv = _smi()
    flop = 2.0 * pixels * 196 * 196 * 9
    res = {"device": smi_conv, "flop_per_pass": flop}
    for fam, d in _by_pass(prof, 5).items():
        t = {"fwd": d.get("fwd_k3", 0.0), "dgrad": d.get("dgrad_k3", 0.0),
             "wgrad": d.get("wgrad_k3", 0.0) + d.get("wgrad_reduce", 0.0)}
        res[fam] = {p: {"ms": round(v, 3), "tflops_fp32_equiv": round(flop / (v * 1e-3) / 1e12, 2)}
                    for p, v in t.items() if v > 0}
    out["layer1_outconv2.0"] = res
    return out


def whole_step(reps):
    """The planted step of train_backbone_probe.py with every device mode on (lazy coarse loss, gt_sparse,
    fine, coarse transformer, keypoint encoder), the backbone in "kernels" and in "tf32x3", alternated."""
    sd = workload.synthetic_state_dict(0)
    data, _ = workload.planted_workload(sd, 512, 512, 7000, 3000, batch=4, seed=5)
    S = 64 * 64
    g = torch.Generator().manual_seed(3)
    cm = torch.zeros(4, 7000, S, dtype=torch.bool)
    cm[torch.randint(0, 4, (2000,), generator=g), torch.randint(0, 7000, (2000,), generator=g),
       torch.randint(0, S, (2000,), generator=g)] = True
    gt = planted_gt(cm)
    models = {}
    for mode in ("kernels", "tf32x3"):
        m = OnePosePlus_model(mrg.train_config())
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
        m.conf_matrix_mode = "lazy"
        m.fine_train_mode = m.coarse_transformer_train_mode = m.kpt_encoder_train_mode = "kernels"
        m.backbone_train_mode = mode
        models[f"all_on_backbone_{mode}"] = m

    def run(name):
        m = models[name]
        d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
        d["gt_sparse"] = gt.to("cuda")
        torch.manual_seed(11)
        m(d)
        train_gt.fine_supervision(d, otg.config())
        losses.Loss(cl.LOSS_CONFIG).train()(d)
        m.zero_grad(set_to_none=True)
        d["loss"].backward()

    out = {"device": None, "B": 4, "H": 512, "W": 512, "N": 7000, "reps": reps}
    peaks, times = {}, {k: [] for k in models}
    for name in models:
        run(name)
        peaks[name] = _peak(lambda: run(name))
    for _ in range(reps):
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
