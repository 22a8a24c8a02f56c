"""Time and memory of the keypoint encoder of a training step, forward + backward, alternating in one
process: train_path.keypoint_encoding by autograd and train_kpt.KeypointEncoderStage (the
opp_kpt_train_* kernels), at B = 4 with N = 7000 (the reference training shape) and N = 20000.  A second
part times one whole model.train() forward + Loss + backward (B = 4, 512 x 512, N = 7000, planted)
with every device mode on, against the same step with only the encoder on autograd.  One JSON line;
card name, power limit and SM clock are read in the same call.

    python scripts/train_kpt_probe.py [--reps 20] [--step-reps 5]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import coarse_loss as cl  # noqa: E402
from oracle import make_reference_golden as mrg  # noqa: E402
from oracle import make_train_kpt_golden as mtk  # noqa: E402
from oracle import oracle, workload  # noqa: E402
from oracle import train_gt as otg  # noqa: E402
from onepose_plus_plus_b200 import OnePosePlus_model, losses, train_gt, train_kpt, train_path  # noqa: E402
from tests.test_train_gt_gpu import planted_gt  # noqa: E402


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


def _summary(times, peak):
    t = sorted(times)
    return {"median_ms": round(t[len(t) // 2], 3), "min_ms": round(t[0], 3), "max_ms": round(t[-1], 3),
            "peak_mib": peak}


def stage(n, reps):
    m = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    m.load_state_dict(workload.synthetic_state_dict(0), strict=True)
    enc = m.kpt_3d_pos_encoding.cuda().train()
    case = {k: v.cuda().float() for k, v in mtk.make_case(seed=1, B=4, N=n).items()}
    up = case["g"].transpose(1, 2).contiguous().transpose(1, 2)      # the rows' gradient, contiguous
    params = train_kpt.params(enc)

    def run(kernels):
        if kernels:
            out = train_kpt.keypoint_encoding(enc, case["kpts"], case["desc"])
        else:
            out = train_path.keypoint_encoding(enc, train_path.normalize_3d_keypoints(case["kpts"]), case["desc"])
        torch.autograd.grad(out, params, up)

    runs = {"autograd": lambda: run(False), "kernels": lambda: run(True)}
    peaks = {}
    for name, fn in runs.items():
        fn()
        peaks[name] = _peak(fn)
    times = {k: [] for k in runs}
    for _ in range(reps):
        for name, fn in runs.items():
            times[name].append(_timed(fn))
    out = {"device": _smi(), "B": 4, "N": n, "reps": reps}
    out.update({name: _summary(times[name], peaks[name]) for name in runs})
    return out


def _model(sd, kpt_mode):
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.conf_matrix_mode = "lazy"
    m.fine_train_mode = m.coarse_transformer_train_mode = m.backbone_train_mode = "kernels"
    m.kpt_encoder_train_mode = kpt_mode
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
    models = {"encoder_autograd": _model(sd, "autograd"), "all_kernels": _model(sd, "kernels")}

    def run(name):
        d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
        d["gt_sparse"] = gt.to("cuda")
        torch.manual_seed(11)
        models[name](d)
        train_gt.fine_supervision(d, otg.config())
        losses.Loss(cl.LOSS_CONFIG).train()(d)
        models[name].zero_grad(set_to_none=True)
        d["loss"].backward()

    peaks, times = {}, {k: [] for k in models}
    for name in models:
        run(name)
        peaks[name] = _peak(lambda: run(name))
    for _ in range(reps):
        for name in models:
            times[name].append(_timed(lambda: run(name)))
    out = {"device": _smi(), "B": 4, "H": 512, "W": 512, "N": 7000, "reps": reps}
    out.update({name: _summary(times[name], peaks[name]) for name in models})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--step-reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    stages = [stage(7000, args.reps), stage(20000, args.reps)]
    print(json.dumps({"stage": stages, "whole_step": whole_step(args.step_reps)}), flush=True)


if __name__ == "__main__":
    main()
