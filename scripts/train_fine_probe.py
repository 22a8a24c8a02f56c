"""Time and memory of the fine level of a training step, forward + backward, at the reference training
shape (B = 4, 512 x 512: a 256 x 256 fine map, stride 4, L = 7000, M = 4915 matches): the autograd
path of train_path (F.unfold + PyTorch layers + fine_matching) against train_fine.FineStage (the
opp_fine_train_* kernels), alternated in one process.  Prints one JSON line.

    python scripts/train_fine_probe.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import make_train_fine_golden as mtf  # noqa: E402
from oracle import workload  # noqa: E402
from onepose_plus_plus_b200 import train_fine, train_path  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    case = mtf.make_case(0, B=4, hc=64, wc=64, stride=4, n3d=7000, M=4915)
    fine = mtf.fine_module(workload.synthetic_state_dict(0), torch.float32, "cuda")
    params = [p for layer in fine.layers for p in train_fine.layer_params(layer)]
    feat = case["feat_f"].cuda().float().requires_grad_(True)
    desc = case["desc3d"].cuda().float().contiguous()
    ids = [case[k].cuda() for k in ("b_ids", "i_ids", "j_ids")]
    w = torch.randn(len(ids[0]), 3, device="cuda")
    data0 = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in mtf.fine_data(case).items()}

    def autograd():
        data = dict(data0)
        f3d, f2d = train_path.fine_preprocess(5, 128, data, desc, feat)
        f3d, f2d = train_path.transformer(fine, f3d, f2d)
        train_path.fine_matching(f3d, f2d, data, True)
        torch.autograd.grad((data["expec_f"] * w).sum(), [feat] + params)

    def kernels():
        expec = train_fine.FineStage.apply(feat, desc, *ids, (64, 64, 4), *params)
        torch.autograd.grad((expec * w).sum(), [feat] + params)

    runs = {"autograd": autograd, "kernels": kernels}
    times = {k: [] for k in runs}
    peaks = {}
    for name, fn in runs.items():          # warm-up and peak memory above the inputs
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    for _ in range(args.reps):
        for name, fn in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        power = "unknown"
    out = {"device": torch.cuda.get_device_name(), "power_limit": power, "B": 4, "fine_hw": [256, 256], "M": 4915,
           "reps": args.reps}
    for name in runs:
        t = sorted(times[name])
        out[name] = {"median_ms": round(t[len(t) // 2], 3), "min_ms": round(t[0], 3), "max_ms": round(t[-1], 3),
                     "peak_mib": round(peaks[name] / 2 ** 20, 1)}
    out["unfold_tensor_mib"] = round(4 * 3200 * 4096 * 4 / 2 ** 20, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
