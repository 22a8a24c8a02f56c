"""Time and memory of the coarse transformer of a training step, forward + backward, at the reference
training shape (B = 4, 512 x 512 images: S = 64 x 64 = 4096 2D tokens, N = 7000 3D tokens, the six
layers of 3 x (self, cross), a pad mask): train_path.transformer by autograd against
train_coarse_tf.CoarseTransformerStage (the opp_coarse_tf_* kernels), alternated in one process.
Prints one JSON line.

    python scripts/train_coarse_tf_probe.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import make_train_coarse_tf_golden as mct  # noqa: E402
from oracle import workload  # noqa: E402
from onepose_plus_plus_b200 import train_coarse_tf, train_fine, train_path  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    B, hc, wc, N = 4, 64, 64, 7000
    case = mct.make_case(seed=1, B=B, hc=hc, wc=wc, N=N)
    tf = mct.coarse_module(workload.synthetic_state_dict(0), torch.float32, "cuda")
    params = [p for layer in tf.layers for p in train_fine.layer_params(layer)]
    d3 = case["desc3d"].cuda().float().requires_grad_(True)
    d2 = case["desc2d"].cuda().float().requires_grad_(True)
    mask = workload.pad_mask(B, hc, wc).reshape(B, hc * wc).cuda()
    w3, w2 = case["w3"].cuda().float(), case["w2"].cuda().float()

    def run(fn):
        o3, o2 = fn(tf, d3, d2, mask)
        torch.autograd.grad((o3 * w3).sum() + (o2 * w2).sum(), [d3, d2] + params)

    runs = {"autograd": lambda: run(train_path.transformer), "kernels": lambda: run(train_coarse_tf.coarse_transformer)}
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
    out = {"device": torch.cuda.get_device_name(), "power_limit": power, "B": B, "S": hc * wc, "N": N,
           "layers": list(tf.layer_names), "masked": True, "reps": args.reps}
    for name in runs:
        t = sorted(times[name])
        out[name] = {"median_ms": round(t[len(t) // 2], 3), "min_ms": round(t[0], 3), "max_ms": round(t[-1], 3),
                     "peak_mib": round(peaks[name] / 2 ** 20, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
