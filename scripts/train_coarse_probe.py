"""Coarse supervision of one training step alone — statistics -> focal loss -> backward to feat3d /
feat2d — at the training shape (B = 4, L = 7000, S = 4096, configs/experiment/train.yaml), for
  eager: the dual-softmax matrix and the reference loss formula in PyTorch (CUDA),
  lazy:  the opp_coarse_focal statistics, loss and backward kernels (no [B, L, S] matrix).
Reports the peak of torch.cuda.max_memory_allocated above the inputs and the time per step (CUDA
events, after warm-up), and prints one JSON line with the device name and power limit.
    python scripts/train_coarse_probe.py [steps]"""
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import coarse_loss as cl  # noqa: E402
from onepose_plus_plus_b200 import losses, train_path  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
B, L, S = 4, 7000, 4096


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


a, b, gt = (t.cuda() for t in cl.make_case("planted", B, L, S, seed=1)[:3])
crit = losses.Loss(cl.LOSS_CONFIG)
cm = types.SimpleNamespace(temperature=cl.TEMPERATURE)


def step(mode):
    fa, fb = a.detach().requires_grad_(True), b.detach().requires_grad_(True)
    if mode == "eager":
        conf = train_path.dual_softmax(cm, fa, fb, None)
    else:
        conf = train_path.TrainConfHandle(cm, fa, fb, None)
    loss = crit.compute_coarse_loss(conf, gt)
    loss.backward()
    return loss.detach()


rows = {}
for mode in ("eager", "lazy"):
    for _ in range(2):
        step(mode)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step(mode)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step(mode)
    e1.record()
    torch.cuda.synchronize()
    rows[mode] = {"ms_per_step": round(e0.elapsed_time(e1) / steps, 3), "peak_mib": round(peak / 2**20, 1),
                  "loss": loss.item()}
print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "B": B, "L": L, "S": S,
                  "steps": steps, "matrix_mib": round(B * L * S * 4 / 2**20, 1), **rows}))
