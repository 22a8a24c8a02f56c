"""Time the LINEMOD metric stage: pose_metrics_batched (opp_pose_metrics) on the device, with CUDA
events after warm-up, against the reference's per-frame CPU path (numpy + scipy cKDTree, restated
in oracle/pose_metrics.py) over the same poses.  Batch 1 and 64, models of 2000 / 8000 / 30000
points, ADD (symmetric = 0) and ADD-S (symmetric = 1).  Prints one JSON line with the device name
and power limit.
    python scripts/pose_metrics_probe.py [iters]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pose_metrics as opm  # noqa: E402  (test infrastructure: seeded models and poses)
from onepose_plus_plus_b200 import pnp  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("pose_metrics_probe needs a CUDA device")
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


rows = []
for V in (2000, 8000, 30000):
    verts = opm.synthetic_model(V, V)
    dia = opm.bbox_diameter(verts)
    pred, gt = opm.metric_frames(verts, dia, 64, seed=V)
    K = np.stack([opm.K_LINEMOD] * 64)
    tv, tp, tg, tK = (torch.as_tensor(x, dtype=torch.float32, device="cuda") for x in (verts, pred, gt, K))
    for B in (1, 64):
        for sym in (False, True):
            def stage():
                return pnp.pose_metrics_batched(tv, tp[:B], tg[:B], tK[:B], sym, dia)
            for _ in range(3):
                stage()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                r = stage()
            e1.record()
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / iters
            t0 = time.perf_counter()
            for b in range(B):   # the reference's per-frame host path
                opm.add_metric(verts, dia, pred[b], gt[b], syn=sym)
                opm.projection_2d_error(verts, pred[b], gt[b], K[b])
            cpu_ms = (time.perf_counter() - t0) * 1e3
            dist = np.array([opm.add_mean_distance(verts, pred[b], gt[b], syn=sym) for b in range(min(B, 4))])
            err = float(np.max(np.abs(r["add_dist"][: len(dist)].cpu().numpy() - dist)))
            rows.append({"V": V, "B": B, "symmetric": sym, "device_ms": round(dev_ms, 4), "cpu_ms": round(cpu_ms, 2),
                         "speedup": round(cpu_ms / dev_ms, 1), "max_abs_err_first4": err})
print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "iters": iters,
                  "rows": rows}))
