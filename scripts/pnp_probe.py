"""Time the pose stage's two solvers: ransac_pnp_batched(solver="opencv") (the reference's
cv2.solvePnPRansac branch) and solver="colmap" (its use_pycolmap_ransac branch), with CUDA events
after warm-up, at batch 1 and 64, 400 and 2000 matches per frame, 30 % outliers (LINEMOD
intrinsics, oracle/pnp_colmap.heavy_tailed_frames).  The CPU column is the reference's per-frame
cv2.solvePnPRansac call (EPnP, 10000 iterations) on the same frames; pycolmap is not part of this
environment, so the colmap branch has no CPU timing.  Prints one JSON line with the device name
and power limit.
    python scripts/pnp_probe.py [iters]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pnp as opnp  # noqa: E402  (test infrastructure: the reference's cv2 call)
from oracle import pnp_colmap as opc  # noqa: E402  (seeded planted frames)
from onepose_plus_plus_b200 import pnp  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("pnp_probe needs a CUDA device")
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


rows = []
for n in (400, 2000):
    b, p3, p2, K, _ = opc.heavy_tailed_frames(64, seed=n, n_range=(n, n))
    tb, t3, t2, tK = (torch.as_tensor(x, device="cuda") for x in (b, p3, p2, K))
    for B in (1, 64):
        sel = tb < B
        args = (tb[sel], t3[sel], t2[sel], tK[:B])
        row = {"matches_per_frame": n, "B": B}
        for solver in ("opencv", "colmap"):
            def stage():
                return pnp.ransac_pnp_batched(*args, reprojection_error=7.0, solver=solver)
            for _ in range(3):
                stage()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                stage()
            e1.record()
            torch.cuda.synchronize()
            row[f"{solver}_us_per_frame"] = round(e0.elapsed_time(e1) * 1e3 / iters / B, 1)
        t0 = time.perf_counter()
        for f in range(B):   # the reference's per-frame host call (cv2 branch)
            m = b == f
            opnp.ransac_pnp(K[f], p2[m], p3[m], scale=1, pnp_reprojection_error=7)
        row["cpu_cv2_us_per_frame"] = round((time.perf_counter() - t0) * 1e6 / B, 1)
        rows.append(row)
print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "iters": iters,
                  "outlier_frac": 0.3, "threshold_px": 7.0,
                  "note": "no pycolmap CPU timing: pycolmap is not installed in this environment", "rows": rows}))
