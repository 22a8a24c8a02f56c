"""Tracking-step probe: the device crop (opp_crop_resize_u8) and the whole PoseTracker.step
(crop -> matcher -> colmap PnP), eager and with CUDA graphs, against the reference's CPU crop
(two cv2.warpAffine calls, the float conversion and the upload of the 512 x 512 crop) on the same host.
Frames of 640 x 480 and 1920 x 1440, B = 1 and 8; the bank is planted (oracle/workload.py, N = 5000)
and each frame holds the planted image under its box, so the matcher finds its usual match count.
Prints one JSON line with the device name and power limit.
    python scripts/track_probe.py [step_iters]"""
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle, workload  # noqa: E402  (planted workloads)
from onepose_plus_plus_b200 import OnePosePlus_model, tracking  # noqa: E402

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 30
CROP = 512


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def device_us(fn, n):
    """Mean device time of fn() in microseconds over n calls (CUDA events, after a warm-up)."""
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / n


def host_us(fn, n, warm=3):
    """Mean wall time of fn() (which ends in a device synchronise) in microseconds."""
    for _ in range(warm):
        fn()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t0) * 1e6 / n


sd = workload.synthetic_state_dict(0)
model = OnePosePlus_model(oracle.DEFAULT_CONFIG)
model.load_state_dict(sd, strict=True)
model = model.eval().cuda()
data, _ = workload.planted_workload(sd, CROP, CROP, 5000, 3000, batch=1, with_scale=False)
model.set_bank(data["keypoints3d"].cuda(), data["descriptors3d_db"].cuda(), data["descriptors3d_coarse_db"].cuda())
base = (data["query_image"][0, 0] * 255).round().to(torch.uint8).numpy()
rng = np.random.default_rng(0)
rows = []
for (H, W), (ox, oy) in (((480, 640), (64, -16)), ((1440, 1920), (700, 460))):
    for B in (1, 8):
        frames = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
        y0, y1 = max(oy, 0), min(oy + CROP, H)
        frames[:, y0:y1, ox:ox + CROP] = base[y0 - oy:y1 - oy]
        boxes = np.array([[ox, oy, ox + CROP, oy + CROP]] * B, dtype=np.int32)
        dframes = torch.from_numpy(frames).cuda()
        rec = tracking.crop_params(boxes, CROP)
        params = tracking._params_tensor(rec).cuda()
        out = torch.empty((B, 1, CROP, CROP), dtype=torch.uint8, device="cuda")
        kernel = device_us(lambda: tracking._launch_crop(dframes, params, out), 200)

        def call():
            tracking.crop_resize_batched(dframes, boxes, CROP)
            torch.cuda.synchronize()
        crop_call = host_us(call, 100)
        # the reference's CPU crop of the same frames: two warps, float conversion, upload
        K = np.array([[600.0, 0, W / 2], [0, 600.0, H / 2], [0, 0, 1]])

        def cpu_crop():
            for b in range(B):
                x0, y0_, x1, y1_ = boxes[b]
                w, h = int(x1 - x0), int(y1_ - y0_)
                s1 = cv2.warpAffine(frames[b], tracking._box_map(boxes[b], (h, w)), (w, h), flags=cv2.INTER_LINEAR)
                s2 = cv2.warpAffine(s1, tracking._box_map(np.array([0, 0, w, h]), (CROP, CROP)), (CROP, CROP),
                                    flags=cv2.INTER_LINEAR)
                torch.from_numpy(s2.astype(np.float32) / 255)[None][None].cuda()
            torch.cuda.synchronize()
        cpu = host_us(cpu_crop, 20)
        # same crop bytes as the reference path (spot check of the timed configuration)
        ref = cv2.warpAffine(cv2.warpAffine(frames[0], tracking._box_map(boxes[0], (CROP, CROP)), (CROP, CROP)),
                             tracking._box_map(np.array([0, 0, CROP, CROP]), (CROP, CROP)), (CROP, CROP))
        same = bool(np.array_equal(out[0, 0].cpu().numpy(), ref))
        row = {"frame": f"{W}x{H}", "B": B, "crop_kernel_us_per_frame": round(kernel / B, 2),
               "crop_call_us_per_frame": round(crop_call / B, 1), "cpu_ref_crop_us_per_frame": round(cpu / B, 1),
               "crop_equal_cv2": same}
        for graphs in (False, True):
            model.enable_cuda_graphs(graphs)
            tr = tracking.PoseTracker(model, K, np.zeros((8, 3)))
            init = list(boxes)
            res = tr.step(dframes, init_bbox=init)
            step = host_us(lambda: tr.step(dframes, init_bbox=init), iters)
            row["step_graphs_us_per_frame" if graphs else "step_eager_us_per_frame"] = round(step / B, 1)
            row["matches_frame0"] = int(res[0]["mkpts_query_f"].shape[0])
        model.enable_cuda_graphs(False)
        rows.append(row)
print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "step_iters": iters,
                  "rows": rows}))
