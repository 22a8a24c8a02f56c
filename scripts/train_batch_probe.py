"""Loader-side cost of the training ground truth and its device replacement; prints one JSON line.

  --cpu  (needs the reference tree) per-item time of the reference item followed by SparseGTDataset's
         conversion of its dense tensors, against ProjectedGTDataset's item, at the training shape
         (512², shape3d 7000, 3000 correspondences), odd items warped.  torch keeps its default thread
         count (a loader worker may have fewer); the host's core count is reported beside the numbers.
  --gpu  prepare_batch at the training shape (B = 4, half the items warped) with CUDA events after a
         warm-up, and one kernel-mode training step (model.train(), conf_matrix_mode "lazy", every
         *_train_mode "kernels", forward + fine supervision + loss + backward) at that shape.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def cpu_probe(n_items):
    from oracle import train_batch as otb
    from onepose_plus_plus_b200 import train_batch, train_gt
    out = {"host_cpus": os.cpu_count(), "torch_threads": torch.get_num_threads()}
    with tempfile.TemporaryDirectory() as root:
        case = otb.make_case(root, seed=11, n_items=n_items, warp=True, shape3d=7000, n_3d=7500, n_corr=3000)
        ds = otb.reference_dataset(case)
        routes = {"reference_item_plus_sparse_conversion": train_gt.SparseGTDataset(ds),
                  "projected_gt_item": train_batch.ProjectedGTDataset(ds)}
        for name, d in routes.items():
            d[0], d[1]                                  # warm-up (file cache, imports)
            ts = []
            for idx in range(2 * n_items):
                t0 = time.perf_counter()
                d[idx]
                ts.append(time.perf_counter() - t0)
            out[name + "_ms"] = round(1e3 * float(np.median(ts)), 2)
    return out


def gpu_probe(warmup, iters):
    from oracle import train_batch as otb
    from oracle import coarse_loss as cl
    from oracle import make_reference_golden as mrg
    from oracle import train_gt as otg
    from oracle import workload
    from onepose_plus_plus_b200 import OnePosePlus_model, losses, train_batch, train_gt
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}
    host = otb.synthetic_batch(1)

    def cuda_batch():
        return {k: (v.to("cuda") if torch.is_tensor(v) or isinstance(v, train_batch.GTSource) else v)
                for k, v in host.items()}

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for k in range(warmup + iters):
        b = cuda_batch()
        torch.cuda.synchronize()
        e0.record()
        train_batch.prepare_batch(b)
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms.append(e0.elapsed_time(e1))
    out["prepare_batch_ms"] = round(float(np.median(ms)), 3)
    out["correspondences"] = len(b["gt_sparse"])
    sd = workload.synthetic_state_dict(0)
    base, _ = workload.planted_workload(sd, 512, 512, 7000, 3000, batch=4, seed=5)
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    m.conf_matrix_mode = "lazy"
    for k in ("fine_train_mode", "coarse_transformer_train_mode", "backbone_train_mode", "kpt_encoder_train_mode"):
        setattr(m, k, "kernels")
    crit = losses.Loss(cl.LOSS_CONFIG).train()
    ms = []
    for k in range(warmup + iters):
        data = {kk: v for kk, v in base.items() if kk not in ("query_image", "keypoints3d")}
        data.update({kk: host[kk] for kk in ("query_image", "keypoints3d", "query_image_scale", "query_intrinsic")})
        data["gt_source"] = host["gt_source"]
        data = {kk: (v.to("cuda") if torch.is_tensor(v) or isinstance(v, train_batch.GTSource) else v)
                for kk, v in data.items()}
        torch.cuda.synchronize()
        e0.record()
        train_batch.prepare_batch(data)
        m(data)
        train_gt.fine_supervision(data, otg.config())
        crit(data)
        m.zero_grad(set_to_none=True)
        data["loss"].backward()
        e1.record()
        torch.cuda.synchronize()
        if k >= warmup:
            ms.append(e0.elapsed_time(e1))
    out["train_step_ms"] = round(float(np.median(ms)), 2)
    out["prepare_share_of_step"] = round(out["prepare_batch_ms"] / out["train_step_ms"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--items", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    res = {}
    if a.cpu:
        res["cpu"] = cpu_probe(a.items)
    if a.gpu:
        res["gpu"] = gpu_probe(a.warmup, a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
