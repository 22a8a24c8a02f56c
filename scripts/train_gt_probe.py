"""Ground truth of one training step, dense (conf_matrix_gt int16 [B, L, S] + fine_location_matrix_gt
fp32 [B, L, S, 2]) against sparse (SparseGT), at the training shape (B = 4, L = 7000, S = 4096,
configs/experiment/train.yaml) with ~3000 correspondences per sample:
  h2d:   bytes per step (from the tensors) and the time of that copy from pinned memory,
  chain: statistics -> focal loss -> backward -> fine supervision with the ground truth resident:
         peak of torch.cuda.max_memory_allocated above the inputs (features + ground truth) and ms per step,
  alone: opp_gt_index and opp_fine_supervision.
The two forms alternate in one process after warm-up; times are CUDA events around work that ends in
a synchronise.  Prints one JSON line with the device name and its power limit.  Needs a GPU.
    python scripts/train_gt_probe.py [steps]"""
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import coarse_loss as cl  # noqa: E402
from oracle import train_gt as otg  # noqa: E402
from onepose_plus_plus_b200 import SparseGT, losses, ops, train_gt, train_path  # noqa: E402

if not torch.cuda.is_available():
    sys.exit("train_gt_probe: no CUDA device (there is nothing to measure without one)")
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
B, L, S, N_POS, HC = 4, 7000, 4096, 3000, 64


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


# features with N_POS planted correspondences per sample, one 3D point per cell (as the dataset yields)
g = torch.Generator().manual_seed(1)
a, b = torch.randn(B, L, 256, generator=g), torch.randn(B, S, 256, generator=g)
ids = []
for bi in range(B):
    ri = torch.randperm(L, generator=g)[:N_POS].sort().values
    cj = torch.randperm(S, generator=g)[:N_POS]
    b[bi, cj] = a[bi, ri] + 0.3 * torch.randn(N_POS, 256, generator=g)
    ids.append((torch.full((N_POS,), bi), ri, cj))
a, b = (a * 0.6).cuda(), (b * 0.6).cuda()
gb, gi, gj = (torch.cat(t) for t in zip(*ids))
xy = torch.stack([gj % HC, gj // HC], 1).float() * 8 + torch.rand(len(gj), 2, generator=g) * 8
host_sparse = SparseGT(gb, gi, gj, xy, (B, L, S)).pin_memory()
host_dense = tuple(t.pin_memory() for t in host_sparse.to_dense())
dense_bytes = sum(t.numel() * t.element_size() for t in host_dense)

# (a) host -> device
h2d_dense = timed(lambda: [t.to("cuda", non_blocking=True) for t in host_dense], 3)
h2d_sparse = timed(lambda: host_sparse.to("cuda", non_blocking=True), 3)

dev_sparse = host_sparse.to("cuda")
dev_dense = tuple(t.cuda() for t in host_dense)
pick = torch.randperm(len(gb), generator=g)[:2000]
matches = {"b_ids": gb[pick].cuda(), "i_ids": gi[pick].cuda(), "j_ids": gj[pick].cuda(), "q_hw_c": (HC, HC)}
crit = losses.Loss(cl.LOSS_CONFIG)
cm = types.SimpleNamespace(temperature=cl.TEMPERATURE)
cfg = otg.config()


def step(mode):
    fa, fb = a.detach().requires_grad_(True), b.detach().requires_grad_(True)
    data = dict(matches)
    if mode == "sparse":
        data["gt_sparse"] = dev_sparse
        gt = dev_sparse
    else:
        data["fine_location_matrix_gt"] = dev_dense[1]
        gt = dev_dense[0]
    loss = crit.compute_coarse_loss(train_path.TrainConfHandle(cm, fa, fb, None), gt)
    loss.backward()
    train_gt.fine_supervision(data, cfg)
    return loss.detach(), data["expec_f_gt"]


rows = {m: {} for m in ("dense", "sparse")}
out = {}
for mode in ("dense", "sparse"):
    for _ in range(2):
        out[mode] = step(mode)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step(mode)
    torch.cuda.synchronize()
    rows[mode]["peak_above_inputs_mib"] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
ms = {m: [] for m in rows}
for _ in range(3):                       # alternate the two forms
    for mode in rows:
        ms[mode].append(timed(lambda: step(mode), steps))
for mode in rows:
    rows[mode]["ms_per_step"] = round(min(ms[mode]), 3)
    rows[mode]["ms_per_step_runs"] = [round(x, 3) for x in ms[mode]]
rows["dense"].update(h2d_bytes=dense_bytes, h2d_ms=round(h2d_dense, 3), resident_mib=round(dense_bytes / 2**20, 1))
rows["sparse"].update(h2d_bytes=host_sparse.nbytes(), h2d_ms=round(h2d_sparse, 3),
                      resident_mib=round(host_sparse.nbytes() / 2**20, 3))
same = bool(torch.equal(out["dense"][0], out["sparse"][0]) and torch.equal(out["dense"][1], out["sparse"][1]))
alone = {"gt_index_ms": round(timed(lambda: ops.gt_index(dev_sparse.b_ids, dev_sparse.i_ids, dev_sparse.j_ids,
                                                         dev_sparse.shape), 50), 4),
         "fine_supervision_ms": round(timed(lambda: train_gt.fine_supervision(
             {**matches, "gt_sparse": dev_sparse}, cfg), 50), 4)}
print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit_w": power_limit(), "B": B, "L": L, "S": S,
                  "positives": len(gb), "matches": len(pick), "steps": steps, "same_loss_and_expec_f_gt_bits": same,
                  "loss": out["sparse"][0].item(), **rows, **alone}))
