"""Bank-set probe: one forward over the frames of K objects (model.set_banks + object_ids) against K
one-object forwards (one model per object with its bank resident, as a caller without bank sets
runs them), eager and with CUDA graphs.  K in {2, 4, 8} objects with N from {3000, 5000, 7000}
points, 1 and 8 frames per object, 512 x 512 planted frames (oracle/workload.py) so the fine stage
sees its usual match count.  Reports ms per frame for both ways and the padding fraction
(K * N_max - sum N_k) / (K * N_max) of the set.  Prints one JSON line with the device name and
power limit.
    python scripts/multi_object_probe.py [iters]"""
import copy
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle, workload  # noqa: E402  (planted workloads)
from onepose_plus_plus_b200 import OnePosePlus_model  # noqa: E402

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
HW = 512
NS = (3000, 5000, 7000)


def power_limit():
    try:   # a query only
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def wall_ms(fn, n, warm=3):
    """Mean wall time of fn() in ms; every forward ends in a host sync (it sizes its outputs)."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


sd = workload.synthetic_state_dict(0)
base = OnePosePlus_model(oracle.DEFAULT_CONFIG)
base.load_state_dict(sd, strict=True)
base = base.eval()
base.conf_matrix_mode = "skip"
objs = []
for k in range(8):
    d, _ = workload.planted_workload(sd, HW, HW, n_points=NS[k % 3], n_planted=2000, batch=1, seed=11 + k,
                                     with_scale=False)
    objs.append(d)
banks = [(o["keypoints3d"].cuda(), o["descriptors3d_db"].cuda(), o["descriptors3d_coarse_db"].cuda()) for o in objs]
singles = []
for k in range(8):
    m = copy.deepcopy(base).cuda()
    m.set_bank(*banks[k])
    singles.append(m)
multi = copy.deepcopy(base).cuda()

rows = []
g = torch.Generator().manual_seed(0)
for K in (2, 4, 8):
    multi.set_banks(banks[:K])
    ns = [banks[k][0].shape[1] for k in range(K)]
    pad = (K * max(ns) - sum(ns)) / (K * max(ns))
    for f in (1, 8):
        oids = [k for k in range(K) for _ in range(f)]
        frames = torch.cat([(objs[o]["query_image"] + 0.01 * torch.randn(1, 1, HW, HW, generator=g)).clamp(0, 1)
                            for o in oids], 0).cuda()
        per_obj = [frames[k * f:(k + 1) * f].contiguous() for k in range(K)]
        oid_dev = torch.tensor(oids, dtype=torch.int32, device="cuda")
        row = {"K": K, "frames_per_object": f, "B": K * f, "N": ns, "padding_fraction": round(pad, 4)}
        # graph mode is the latency mode: the capture of a 64-frame batch (fine stage at its
        # capacity of B * min(N, S) windows, plus the capture pool) does not fit next to nine models
        for graphs in ((False, True) if K * f <= 32 else (False,)):
            multi.enable_cuda_graphs(graphs)
            for m in singles[:K]:
                m.enable_cuda_graphs(graphs)
            matches = {}

            def run_multi():
                d = {"query_image": frames, "object_ids": oid_dev}
                multi(d)
                matches["multi"] = d["b_ids"].numel()

            def run_singles():
                tot = 0
                for k in range(K):
                    d = {"query_image": per_obj[k]}
                    singles[k](d)
                    tot += d["b_ids"].numel()
                matches["single"] = tot

            t_multi = wall_ms(run_multi, iters)
            t_single = wall_ms(run_singles, iters)
            tag = "graphs" if graphs else "eager"
            row[tag] = {"multi_ms_per_frame": round(t_multi / (K * f), 3),
                        "single_ms_per_frame": round(t_single / (K * f), 3),
                        "speedup": round(t_single / t_multi, 3), "matches": [matches["multi"], matches["single"]]}
            multi.enable_cuda_graphs(False)
            for m in singles[:K]:
                m.enable_cuda_graphs(False)
        rows.append(row)
        print(row, file=sys.stderr, flush=True)
        for m in singles + [multi]:     # nine models' workspaces: keep only one row's at a time
            m.clear_workspace()
        torch.cuda.empty_cache()

print(json.dumps({"probe": "multi_object", "device": torch.cuda.get_device_name(),
                  "power_limit_w": power_limit(), "image": [HW, HW], "iters": iters,
                  "precision": base.precision, "conf_matrix_mode": "skip", "rows": rows}))
