"""Stage time of the SfM coarse matching on a synthetic object; prints one JSON line.

The object: --images uint8 views of 512^2 cropped from one seeded canvas at random 8-px shifts
(planted translations), each image paired with its next --covis images (about images x covis pairs),
and the planted checkpoint of workload.planted_loftr.  Two routes over the same pairs and the same
pair order, each timed once after a warm-up on a few pairs, with the device's peak memory:

  per_pair   the reference's flow: one LoFTR_for_OnePose_Plus(enable_fine_matching=False) forward per
             pair on images sent as float /255 (the reference's input), its matches copied to the
             host, then the merge restated in NumPy (oracle/sfm_coarse.py).
  batched    sfm_coarse.coarse_match_pairs: each image's coarse backbone once, pairs in batches,
             the merge on the device.

Both routes' outputs are compared: the coarse coordinates, the largest mconf difference, and the
keypoints (ids can swap where two scores differ in the last bits, so the sets are compared too).
The card's name and power limit are read in the same call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def synthetic_object(n, size, covis, seed=0):
    g = torch.Generator().manual_seed(seed)
    canvas = torch.rand(size + 256, size + 256, generator=g)
    shifts = torch.randint(0, 32, (n, 2), generator=g) * 8
    imgs = torch.stack([(canvas[dy:dy + size, dx:dx + size] * 255).round().to(torch.uint8)
                        for dy, dx in shifts.tolist()])[:, None]
    names = [f"obj/{i:04d}.png" for i in range(n)]
    pairs = [f"{names[i]} {names[(i + k) % n]}" for i in range(n) for k in range(1, covis + 1)]
    return imgs, names, pairs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=150)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--covis", type=int, default=10)
    ap.add_argument("--pair-batch", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sfm_coarse_probe needs a CUDA device")
    from oracle import sfm_coarse as osc
    from oracle import workload
    from onepose_plus_plus_b200 import LoFTR_for_OnePose_Plus, sfm_coarse
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q, "images": args.images, "size": args.size,
           "covis": args.covis, "pair_batch": args.pair_batch}
    sd, _ = workload.planted_loftr(256, 320, seed=0)
    m = LoFTR_for_OnePose_Plus(sfm_coarse.default_cfg, enable_fine_matching=False)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    imgs, names, pairs = synthetic_object(args.images, args.size, args.covis)
    scales = torch.ones(args.images, 2)
    out["pairs"] = len(pairs)
    ids = {n: i for i, n in enumerate(names)}

    def per_pair(plist):
        matches = {}
        for p in plist:
            a, b = (ids[x] for x in p.split(" "))
            d = {"image0": (imgs[a:a + 1].float() / 255).cuda(), "image1": (imgs[b:b + 1].float() / 255).cuda(),
                 "scale0": scales[a:a + 1].cuda(), "scale1": scales[b:b + 1].cuda()}
            with torch.no_grad():
                m(d)
            matches[p] = np.concatenate([d["mkpts0_f"].cpu().numpy(), d["mkpts1_f"].cpu().numpy(),
                                         d["mconf"].cpu().numpy()[:, None]], -1)
        return matches, osc.merge(matches, names) if len(plist) == len(pairs) else None

    def batched(plist):
        used = sorted({i for p in plist for i in (ids[x] for x in p.split(" "))})
        sub = [names[i] for i in used]
        return sfm_coarse.coarse_match_pairs(m, sub, plist, args.pair_batch,
                                             images=(imgs[used], scales[used]))

    warm = [p for p in pairs if p.split(" ")[0] in names[:4]][:8]
    routes = {}
    for name, fn in (("per_pair", per_pair), ("batched", batched)):
        fn(warm)
        m.clear_workspace()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        res = fn(pairs)
        torch.cuda.synchronize()
        out[name + "_s"] = round(time.perf_counter() - t0, 3)
        out[name + "_peak_mib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        routes[name] = res
    rm, (rk, rs, ri) = routes["per_pair"]
    bm, bk, bs, bi = routes["batched"]
    same = all(np.array_equal(rm[p][:, :4], bm[p][:, :4]) for p in pairs)
    out["matches"] = int(sum(len(v) for v in bm.values()))
    out["keypoints"] = int(sum(len(v) for v in bk.values()))
    out["same_coarse_matches"] = bool(same)
    out["max_mconf_diff"] = float(max((np.abs(rm[p][:, 4] - bm[p][:, 4]).max() for p in pairs if len(bm[p])),
                                      default=0.0)) if same else None
    out["same_keypoints"] = bool(same and all(np.array_equal(rk[n], bk[n]) for n in names))
    out["same_keypoint_sets"] = bool(same and all(np.array_equal(np.unique(rk[n], axis=0), np.unique(bk[n], axis=0))
                                                  for n in names))
    out["speedup"] = round(out["per_pair_s"] / out["batched_s"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
