"""Stage time of the SfM refinement (2D refinement + feature update) on a synthetic object; prints
one JSON line.

The object: --images uint8 views of 512^2 cropped from one seeded canvas (as sfm_coarse_probe.py),
with the planted checkpoint of workload.planted_loftr, and a seeded reconstruction
(oracle/sfm_refine.py:seeded_reconstruction) of --points tracks of 2 to --max-track images drawn from
a covisible neighbourhood of --window images, --kpts keypoints per image.  Two routes over the same
reconstruction, alternated --runs times, each timed after a warm-up, with the device's peak memory:

  per_pair   the reference's flow: the pair lists built per keypoint (the restatement of
             MatchingPairData.__getitem__), one fine-only LoFTR_for_OnePose_Plus forward with both
             extractions per pair on float / 255 images (the reference's input), its results copied
             to the host, then the per-point aggregation loop (the restatement of
             feature_aggregation_and_update).
  batched    sfm_refine.fine_matcher + sfm_refine.feature_aggregation_and_update: each image's
             backbone once, pairs in batches, the lookups and means on the device.

The feature files live in memory (an h5py stand-in) for both routes.  Both routes' results are
compared: equal ids and keypoints, the largest mkpts1_f and feature differences.  The card's name and
power limit are read in the same call.
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


def object_images(n, size, seed=0):
    g = torch.Generator().manual_seed(seed)
    canvas = torch.rand(size + 256, size + 256, generator=g)
    shifts = torch.randint(0, 32, (n, 2), generator=g) * 8
    return np.stack([(canvas[dy:dy + size, dx:dx + size] * 255).round().to(torch.uint8).numpy()
                     for dy, dx in shifts.tolist()])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=150)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--points", type=int, default=20000)
    ap.add_argument("--kpts", type=int, default=1500)
    ap.add_argument("--max-track", type=int, default=12)
    ap.add_argument("--window", type=int, default=7)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--pair-batch", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sfm_refine_probe needs a CUDA device")
    from oracle import sfm_refine as osr
    from oracle import workload
    from onepose_plus_plus_b200 import LoFTR_for_OnePose_Plus, sfm_refine
    from onepose_plus_plus_b200.sfm_coarse import default_cfg
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    sys.modules["h5py"] = osr.fake_h5py()
    sd, _ = workload.planted_loftr(256, 320, seed=0)
    m = LoFTR_for_OnePose_Plus(default_cfg, enable_fine_matching=True)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    imgs = object_images(args.images, args.size)
    ds, feats = osr.seeded_reconstruction(0, n_images=args.images, n_points=args.points, n_kpts=args.kpts,
                                          h=args.size, w=args.size, max_track=args.max_track, window=args.window,
                                          scale=(1.0 / 0.75, 1.0), images=imgs)
    names = list(feats)
    out = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q, "images": args.images, "size": args.size,
           "pairs": len(ds.all_pairs), "tracks": len(ds.point_cloud_assigned_imgID_kptID),
           "pair_batch": args.pair_batch}

    def per_pair(sub):
        lists = osr.pair_lists(sub)
        res = {}
        for (left, right), (mk0, mk1, idx) in zip(sub.all_pairs, lists):
            a, b = sub[sub.colmapID2frameID_dict[left]], sub[sub.colmapID2frameID_dict[right]]
            d = {"image0": a["image"].cuda(), "image1": b["image"].cuda(), "scale0": a["scale"].cuda(),
                 "scale1": b["scale"].cuda(), "mkpts0_c": torch.from_numpy(mk0).cuda(),
                 "mkpts1_c": torch.from_numpy(mk1).cuda()}
            with torch.no_grad():
                m(d, extract_coarse_feature=True, extract_fine_feature=True)
            h = {k: d[k].cpu().numpy() for k in ("mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts1_f", "scale0", "scale1")}
            h.update({"mkpts0_idx": idx, "feature_c0": d["feat_coarse_b_0"].cpu().numpy(),
                      "feature_c1": d["feat_coarse_b_1"].cpu().numpy(), "feature0": d["feat_ext0"].cpu().numpy(),
                      "feature1": d["feat_ext1"].cpu().numpy()})
            res[f"{left}-{right}"] = h
        if sub is ds:
            return res, osr.aggregate(sub, res, feats)
        return res, None

    def batched(sub):
        res = sfm_refine.fine_matcher({"model": None}, sub, verbose=False, matcher=m, pair_batch=args.pair_batch)
        if sub is not ds:
            return res, None
        osr.FakeH5.store("/probe/feats_coarse.h5", feats)
        sfm_refine.feature_aggregation_and_update(ds, res, "/probe/feats.h5", names, verbose=False)
        return res, (osr.FakeH5.files["/probe/feats_coarse.h5"], osr.FakeH5.files["/probe/feats.h5"])

    warm = osr.Recon(**{**ds.__dict__, "all_pairs": ds.all_pairs[:4]})
    routes = {}
    for run in range(args.runs):
        for name, fn in (("per_pair", per_pair), ("batched", batched)):
            fn(warm)
            m.clear_workspace()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            routes[name] = fn(ds)
            torch.cuda.synchronize()
            out.setdefault(name + "_s", []).append(round(time.perf_counter() - t0, 3))
            out.setdefault(name + "_peak_mib", []).append(round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1))
    (rr, (rc, rf)), (br, (bc, bf)) = routes["per_pair"], routes["batched"]
    out["matches"] = int(sum(len(v["mkpts0_idx"]) for v in br.values()))
    out["same_keypoints_and_ids"] = bool(all(np.array_equal(rr[p][k], br[p][k]) for p in rr
                                             for k in ("mkpts0_c", "mkpts1_c", "mkpts0_idx")))
    out["max_mkpts1_f_diff"] = float(max(np.abs(rr[p]["mkpts1_f"] - br[p]["mkpts1_f"]).max() for p in rr))
    out["max_feature_diff"] = float(max(np.abs(rr[p][k] - br[p][k]).max() for p in rr
                                        for k in ("feature_c0", "feature_c1", "feature0", "feature1")))
    out["max_descriptor_diff"] = float(max(np.abs(a[n]["descriptors"] - b[n]["descriptors"]).max()
                                           for a, b in ((rc, bc), (rf, bf)) for n in names))
    out["speedup"] = round(min(out["per_pair_s"]) / min(out["batched_s"]), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
