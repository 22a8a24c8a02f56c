"""Drop-in for the first stage of OnePose++'s keypoint-free SfM mapping,
``detector_free_coarse_matching`` (src/KeypointFreeSfM/coarse_match/coarse_match.py:35-215): LoFTR
coarse matches for every covisible pair and the merge of their endpoints into per-image 2D
keypoints, on the device.

The reference matches one pair per forward (the backbone of an image is recomputed for each of its
~2 covis_num pairs and each call writes the [1, S, S] confidence matrix), then merges the
keypoints in Python over dicts of tuples.  Here each image goes through the coarse backbone once,
pairs run in batches through the coarse transformer and the matrix-free dual softmax
(LoFTR_for_OnePose_Plus.coarse_matches_for_pairs), and the merge runs on all pairs at once
(opp_sfm_points.cu).  Results, files and the pair order are the reference's; oracle/sfm_coarse.py
states the merge's rules.

Not built: padding masks and images of different sizes (mapping crops are all one size).  Inputs
the reference would fail on late, or silently get wrong, raise ValueError before any launch.
"""
import os
import os.path as osp
import random

import numpy as np
import torch

from . import ops
from .loftr import LoFTR_for_OnePose_Plus

__all__ = ["cfgs", "default_cfg", "detector_free_coarse_matching", "coarse_match_pairs", "read_pair_list",
           "read_images", "build_matcher", "names_to_pair", "write_outputs"]

cfgs = {
    "data": {"img_resize": None, "df": 8, "shuffle": True},
    "matcher": {"model": {"weight_path": "weight/LoFTR_wsize9.ckpt", "seed": 666}, "pair_name_split": " "},
    "coarse_match_debug": True,
}

# src/KeypointFreeSfM/loftr_for_sfm/utils/loftr_for_onepose_plus_cfg.py, lower-cased
default_cfg = {
    "backbone_type": "ResNetFPN", "resolution": (8, 2), "fine_window_size": 9, "fine_concat_coarse_feat": False,
    "resnetfpn": {"initial_dim": 128, "block_dims": [128, 196, 256]},
    "coarse": {"d_model": 256, "d_ffn": 256, "nhead": 8, "layer_names": ["self", "cross"] * 4,
               "attention": "linear", "temp_bug_fix": False},
    "match_coarse": {"thr": 0.2, "border_rm": 2, "match_type": "dual_softmax", "dsmax_temperature": 0.1,
                     "skh_iters": 3, "skh_init_bin_score": 1.0, "skh_prefilter": True,
                     "train_coarse_percent": 0.4, "train_pad_num_gt_min": 200},
    "fine": {"d_model": 128, "d_ffn": 128, "nhead": 8, "layer_names": ["self", "cross"], "attention": "linear"},
}

PAIR_BATCH = 32


def names_to_pair(name0, name1):
    return "_".join((name0.replace("/", "-"), name1.replace("/", "-")))


def read_pair_list(covis_pairs, shuffle=True):
    """LoftrCoarseDataset's pair list: a list is taken as is, a path is read, its trailing newlines
    dropped and split into lines; then Python's random.shuffle, the call the reference makes."""
    if isinstance(covis_pairs, list):
        pair_list = covis_pairs
    else:
        with open(covis_pairs, "r") as f:
            pair_list = f.read().rstrip("\n").split("\n")
    if shuffle:
        random.shuffle(pair_list)
    return pair_list


def _pair_index(image_lists, pair_list, split):
    """int64 [P, 2] image indices of the pair lines.  ValueError for a line that is not two names, a
    name outside image_lists, a repeated line, or an image no pair names."""
    ids = {}
    for i, name in enumerate(image_lists):
        ids.setdefault(name, i)
    if len(ids) != len(image_lists):
        raise ValueError("image_lists names an image twice")
    out, seen = [], set()
    for line in pair_list:
        names = line.split(split)
        if len(names) != 2:
            raise ValueError(f"pair line {line!r} is not two image names separated by {split!r}")
        for n in names:
            if n not in ids:
                raise ValueError(f"pair {line!r} names {n!r}, which is not in image_lists")
        if line in seen:
            raise ValueError(f"pair {line!r} is listed twice")
        seen.add(line)
        out.append((ids[names[0]], ids[names[1]]))
    idx = np.asarray(out, np.int64).reshape(-1, 2)
    unused = np.setdiff1d(np.arange(len(image_lists)), idx.reshape(-1))
    if len(unused):
        raise ValueError(f"image {image_lists[unused[0]]!r} is in no pair, so it would have no keypoint")
    return idx


def read_images(image_lists, df=8):
    """read_grayscale(path, None, df, ret_scales=True) for every image, kept as uint8 (the kernels fold
    the /255 into conv1): cv2 decode, cv2.resize only when a side is not a multiple of df.  Returns
    (uint8 [N, 1, H, W] host tensor, fp32 [N, 2] scales [h / h_new, w / w_new]).  Images of different
    sizes raise NotImplementedError."""
    import cv2
    frames, scales = [], []
    for path in image_lists:
        image = cv2.imread(str(path), cv2.IMREAD_GRAYSCALE)
        if image is None:
            raise ValueError(f"cannot read image {path!r}")
        h, w = image.shape
        h_new, w_new = h // df * df, w // df * df
        if (h_new, w_new) != (h, w):
            image = cv2.resize(image, (w_new, h_new))
        frames.append(image)
        scales.append([float(h) / float(h_new), float(w) / float(w_new)])
    if len({f.shape for f in frames}) > 1:
        raise NotImplementedError("images of different sizes are not built: mapping crops are all one size")
    return torch.from_numpy(np.stack(frames))[:, None], torch.tensor(scales, dtype=torch.float32)


def build_matcher(args=None, device="cuda"):
    """build_model (coarse_match_worker.py:16-27) without Lightning: seed torch, random and numpy,
    load the checkpoint with the "matcher." prefix stripped, strictly, coarse-only, eval, on device."""
    args = args or cfgs["matcher"]["model"]
    torch.manual_seed(args["seed"])
    random.seed(args["seed"])
    np.random.seed(args["seed"])
    matcher = LoFTR_for_OnePose_Plus(config=default_cfg, enable_fine_matching=False)
    state_dict = torch.load(args["weight_path"], map_location="cpu")["state_dict"]
    state_dict = {k.replace("matcher.", ""): v for k, v in state_dict.items()}
    matcher.load_state_dict(state_dict, strict=True)
    return matcher.eval().to(device)


def _merge(matches, offsets, pair_idx, image_lists):
    """The device merge of all pairs (ops.sfm_points) -> (keypoints, scores, index matches) as the
    reference's dicts; offsets int64 [P + 1] on the host."""
    counts = np.bincount(pair_idx[np.diff(offsets) > 0].reshape(-1), minlength=len(image_lists))
    if (counts == 0).any():
        raise ValueError(f"image {image_lists[int(np.argmin(counts))]!r} has no keypoint: all its pairs are empty")
    dev = matches.device
    kpts, scores, img_off, idx, status = ops.sfm_points(
        matches, torch.from_numpy(offsets).to(dev), torch.from_numpy(pair_idx.astype(np.int32)).to(dev),
        len(image_lists))
    kpts, scores, img_off, idx = kpts.cpu().numpy(), scores.cpu().numpy(), img_off.cpu().numpy(), idx.cpu().numpy()
    if int(status.item()):
        raise RuntimeError("opp_sfm_points_remap: a match endpoint is missing from its image's keypoints")
    keypoints = {n: kpts[img_off[i]:img_off[i + 1]] for i, n in enumerate(image_lists)}
    kp_scores = {n: scores[img_off[i]:img_off[i + 1]] for i, n in enumerate(image_lists)}
    return keypoints, kp_scores, idx


@torch.no_grad()
def coarse_match_pairs(matcher, image_lists, pair_list, pair_batch=PAIR_BATCH, images=None):
    """The core of detector_free_coarse_matching for `pair_list` in its final order.  matcher: a
    loaded LoFTR_for_OnePose_Plus in eval mode on CUDA.  images: (uint8 [N, 1, H, W], fp32 [N, 2])
    as read_images returns them (read from image_lists when None).  Returns (matches
    {"p0 p1": fp32 [M, 5] x0, y0, x1, y1, mconf}, keypoints {name: fp32 [K, 2]}, scores
    {name: fp32 [K]}, index matches {"p0 p1": int64 [M, 2]})."""
    split = cfgs["matcher"]["pair_name_split"]
    pair_idx = _pair_index(list(image_lists), pair_list, split)
    frames, scales = images if images is not None else read_images(image_lists, cfgs["data"]["df"])
    if len(frames) != len(image_lists):
        raise ValueError(f"{len(frames)} images for {len(image_lists)} names")
    dev = next(matcher.parameters()).device
    if dev.type != "cuda" or matcher.training:
        raise RuntimeError("coarse_match_pairs needs the matcher in eval mode on a CUDA device")
    res = matcher.coarse_matches_for_pairs(frames.to(dev), scales, torch.from_numpy(pair_idx), pair_batch)
    offsets = res["offsets"].numpy()
    flat = torch.cat([res["mkpts0_c"], res["mkpts1_c"], res["mconf"][:, None]], 1).contiguous()
    keypoints, scores, idx = _merge(flat, offsets, pair_idx, list(image_lists))
    flat = flat.cpu().numpy()
    matches = {line: flat[offsets[p]:offsets[p + 1]] for p, line in enumerate(pair_list)}
    index_matches = {line: idx[offsets[p]:offsets[p + 1]] for p, line in enumerate(pair_list)}
    return matches, keypoints, scores, index_matches


def write_outputs(feature_out, match_out, raw_out, matches, keypoints, index_matches):
    """The reference's three files: raw_matches.h5 (save_h5, "/" -> "+"), the feature file (per
    image: keypoints, zero descriptors fp64 [256, K], unit scores) and the match file (per
    names_to_pair group: matches, unit matching_scores, matches0)."""
    import h5py
    split = cfgs["matcher"]["pair_name_split"]
    with h5py.File(raw_out, "w") as f:
        for key, v in matches.items():
            f.create_dataset(key.replace("/", "+"), data=v)
    with h5py.File(feature_out, "w") as f:
        for name, kp in keypoints.items():
            grp = f.create_group(name)
            grp.create_dataset("keypoints", data=kp)
            grp.create_dataset("descriptors", data=np.zeros((256, kp.shape[0])))
            grp.create_dataset("scores", data=np.ones((kp.shape[0],)))
    with h5py.File(match_out, "w") as f:
        for key, m in index_matches.items():
            name0, name1 = key.split(split)
            grp = f.create_group(names_to_pair(name0, name1))
            grp.create_dataset("matches", data=m)
            grp.create_dataset("matching_scores", data=np.ones((m.shape[0],)))
            grp.create_dataset("matches0", data=m)


def detector_free_coarse_matching(image_lists, covis_pairs_out, feature_out, match_out, use_ray=False,
                                  verbose=False, matcher=None):
    """coarse_match.detector_free_coarse_matching on the device.  use_ray is accepted and ignored (one
    process drives the GPU).  matcher: a loaded LoFTR_for_OnePose_Plus to use instead of building
    one from cfgs["matcher"]["model"].  Returns (final_keypoints, updated_matches)."""
    image_lists = list(image_lists)
    pair_list = read_pair_list(covis_pairs_out, cfgs["data"]["shuffle"])    # before the seeding, as the reference
    _pair_index(image_lists, pair_list, cfgs["matcher"]["pair_name_split"])
    images = read_images(image_lists, cfgs["data"]["df"])
    base_dir = feature_out.rsplit("/", 1)[0]
    os.makedirs(base_dir, exist_ok=True)
    if matcher is None:
        matcher = build_matcher()
    matches, keypoints, scores, index_matches = coarse_match_pairs(matcher, image_lists, pair_list, images=images)
    if verbose:
        print(f"coarse matching: {len(pair_list)} pairs, {sum(len(m) for m in matches.values())} matches, "
              f"{sum(len(k) for k in keypoints.values())} keypoints")
    write_outputs(feature_out, match_out, osp.join(base_dir, "raw_matches.h5"), matches, keypoints, index_matches)
    return keypoints, index_matches
