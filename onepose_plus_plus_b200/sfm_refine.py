"""Drop-ins for the 2D refinement and the feature update of OnePose++'s keypoint-free SfM
post-optimisation (src/KeypointFreeSfM/post_optimization/post_optimization.py:62-152):
``fine_matcher`` (matcher_model/fine_match.py) and ``feature_aggregation_and_update``
(feature_aggregation.py:10-180), on the device.

The reference runs one LoFTR forward per keyframe pair, so every image's full backbone (1/2
resolution FPN branch included) is recomputed for every pair it takes part in, and it builds the
pair lists and averages the track features in Python loops of ``np.argwhere``.  Here each image goes
through the backbone once (LoFTR_for_OnePose_Plus.fine_matches_for_pairs keeps its fine map and raw
coarse map), the pair lists come from vectorised NumPy, and the (pair, keypoint) lookups, the
gathers and the track means run on the device (opp_sfm_refine.cu).  Arguments, return values and
files are the reference's; oracle/sfm_refine.py states the rules.

Not built: ray (``use_ray`` is ignored: one process drives the GPU), padding masks, images of
different sizes, ``keypoints_update_method`` other than the default and ``aggregation_method`` other
than "avg".  Inputs the reference would fail on late raise ValueError before any launch.
"""
import os.path as osp
import random
from copy import deepcopy

import numpy as np
import torch

from . import ops
from .loftr import LoFTR_for_OnePose_Plus
from .sfm_coarse import default_cfg

__all__ = ["fine_matcher", "feature_aggregation_and_update", "pair_lists", "build_model", "PAIR_BATCH"]

PAIR_BATCH = 32


def build_model(args, device="cuda"):
    """build_model (fine_match_worker.py:11-21) without Lightning: seed random, numpy and torch, load
    the checkpoint with the "matcher." prefix stripped, strictly, with the fine level, eval."""
    random.seed(args["seed"])
    np.random.seed(args["seed"])
    torch.manual_seed(args["seed"])
    matcher = LoFTR_for_OnePose_Plus(config=default_cfg, enable_fine_matching=True)
    state_dict = torch.load(args["weight_path"], map_location="cpu")["state_dict"]
    state_dict = {k.replace("matcher.", ""): v for k, v in state_dict.items()}
    matcher.load_state_dict(state_dict, strict=True)
    return matcher.eval().to(device)


def _first_members(colmap_3ds, point_ids):
    """Sorted keys point << 32 | image of the given points' track members and the point2D index of
    each key's FIRST member (related_index[0] in MatchingPairData.__getitem__)."""
    pts = [colmap_3ds[int(p)] for p in point_ids]
    lens = np.fromiter((len(p.image_ids) for p in pts), np.int64, len(pts))
    img = np.concatenate([np.asarray(p.image_ids, np.int64) for p in pts]) if pts else np.zeros(0, np.int64)
    p2d = np.concatenate([np.asarray(p.point2D_idxs, np.int64) for p in pts]) if pts else np.zeros(0, np.int64)
    key = (np.repeat(np.asarray(point_ids, np.int64), lens) << 32) | img
    ukey, first = np.unique(key, return_index=True)
    return ukey, p2d[first]


def pair_lists(matching_pairs_dataset):
    """MatchingPairData.__getitem__'s coarse matches of every pair, vectorised: (pairs [(left, right)
    colmap ids], mkpts0_c list, mkpts1_c list, mkpts0_idx list) in all_pairs order and, within a pair,
    in the left frame's keypoint order, with the reference's dtypes (the left frame's keypoints, the
    right image's xys, int64 indices).  ValueError for a pair with no shared track or a track whose
    assigned image is not the pair's left image (the reference fails on both)."""
    ds = matching_pairs_dataset
    frames, images = ds.colmap_frame_dict, ds.colmap_images
    assigned = ds.colmap_image_dataset.point_cloud_assigned_imgID_kptID
    lefts = sorted({int(l) for l, _ in ds.all_pairs})
    status = {l: np.asarray(frames[l]["all_kpt_status"]) for l in lefts}
    needed = np.unique(np.concatenate([s[s >= 0] for s in status.values()]).astype(np.int64)) if lefts \
        else np.zeros(0, np.int64)
    ukey, p2d_first = _first_members(ds.colmap_3ds, needed)
    owner = np.asarray([assigned[int(p)][0] for p in needed], np.int64)
    pairs, mk0, mk1, idx0 = [], [], [], []
    for left, right in ds.all_pairs:
        st = status[int(left)]
        valid = st >= 0
        vidx = np.arange(st.shape[0])[valid]
        rel = st[valid].astype(np.int64)
        q = (rel << 32) | int(right)
        pos = np.minimum(np.searchsorted(ukey, q), max(len(ukey) - 1, 0))
        found = ukey[pos] == q if len(ukey) else np.zeros(len(q), bool)
        if not found.any():
            raise ValueError(f"pair ({left}, {right}) shares no track: the reference cannot stack its matches")
        if (owner[np.searchsorted(needed, rel[found])] != int(left)).any():
            raise ValueError(f"pair ({left}, {right}): a track of the left frame is assigned to another image")
        pairs.append((left, right))
        mk0.append(frames[left]["keypoints"][valid][found])
        mk1.append(images[right].xys[p2d_first[pos[found]]])
        idx0.append(vidx[found])
    return pairs, mk0, mk1, idx0


def _read_images(dataset, colmap_ids):
    """colmap_image_dataset[frame_id] once per image -> (uint8 [N, 1, H, W] host, fp32 [N, 2] scales).
    read_grayscale returns the pixels / 255 in fp32; they are returned to uint8 exactly (the kernels
    fold the / 255 into conv1).  ValueError for images of different sizes."""
    frames, scales = [], []
    for cid in colmap_ids:
        item = dataset[dataset.colmapID2frameID_dict[cid]]
        img = torch.as_tensor(item["image"]).reshape(-1, *item["image"].shape[-2:])
        u8 = torch.round(img.float() * 255).clamp_(0, 255).to(torch.uint8)
        if not torch.equal(torch.from_numpy(u8.numpy() / 255.).float(), img.float()):
            raise ValueError(f"image of colmap id {cid} is not an 8-bit grayscale image / 255")
        frames.append(u8)
        scales.append(torch.as_tensor(item["scale"], dtype=torch.float32).reshape(2))
    if len({tuple(f.shape) for f in frames}) > 1:
        raise ValueError("images of different sizes are not built: mapping crops are all one size")
    return torch.stack(frames), torch.stack(scales)


@torch.no_grad()
def fine_matcher(cfgs, matching_pairs_dataset, use_ray=False, verbose=True, matcher=None, pair_batch=PAIR_BATCH):
    """matcher_model/fine_match.py:fine_matcher on the device: returns {"left-right": the 11 arrays of
    matchWorker} for every pair of matching_pairs_dataset.all_pairs.  use_ray is accepted and
    ignored.  matcher: a loaded LoFTR_for_OnePose_Plus to use instead of building one from
    cfgs["model"]."""
    if cfgs.get("extract_feature_method", "fine_match_backbone") != "fine_match_backbone":
        raise NotImplementedError("only extract_feature_method 'fine_match_backbone' exists in the reference")
    ds = matching_pairs_dataset
    pairs, mk0, mk1, idx0 = pair_lists(ds)
    if not pairs:
        return {}
    for side, arrs in (("left keypoints", mk0), ("right xys", mk1)):
        if len({a.dtype for a in arrs}) != 1 or arrs[0].dtype not in (np.float32, np.float64):
            raise ValueError(f"the {side} must all be float32 or all float64")
    cids = sorted({int(c) for p in pairs for c in p})
    slot = {c: i for i, c in enumerate(cids)}
    frames, scales = _read_images(ds.colmap_image_dataset, cids)
    if matcher is None:
        matcher = build_model(cfgs["model"])
    dev = next(matcher.parameters()).device
    if dev.type != "cuda" or matcher.training:
        raise RuntimeError("fine_matcher needs the matcher in eval mode on a CUDA device")
    counts = np.asarray([len(a) for a in mk0], np.int64)
    offsets = np.concatenate([[0], np.cumsum(counts)])
    pair_idx = torch.tensor([[slot[int(l)], slot[int(r)]] for l, r in pairs], dtype=torch.int64)
    m0 = torch.from_numpy(np.concatenate(mk0)).to(dev)
    m1 = torch.from_numpy(np.concatenate(mk1)).to(dev)
    res = matcher.fine_matches_for_pairs(frames.to(dev), scales, pair_idx, m0, m1, torch.from_numpy(offsets),
                                         pair_batch=pair_batch)
    host = {k: res[k].cpu().numpy() for k in ("mkpts1_f", "feat_coarse_b_0", "feat_coarse_b_1", "feat_ext0",
                                              "feat_ext1")}
    m0, m1 = m0.cpu().numpy(), m1.cpu().numpy()
    sc = scales.numpy()
    out = {}
    for p, (left, right) in enumerate(pairs):
        a, b = offsets[p], offsets[p + 1]
        out["-".join([str(left), str(right)])] = {
            "mkpts0_c": m0[a:b], "mkpts1_c": m1[a:b], "mkpts0_f": m0[a:b].copy(), "mkpts1_f": host["mkpts1_f"][a:b],
            "mkpts0_idx": idx0[p], "scale0": sc[slot[int(left)]][None].copy(), "scale1": sc[slot[int(right)]][None].copy(),
            "feature_c0": host["feat_coarse_b_0"][a:b], "feature_c1": host["feat_coarse_b_1"][a:b],
            "feature0": host["feat_ext0"][a:b], "feature1": host["feat_ext1"][a:b]}
    if verbose:
        print(f"fine matching: {len(pairs)} pairs, {int(offsets[-1])} matches, {len(cids)} images")
    return out


def track_members(colmap_image_dataset, fine_match_results_dict):
    """The per-point loop of feature_aggregation_and_update flattened.  Returns a dict of int64 arrays:
    per track t (in point_cloud_assigned_imgID_kptID order) its assigned image / keypoint and member
    range; per member k (the track's other observations, in track order) its image, keypoint, pair
    index into the results dict's order and the query key pair << 32 | assigned keypoint; and the row
    keys pair << 32 | mkpts0_idx of all result rows in order.  ValueError for a track with no other
    image and for a pair missing from the results (the reference asserts on both)."""
    colmap_3ds = colmap_image_dataset.colmap_3ds
    items = list(colmap_image_dataset.point_cloud_assigned_imgID_kptID.items())
    names = list(fine_match_results_dict)
    pk = np.asarray([(int(a) << 32) | int(b) for a, b in (n.split("-") for n in names)], np.int64)
    porder = np.argsort(pk, kind="stable")
    T = len(items)
    a_img = np.fromiter((int(s[0]) for _, s in items), np.int64, T)
    a_kpt = np.fromiter((int(s[1]) for _, s in items), np.int64, T)
    pts = [colmap_3ds[p] for p, _ in items]
    lens = np.fromiter((len(p.image_ids) for p in pts), np.int64, T)
    img = np.concatenate([np.asarray(p.image_ids, np.int64) for p in pts]) if T else np.zeros(0, np.int64)
    kpt = np.concatenate([np.asarray(p.point2D_idxs, np.int64) for p in pts]) if T else np.zeros(0, np.int64)
    t_of = np.repeat(np.arange(T), lens)
    keep = img != a_img[t_of]
    img, kpt, t_of = img[keep], kpt[keep], t_of[keep]
    track_off = np.zeros(T + 1, np.int64)
    np.cumsum(np.bincount(t_of, minlength=T), out=track_off[1:])
    if T and (np.diff(track_off) == 0).any():
        t = int(np.argmax(np.diff(track_off) == 0))
        raise ValueError(f"3D point {items[t][0]} has no observation outside its assigned image")
    want = (a_img[t_of] << 32) | img
    pos = np.minimum(np.searchsorted(pk[porder], want), max(len(pk) - 1, 0))
    ok = pk[porder][pos] == want if len(pk) else np.zeros(len(want), bool)
    if not ok.all():
        k = int(np.argmin(ok))
        raise ValueError(f"pair {a_img[t_of[k]]}-{img[k]} is not in the fine match results")
    pair = porder[pos]
    rows = [np.asarray(fine_match_results_dict[n]["mkpts0_idx"], np.int64) for n in names]
    row_key = np.concatenate([(np.full(len(r), p, np.int64) << 32) | r for p, r in enumerate(rows)]) if rows \
        else np.zeros(0, np.int64)
    return {"a_img": a_img, "a_kpt": a_kpt, "track_off": track_off, "img": img, "kpt": kpt, "t_of": t_of,
            "pair": pair, "query": (pair << 32) | a_kpt[t_of], "row_key": row_key, "names": names}


def _device_means(fine_match_results_dict, tm):
    """The lookup and the aggregation on the device -> (mean_c, mean_f, ref_c, ref_f) host fp32."""
    names = tm["names"]
    cat = lambda k: torch.from_numpy(np.ascontiguousarray(                      # noqa: E731
        np.concatenate([np.asarray(fine_match_results_dict[n][k], np.float32) for n in names]))).cuda()
    row = ops.sfm_refine_lookup(torch.from_numpy(tm["row_key"]).cuda(), torch.from_numpy(tm["query"]).cuda())
    bad = row.min().item() if row.numel() else 0
    if bad < 0:
        k = int(torch.argmin(row).item())
        raise ValueError(f"pair {tm['names'][tm['pair'][k]]}: keypoint {tm['query'][k] & 0xffffffff} is "
                         f"{'missing from' if bad == -1 else 'repeated in'} mkpts0_idx (the reference asserts one row)")
    c0, c1, f0, f1 = cat("feature_c0"), cat("feature_c1"), cat("feature0"), cat("feature1")
    out = ops.sfm_refine_aggregate(c0, c1, f0, f1, row, torch.from_numpy(tm["track_off"]).cuda())
    return tuple(o.cpu().numpy() for o in out)


def apply_updates(feature_dict_coarse, feature_dict_fine, colmap_images, tm, mean_c, mean_f, ref_c, ref_f):
    """Writes the aggregation into the two feature dicts as the reference's per-point loop leaves them:
    descriptors re-zeroed (fp64 [dim, K]) where the loaded dimension differs, at the first touch of
    an image (the fine keypoint count is the COLMAP one after the first point); the reference sides'
    rows and the track means written in loop order, the last write of a column winning; the assigned
    keypoints' scores zeroed; the fine keypoints replaced by the COLMAP xys (after any point)."""
    T = len(tm["a_img"])
    if T == 0:
        return
    name_of = {}

    def name(cid):
        if cid not in name_of:
            name_of[cid] = colmap_images[int(cid)].name
        return name_of[cid]

    w_img = np.concatenate([tm["img"], tm["a_img"]])
    w_col = np.concatenate([tm["kpt"], tm["a_kpt"]])
    w_t = np.concatenate([tm["t_of"], np.arange(T)])
    w_type = np.concatenate([np.zeros(len(tm["img"]), np.int64), np.ones(T, np.int64)])
    order = np.lexsort((np.arange(len(w_img)), w_type, w_t))
    w_img, w_col, w_t = w_img[order], w_col[order], w_t[order]
    vals_c, vals_f = np.concatenate([ref_c, mean_c])[order], np.concatenate([ref_f, mean_f])[order]
    first_t = {}
    for cid, t in zip(*np.unique(w_img, return_index=True)):
        first_t[int(cid)] = int(w_t[t])
    xys_count = {int(i): im.xys.shape[0] for i, im in colmap_images.items()}
    dc, df = vals_c.shape[1], vals_f.shape[1]
    for cid, t0 in first_t.items():
        n = name(cid)
        if feature_dict_coarse[n]["descriptors"].shape[0] != dc:
            feature_dict_coarse[n]["descriptors"] = np.zeros((dc, feature_dict_coarse[n]["keypoints"].shape[0]))
        if feature_dict_fine[n]["descriptors"].shape[0] != df:
            nk = feature_dict_fine[n]["keypoints"].shape[0] if t0 == 0 else xys_count[cid]
            feature_dict_fine[n]["descriptors"] = np.zeros((df, nk))
    key = (w_img << 32) | w_col
    rev = len(key) - 1 - np.unique(key[::-1], return_index=True)[1]       # the last write of each column
    last = np.sort(rev)
    for cid in np.unique(w_img[last]):
        sel = last[w_img[last] == cid]
        n = name(int(cid))
        feature_dict_coarse[n]["descriptors"][:, w_col[sel]] = vals_c[sel].T
        feature_dict_fine[n]["descriptors"][:, w_col[sel]] = vals_f[sel].T
    for cid in np.unique(tm["a_img"]):
        n = name(int(cid))
        cols = tm["a_kpt"][tm["a_img"] == cid]
        feature_dict_coarse[n]["scores"][cols] = 0
        feature_dict_fine[n]["scores"][cols] = 0
    for _, im in colmap_images.items():
        feature_dict_fine[im.name]["keypoints"] = im.xys


def _feature_load(path, names):
    import h5py
    with h5py.File(path, "r") as f:
        return {n: {k: v.__array__() for k, v in f[n].items()} for n in names}


def _feature_save(feature_dict, path):
    import h5py
    with h5py.File(path, "w") as f:
        for key, value in feature_dict.items():
            grp = f.create_group(key)
            for k, v in value.items():
                grp.create_dataset(k, data=v)


def feature_aggregation_and_update(colmap_image_dataset, fine_match_results_dict, feature_out_pth, image_lists,
                                   keypoints_update_method="colmap_updated_keypoints", aggregation_method="avg",
                                   verbose=True):
    """feature_aggregation.py:feature_aggregation_and_update on the device: reads
    <feature_out_pth stem>_coarse<ext>, writes it back with the reference images' coarse features and
    the tracks' mean coarse features, and writes feature_out_pth with the fine ones and the COLMAP
    keypoints."""
    if aggregation_method != "avg":
        raise NotImplementedError(f"aggregation_method {aggregation_method!r} (the reference builds 'avg' only)")
    if keypoints_update_method != "colmap_updated_keypoints":
        raise NotImplementedError("only keypoints_update_method 'colmap_updated_keypoints' is built")
    stem, ext = osp.splitext(feature_out_pth)
    coarse_path = stem + "_coarse" + ext
    feature_dict_coarse = _feature_load(coarse_path, image_lists)
    feature_dict_fine = deepcopy(feature_dict_coarse)
    tm = track_members(colmap_image_dataset, fine_match_results_dict)
    if len(tm["a_img"]):
        mean_c, mean_f, ref_c, ref_f = _device_means(fine_match_results_dict, tm)
        apply_updates(feature_dict_coarse, feature_dict_fine, colmap_image_dataset.colmap_images, tm, mean_c, mean_f,
                      ref_c, ref_f)
    if verbose:
        print(f"feature aggregation: {len(tm['a_img'])} tracks, {len(tm['img'])} observations")
    _feature_save(feature_dict_coarse, coarse_path)
    _feature_save(feature_dict_fine, feature_out_pth)
