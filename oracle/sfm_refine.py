"""NumPy restatement of the keypoint-free SfM refinement's bookkeeping and sampling
(onepose_plus_plus_b200/sfm_refine.py, loftr.py's fine-only branch, opp_sfm_refine.cu), written
after the reference's loops:

  pair_lists     MatchingPairData.__getitem__ (construct_matching_data.py:41-84): per valid left
                 keypoint, the FIRST member of its track in the right image.
  cells          loftr.py:87-109: clip to [0, hw - 2], round(mkpts / (8 * scale[[1, 0]])) half to
                 even, y * wc + x (an x that rounds to wc wraps into the next row).
  sample         sample_feature_from_featuremap: coord_normalization in the keypoints' dtype, then
                 fp32 grid_sample(align_corners=True, zeros): (g + 1) * ((n - 1) / 2), nearest
                 half-to-even or bilinear nw, ne, sw, se summed in that order, one rounding each.
  aggregate      feature_aggregation_and_update's per-point loop with a dict instead of argwhere.
  seeded_reconstruction  a synthetic COLMAP-like reconstruction with the attributes the stage reads.
"""
from copy import deepcopy
from types import SimpleNamespace

import numpy as np
import torch


# the end-to-end case of tests/golden/reference/sfm_refine.npz (oracle/make_sfm_refine_golden.py)
E2E_RECON = dict(seed=5, n_images=4, n_points=10, n_kpts=24, max_track=4, scale=(1.0 / 0.75, 1.0))


class Recon(SimpleNamespace):
    """The stub reconstruction: CoarseReconDataset's attributes; indexing by frame id gives
    read_grayscale's item (pixels / 255 in fp32 [1, 1, H, W], scale fp32 [1, 2]) when images are set."""

    def __getitem__(self, i):
        cid = [c for c, f in self.colmapID2frameID_dict.items() if f == i][0]
        return {"image": torch.from_numpy(self.images[i] / 255.).float()[None, None],
                "scale": torch.tensor([list(self.scale)], dtype=torch.float32),
                "img_path": self.colmap_images[cid].name}


class FakeH5:
    """The part of h5py.File the feature readers and writers use; files live in FakeH5.files."""
    files = {}

    class _Group(dict):
        def create_group(self, name):
            g = self[name] = FakeH5._Group()
            return g

        def create_dataset(self, name, data):
            self[name] = np.array(data)

    class _Dataset:
        def __init__(self, a):
            self.a = a

        def __array__(self, *args, **kwargs):
            return self.a.copy()

    class _Reader:
        def __init__(self, root):
            self.root = root

        def __getitem__(self, name):
            return {k: FakeH5._Dataset(v) for k, v in self.root[name].items()}

    def __init__(self, path, mode):
        if mode == "w":
            self.root = FakeH5.files[path] = FakeH5._Group()
            self.view = self.root
        else:
            self.view = FakeH5._Reader(FakeH5.files[path])

    def __enter__(self):
        return self.view

    def __exit__(self, *a):
        return False

    @staticmethod
    def store(path, feature_dict):
        root = FakeH5.files[path] = FakeH5._Group()
        for n, d in feature_dict.items():
            g = root.create_group(n)
            for k, v in d.items():
                g.create_dataset(k, v)


def fake_h5py():
    return SimpleNamespace(File=FakeH5)


def pair_lists(ds):
    frames, images = ds.colmap_frame_dict, ds.colmap_images
    out = []
    for left, right in ds.all_pairs:
        st = frames[left]["all_kpt_status"]
        mk0, mk1, idx = [], [], []
        for i in range(st.shape[0]):
            if st[i] < 0:
                continue
            p = ds.colmap_3ds[int(st[i])]
            hit = [k for k, im in enumerate(p.image_ids) if im == right]
            if hit:
                mk0.append(frames[left]["keypoints"][i])
                mk1.append(images[right].xys[p.point2D_idxs[hit[0]]])
                idx.append(i)
        out.append((np.stack(mk0), np.stack(mk1), np.asarray(idx, np.int64)))
    return out


def cells(mk, h, w, hc, wc, scale=None):
    """-> (clipped copy of mk, int64 cell ids).  scale: the image's (h, w) scale, fp32 [2], or None."""
    mk = mk.copy()
    mk[:, 0] = np.clip(mk[:, 0], 0, w - 2)
    mk[:, 1] = np.clip(mk[:, 1], 0, h - 2)
    s = h / hc
    div = (np.float32(s) * np.asarray(scale, np.float32)[[1, 0]]).astype(np.float32) if scale is not None else s
    r = np.round(mk / div)
    return mk, (r[:, 1] * wc + r[:, 0]).astype(np.int64)


def _normalise(k, size):
    t = k.dtype.type
    r = t(np.float32(size) - np.float32(1))
    v = (k - t(0.5)) + t(0.5)
    v = v / r
    return (v * t(2) - t(1)).astype(np.float32)


def sample(fmap, kpts, imghw, nearest):
    """fmap fp32 [C, H, W]; kpts [n, 2] fp32 or fp64; imghw fp32 (h, w).  -> fp32 [n, C]."""
    C, H, W = fmap.shape
    f32 = np.float32
    gx, gy = _normalise(kpts[:, 0], imghw[1]), _normalise(kpts[:, 1], imghw[0])
    ix = (gx + f32(1)) * f32((W - 1) / 2)
    iy = (gy + f32(1)) * f32((H - 1) / 2)
    n = len(kpts)
    out = np.zeros((n, C), np.float32)

    def tap(y, x):
        ok = (x > -1) & (x < W) & (y > -1) & (y < H)
        v = np.zeros((n, C), np.float32)
        v[ok] = fmap[:, y[ok].astype(np.int64), x[ok].astype(np.int64)].T
        return v

    with np.errstate(invalid="ignore"):
        if nearest:
            xr, yr = np.rint(ix), np.rint(iy)
            return tap(yr, xr)
        xw, yn = np.floor(ix), np.floor(iy)
        w = ix - xw
        e = f32(1) - w
        nn = iy - yn
        s = f32(1) - nn
        wnw, wne, wsw, wse = (s * e)[:, None], (s * w)[:, None], (nn * e)[:, None], (nn * w)[:, None]
        out = tap(yn, xw) * wnw + tap(yn, xw + 1) * wne
        out = out + tap(yn + 1, xw) * wsw
        return out + tap(yn + 1, xw + 1) * wse


def aggregate(colmap_image_dataset, results, feature_dict_coarse):
    """-> (coarse, fine) feature dicts as feature_aggregation_and_update leaves them (default method)."""
    coarse = deepcopy(feature_dict_coarse)
    fine = deepcopy(coarse)
    c3, ims = colmap_image_dataset.colmap_3ds, colmap_image_dataset.colmap_images
    row = {name: {int(k): i for i, k in enumerate(r["mkpts0_idx"])} for name, r in results.items()}
    for t, (pid, (a, q)) in enumerate(colmap_image_dataset.point_cloud_assigned_imgID_kptID.items()):
        fc, ff = [], []
        ln = ims[int(a)].name
        for im, kp in zip(c3[pid].image_ids.tolist(), c3[pid].point2D_idxs.tolist()):
            if im == a:
                continue
            r = results[f"{a}-{im}"]
            i = row[f"{a}-{im}"][q]
            fc.append(r["feature_c0"][i])
            ff.append(r["feature0"][i])
            rn = ims[int(im)].name
            for d, f in ((coarse, r["feature_c1"][i]), (fine, r["feature1"][i])):
                if d[rn]["descriptors"].shape[0] != f.shape[0]:
                    d[rn]["descriptors"] = np.zeros((f.shape[0], d[rn]["keypoints"].shape[0]))
                d[rn]["descriptors"][:, kp] = f
        for d, fs in ((coarse, fc), (fine, ff)):
            if d[ln]["descriptors"].shape[0] != fs[0].shape[0]:
                d[ln]["descriptors"] = np.zeros((fs[0].shape[0], d[ln]["keypoints"].shape[0]))
            acc = fs[0].copy()
            for f in fs[1:]:
                acc = acc + f
            d[ln]["descriptors"][:, q] = acc / np.float32(len(fs))
            d[ln]["scores"][q] = 0
        for im in ims.values():
            fine[im.name]["keypoints"] = im.xys
    return coarse, fine


def seeded_reconstruction(seed, n_images=8, n_points=60, n_kpts=80, h=96, w=128, max_track=12, scale=(1.0, 1.0),
                          left_f32=True, images=None, window=None):
    """A synthetic reconstruction: stub dataset with colmap_frame_dict, colmap_3ds, colmap_images,
    point_cloud_assigned_imgID_kptID, colmapID2frameID_dict and all_pairs.  Every 2D point is in at most
    one track except that the first track holds its second image twice; keypoints are planted on the
    clip edge, at .5 cell positions and at the wc wrap.  Colmap ids are 1-based and not contiguous
    with the frame ids.  Returns (dataset stub, {image name: feature dict of the coarse stage})."""
    pixels = images
    rng = np.random.default_rng(seed)
    cids = [3 * i + 1 for i in range(n_images)]
    xys = {c: np.stack([rng.uniform(0, w - 1, n_kpts), rng.uniform(0, h - 1, n_kpts)], 1) for c in cids}
    special = np.array([[w - 2, h - 2], [w - 1.0, 0.0], [4.0 * 1.0, 12.0], [12.0, 20.0], [w - 4.0, 5.0],
                        [w - 3.999, 9.5], [0.0, 0.0], [-0.5, h + 3.0]])
    for c in cids:
        xys[c][:len(special)] = special
    free = {c: list(rng.permutation(n_kpts)) for c in cids}
    status = {c: np.full(n_kpts, -1, np.int64) for c in cids}
    c3, assigned = {}, {}
    lengths = rng.integers(2, max_track + 1, n_points)
    lengths[0] = max(lengths[0], 3)
    for p in range(n_points):
        pid = 10 + 2 * p
        L = int(min(lengths[p], n_images))
        if window:      # covisible neighbourhood: the track's images within `window` of a random start
            start = int(rng.integers(n_images))
            L = min(L, window)
            imgs = [cids[(start + i) % n_images] for i in rng.choice(window, L, replace=False)]
        else:
            imgs = [cids[i] for i in rng.choice(n_images, L, replace=False)]
        imgs = [c for c in imgs if free[c]]
        if len(imgs) < 2:
            continue
        kp = [int(free[c].pop()) for c in imgs]
        if p == 0 and free[imgs[1]]:          # the right image twice in one track
            imgs.insert(2, imgs[1])
            kp.insert(2, int(free[imgs[1]].pop()))
        c3[pid] = SimpleNamespace(image_ids=np.asarray(imgs, np.int64), point2D_idxs=np.asarray(kp, np.int64))
        assigned[pid] = (imgs[0], kp[0])
        status[imgs[0]][kp[0]] = pid
    images = {c: SimpleNamespace(name=f"img/{c}.png", xys=xys[c]) for c in cids}
    frame_dict = {}
    for c in cids:
        related = sorted({int(i) for pid, (a, _) in assigned.items() if a == c for i in c3[pid].image_ids if i != c})
        kps = xys[c].astype(np.float32) if left_f32 else xys[c].copy()
        frame_dict[c] = {"is_keyframe": bool(related), "related_frameID": related, "keypoints": kps,
                         "all_kpt_status": status[c]}
    all_pairs = [[c, r] for c in cids if frame_dict[c]["is_keyframe"] for r in frame_dict[c]["related_frameID"]]
    ds = Recon(colmap_frame_dict=frame_dict, colmap_cameras={}, colmap_3ds=c3, colmap_images=images, all_pairs=all_pairs,
                         point_cloud_assigned_imgID_kptID=assigned,
                         colmapID2frameID_dict={c: i for i, c in enumerate(cids)}, scale=tuple(scale),
                         images=pixels)
    ds.colmap_image_dataset = ds
    feats = {im.name: {"descriptors": np.zeros((256, n_kpts)), "keypoints": xys[c].astype(np.float32),
                       "scores": np.ones(n_kpts)} for c, im in images.items()}
    return ds, feats


def synthetic_results(ds, seed, dc=256, df=128):
    """Fine match results with random features over the pair lists of ds (for the aggregation)."""
    rng = np.random.default_rng(seed)
    out = {}
    for (left, right), (mk0, mk1, idx) in zip(ds.all_pairs, pair_lists(ds)):
        m = len(idx)
        out[f"{left}-{right}"] = {"mkpts0_idx": idx, **{k: rng.standard_normal((m, d)).astype(np.float32) for k, d in
                                  (("feature_c0", dc), ("feature_c1", dc), ("feature0", df), ("feature1", df))}}
    return out
