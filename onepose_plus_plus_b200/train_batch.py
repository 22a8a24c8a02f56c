"""Training batches with the ground truth built on the device: the homography augmentation of the
query image and the correspondences projected from the pose, which the reference dataset computes
per item in the loader workers (OnePosePlusDataset.read_anno, src/datasets/OnePosePlus_dataset.py:
341-444, build_assignmatrix :174-236) before writing them into two dense [shape3d, h_c * w_c]
tensors (57 MB + 229 MB per item at shape3d 7000, 512²).

  * ProjectedGTDataset wraps a OnePosePlusDataset.  Its train items stop before the projection: they
    carry the unwarped query_image and, in item["gt_source"], what the projection needs — the
    correspondences (after the 3D padding's remap), the pose, K_crop and the sampled homography.
  * collate joins the items (torch's default collation, gt_source joined with per-item offsets).
  * prepare_batch, the first line of training_step after the device transfer, warps the images of
    the items with a homography, sets their query_intrinsic to H @ K and writes batch["gt_sparse"],
    the SparseGT (train_gt.py) that SparseGT.from_dense gives on the reference's collated dense
    tensors.  CUDA batches run opp_homography_warp_f32 / opp_train_gt_build / opp_train_gt_compact
    (one host synchronisation, for the list length); CPU batches run the same fp32 steps in torch.

The arithmetic is fp32 with one rounding per operation in the order of opp_train_batch.cu.  The
reference multiplies its 3x3 matrices with BLAS, so its projected coordinates can differ from these
in the last bits; the rounding, the filters, the tie rules and the cell arithmetic are the
reference's elementwise operations and agree exactly on the same coordinates.  The 3x3 algebra of
the homography (normalize_homography, its inverse, normal_transform_pixel and N^-1 . Hn) runs on
the host per item with the reference's calls and dtypes.
"""
import sys

import numpy as np
import torch

from .train_gt import SparseGT

COARSE_STRIDE = 8          # int(1 / coarse_scale) at the training config's coarse_scale 0.125
PACK = 44                  # floats per item of the kernels' parameter pack (opp_train_batch.cu)
_ERR_CELL, _ERR_2D, _ERR_3D = 1, 2, 4


# ---- kornia 0.4.1 (kornia.geometry.conversions / transform), the three calls of :359-385 --------

def normal_transform_pixel(height, width):
    """fp32 [1, 3, 3]: pixel -> [-1, 1] coordinates (kornia normal_transform_pixel)."""
    tr = torch.tensor([[1.0, 0.0, -1.0], [0.0, 1.0, -1.0], [0.0, 0.0, 1.0]])
    tr[0, 0] = tr[0, 0] * 2.0 / (width - 1.0)
    tr[1, 1] = tr[1, 1] * 2.0 / (height - 1.0)
    return tr.unsqueeze(0)


def normalize_homography(dst_pix_trans_src_pix, dsize_src, dsize_dst):
    """[B, 3, 3] pixel homography -> the same map in normalised coordinates (kornia normalize_homography)."""
    (src_h, src_w), (dst_h, dst_w) = dsize_src, dsize_dst
    src_norm_trans_src_pix = normal_transform_pixel(src_h, src_w).to(dst_pix_trans_src_pix)
    src_pix_trans_src_norm = torch.inverse(src_norm_trans_src_pix)
    dst_norm_trans_dst_pix = normal_transform_pixel(dst_h, dst_w).to(dst_pix_trans_src_pix)
    return dst_norm_trans_dst_pix @ (dst_pix_trans_src_pix @ src_pix_trans_src_norm)


# ---- worker side ---------------------------------------------------------------------------------

class ProjectedGTDataset(torch.utils.data.Dataset):
    """Wraps a OnePosePlusDataset.  A train item is the reference item without conf_matrix_gt and
    fine_location_matrix_gt, with the unwarped query_image and query_intrinsic = K_crop, plus
    item["gt_source"]: assign int64 [2, k] (2D keypoint, 3D point after the padding's remap),
    n_2d, K_crop fp64 [3, 3], pose_gt fp64 [4, 4] and homography (the sampled fp64 [3, 3], or None).
    It makes the reference's file reads and RNG draws in the same order (torch in read_anno3d's
    padding, then np.random in sample_homography_sap).  Items of other splits pass through."""

    def __init__(self, dataset):
        self.dataset = dataset

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, index):
        ds = self.dataset
        if ds.split != "train":
            return ds[index]
        # __getitem__ :448-455
        if ds.image_warp_adapt:
            return self._read(ds.anns[index // 2], (index % 2) != 0)
        return self._read(ds.anns[index], False)

    def _read(self, img_id, image_warp_adapt):
        ds = self.dataset
        mod = sys.modules[type(ds).__module__]
        if not ds.load_pose_gt:
            raise ValueError("ProjectedGTDataset: the train split projects with the pose; set load_pose_gt")
        if abs(ds.coarse_scale * COARSE_STRIDE - 1.0) > 0:
            raise ValueError(f"ProjectedGTDataset: coarse_scale must be 1/{COARSE_STRIDE}, got {ds.coarse_scale}")
        # read_anno :255-268
        anno = ds.coco.loadAnns(ds.coco.getAnnIds(imgIds=img_id))[0]
        color_path = ds.coco.loadImgs(int(img_id))[0]["img_file"]
        query_img, query_img_scale, query_img_mask = mod.read_grayscale(
            color_path, resize=ds.img_resize, pad_to=ds.img_resize if ds.img_pad else None, ret_scales=True,
            ret_pad_mask=True, df=ds.df, augmentor=ds.augmentor)
        data = {}
        if query_img_mask is not None:                                         # :282-283
            data["query_image_mask"] = query_img_mask
        K_crop = ds.get_intrin_by_color_pth(color_path)                        # :285-289
        pose_gt = ds.get_gt_pose_by_color_pth(color_path)
        data.update({"query_intrinsic": K_crop, "query_pose_gt": pose_gt})
        # :292-303: the coarse 2D annotation
        anno2d_coarse_file = anno["anno2d_file"].replace("/anno_loftr/", "/anno_loftr_coarse/")
        keypoints2d_coarse, _, assign_matrix, _ = ds.read_anno2d(anno2d_coarse_file)
        n_2d = keypoints2d_coarse.shape[0]
        am = assign_matrix.long()
        if am.numel() and bool((am[0] < 0).any() | (am[0] >= n_2d).any()):
            raise ValueError(f"{anno2d_coarse_file}: assign_matrix[0] outside the {n_2d} 2D keypoints")
        n_3d = np.load(anno["avg_anno3d_file"])["keypoints3d"].shape[0]
        if am.numel() and bool((am[1] < 0).any() | (am[1] >= n_3d).any()):
            raise ValueError(f"{anno2d_coarse_file}: assign_matrix[1] outside the {n_3d} 3D points")
        # :308-321: read and pad the 3D points (the torch RNG draws of the padding)
        keypoints3d, desc3d, desc3d_coarse, scores3d, assign_matrix = ds.read_anno3d(
            anno["avg_anno3d_file"], pad=ds.pad, assignmatrix=assign_matrix, load_3d_coarse=ds.load_3d_coarse)
        data.update({"keypoints3d": keypoints3d, "descriptors3d_db": desc3d, "scores3d_db": scores3d.squeeze(1),
                     "query_image": query_img, "query_image_scale": query_img_scale,
                     "query_image_path": color_path})                          # :323-332
        if desc3d_coarse is not None:                                          # :334-339
            data["descriptors3d_coarse_db"] = desc3d_coarse
        assign = assign_matrix.long()                                          # :342
        if assign.numel() and bool((assign[1] >= keypoints3d.shape[0]).any()):
            raise ValueError("assign_matrix[1] outside the padded 3D points")
        # :357-358: the homography draw (np.random); the warp itself runs in prepare_batch
        homography = None
        if image_warp_adapt:
            homography = torch.from_numpy(np.asarray(mod.sample_homography_sap(query_img.shape[1],
                                                                               query_img.shape[2])))
        data["gt_source"] = {"assign": assign.contiguous(), "n_2d": int(n_2d), "K_crop": K_crop,
                             "pose_gt": pose_gt, "homography": homography}
        return data


class GTSource:
    """The gt_source of a batch: assign int64 [2, N] (items joined), offsets int64 [B + 1] (item b
    owns assign[:, offsets[b]:offsets[b + 1]]), kp_offsets int64 [B + 1] (the items' 2D keypoint
    counts n_2d, cumulated), and per item K_crop, pose_gt and homography.  .to() / .pin_memory()
    move the three index tensors; the per-item 3x3 matrices stay on the host, where prepare_batch's
    3x3 algebra reads them."""

    def __init__(self, assign, offsets, kp_offsets, n_kp, K_crop, pose_gt, homography):
        self.assign, self.offsets, self.kp_offsets, self.n_kp = assign, offsets, kp_offsets, int(n_kp)
        self.K_crop, self.pose_gt, self.homography = K_crop, pose_gt, list(homography)

    @classmethod
    def collate(cls, sources):
        counts = torch.tensor([0] + [s["assign"].shape[1] for s in sources], dtype=torch.int64)
        n_2d = torch.tensor([0] + [int(s["n_2d"]) for s in sources], dtype=torch.int64)
        assign = torch.cat([s["assign"].long().reshape(2, -1) for s in sources], 1)
        return cls(assign, counts.cumsum(0), n_2d.cumsum(0), int(n_2d.sum()),
                   torch.stack([s["K_crop"] for s in sources]), torch.stack([s["pose_gt"] for s in sources]),
                   [s["homography"] for s in sources])

    def __len__(self):
        return len(self.homography)

    def _map(self, fn):
        return GTSource(*(fn(t) for t in (self.assign, self.offsets, self.kp_offsets)), self.n_kp, self.K_crop,
                        self.pose_gt, self.homography)

    def to(self, device, non_blocking=False):
        return self._map(lambda t: t.to(device, non_blocking=non_blocking))

    def pin_memory(self):
        return self._map(lambda t: t.pin_memory())

    @property
    def device(self):
        return self.assign.device


def collate(items):
    """collate_fn of a DataLoader over ProjectedGTDataset: torch's default collation, with the
    gt_source items joined into a GTSource."""
    from torch.utils.data import default_collate
    sources = [it["gt_source"] for it in items if "gt_source" in it]
    if sources and len(sources) != len(items):
        raise ValueError("collate: some items of the batch have gt_source and some do not")
    batch = default_collate([{k: v for k, v in it.items() if k != "gt_source"} for it in items])
    if sources:
        batch["gt_source"] = GTSource.collate(sources)
    return batch


# ---- after the device transfer -------------------------------------------------------------------

def _pack(src, h, w):
    """fp32 [B, PACK] on the host: R, t, K, M = N^-1 . Hn, N's four entries, A = Hn^-1, warp flag;
    and the per-item H @ K (fp32, None for unwarped items) — :344-346, :359-403."""
    B = len(src)
    pack = torch.zeros(B, PACK, dtype=torch.float32)
    hk = [None] * B
    pose, K = src.pose_gt.cpu(), src.K_crop.cpu()
    for b in range(B):
        Kf = K[b].to(torch.float)
        pack[b, 0:9] = pose[b, :3, :3].to(torch.float).reshape(9)
        pack[b, 9:12] = pose[b, :3, 3].to(torch.float)
        pack[b, 12:21] = Kf.reshape(9)
        H = src.homography[b]
        if H is None:
            continue
        H = torch.as_tensor(H).cpu()
        Hn = normalize_homography(H[None].to(torch.float32), (h, w), (h, w))
        N = normal_transform_pixel(h, w)
        pack[b, 21:30] = (N[0].inverse() @ Hn[0]).reshape(9)
        pack[b, 30:34] = torch.stack([N[0, 0, 0], N[0, 0, 2], N[0, 1, 1], N[0, 1, 2]])
        pack[b, 34:43] = torch.linalg.inv(Hn)[0].reshape(9)
        pack[b, 43] = 1.0
        hk[b] = H.to(torch.float32) @ Kf          # :401-403, FIXME of the reference kept: H @ K
    return pack, hk


def _raise_status(bits):
    if bits & _ERR_2D:
        raise ValueError("prepare_batch: assign[0] outside the item's 2D keypoints")
    if bits & _ERR_3D:
        raise ValueError("prepare_batch: assign[1] outside the 3D points")
    if bits & _ERR_CELL:
        raise ValueError("prepare_batch: a correspondence's coarse cell index is the grid size or negative "
                         "(the reference writes out of bounds there)")


@torch.no_grad()
def prepare_batch(batch):
    """In place, after the device transfer and before the matcher: warp the query images of the
    items with a homography, set their query_intrinsic to H @ K, and replace batch["gt_source"] by
    batch["gt_sparse"] (a SparseGT of shape (B, L, h_c * w_c)).  A batch without gt_source is
    returned unchanged."""
    src = batch.pop("gt_source", None)
    if src is None:
        return batch
    img = batch["query_image"]
    B, _, h, w = img.shape
    if len(src) != B:
        raise ValueError(f"prepare_batch: gt_source has {len(src)} items, query_image {B}")
    kp3d = batch["keypoints3d"]
    L = kp3d.shape[1]
    h_c, w_c = int(h / COARSE_STRIDE), int(w / COARSE_STRIDE)
    S = h_c * w_c
    if S == 0:
        raise ValueError(f"prepare_batch: a {h}x{w} query image has no {COARSE_STRIDE}-px coarse cell")
    pack, hk = _pack(src, h, w)
    dev = img.device
    scale = batch["query_image_scale"].to(torch.float32)
    if any(m is not None for m in hk):
        intr = batch["query_intrinsic"]
        for b, m in enumerate(hk):
            if m is not None:
                intr[b] = m.to(intr.dtype)
    if img.is_cuda:
        from . import ops
        pack_d = pack.to(dev)
        if pack[:, 43].any():
            batch["query_image"] = ops.homography_warp(img.contiguous(), pack_d)
        b_ids, i_ids, j_ids, fine_xy, status = ops.train_gt(
            kp3d.to(torch.float32).contiguous(), src.assign.to(dev).contiguous(), src.offsets.to(dev),
            src.kp_offsets.to(dev), src.n_kp, pack_d, scale.contiguous(), (h, w), w_c, S)
        bits, n = (int(v) for v in status.cpu())
        _raise_status(bits)
        batch["gt_sparse"] = SparseGT(b_ids[:n], i_ids[:n], j_ids[:n], fine_xy[:n], (B, L, S))
        return batch
    if pack[:, 43].any():
        batch["query_image"] = warp_images_torch(img, pack)
    b_ids, i_ids, j_ids, fine_xy = gt_list_torch(kp3d.to(torch.float32), src, pack, scale, (h, w), L, w_c, S)
    batch["gt_sparse"] = SparseGT(b_ids, i_ids, j_ids, fine_xy, (B, L, S))
    return batch


# ---- the same steps in torch (CPU batches) -------------------------------------------------------

def _linspace_pm1(n):
    i = torch.arange(n)
    step = torch.tensor(2.0, dtype=torch.float32) / float(n - 1)
    lo = -1.0 + step * i.float()
    hi = 1.0 - step * (n - 1 - i).float()
    return torch.where(i < n // 2, lo, hi)


def _mad3(a0, x, a1, y, a2, z):
    return (a0 * x + a1 * y) + a2 * z


def warp_images_torch(img, pack):
    """opp_homography_warp_f32 in torch ops: img fp32 [B, 1, h, w]."""
    B, _, h, w = img.shape
    out = img.clone()
    gx, gy = _linspace_pm1(w)[None, :], _linspace_pm1(h)[:, None]
    one = torch.ones((), dtype=torch.float32)
    for b in range(B):
        if pack[b, 43] == 0:
            continue
        A = pack[b, 34:43]
        sx = _mad3(A[0], gx, A[1], gy, A[2], one)
        sy = _mad3(A[3], gx, A[4], gy, A[5], one)
        sz = _mad3(A[6], gx, A[7], gy, A[8], one)
        s = torch.where(sz.abs() > 1e-8, 1.0 / sz, one)
        ix = (s * sx + 1.0) * (0.5 * w) - 0.5
        iy = (s * sy + 1.0) * (0.5 * h) - 0.5
        inside = (ix > -1) & (ix < w) & (iy > -1) & (iy < h)
        fx, fy = torch.floor(ix), torch.floor(iy)
        wx, ny = ix - fx, iy - fy
        ex, sy_ = 1.0 - wx, 1.0 - ny
        x0 = torch.where(inside, fx, -2).long()
        y0 = torch.where(inside, fy, -2).long()
        src = img[b, 0]

        def tap(xx, yy):
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            return torch.where(ok, src[yy.clamp(0, h - 1), xx.clamp(0, w - 1)], 0.0)

        val = ((sy_ * ex) * tap(x0, y0) + (sy_ * wx) * tap(x0 + 1, y0)) + (ny * ex) * tap(x0, y0 + 1)
        val = val + (ny * wx) * tap(x0 + 1, y0 + 1)
        out[b, 0] = torch.where(inside, val, 0.0)
    return out


def gt_list_torch(kp3d, src, pack, img_scale, hw, L, w_c, S):
    """opp_train_gt_build + sort + opp_train_gt_compact in torch ops (CPU)."""
    h, w = hw
    B = kp3d.shape[0]
    ncx, ncy = (w - 1) // COARSE_STRIDE + 1, (h - 1) // COARSE_STRIDE + 1
    ranks = ncx * ncy
    assign, offsets, kp_off = src.assign.cpu(), src.offsets.cpu(), src.kp_offsets.cpu()
    n = assign.shape[1]
    b = torch.repeat_interleave(torch.arange(B), offsets[1:] - offsets[:-1])
    a0, a1 = assign[0], assign[1]
    if bool(((a0 < 0) | (a0 >= (kp_off[1:] - kp_off[:-1])[b])).any()):
        _raise_status(_ERR_2D)
    if bool(((a1 < 0) | (a1 >= L)).any()):
        _raise_status(_ERR_3D)
    p = pack[b]                                               # [n, PACK]
    X = kp3d[b, a1]                                           # [n, 3]
    cam = [_mad3(p[:, 3 * r], X[:, 0], p[:, 3 * r + 1], X[:, 1], p[:, 3 * r + 2], X[:, 2]) + p[:, 9 + r]
           for r in range(3)]
    q = [_mad3(p[:, 12 + 3 * r], cam[0], p[:, 13 + 3 * r], cam[1], p[:, 14 + 3 * r], cam[2]) for r in range(3)]
    zd = q[2] + torch.tensor(1e-6, dtype=torch.float32)
    x, y = q[0] / zd, q[1] / zd
    warped = p[:, 43] != 0
    keep = torch.ones(n, dtype=torch.bool)
    if bool(warped.any()):
        xn = p[:, 30] * x + p[:, 31]
        yn = p[:, 32] * y + p[:, 33]
        one = torch.ones((), dtype=torch.float32)
        wv = [_mad3(p[:, 21 + 3 * r], xn, p[:, 22 + 3 * r], yn, p[:, 23 + 3 * r], one) for r in range(3)]
        xw, yw = wv[0] / wv[2], wv[1] / wv[2]
        oob = (xw < 0) | (xw > w - 1) | (yw < 0) | (yw > h - 1)
        x, y = torch.where(warped, xw, x), torch.where(warped, yw, y)
        keep &= ~(warped & oob)
    cx, cy = torch.round(x * 0.125), torch.round(y * 0.125)
    rx, ry = cx * 8.0, cy * 8.0
    keep &= (rx >= 0) & (rx <= w - 1) & (ry >= 0) & (ry <= h - 1)
    rank = torch.where(keep, cx.nan_to_num(0).long() * ncy + cy.nan_to_num(0).long(), 0)
    # first correspondence per (b, cell) among the kept ones
    c = torch.arange(n)
    cell = b * ranks + rank
    owner = torch.full((B * ranks,), n, dtype=torch.int64)
    owner.scatter_reduce_(0, cell[keep], c[keep], "amin")
    surv = keep & (owner[cell] == c)
    # last writer (largest rank) per 2D keypoint
    kp = kp_off[b] + a0
    kp_owner = torch.full((max(int(kp_off[-1]), 1),), -1, dtype=torch.int64)
    kp_owner.scatter_reduce_(0, kp[surv], rank[surv], "amax")
    won = kp_owner[kp].clamp(min=0)
    cw = owner[b * ranks + won].clamp(max=max(n - 1, 0))
    px, py = (won // ncy).float() * 8.0, (won % ncy).float() * 8.0
    s = img_scale.cpu().to(torch.float32)[b]
    jx = torch.round(px / s[:, 1] * 0.125)
    jy = torch.round(py / s[:, 0] * 0.125)
    j = (jy * float(w_c) + jx).long()
    emit = surv & (a1 < L) & ~(j > S)
    if bool((emit & ((j == S) | (j < 0))).any()):
        _raise_status(_ERR_CELL)
    key = ((b * L + a1) * S + j) * ranks + rank
    fxy = torch.stack([x, y], 1)[cw] if n else torch.zeros(0, 2)
    key, fxy = key[emit], fxy[emit]
    order = torch.argsort(key)
    key, fxy = key[order], fxy[order]
    cellkey = key // ranks
    last = torch.ones(len(key), dtype=torch.bool)
    last[:-1] = cellkey[1:] != cellkey[:-1]
    cellkey, fxy = cellkey[last], fxy[last].contiguous()
    return cellkey // (L * S), (cellkey // S) % L, cellkey % S, fxy
