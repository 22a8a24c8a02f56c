"""NumPy restatement of the training batch's ground truth built on the device
(onepose_plus_plus_b200/train_batch.py, csrc/opp_train_batch.cu): the homography warp of the query
image and the correspondences projected from the pose (OnePosePlusDataset.read_anno,
src/datasets/OnePosePlus_dataset.py:341-444, build_assignmatrix :174-236).  Elementwise fp32
operations in the kernels' order — no `@` — so kernels and restatement agree bit for bit.

Also here, for the build container only:
  * install_kornia(): kornia 0.4.1's normal_transform_pixel, normalize_homography and
    homography_warp, restated from its published definitions (kornia is not installed here), put
    on the stand-in `kornia` module of ref_shims and on the reference dataset module;
  * make_case(): a seeded on-disk stand-in of the dataset (PNG, anno2d JSON, anno3d npz and its
    _coarse file, intrin_ba / poses_ba txt, a COCO stand-in) whose projected coordinates keep a
    margin from every rounding boundary and border threshold;
  * reference_dataset(): the live reference OnePosePlusDataset over such a case.
"""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

f32 = np.float32
PACK = 44
MARGIN = 1e-2          # px: distance kept from x = 4 (mod 8) and from each border threshold


# ---- the restatement -----------------------------------------------------------------------------

def normal_transform_pixel(height, width):
    tr = torch.tensor([[1.0, 0.0, -1.0], [0.0, 1.0, -1.0], [0.0, 0.0, 1.0]])
    tr[0, 0] = tr[0, 0] * 2.0 / (width - 1.0)
    tr[1, 1] = tr[1, 1] * 2.0 / (height - 1.0)
    return tr.unsqueeze(0)


def normalize_homography(dst_pix_trans_src_pix, dsize_src, dsize_dst):
    (src_h, src_w), (dst_h, dst_w) = dsize_src, dsize_dst
    src_norm_trans_src_pix = normal_transform_pixel(src_h, src_w).to(dst_pix_trans_src_pix)
    src_pix_trans_src_norm = torch.inverse(src_norm_trans_src_pix)
    dst_norm_trans_dst_pix = normal_transform_pixel(dst_h, dst_w).to(dst_pix_trans_src_pix)
    return dst_norm_trans_dst_pix @ (dst_pix_trans_src_pix @ src_pix_trans_src_norm)


def homography_warp(patch_src, src_homo_dst, dsize, mode="bilinear", padding_mode="zeros", align_corners=False):
    """kornia 0.4.1 homography_warp: meshgrid(linspace(-1, 1)) through src_homo_dst [B, 3, 3] by
    matmul, the division by z (scale 1 where |z| <= 1e-8), grid_sample."""
    height, width = dsize
    xs = torch.linspace(-1, 1, width, dtype=torch.float)
    ys = torch.linspace(-1, 1, height, dtype=torch.float)
    grid = torch.stack(torch.meshgrid([xs, ys], indexing="ij")).transpose(1, 2)[None].permute(0, 2, 3, 1)
    B = src_homo_dst.shape[0]
    pts = torch.cat([grid.expand(B, -1, -1, -1), torch.ones(B, height, width, 1)], -1).to(src_homo_dst)
    ph = torch.matmul(src_homo_dst[:, None, None], pts[..., None])[..., 0]
    z = ph[..., -1:]
    mask = torch.abs(z) > 1e-8
    scale = torch.ones_like(z).masked_scatter_(mask, torch.tensor(1.0) / z[mask])
    flow = scale * ph[..., :-1]
    return F.grid_sample(patch_src, flow, mode=mode, padding_mode=padding_mode, align_corners=align_corners)


def pack_item(pose_gt, K_crop, homography, h, w):
    """fp32 [PACK]: the kernels' per-item parameters from the pose (fp64 [4, 4]), K_crop (fp64 [3, 3])
    and the sampled homography (fp64 [3, 3] or None) — the reference's 3x3 calls and dtypes."""
    pose, K = torch.as_tensor(pose_gt), torch.as_tensor(K_crop)
    p = torch.zeros(PACK, dtype=torch.float32)
    p[0:9] = pose[:3, :3].to(torch.float).reshape(9)
    p[9:12] = pose[:3, 3].to(torch.float)
    p[12:21] = K.to(torch.float).reshape(9)
    if homography is not None:
        Hn = normalize_homography(torch.as_tensor(np.asarray(homography))[None].to(torch.float32), (h, w), (h, w))
        N = normal_transform_pixel(h, w)
        p[21:30] = (N[0].inverse() @ Hn[0]).reshape(9)
        p[30:34] = torch.stack([N[0, 0, 0], N[0, 0, 2], N[0, 1, 1], N[0, 1, 2]])
        p[34:43] = torch.linalg.inv(Hn)[0].reshape(9)
        p[43] = 1.0
    return p.numpy()


def linspace_pm1(n):
    i = np.arange(n)
    step = f32(2) / f32(n - 1)
    return np.where(i < n // 2, f32(-1) + step * i.astype(f32), f32(1) - step * (n - 1 - i).astype(f32)).astype(f32)


def _mad3(a0, x, a1, y, a2, z, dt=f32):
    return ((a0 * x + a1 * y) + a2 * z).astype(dt)


def warp_image(img, pack):
    """img fp32 [h, w] -> the kernel's warp (a copy when the pack's warp flag is 0)."""
    img = np.asarray(img, dtype=f32)
    p = np.asarray(pack, dtype=f32)
    if p[43] == 0:
        return img.copy()
    h, w = img.shape
    gx, gy = linspace_pm1(w)[None, :], linspace_pm1(h)[:, None]
    A = p[34:43]
    one = f32(1)
    sx, sy, sz = (_mad3(A[3 * r], gx, A[3 * r + 1], gy, A[3 * r + 2], one) for r in range(3))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = np.where(np.abs(sz) > f32(1e-8), one / sz, one).astype(f32)
        ix = ((s * sx + one) * f32(0.5 * w) - f32(0.5)).astype(f32)
        iy = ((s * sy + one) * f32(0.5 * h) - f32(0.5)).astype(f32)
    inside = (ix > -1) & (ix < w) & (iy > -1) & (iy < h)
    fx = np.floor(np.where(inside, ix, f32(-2))).astype(f32)
    fy = np.floor(np.where(inside, iy, f32(-2))).astype(f32)
    wx, ny = (ix - fx).astype(f32), (iy - fy).astype(f32)
    ex, sy_ = (one - wx).astype(f32), (one - ny).astype(f32)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)

    def tap(xx, yy):
        ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
        return np.where(ok, img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)], f32(0)).astype(f32)

    val = ((sy_ * ex) * tap(x0, y0) + (sy_ * wx) * tap(x0 + 1, y0)) + (ny * ex) * tap(x0, y0 + 1)
    val = (val + (ny * wx) * tap(x0 + 1, y0 + 1)).astype(f32)
    return np.where(inside, val, f32(0)).astype(f32)


def project(kp3d, assign, pack, hw, dt=f32):
    """One item: (x, y [k], kept bool [k]) — the projection, the warp and its out-of-bounds filter
    (:342-400), before the rounding.  dt=np.float64 runs the same operations in fp64 on the fp32
    inputs (the pack, the points and the 1e-6 promoted), for error bounds of the fp32 kernels."""
    h, w = hw
    p = np.asarray(pack, dtype=f32).astype(dt)
    X = np.asarray(kp3d, dtype=f32).astype(dt)[np.asarray(assign)[1]]
    cam = [(_mad3(p[3 * r], X[:, 0], p[3 * r + 1], X[:, 1], p[3 * r + 2], X[:, 2], dt) + p[9 + r]).astype(dt)
           for r in range(3)]
    q = [_mad3(p[12 + 3 * r], cam[0], p[13 + 3 * r], cam[1], p[14 + 3 * r], cam[2], dt) for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        zd = (q[2] + dt(f32(1e-6))).astype(dt)
        x, y = (q[0] / zd).astype(dt), (q[1] / zd).astype(dt)
        kept = np.ones(len(x), dtype=bool)
        if p[43] != 0:
            xn = (p[30] * x + p[31]).astype(dt)
            yn = (p[32] * y + p[33]).astype(dt)
            wv = [_mad3(p[21 + 3 * r], xn, p[22 + 3 * r], yn, p[23 + 3 * r], dt(1), dt) for r in range(3)]
            x, y = (wv[0] / wv[2]).astype(dt), (wv[1] / wv[2]).astype(dt)
            kept = ~((x < 0) | (x > w - 1) | (y < 0) | (y > h - 1))
    return x, y, kept


def item_list(kp3d, assign, pack, scale, hw, L, dt=f32):
    """One item's correspondences as build_assignmatrix writes them: (i, j int64, fine_xy [n, 2])
    sorted by (i, j), the later write of a cell kept (dt as in project)."""
    h, w = hw
    w_c, S = int(w * 0.125), int(h * 0.125) * int(w * 0.125)
    assign = np.asarray(assign, dtype=np.int64).reshape(2, -1)
    x, y, kept = project(kp3d, assign, pack, hw, dt)
    with np.errstate(invalid="ignore"):
        rx = (np.round((x * dt(0.125)).astype(dt)) * dt(8)).astype(dt)
        ry = (np.round((y * dt(0.125)).astype(dt)) * dt(8)).astype(dt)
        kept &= (rx >= 0) & (rx <= w - 1) & (ry >= 0) & (ry <= h - 1)                 # :411-424
    idx = np.nonzero(kept)[0]
    rounded = np.stack([rx[idx], ry[idx]], 1) + dt(0)       # + 0: -0.0 -> 0.0, the same row for np.unique
    _, first = np.unique(rounded, return_index=True, axis=0)                             # :426
    order = idx[first]                      # survivors in np.unique's (x, y) row order
    a0, a1 = assign[0][order], assign[1][order]
    coarse = np.zeros((a0.max() + 1 if len(a0) else 0, 2), dtype=dt)
    fine = np.zeros_like(coarse)
    for c, k in zip(order, a0):             # :431-433, the later write wins
        coarse[k] = (rx[c], ry[c])
        fine[k] = (x[c], y[c])
    ok = a1 < L                                                                          # :195-196
    a0, a1 = a0[ok], a1[ok]
    s = np.asarray(scale, dtype=f32).astype(dt)[[1, 0]]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        cell = np.round(((coarse[a0] / s).astype(dt) * dt(0.125)).astype(dt))          # :205-212
        j = (cell[:, 1] * dt(w_c) + cell[:, 0]).astype(dt).astype(np.int64)             # :219-223
    ok = ~(j > S)                                                                        # :225-228
    i, j, xy = a1[ok], j[ok], fine[a0][ok]
    if ((j == S) | (j < 0)).any():
        raise ValueError("cell index == S or < 0")
    key = i * S + j
    o = np.argsort(key, kind="stable")
    key = key[o]
    last = np.ones(len(key), dtype=bool)
    last[:-1] = key[1:] != key[:-1]
    o = o[last]
    return i[o], j[o], xy[o]


def batch_list(kp3d, assigns, packs, scales, hw, dt=f32):
    """(b, i, j int64, fine_xy [G, 2]) of a batch, ascending in (b, i, j)."""
    L = np.asarray(kp3d).shape[1]
    out = [item_list(kp3d[b], assigns[b], packs[b], scales[b], hw, L, dt) for b in range(len(assigns))]
    bb = np.concatenate([np.full(len(o[0]), b, dtype=np.int64) for b, o in enumerate(out)])
    return (bb, np.concatenate([o[0] for o in out]).astype(np.int64),
            np.concatenate([o[1] for o in out]).astype(np.int64),
            np.concatenate([o[2] for o in out]).reshape(-1, 2).astype(dt))


# ---- the scratch arrays of opp_train_gt_build ------------------------------------------------------

ERR_CELL, ERR_2D, ERR_3D = 1, 2, 4
CELL_FREE = 0x7f7f7f7f                  # cell_owner of a cell no correspondence rounds to
KEY_DROPPED = np.iinfo(np.int64).max


def item_scratch(kp3d, assign, pack, scale, hw, L, n_2d):
    """One item's share of opp_train_gt_build's scratch arrays, restated per correspondence in
    build_assignmatrix's terms rather than by atomics:
      rank_of int32 [k]: the cell cx * ncy + cy of the rounded location, -1 without one;
      cell_owner int32 [R]: np.unique's first index of each cell (local), CELL_FREE if empty;
      kp_owner int32 [n_2d]: the rank of the sequentially last survivor written to each 2D keypoint, -1 if none;
      fine fp32 [k, 2]: the unrounded location where rank_of >= 0 (NaN elsewhere);
      j int64 [k]: the emitted coarse cell (-1: not emitted, -2: an ERR_CELL), xy fp32 [k, 2] its
      fine location;
      bits: the status bits (ERR_*) the item sets."""
    h, w = hw
    ncx, ncy = (w - 1) // 8 + 1, (h - 1) // 8 + 1
    w_c, S = int(w * 0.125), int(h * 0.125) * int(w * 0.125)
    assign = np.asarray(assign, dtype=np.int64).reshape(2, -1)
    k = assign.shape[1]
    a0, a1 = assign
    bad2 = (a0 < 0) | (a0 >= n_2d)
    bad3 = ~bad2 & ((a1 < 0) | (a1 >= L))
    bits = (ERR_2D if bad2.any() else 0) | (ERR_3D if bad3.any() else 0)
    valid = ~(bad2 | bad3)
    x, y, kept = project(kp3d, np.stack([a0, np.where(valid, a1, 0)]), pack, hw)
    with np.errstate(invalid="ignore"):
        cx, cy = np.round((x * f32(0.125)).astype(f32)), np.round((y * f32(0.125)).astype(f32))
        rx, ry = (cx * f32(8)).astype(f32), (cy * f32(8)).astype(f32)
        kept &= valid & (rx >= 0) & (rx <= w - 1) & (ry >= 0) & (ry <= h - 1)
    rank_of = np.full(k, -1, np.int32)
    rank_of[kept] = cx[kept].astype(np.int64) * ncy + cy[kept].astype(np.int64)
    fine = np.full((k, 2), np.nan, f32)
    fine[kept] = np.stack([x, y], 1)[kept]
    cell_owner = np.full(ncx * ncy, CELL_FREE, np.int32)
    idx = np.nonzero(kept)[0]
    cells, first = np.unique(rank_of[idx], return_index=True)
    cell_owner[cells] = idx[first]
    surv = kept.copy()
    surv[idx] = cell_owner[rank_of[idx]] == idx
    kp_owner = np.full(n_2d, -1, np.int32)
    for c in sorted(np.nonzero(surv)[0], key=lambda c: rank_of[c]):     # :431-433, in np.unique's row order
        kp_owner[a0[c]] = rank_of[c]
    j = np.full(k, -1, np.int64)
    xy = np.full((k, 2), np.nan, f32)
    s = np.asarray(scale, dtype=f32)
    for c in np.nonzero(surv & (a1 < L))[0]:
        won = int(kp_owner[a0[c]])
        px, py = f32(won // ncy) * f32(8), f32(won % ncy) * f32(8)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            jx = np.round(f32(px / s[1]) * f32(0.125))
            jy = np.round(f32(py / s[0]) * f32(0.125))
            jf = f32(f32(jy * f32(w_c)) + jx)
        if not (jf > f32(-9.2e18) and jf < f32(9.2e18)):
            bits |= ERR_CELL
            j[c] = -2
            continue
        jc = int(jf)
        if jc > S:
            continue
        if jc == S or jc < 0:
            bits |= ERR_CELL
            j[c] = -2
            continue
        j[c] = jc
        xy[c] = fine[cell_owner[won]]
    return {"rank_of": rank_of, "cell_owner": cell_owner, "kp_owner": kp_owner, "fine": fine, "j": j, "xy": xy,
            "bits": bits}


def batch_scratch(kp3d, assign, offsets, kp_offsets, packs, scales, hw):
    """item_scratch over a batch, joined as the kernels lay it out: cell_owner [B * R], kp_owner
    [n_kp], rank_of / fine / key / key_xy per correspondence (key ((b L + i) S + j) R + rank,
    KEY_DROPPED where nothing is emitted), and the status bits of all items."""
    h, w = hw
    B, L = np.asarray(kp3d).shape[:2]
    R = ((w - 1) // 8 + 1) * ((h - 1) // 8 + 1)
    S = int(h * 0.125) * int(w * 0.125)
    parts = [item_scratch(kp3d[b], assign[:, offsets[b]:offsets[b + 1]], packs[b], scales[b], hw, L,
                          int(kp_offsets[b + 1] - kp_offsets[b])) for b in range(B)]
    out = {k: np.concatenate([p[k] for p in parts]) for k in ("rank_of", "cell_owner", "kp_owner", "fine", "xy")}
    key = np.full(assign.shape[1], KEY_DROPPED, np.int64)
    for b, p in enumerate(parts):
        c = np.nonzero(p["j"] >= 0)[0]
        i = assign[1, offsets[b] + c]
        key[offsets[b] + c] = ((b * L + i) * S + p["j"][c]) * R + p["rank_of"][c]
    out["key"], out["key_xy"] = key, out.pop("xy")
    out["bits"] = int(np.bitwise_or.reduce([p["bits"] for p in parts])) if parts else 0
    return out


# ---- a synthetic batch at the training shape (no reference needed) ---------------------------------

def random_homography(g, h, w):
    """a similarity + shear + perspective about the image centre (the kind sample_homography_sap draws)"""
    a, s = g.uniform(-np.pi, np.pi), g.uniform(0.4, 1.0)
    m = max(h, w) / 2
    Tn = np.array([[1 / m, 0, -w / 2 / m], [0, 1 / m, -h / 2 / m], [0, 0, 1]])
    S = np.array([[s * np.cos(a), -s * np.sin(a), g.uniform(-0.25, 0.25)],
                  [s * np.sin(a), s * np.cos(a), g.uniform(-0.25, 0.25)], [0, 0, 1]])
    A = np.array([[1, g.uniform(-0.1, 0.1), 0], [0, 1, 0], [0, 0, 1]])
    P = np.array([[1, 0, 0], [0, 1, 0], [g.uniform(-0.5, 0.5), g.uniform(-0.5, 0.5), 1]])
    return np.linalg.inv(Tn) @ S @ A @ P @ Tn


def synthetic_batch(seed, B=4, hw=(512, 512), L=7000, n_corr=3000, n_2d=3500, scale=(1.0, 1.0)):
    """The training shape without the reference: poses, K, 3D points in front of the camera (a few
    behind and outside), random homographies on the odd items, repeated 2D keypoints."""
    g = np.random.default_rng(seed)
    h, w = hw
    kp3d = np.zeros((B, L, 3), np.float32)
    assign, Ks, poses, hs = [], [], [], []
    for b in range(B):
        K = np.array([[g.uniform(450, 600), 0, w / 2], [0, g.uniform(450, 600), h / 2], [0, 0, 1]])
        a = np.deg2rad(g.uniform(-20, 20))
        R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        t = np.array([0.01, -0.02, 0.6])
        uv = g.uniform([-40, -40], [w + 40, h + 40], (L, 2))
        d = g.uniform(0.4, 0.8, L)
        d[:20] *= -1
        cam = d[:, None] * (np.linalg.inv(K) @ np.concatenate([uv, np.ones((L, 1))], 1).T).T
        kp3d[b] = ((cam - t) @ R).astype(np.float32)
        a1 = g.choice(L, n_corr, replace=False)
        a0 = g.integers(0, n_2d, n_corr)
        assign.append(np.stack([a0, a1]))
        pose = np.eye(4)
        pose[:3, :3], pose[:3, 3] = R, t
        Ks.append(K), poses.append(pose)
        hs.append(torch.from_numpy(random_homography(g, h, w)) if b % 2 else None)
    yy, xx = np.mgrid[0:h, 0:w]
    img = (0.5 + 0.4 * np.sin(xx[None] / 17.0 + np.arange(B)[:, None, None]) * np.cos(yy[None] / 23.0))
    counts = np.cumsum([0] + [a.shape[1] for a in assign])
    from onepose_plus_plus_b200 import train_batch
    src = train_batch.GTSource(torch.from_numpy(np.concatenate(assign, 1)), torch.from_numpy(counts),
                               torch.arange(B + 1) * n_2d, B * n_2d, torch.from_numpy(np.stack(Ks)),
                               torch.from_numpy(np.stack(poses)), hs)
    return {"query_image": torch.from_numpy(img[:, None].astype(np.float32)), "keypoints3d": torch.from_numpy(kp3d),
            "query_image_scale": torch.tensor([scale] * B, dtype=torch.float32),
            "query_intrinsic": torch.from_numpy(np.stack(Ks)), "gt_source": src}


def planted_batch(seed, B=4, hw=(512, 512), L=7000, n_corr=3000, n_2d=3500):
    """synthetic_batch's training shape with every correspondence planted as make_case plants them:
    its projection (and, on the warped odd items, its warped position) keeps MARGIN px from x = 4
    (mod 8) and from the border thresholds, so an fp64 run of the same steps rounds to the same cells."""
    g = np.random.default_rng(seed)
    h, w = hw
    items = []
    for b in range(B):
        it = _random_item(g, hw, L, L, n_2d, b % 2 == 1, behind=20)
        p = pack_item(it["pose"], it["K"], None, h, w).astype(np.float64)
        X = it["kp3d"].astype(np.float64)
        q = (X @ p[0:9].reshape(3, 3).T + p[9:12]) @ p[12:21].reshape(3, 3).T
        u, v = q[:, 0] / (q[:, 2] + 1e-6), q[:, 1] / (q[:, 2] + 1e-6)
        ok = _margin_ok(u, v, h, w)
        if it["H"] is not None:
            r = np.stack([u, v, np.ones_like(u)], 1) @ it["H"].T
            ok &= _margin_ok(r[:, 0] / r[:, 2], r[:, 1] / r[:, 2], h, w)
        a1 = g.choice(np.nonzero(ok)[0], n_corr, replace=False)
        it["assign"] = np.stack([g.integers(0, n_2d, n_corr), a1])
        items.append(it)
    return _assemble(items, hw, L, (1.0, 1.0), seed)


# ---- edge batches: the shapes, scales, ties and rounding edges where the kernels can go wrong -------

def _assemble(items, hw, L, scale, seed):
    """a host batch from per-item dicts (kp3d fp32 [L, 3], assign int64 [2, k], n_2d, K, pose fp64, H)"""
    g = np.random.default_rng(seed)
    h, w = hw
    B = len(items)
    counts = np.cumsum([0] + [it["assign"].shape[1] for it in items])
    n2d = np.cumsum([0] + [it["n_2d"] for it in items])
    assign = np.concatenate([it["assign"] for it in items], 1).astype(np.int64).reshape(2, -1)
    src = _gt_source(assign, counts, n2d, [it["K"] for it in items], [it["pose"] for it in items],
                     [it["H"] for it in items])
    return {"query_image": torch.from_numpy(g.random((B, 1, h, w), dtype=np.float32)),
            "keypoints3d": torch.from_numpy(np.stack([it["kp3d"] for it in items]).astype(f32)),
            "query_image_scale": torch.tensor([scale] * B, dtype=torch.float32),
            "query_intrinsic": torch.from_numpy(np.stack([it["K"] for it in items])), "gt_source": src}


def _gt_source(assign, counts, n2d, Ks, poses, hs):
    from onepose_plus_plus_b200 import train_batch
    return train_batch.GTSource(torch.from_numpy(assign), torch.from_numpy(np.asarray(counts, np.int64)),
                                torch.from_numpy(np.asarray(n2d, np.int64)), int(n2d[-1]),
                                torch.from_numpy(np.stack(Ks)), torch.from_numpy(np.stack(poses)),
                                [None if H is None else torch.from_numpy(H) for H in hs])


def _random_item(g, hw, L, n_corr, n_2d, warp, behind=10, pad=40):
    """synthetic_batch's item at any size: a random camera, points over the image and pad px around
    it (behind of them behind the camera), a random homography when warp"""
    h, w = hw
    f = g.uniform(0.9, 1.2) * max(h, w)
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    a = np.deg2rad(g.uniform(-20, 20))
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    t = np.array([0.01, -0.02, 0.6])
    uv = g.uniform([-pad, -pad], [w + pad, h + pad], (L, 2))
    d = g.uniform(0.4, 0.8, L)
    d[:behind] *= -1
    cam = d[:, None] * (np.linalg.inv(K) @ np.concatenate([uv, np.ones((L, 1))], 1).T).T
    pose = np.eye(4)
    pose[:3, :3], pose[:3, 3] = R, t
    a1 = g.choice(L, min(n_corr, L), replace=False) if n_corr <= L else g.integers(0, L, n_corr)
    return {"kp3d": ((cam - t) @ R).astype(f32), "assign": np.stack([g.integers(0, n_2d, len(a1)), a1]),
            "n_2d": n_2d, "K": K, "pose": pose, "H": random_homography(g, h, w) if warp else None}


def _identity_item(L, n_2d):
    """identity pose and K: the point (X0, X1, 1) projects to (X0, X1) / fl(1 + 1e-6)"""
    return {"kp3d": np.zeros((L, 3), f32) + np.array([0, 0, 1], f32), "assign": np.zeros((2, 0), np.int64),
            "n_2d": n_2d, "K": np.eye(3), "pose": np.eye(4), "H": None}


def _place(item, pts, a0, a1):
    """append correspondences (a0, a1) whose 3D points are pts fp32 [k, 3]"""
    item["kp3d"][a1] = np.asarray(pts, f32).reshape(-1, 3)
    item["assign"] = np.concatenate([item["assign"], np.stack([a0, a1]).astype(np.int64)], 1)


_ZD = f32(f32(1) + f32(1e-6))


def at_pixels(uv):
    """the identity item's 3D points (fp32 [k, 3]) that project to about the pixels uv [k, 2]"""
    uv = np.asarray(uv, np.float64).reshape(-1, 2)
    return np.concatenate([(uv * float(_ZD)).astype(f32), np.ones((len(uv), 1), f32)], 1)


def land(pack, hw, axis, target, other):
    """An fp32 point of the identity item whose projection (through the pack's warp, if set) has
    coordinate `axis` exactly `target` (sign included) and the other about `other`: a search over
    neighbouring fp32 inputs, run through project().  Raises if no input lands there."""
    p = np.asarray(pack, np.float64)
    tgt = np.array([target, other] if axis == 0 else [other, target], np.float64)
    if p[43]:
        v = np.linalg.solve(p[21:30].reshape(3, 3), [tgt[0], tgt[1], 1.0])
        tgt = np.array([(v[0] / v[2] - p[31]) / p[30], (v[1] / v[2] - p[33]) / p[32]])
    start = (tgt * float(_ZD)).astype(f32)
    if start[axis] == 0:
        start[axis] = np.copysign(f32(0), target)
        if not p[43]:
            return np.array([*start, 1.0], f32)

    def around(v, n):
        bits = np.asarray(v, f32).reshape(1).view(np.int32)[0]
        return (bits + np.arange(-n, n + 1, dtype=np.int32)).view(f32)

    mine, theirs = around(start[axis], 2048), around(start[1 - axis], 8)
    A, O = np.meshgrid(mine, theirs, indexing="ij")
    X = np.zeros((A.size, 3), f32)
    X[:, axis], X[:, 1 - axis], X[:, 2] = A.ravel(), O.ravel(), 1
    xy = project(X, np.stack([np.zeros(len(X), np.int64), np.arange(len(X))]), pack, hw)[:2]
    hit = (xy[axis] == f32(target)) & (np.signbit(xy[axis]) == np.signbit(f32(target)))
    if not hit.any():
        raise ValueError(f"land: no fp32 input projects to {target!r} on axis {axis}")
    return X[np.nonzero(hit)[0][0]]


def _prune_cell_errors(items, hw, L, scale):
    """drop the correspondences whose emitted cell would be the grid size or negative, until none is"""
    for it in items:
        pack = pack_item(it["pose"], it["K"], it["H"], *hw)
        for _ in range(200):
            sc = item_scratch(it["kp3d"], it["assign"], pack, scale, hw, L, it["n_2d"])
            if not sc["bits"]:
                break
            it["assign"] = it["assign"][:, sc["j"] != -2]
        else:
            raise RuntimeError("_prune_cell_errors did not converge")


def _perspective_flip(h, w, a):
    """a pixel homography whose normalised form is [[1, 0, 0], [0, 1, 0], [a, 0, 1]]: with |a| > 1 the
    warp's z (1 - a gx) and the points' w2 (a xn + 1) change sign inside the image"""
    N = normal_transform_pixel(h, w)[0].double().numpy()
    Hn = np.array([[1, 0, 0], [0, 1, 0], [a, 0, 1.0]])
    return np.linalg.inv(N) @ Hn @ N


def edge_batch(name):
    """(host batch, expected error): the seeded edge case `name` of EDGE_CASES.  The expected error
    is None (a list), "grid size" (a cell index equals the grid size: the restatement, the CPU path
    and the device path raise ValueError) or "coarse cell" (S = 0: prepare_batch refuses the image
    before any step)."""
    kind, kw = EDGE_CASES[name]
    g = np.random.default_rng(sum(map(ord, name)))
    hw, L, scale = kw.get("hw", (96, 128)), kw.get("L", 600), kw.get("scale", (1.0, 1.0))
    h, w = hw
    expect = None
    if kind == "size":
        B = kw.get("B", 3)
        items = [_random_item(g, hw, L, kw.get("n", 400), 300, b % 2 == 1, pad=max(8, w // 8)) for b in range(B)]
        _prune_cell_errors(items, hw, L, scale)
        if int(h * 0.125) * int(w * 0.125) == 0:
            expect = "coarse cell"
    elif kind == "cell_S":
        # 97 x 131: w_c = 16, h_c = 12, ncy = 13; the point rounded to (0, 96) has j = 12 * 16 = S
        it = _random_item(g, hw, L, 200, 300, False)
        _prune_cell_errors([it], hw, L, scale)
        edge = _identity_item(L, 8)
        y = 96.4 if kw["hit"] else 88.4
        _place(edge, at_pixels([(1.3, y), (20.2, 40.3)]), np.array([0, 1]), np.array([3, 4]))
        items, expect = [it, edge], "grid size" if kw["hit"] else None
    elif kind == "scale":
        items = [_random_item(g, hw, L, 300, 200, b % 2 == 1) for b in range(3)]
        if kw.get("merge"):
            # scale 2: the cells cx = 3, 4, 5 all give jx = 2, so three 3D points share one j
            edge = _identity_item(L, 10)
            _place(edge, at_pixels([(24.5, 17.0), (33.0, 17.2), (41.3, 16.6)]), np.array([0, 1, 2]),
                   np.array([5, 6, 7]))
            items.append(edge)
        _prune_cell_errors(items, hw, L, scale)
    elif kind == "contention":
        # item 0: 2500 correspondences in the cell (10, 10) and 2100 survivors of one 2D keypoint, shuffled
        # over 19 CTAs; 300 more share another 2D keypoint; item 1 warped
        edge = _identity_item(L, 3000)
        n0, n1, n2 = 2500, 2100, 300
        cells = g.permutation(64 * 64)[:n1 + n2 + 1]
        cells = cells[cells != 10 * 64 + 10][:n1 + n2]
        uv = np.concatenate([80 + g.uniform(-3.4, 3.4, (n0, 2)),
                             np.stack([cells // 64 * 8, cells % 64 * 8], 1) + g.uniform(-3.4, 3.4, (n1 + n2, 2))])
        a0 = np.concatenate([g.permutation(3000)[:n0], np.full(n1, 7), np.full(n2, 9)])
        a1 = g.permutation(L)[:n0 + n1 + n2]
        o = g.permutation(n0 + n1 + n2)
        _place(edge, at_pixels(uv[o]), a0[o], a1[o])
        items = [edge, _random_item(g, hw, L, 3000, 3500, True)]
        _prune_cell_errors(items, hw, L, scale)
    elif kind == "rounding":
        # (89, 97): h - 1 = 88 and w - 1 = 96 are cell centres, so the border filters decide alone
        items = []
        for warp in (False, True):
            it = _identity_item(L, 64)
            # -0.0 off the diagonals and in t keep a -0.0 input coordinate -0.0 through the projection
            it["pose"] = np.where(np.eye(4) == 0, -0.0, np.eye(4))
            it["pose"][3, :3] = 0.0
            it["K"] = np.where(np.eye(3) == 0, -0.0, np.eye(3))
            it["K"][2, :2] = 0.0
            if warp:
                it["H"] = random_homography(g, h, w)
            pack = pack_item(it["pose"], it["K"], it["H"], h, w)
            pts = []
            for axis, n in ((0, w), (1, h)):
                other = 41.3 if axis == 0 else 49.7
                for t in (4.0, 12.0, 20.0, 28.0, 0.0, -0.0, float(n - 1), float(np.nextafter(f32(n - 1), f32(n))),
                          float(-np.nextafter(f32(0), f32(1))), 8.0 * (n // 16) + 4.0):
                    if warp and t == 0.0 and np.signbit(t):
                        continue           # -0.0 needs w0 = +0 over a negative w2; no such point here
                    try:
                        pts.append(land(pack, hw, axis, t, other))
                    except ValueError:
                        if not warp:
                            raise
            k = len(pts)
            _place(it, np.stack(pts), np.arange(k), np.arange(k) + 1)
            items.append(it)
        _prune_cell_errors(items, hw, L, scale)
    elif kind == "flip":
        # the warp's z and the points' w2 change sign in the image; points behind the camera, and
        # zd = 0 exactly (X2 = -1e-6: x = +-inf, y = NaN)
        items = [_random_item(g, hw, L, 400, 300, False, behind=60), _random_item(g, hw, L, 400, 300, False, behind=60)]
        items[1]["H"] = _perspective_flip(h, w, kw["a"])
        for it in items:
            z = _identity_item(L, 300)
            it["kp3d"][:4] = z["kp3d"][:4]
        zero = _identity_item(L, 300)
        _place(zero, np.array([[5, 0, -1e-6], [0, 0, -1e-6], [-3, 7, -1e-6], [10, 20, 1]], f32), np.arange(4),
               np.arange(4))
        zero["H"] = _perspective_flip(h, w, kw["a"])
        items.append(zero)
        _prune_cell_errors(items, hw, L, scale)
    elif kind == "empty":
        B = kw["B"]
        items = []
        for b in range(B):
            if b in kw["empty"]:
                it = _random_item(g, hw, L, 0, 0 if b % 2 else 5, False)
            else:
                it = _random_item(g, hw, L, kw.get("n", 120), 100, b % 2 == 1)
                if kw.get("outside"):
                    # everything behind the camera and far outside, or past L: nothing survives
                    it["kp3d"][:] = np.array([1e4, -1e4, 1.0], f32)
            items.append(it)
        _prune_cell_errors(items, hw, L, scale)
    else:
        raise KeyError(name)
    return _assemble(items, hw, L, scale, sum(map(ord, name)) + 1), expect


EDGE_CASES = {
    # the warp's 32 x 8 tile and the 8-px grid do not divide the image
    "size_2x2": ("size", dict(hw=(2, 2), B=2, n=20, L=40)),           # S = 0: no coarse cell
    "size_7x33": ("size", dict(hw=(7, 33), n=60, L=80)),
    "size_97x131": ("size", dict(hw=(97, 131))),
    "size_100x100": ("size", dict(hw=(100, 100))),
    "size_511x509": ("size", dict(hw=(511, 509), n=3000, L=4000)),
    "size_8x1000": ("size", dict(hw=(8, 1000), n=500)),
    # the rounded point (0, 96) reaches j == S, or (0, 88) stays below it
    "cell_S_hit": ("cell_S", dict(hw=(97, 131), hit=True)),
    "cell_S_avoid": ("cell_S", dict(hw=(97, 131), hit=False)),
    # non-square and merging query_image_scale
    "scale_0.75_1.5": ("scale", dict(hw=(96, 128), scale=(0.75, 1.5))),
    "scale_2_2": ("scale", dict(hw=(64, 64), scale=(2.0, 2.0), merge=True)),
    "scale_0.5_0.5": ("scale", dict(hw=(128, 128), scale=(0.5, 0.5))),
    # atomicMin / atomicMax over many CTAs
    "contention": ("contention", dict(hw=(512, 512), L=7000)),
    # projections exactly at 8k + 4, 0, -0.0, w - 1 and one ulp past it, unwarped and warped
    "rounding": ("rounding", dict(hw=(89, 97), L=64)),
    # sign changes of z / w2 in the image, points behind the camera, zd = 0
    "flip": ("flip", dict(hw=(96, 128), a=1.6)),
    # empty items first, in the middle and last; B = 1 and B = 17; n > 0 and no survivor
    "empty_b17": ("empty", dict(hw=(64, 80), B=17, empty=(0, 8, 15, 16), L=150)),
    "b1": ("empty", dict(hw=(96, 128), B=1, empty=(), n=300)),
    "no_survivor": ("empty", dict(hw=(96, 128), B=3, empty=(1,), outside=True)),
}



# ---- the live reference (build container only) ---------------------------------------------------

class StandInCOCO:
    """The four pycocotools.coco.COCO calls of the dataset, over a JSON of images and annotations."""

    def __init__(self, anno_file):
        with open(anno_file) as f:
            d = json.load(f)
        self.imgs = {im["id"]: im for im in d["images"]}
        self.anns = d["annotations"]

    def getImgIds(self):
        return sorted(self.imgs)

    def getAnnIds(self, imgIds):
        return [k for k, a in enumerate(self.anns) if a["image_id"] == imgIds]

    def loadAnns(self, ids):
        return [self.anns[k] for k in ids]

    def loadImgs(self, img_id):
        return [self.imgs[img_id]]


def install_kornia():
    from . import ref_shims
    ref_shims.install()
    for name, attrs in (("pycocotools", ()), ("pycocotools.coco", ("COCO",)), ("h5py", ())):
        try:
            __import__(name)
        except ImportError:
            mod = types.ModuleType(name)
            for a in attrs:
                setattr(mod, a, None)
            sys.modules[name] = mod
    fns = {"homography_warp": homography_warp, "normalize_homography": normalize_homography,
           "normal_transform_pixel": normal_transform_pixel}
    for k, v in fns.items():
        setattr(sys.modules["kornia"], k, v)
    import importlib
    dmod = importlib.import_module("src.datasets.OnePosePlus_dataset")
    for k, v in fns.items():
        setattr(dmod, k, v)
    dmod.COCO = StandInCOCO
    return dmod


def reference_dataset(case, **kw):
    """The live OnePosePlusDataset over a make_case() directory (split train, poses loaded)."""
    dmod = install_kornia()
    args = dict(pad=True, img_pad=False, img_resize=case["img_resize"], coarse_scale=0.125, df=8,
                shape3d=case["shape3d"], percent=1.0, split="train", load_pose_gt=True,
                load_3d_coarse_feature=True, image_warp_adapt=case["warp"], augmentor=None)
    args.update(kw)
    return dmod.OnePosePlusDataset(case["anno_file"], **args)


def _rot(g, deg):
    a = np.deg2rad(g.uniform(-deg, deg, 3))
    cx, cy, cz, sx, sy, sz = *np.cos(a), *np.sin(a)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _sample_homography(seed, h, w):
    """the homography the reference draws after np.random.seed(seed) (sample_homography_sap)"""
    install_kornia()
    from src.utils.sample_homo import sample_homography_sap   # type: ignore
    st = np.random.get_state()
    np.random.seed(seed)
    H = sample_homography_sap(h, w)
    np.random.set_state(st)
    return H


def _margin_ok(u, v, h, w):
    """every coordinate at least MARGIN from x = 4 (mod 8) and from the thresholds 0 and w - 1"""
    ok = np.ones(len(u), dtype=bool)
    for c, n in ((u, w), (v, h)):
        ok &= np.abs(np.mod(c, 8.0) - 4.0) >= MARGIN
        ok &= (np.abs(c) >= MARGIN) & (np.abs(c - (n - 1)) >= MARGIN)
    return ok


def make_case(root, seed=0, n_items=2, warp=False, src_hw=(512, 512), img_resize=(512, 512), shape3d=300,
              n_3d=400, n_corr=120, n_2d=None, collide=0, repeat_2d=0, behind=0, outside=0, empty_items=(),
              exact=False, item_seeds=None):
    """Write a seeded dataset stand-in under `root`; returns its description (paths, sizes, seeds).

    Each item has n_3d points (more or fewer than shape3d picks the padding branch) and n_corr
    correspondences whose projections (and, with warp, their warped positions under the homography
    the reference draws for the item's seed) keep MARGIN px from the rounding boundaries and the
    border thresholds; closer draws are rejected and counted in case["rejected"].  collide pairs
    share a coarse cell, repeat_2d pairs share a 2D keypoint, behind / outside points lie behind the
    camera / outside the image, and the items in empty_items project entirely outside.  exact=True
    uses an identity rotation, zero translation, unit depth and dyadic pixel coordinates, so every
    matmul of the reference is exact and its coordinates equal the restatement's bit for bit."""
    g = np.random.default_rng(seed)
    H0, W0 = src_hw
    w, h = img_resize
    item_seeds = list(item_seeds) if item_seeds is not None else [1000 * seed + k for k in range(n_items)]
    images, annos, rejected = [], [], 0
    for k in range(n_items):
        base = os.path.join(root, f"obj{k}")
        for d in ("color", "intrin_ba", "poses_ba", "anno_loftr", "anno_loftr_coarse", "anno3d"):
            os.makedirs(os.path.join(base, d), exist_ok=True)
        # a smooth image that fades to 0 at the borders: the reference's matmul grid differs from the
        # restatement's by up to ~1e-3 px where its terms cancel, which moves a bilinear sample by
        # (gradient) x (that distance); zero padding makes the border a step unless the image is 0 there
        yy, xx = np.mgrid[0:H0, 0:W0]
        ph = g.uniform(0, 2 * np.pi, 2)
        win = np.sin(np.pi * xx / (W0 - 1)) * np.sin(np.pi * yy / (H0 - 1))
        img = 255 * win * (0.6 + 0.25 * np.sin(xx / 90.0 + ph[0]) * np.cos(yy / 70.0 + ph[1]))
        color = os.path.join(base, "color", f"{k}.png")
        import cv2
        cv2.imwrite(color, np.clip(np.round(img), 0, 255).astype(np.uint8))
        if exact:
            R, t = np.eye(3), np.zeros(3)
            f, cxk, cyk = 1.0, 0.0, 0.0
        else:
            R, t = _rot(g, 25), np.array([g.uniform(-0.05, 0.05), g.uniform(-0.05, 0.05), g.uniform(0.55, 0.7)])
            f, cxk, cyk = g.uniform(450, 600), w / 2 + g.uniform(-8, 8), h / 2 + g.uniform(-8, 8)
        K = np.array([[f, 0, cxk], [0, f, cyk], [0, 0, 1.0]])
        pose = np.eye(4)
        pose[:3, :3], pose[:3, 3] = R, t
        np.savetxt(color.replace("/color/", "/intrin_ba/").replace(".png", ".txt"), K)
        np.savetxt(color.replace("/color/", "/poses_ba/").replace(".png", ".txt"), pose)
        Hs = _sample_homography(item_seeds[k], h, w) if warp else None
        R32, t32, K32 = R.astype(f32).astype(np.float64), t.astype(f32).astype(np.float64), K.astype(f32).astype(
            np.float64)

        def proj(X):
            cam = X @ R32.T + t32
            q = cam @ K32.T
            u, v = q[:, 0] / (q[:, 2] + 1e-6), q[:, 1] / (q[:, 2] + 1e-6)
            ok = _margin_ok(u, v, h, w)
            if Hs is not None:
                p = np.stack([u, v, np.ones_like(u)], 1) @ Hs.T
                ok &= _margin_ok(p[:, 0] / p[:, 2], p[:, 1] / p[:, 2], h, w)
            return ok

        def draw(n, kind):
            nonlocal rejected
            out = []
            while len(out) < n:
                if exact:
                    uv = g.integers(0, 4 * (min(w, h) + 40), (1, 2)) / 4.0 - 20 if kind != "in" else \
                        g.integers(4, 4 * (min(w, h) - 4), (1, 2)) / 4.0
                    X = np.array([[uv[0, 0], uv[0, 1], 1.0]]).astype(f32)
                else:
                    if kind == "behind":
                        uv, d = g.uniform(0, [w, h], (1, 2)), -g.uniform(0.2, 0.5)
                    elif kind == "outside":
                        uv, d = g.uniform(-0.6, 1.6, (1, 2)) * [w, h], g.uniform(0.5, 0.8)
                        if 0 <= uv[0, 0] < w and 0 <= uv[0, 1] < h:
                            continue
                    else:
                        uv, d = g.uniform(2, [w - 2, h - 2], (1, 2)), g.uniform(0.5, 0.8)
                    cam = d * (np.linalg.inv(K32) @ np.array([uv[0, 0], uv[0, 1], 1.0]))
                    X = (R32.T @ (cam - t32))[None].astype(f32)
                if proj(X.astype(np.float64))[0]:
                    out.append(X[0])
                else:
                    rejected += 1
            return np.array(out, dtype=f32).reshape(-1, 3)

        if k in empty_items:
            pts = draw(n_corr, "outside") if not exact else draw(n_corr, "out")
        else:
            parts = [draw(n_corr - behind - outside, "in"), draw(behind, "behind"), draw(outside, "outside")]
            pts = np.concatenate(parts)
        nc = len(pts)
        # collisions: the last points take the first ones' pixels moved by a quarter pixel (same
        # 8-px cell unless that breaks a margin, then the point is left as drawn) at another depth
        for c in range(min(collide, nc // 2)):
            X = pts[c].astype(np.float64)
            q = (X @ R32.T + t32) @ K32.T
            uv = q[:2] / (q[2] + 1e-6) + 0.25
            cam = 1.0 if exact else g.uniform(0.5, 0.8)
            Y = (R32.T @ (cam * (np.linalg.inv(K32) @ np.array([uv[0], uv[1], 1.0])) - t32))[None].astype(f32)
            if exact:
                Y = (pts[c] + f32(0.25))[None]
                Y[0, 2] = 1.0
            if proj(Y.astype(np.float64))[0]:
                pts[nc - 1 - c] = Y[0]
        extra = draw(n_3d - nc, "in") if n_3d > nc else np.zeros((0, 3), f32)
        kp3d = np.concatenate([pts, extra])[:n_3d]
        perm = g.permutation(n_3d)
        inv = np.argsort(perm)
        kp3d = kp3d[perm]
        a1 = inv[np.arange(nc)]
        n2 = n_2d or nc + 20
        a0 = g.permutation(n2)[:nc]
        for c in range(min(repeat_2d, nc // 2)):
            a0[nc - 1 - c] = a0[c]
        kp2d = g.uniform(0, [w, h], (n2, 2))
        anno2d = {"keypoints2d": kp2d.tolist(), "scores2d": g.uniform(0, 1, (n2, 1)).tolist(),
                  "assign_matrix": [a0.tolist(), a1.tolist()]}
        a2f = os.path.join(base, "anno_loftr", f"{k}.json")
        for path in (a2f, a2f.replace("/anno_loftr/", "/anno_loftr_coarse/")):
            with open(path, "w") as fh:
                json.dump(anno2d, fh)
        a3 = os.path.join(base, "anno3d", "anno_3d_average.npz")
        for path, dim in ((a3, 16), (a3.replace(".npz", "_coarse.npz"), 8)):
            np.savez(path, keypoints3d=kp3d, descriptors3d=g.standard_normal((dim, n_3d)).astype(f32),
                     scores3d=g.uniform(0, 1, (n_3d, 1)).astype(f32))
        images.append({"id": k, "img_file": color})
        annos.append({"image_id": k, "anno2d_file": a2f, "avg_anno3d_file": a3})
    anno_file = os.path.join(root, "train.json")
    with open(anno_file, "w") as fh:
        json.dump({"images": images, "annotations": annos}, fh)
    if rejected:
        print(f"make_case(seed={seed}): rejected {rejected} points within {MARGIN} px of a rounding boundary "
              f"or border threshold", file=sys.stderr)
    return {"anno_file": anno_file, "img_resize": list(img_resize), "shape3d": shape3d, "warp": warp,
            "item_seeds": item_seeds, "rejected": rejected, "n_items": n_items}
