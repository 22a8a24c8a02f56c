"""NumPy restatement of the sparse ground truth of training (onepose_plus_plus_b200/train_gt.py):

  * assign_list      — the correspondences OnePosePlusDataset.build_assignmatrix
                       (src/datasets/OnePosePlus_dataset.py:174-236) writes into its two matrices, as
                       a list sorted by (i, j)
  * lookup           — fine_location_matrix_gt[b, i, j] from the list (-50 where there is none)
  * fine_supervision — src/models/OnePosePlus/utils/fine_supervision.py:18-28 on that lookup, fp32,
                       one rounding per operation in the reference's order

and the two reference functions imported live (reference_*), which tests/test_train_gt_cpu.py pins
the restatement to.  make_case() is the seeded input of tests/golden/reference/train_gt.npz
(oracle/make_train_gt_golden.py).
"""
import sys
import types

import numpy as np

FINE_FILL = np.float32(-50.0)
RESOLUTION = (8, 2)          # loftr_backbone.resolution


def assign_list(keypoints2d_coarse, keypoints2d_fine, assign_matrix, shape3d, n_grid, w_c, query_img_scale,
                coarse_scale):
    """(i_ids, j_ids int64 [n], fine_xy fp32 [n, 2]) sorted by (i, j): what build_assignmatrix sets to 1
    in conf_matrix and writes into fine_location_matrix.  assign_matrix int [2, k] = (2D keypoint, 3D
    point); a 3D point >= shape3d and a cell index > n_grid drop out; of two correspondences of one
    (i, j) the later one's location stays."""
    am = np.asarray(assign_matrix).astype(np.int64)
    am = am[:, am[1] < shape3d]
    coarse = np.asarray(keypoints2d_coarse, dtype=np.float32)[am[0]]
    fine = np.asarray(keypoints2d_fine, dtype=np.float32)[am[0]]
    scale = np.asarray(query_img_scale, dtype=np.float32)[[1, 0]]
    cell = np.round(coarse / scale * np.float32(coarse_scale))     # fp32, half to even as torch.round
    j = (cell[:, 1] * w_c + cell[:, 0]).astype(np.int64)
    ok = ~(j > n_grid)
    i, j, fine = am[1][ok], j[ok], fine[ok]
    key = i * n_grid + j
    order = np.argsort(key, kind="stable")
    key = key[order]
    last = np.ones(len(key), dtype=bool)
    last[:-1] = key[1:] != key[:-1]
    order = order[last]
    return i[order], j[order], fine[order]


def lookup(gt, matches, shape):
    """gt = (b, i, j, fine_xy) sorted by (b, i, j); matches = (b, i, j) -> fp32 [M, 2]"""
    B, L, S = shape
    gb, gi, gj, xy = (np.asarray(t) for t in gt)
    mb, mi, mj = (np.asarray(t).astype(np.int64) for t in matches)
    key = (gb.astype(np.int64) * L + gi) * S + gj
    want = (mb * L + mi) * S + mj
    out = np.full((len(want), 2), FINE_FILL, dtype=np.float32)
    if len(key):
        pos = np.minimum(np.searchsorted(key, want), len(key) - 1)
        hit = key[pos] == want
        out[hit] = xy[pos[hit]]
    return out


def fine_supervision(gt, matches, shape, w_c, window_size, query_image_scale=None, resolution=RESOLUTION):
    """expec_f_gt fp32 [M, 2].  Without query_image_scale the reference uses the FINE resolution as the
    coarse scale (fine_supervision.py:18, the `else` of the conditional); reproduced."""
    f32 = np.float32
    coarse_res, fine_res = resolution
    radius = window_size // 2
    mb, _, mj = (np.asarray(t).astype(np.int64) for t in matches)
    loc = lookup(gt, matches, shape)
    cell = np.stack([mj % w_c, mj // w_c], 1)
    if query_image_scale is not None:
        s = np.asarray(query_image_scale, dtype=f32)[mb][:, [1, 0]]
        coarse_scale, fine_scale = f32(coarse_res) * s, f32(fine_res) * s
        mk = cell.astype(f32) * coarse_scale
    else:
        fine_scale = f32(fine_res)
        mk = (cell * fine_res).astype(f32)
    return ((loc - mk) / fine_scale / f32(radius)).astype(f32)


def config(window_size=5, resolution=RESOLUTION):
    """the keys fine_supervision reads from the experiment config"""
    return {"OnePosePlus": {"loftr_backbone": {"resolution": list(resolution)},
                            "loftr_fine": {"window_size": window_size}}}


def make_case(seed=0, B=2, L=300, hc=12, wc=16, n_gt=70, n_pred=40, with_scale=False):
    """Seeded ground-truth list and matches: one 3D point per chosen cell, locations around the cell
    origin (some outside the fine window), matches = a subset of the ground truth + predictions that
    are not ground truth.  Returns a dict of numpy arrays."""
    g = np.random.default_rng(seed)
    S = hc * wc
    gb, gi, gj = [], [], []
    for b in range(B):
        n = n_gt if b else n_gt // 2
        i = np.sort(g.choice(L, n, replace=False))
        j = g.choice(S, n, replace=False)
        gb.append(np.full(n, b)), gi.append(i), gj.append(j)
    gb, gi, gj = (np.concatenate(t).astype(np.int64) for t in (gb, gi, gj))
    scale = (np.array([[1.0, 1.0], [1.25, 0.75]], dtype=np.float32)[:B] if with_scale else None)
    cell = np.stack([gj % wc, gj // wc], 1).astype(np.float32) * 8
    if with_scale:
        cell = cell * scale[gb][:, [1, 0]]
    xy = (cell + g.uniform(-6, 10, cell.shape)).astype(np.float32)
    take = g.choice(len(gb), n_pred, replace=False)
    pb, pi, pj = g.integers(0, B, n_pred), g.integers(0, L, n_pred), g.integers(0, S, n_pred)
    mb, mi, mj = (np.concatenate(t).astype(np.int64) for t in ((gb[take], pb), (gi[take], pi), (gj[take], pj)))
    return {"shape": np.array([B, L, S]), "hw_c": np.array([hc, wc]), "b_ids": gb, "i_ids": gi, "j_ids": gj,
            "fine_xy": xy, "m_b": mb, "m_i": mi, "m_j": mj, **({"scale": scale} if with_scale else {})}


# ---- the reference's own functions, imported live (build container only) --------------------------

def reference_fine_supervision(data, cfg):
    from . import ref_shims
    ref_shims.install()
    from src.models.OnePosePlus.utils.fine_supervision import fine_supervision as ref   # type: ignore
    ref(data, cfg)
    return data["expec_f_gt"]


def reference_build_assignmatrix(keypoints2d_coarse, keypoints2d_fine, assign_matrix, shape3d, n_grid, w_c,
                                 query_img_scale, coarse_scale):
    """OnePosePlusDataset.build_assignmatrix on a stand-in `self` with the attributes it reads.  The
    dataset module imports packages this image lacks (pycocotools, h5py, three kornia functions);
    none of them is touched by build_assignmatrix, so empty stand-ins are registered when missing."""
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
    kornia = sys.modules["kornia"]
    for a in ("homography_warp", "normalize_homography", "normal_transform_pixel"):
        if not hasattr(kornia, a):
            setattr(kornia, a, None)
    from src.datasets.OnePosePlus_dataset import OnePosePlusDataset   # type: ignore
    me = types.SimpleNamespace(shape3d=shape3d, n_query_coarse_grid=n_grid, w_c=w_c,
                               query_img_scale=query_img_scale, coarse_scale=coarse_scale)
    return OnePosePlusDataset.build_assignmatrix(me, keypoints2d_coarse, keypoints2d_fine, assign_matrix, pad=True)
