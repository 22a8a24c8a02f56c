"""Pose from the matches on the device — drop-in front end for the reference's per-frame CPU
RANSAC-PnP (src/utils/metric_utils.py:121-204 ``ransac_PnP``, :207-292
``compute_query_pose_errors``; demo.py:132) and for its LINEMOD pose metrics (:31-88
``projection_2d_error`` / ``add_metric``, the ``eval_ADD_metric`` branch :233-289).

The reference copies the match lists to the host after every forward and runs
``cv2.solvePnPRansac(EPnP, iterationsCount=10000)`` frame by frame; at the matcher's GPU
throughput that CPU stage is the whole per-frame latency.  Here the batch is solved by one kernel
launch (``opp_pnp_ransac``: one CTA per image, P3P hypotheses + inlier scoring + Gauss-Newton
refinement on the inliers) reading ``m_bids / mkpts_3d_db / mkpts_query_f`` where the matcher left
them; nothing synchronises until the caller reads the poses.  The ADD / ADD-S / proj2D metrics of
the batch follow in one more call (``opp_pose_metrics``) that reads the poses where the PnP
launch left them; ADD-S, a per-frame cKDTree in the reference, is a brute-force nearest-neighbour
search on the device.
"""
import collections
import ctypes
import logging
import os
import os.path as osp

import numpy as np
import torch

from . import _lib, cad

__all__ = ["ransac_pnp_batched", "pose_metrics_batched", "ransac_PnP", "compute_query_pose_errors",
           "query_pose_error"]

logger = logging.getLogger(__name__)


SOLVERS = ("opencv", "colmap")


def ransac_pnp_batched(m_bids, mkpts_3d, mkpts_2d, intrinsics, scale=1.0, reprojection_error=5.0,
                       hypotheses=1024, seed=0, refine_rounds=3, solver="opencv"):
    """m_bids int64 [M] ascending, mkpts_3d fp32 [M, 3], mkpts_2d fp32 [M, 2], intrinsics fp32
    [B, 3, 3] (all CUDA).  Returns a dict of CUDA tensors: pose [B, 3, 4], pose_homo [B, 4, 4],
    n_inliers int32 [B], inlier_mask bool [M], state bool [B].  No host synchronisation.

    solver="opencv" (``opp_pnp_ransac``) is the reference's cv2.solvePnPRansac branch: full K, the
    points multiplied by ``scale`` and t divided by it.  solver="colmap" (``opp_pnp_ransac_colmap``)
    is its ``use_pycolmap_ransac`` branch: a SIMPLE_PINHOLE camera (f = K[0, 0]; K[1, 1] is not
    read), ``scale`` not applied, LO-RANSAC with ``refine_rounds`` local-optimisation rounds, then
    the pose refined on the RANSAC inliers under the per-point Cauchy loss; inlier_mask and
    n_inliers are those of the RANSAC model."""
    if solver not in SOLVERS:
        raise ValueError(f"solver must be one of {SOLVERS}, got {solver!r}")
    K = intrinsics
    if not K.is_cuda:
        raise RuntimeError("ransac_pnp_batched has no CPU path: pass CUDA tensors")
    if K.dim() != 3 or K.shape[1:] != (3, 3):
        raise ValueError(f"intrinsics must be [B, 3, 3], got {tuple(K.shape)}")
    B, M = K.shape[0], m_bids.numel()
    if mkpts_3d.shape != (M, 3) or mkpts_2d.shape != (M, 2):
        raise ValueError("mkpts_3d / mkpts_2d must be [M, 3] / [M, 2] with M = len(m_bids)")
    dev = K.device
    with torch.cuda.device(dev):
        K32 = K.to(torch.float32).contiguous()
        p3 = mkpts_3d.to(torch.float32).contiguous()
        p2 = mkpts_2d.to(torch.float32).contiguous()
        mb = m_bids.to(torch.int64).contiguous()
        pose = torch.empty((B, 3, 4), dtype=torch.float32, device=dev)
        n_inl = torch.empty(B, dtype=torch.int32, device=dev)
        status = torch.empty(B, dtype=torch.int32, device=dev)
        mask = torch.empty(max(M, 1), dtype=torch.uint8, device=dev)
        if solver == "colmap":
            _lib.call("opp_pnp_ransac_colmap", _lib.ptr(p3), _lib.ptr(p2), _lib.ptr(mb), M, _lib.ptr(K32), B,
                      float(reprojection_error), int(hypotheses), ctypes.c_uint(seed & 0xFFFFFFFF),
                      int(refine_rounds), _lib.ptr(pose), _lib.ptr(n_inl), _lib.ptr(mask), _lib.ptr(status),
                      _lib.stream())
        else:
            _lib.call("opp_pnp_ransac", _lib.ptr(p3), _lib.ptr(p2), _lib.ptr(mb), M, _lib.ptr(K32), B,
                      float(scale), float(reprojection_error), int(hypotheses), ctypes.c_uint(seed & 0xFFFFFFFF),
                      int(refine_rounds), _lib.ptr(pose), _lib.ptr(n_inl), _lib.ptr(mask), _lib.ptr(status),
                      _lib.stream())
        homo = torch.zeros((B, 4, 4), dtype=torch.float32, device=dev)
        homo[:, :3] = pose
        homo[:, 3, 3] = 1.0
    return {"pose": pose, "pose_homo": homo, "n_inliers": n_inl, "inlier_mask": mask[:M].bool(),
            "state": status.bool()}


def pose_metrics_batched(verts, pose_pred, pose_gt, K_origin, symmetric, diameter):
    """LINEMOD metrics of B frames of one object model (metric_utils.py:31-88), one
    ``opp_pose_metrics`` call.  verts [V, 3] model points; pose_pred, pose_gt [B, 3, 4] or [B, 4, 4];
    K_origin [B, 3, 3] the original intrinsics (all CUDA); symmetric: one bool for every frame or
    B of them (ADD-S instead of ADD); diameter: a number or a CUDA tensor [B].  Returns CUDA tensors:
    add_dist fp64 [B] (ADD or ADD-S mean distance), add_pass bool [B] = add_dist < 0.1 * diameter,
    proj2d fp64 [B] (mean pixel distance).  No host synchronisation."""
    if not all(torch.is_tensor(t) and t.is_cuda for t in (verts, pose_pred, pose_gt, K_origin)):
        raise RuntimeError("pose_metrics_batched has no CPU path: pass CUDA tensors")
    if verts.dim() != 2 or verts.shape[1] != 3 or verts.shape[0] == 0:
        raise ValueError(f"verts must be a non-empty [V, 3] model, got {tuple(verts.shape)}")
    B = pose_pred.shape[0]
    for name, t in (("pose_pred", pose_pred), ("pose_gt", pose_gt)):
        if t.dim() != 3 or t.shape[0] != B or tuple(t.shape[1:]) not in ((3, 4), (4, 4)):
            raise ValueError(f"{name} must be [B, 3, 4] or [B, 4, 4] with B = {B}, got {tuple(t.shape)}")
    if tuple(K_origin.shape) != (B, 3, 3):
        raise ValueError(f"K_origin must be [{B}, 3, 3], got {tuple(K_origin.shape)}")
    dev = verts.device
    if torch.is_tensor(symmetric) and symmetric.is_cuda:
        sym = symmetric.to(torch.uint8)
    elif isinstance(symmetric, (bool, int, np.bool_)):
        sym = torch.full((B,), int(bool(symmetric)), dtype=torch.uint8, device=dev)
    else:
        sym = torch.as_tensor(np.asarray(symmetric, dtype=bool), dtype=torch.uint8).to(dev)
    if tuple(sym.shape) != (B,):
        raise ValueError(f"symmetric must be one flag or {B} of them, got shape {tuple(sym.shape)}")
    if not torch.is_tensor(diameter):
        # numpy arithmetic as in add_metric: a float32 diameter (model_diameter_from_bbox) gives a
        # float32 threshold
        thr = float(np.asarray(diameter)[()] * 0.1)
    elif tuple(diameter.shape) in ((), (B,)):
        thr = diameter * 0.1
    else:
        raise ValueError(f"diameter must be a number or [{B}], got {tuple(diameter.shape)}")
    if B == 0:
        empty = torch.empty(0, dtype=torch.float64, device=dev)
        return {"add_dist": empty, "add_pass": empty.bool(), "proj2d": empty.clone()}
    with torch.cuda.device(dev):
        v = verts.to(torch.float32).contiguous()
        P = pose_pred[:, :3].to(torch.float32).contiguous()
        G = pose_gt[:, :3].to(torch.float32).contiguous()
        K = K_origin.to(torch.float32).contiguous()
        sym = sym.contiguous()
        V = v.shape[0]
        nbytes = _lib.load().opp_pose_metrics_scratch_bytes(V, B)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        add = torch.empty(B, dtype=torch.float64, device=dev)
        proj = torch.empty(B, dtype=torch.float64, device=dev)
        _lib.call("opp_pose_metrics", _lib.ptr(v), V, _lib.ptr(P), _lib.ptr(G), _lib.ptr(K), _lib.ptr(sym), B,
                  _lib.ptr(scratch), nbytes, _lib.ptr(add), _lib.ptr(proj), _lib.stream())
    return {"add_dist": add, "add_pass": add < thr, "proj2d": proj}


# device copies of CAD model vertices, keyed by absolute path (and mtime / size, so that a model
# file rewritten in place is read again): the reference flow calls once per frame
_MODEL_CACHE = collections.OrderedDict()
_MODEL_CACHE_SIZE = 16


def _model_vertices(model_path, device):
    path = osp.abspath(model_path)
    st = os.stat(path)
    key = (path, st.st_mtime_ns, st.st_size, str(device))
    hit = _MODEL_CACHE.get(key)
    if hit is None:
        verts, bbox = cad.load_points_from_cad(path)
        hit = (torch.from_numpy(verts).to(device), bbox)
        _MODEL_CACHE[key] = hit
        while len(_MODEL_CACHE) > _MODEL_CACHE_SIZE:
            _MODEL_CACHE.popitem(last=False)
    else:
        _MODEL_CACHE.move_to_end(key)
    return hit


def _add_metric_models(image_paths, batch, device):
    """The model lookup of metric_utils.py:236-252 for every frame: [(frame indices, vertices,
    diameter, symmetric flags)] per model file, or None (after logging) when a model is missing."""
    if isinstance(image_paths, str):
        image_paths = [image_paths] * batch
    image_paths = list(image_paths)
    if len(image_paths) != batch:
        raise ValueError(f"query_image_path has {len(image_paths)} entries for {batch} frames")
    groups = collections.OrderedDict()
    for b, image_path in enumerate(image_paths):
        obj_dir = image_path.rsplit("/", 3)[0]
        model_path = osp.join(obj_dir, "model_eval.ply")
        if not osp.exists(model_path):
            model_path = osp.join(obj_dir, "model.ply")
        if not osp.exists(model_path):
            logger.error(f"want to eval add metric, however model_eval.ply path:{model_path} not exists!")
            return None
        g = groups.setdefault(model_path, (obj_dir, [], []))
        g[1].append(b)
        g[2].append(("0810-" in image_path) or ("0811-" in image_path))   # symmetric LINEMOD objects
    out = []
    for model_path, (obj_dir, idx, sym) in groups.items():
        verts, bbox = _model_vertices(model_path, device)
        diameter_path = osp.join(obj_dir, "diameter.txt")
        diameter = np.loadtxt(diameter_path) if osp.exists(diameter_path) else cad.model_diameter_from_bbox(bbox)
        out.append((idx, verts, diameter, sym))
    return out


def ransac_PnP(K, pts_2d, pts_3d, scale=1, pnp_reprojection_error=5, img_hw=None,
               use_pycolmap_ransac=False):
    """Signature and return values of the reference's ``ransac_PnP`` (metric_utils.py:121-204) for
    one frame, numpy in / numpy out: (pose [3,4], pose_homo [4,4], inlier indices, state).

    ``use_pycolmap_ransac=True`` runs the pycolmap branch (``ransac_pnp_batched(solver="colmap")``):
    ``img_hw`` must then be a pair, as the reference asserts (it does not change the estimate),
    ``scale`` is not applied, and the inliers are 1-D int64 indices.  Otherwise the cv2 branch runs
    and the inliers are ``[n, 1]`` int32 like cv2's.  A frame that fails returns the identity pose
    and ``state`` False in both modes; pycolmap itself reports ``success: False`` there and the
    reference then raises ``KeyError`` on ``ret["qvec"]``."""
    if use_pycolmap_ransac and (img_hw is None or len(img_hw) != 2):
        raise ValueError(f"use_pycolmap_ransac needs img_hw = (height, width), got {img_hw!r}")
    dev = torch.device("cuda", torch.cuda.current_device())
    p2 = torch.as_tensor(np.ascontiguousarray(pts_2d), dtype=torch.float32, device=dev).reshape(-1, 2)
    p3 = torch.as_tensor(np.ascontiguousarray(pts_3d), dtype=torch.float32, device=dev).reshape(-1, 3)
    Kt = torch.as_tensor(np.asarray(K), dtype=torch.float32, device=dev).reshape(1, 3, 3)
    r = ransac_pnp_batched(torch.zeros(p2.shape[0], dtype=torch.int64, device=dev), p3, p2, Kt, scale=scale,
                           reprojection_error=pnp_reprojection_error,
                           solver="colmap" if use_pycolmap_ransac else "opencv")
    if not bool(r["state"][0].item()):
        return np.eye(4)[:3], np.eye(4), np.array([]).astype(bool), False
    if use_pycolmap_ransac:
        inliers = torch.nonzero(r["inlier_mask"])[:, 0].cpu().numpy()   # np.arange(n)[mask] like the reference
    else:
        inliers = torch.nonzero(r["inlier_mask"]).cpu().numpy().astype(np.int32)   # [n, 1] like cv2
    return (r["pose"][0].double().cpu().numpy(), r["pose_homo"][0].double().cpu().numpy(), inliers, True)


def query_pose_error(pose_pred, pose_gt, unit="m"):
    """metric_utils.py:91-118: (angular error in degrees, translation error in cm)."""
    pose_pred, pose_gt = np.asarray(pose_pred)[:3], np.asarray(pose_gt)[:3]
    factor = {"m": 100.0, "cm": 1.0, "mm": 0.1}
    if unit not in factor:
        raise NotImplementedError
    t_err = np.linalg.norm(pose_pred[:, 3] - pose_gt[:, 3]) * factor[unit]
    trace = min(np.trace(pose_pred[:, :3] @ pose_gt[:, :3].T), 3.0)
    return np.rad2deg(np.arccos((trace - 1.0) / 2.0)), t_err


@torch.no_grad()
def compute_query_pose_errors(data, configs, training=False):
    """``compute_query_pose_errors`` (metric_utils.py:207-292) with the PnP stage on the device: all
    frames of the batch are solved by one launch, then ONE device->host copy brings back the poses
    and inlier masks.  Writes R_errs, t_errs, inliers, pose_pred (and the empty *_c lists the
    reference initialises).  ``configs["use_pycolmap_ransac"]`` true selects the pycolmap solver
    (``solver="colmap"``, see ``ransac_pnp_batched``; ``point_cloud_rescale`` is then not applied and
    ``inliers`` holds 1-D index arrays); ``q_hw_i`` / ``query_image_scale``, which the reference
    reads only to build pycolmap's image size, are not needed.

    With ``configs["eval_ADD_metric"]`` true and ``training`` false (the LINEMOD evaluation), also
    writes ``data["ADD"]`` (one bool per frame: ADD, or ADD-S for the symmetric objects 0810 / 0811,
    below 0.1 x the model diameter) and ``data["proj2D"]`` (one float per frame: mean reprojection
    distance of the model under ``query_intrinsic_origin``), scored at the pose this function
    computes (identity for a failed frame, like the reference).  The model is
    ``<image_path.rsplit('/', 3)[0]>/model_eval.ply``, else ``model.ply`` beside it; the diameter is
    ``diameter.txt`` there, else the model's bounding-box diagonal.  ``data["query_image_path"]`` is
    one path for the whole batch or one per frame; frames of the same model are scored by one
    ``pose_metrics_batched`` call.  If a model file is missing the error is logged and neither key
    is written."""
    unit = configs["model_unit"] if "model_unit" in configs else "m"
    K = data["query_intrinsic"]
    dev = data["m_bids"].device
    colmap = bool(configs.get("use_pycolmap_ransac", False))
    kw = {"solver": "colmap"} if colmap else {}
    r = ransac_pnp_batched(data["m_bids"], data["mkpts_3d_db"], data["mkpts_query_f"], K.to(dev),
                           scale=configs.get("point_cloud_rescale", 1.0),
                           reprojection_error=configs["pnp_reprojection_error"], **kw)
    metrics = None
    if "eval_ADD_metric" in configs and configs["eval_ADD_metric"] and not training:
        models = _add_metric_models(data["query_image_path"], K.shape[0], dev)
        if models is not None:
            add_pass = torch.empty(K.shape[0], dtype=torch.bool, device=dev)
            proj2d = torch.empty(K.shape[0], dtype=torch.float64, device=dev)
            K_origin = data["query_intrinsic_origin"].to(dev)
            pose_gt = data["query_pose_gt"].to(dev)
            for idx, verts, diameter, sym in models:
                sel = torch.tensor(idx, dtype=torch.int64, device=dev)
                m = pose_metrics_batched(verts, r["pose"][sel], pose_gt[sel], K_origin[sel], sym, diameter)
                add_pass[sel] = m["add_pass"]
                proj2d[sel] = m["proj2d"]
            metrics = (add_pass, proj2d)
    poses = r["pose_homo"].double().cpu().numpy()
    state = r["state"].cpu().numpy()
    mask = r["inlier_mask"].cpu().numpy()
    m_bids = data["m_bids"].cpu().numpy()
    gt = data["query_pose_gt"].cpu().numpy()
    data.update({"R_errs": [], "t_errs": [], "inliers": [], "R_errs_c": [], "t_errs_c": [], "inliers_c": []})
    if metrics is not None:
        data.update({"ADD": [bool(x) for x in metrics[0].cpu().tolist()], "proj2D": metrics[1].cpu().tolist()})
    for b in range(K.shape[0]):
        if not state[b]:
            data["R_errs"].append(np.inf)
            data["t_errs"].append(np.inf)
            data["inliers"].append(np.array([]).astype(bool))
            continue
        R_err, t_err = query_pose_error(poses[b][:3], gt[b], unit=unit)
        data["R_errs"].append(R_err)
        data["t_errs"].append(t_err)
        idx = np.nonzero(mask[m_bids == b])[0]
        data["inliers"].append(idx if colmap else idx[:, None].astype(np.int32))
    data["pose_pred"] = poses
