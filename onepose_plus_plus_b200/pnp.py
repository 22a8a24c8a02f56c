"""Pose from the matches on the device — drop-in front end for the reference's per-frame CPU
RANSAC-PnP (src/utils/metric_utils.py:121-204 ``ransac_PnP``, :207-292
``compute_query_pose_errors``; demo.py:132).

The reference copies the match lists to the host after every forward and runs
``cv2.solvePnPRansac(EPnP, iterationsCount=10000)`` frame by frame; at the matcher's GPU
throughput that CPU stage is the whole per-frame latency.  Here the batch is solved by one kernel
launch (``opp_pnp_ransac``: one CTA per image, P3P hypotheses + inlier scoring + Gauss-Newton
refinement on the inliers) reading ``m_bids / mkpts_3d_db / mkpts_query_f`` where the matcher left
them; nothing synchronises until the caller reads the poses.
"""
import ctypes

import numpy as np
import torch

from . import _lib

__all__ = ["ransac_pnp_batched", "ransac_PnP", "compute_query_pose_errors", "query_pose_error"]


def ransac_pnp_batched(m_bids, mkpts_3d, mkpts_2d, intrinsics, scale=1.0, reprojection_error=5.0,
                       hypotheses=1024, seed=0, refine_rounds=3):
    """m_bids int64 [M] ascending, mkpts_3d fp32 [M, 3], mkpts_2d fp32 [M, 2], intrinsics fp32
    [B, 3, 3] (all CUDA).  Returns a dict of CUDA tensors: pose [B, 3, 4], pose_homo [B, 4, 4],
    n_inliers int32 [B], inlier_mask bool [M], state bool [B].  No host synchronisation."""
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
        _lib.call("opp_pnp_ransac", _lib.ptr(p3), _lib.ptr(p2), _lib.ptr(mb), M, _lib.ptr(K32), B,
                  float(scale), float(reprojection_error), int(hypotheses), ctypes.c_uint(seed & 0xFFFFFFFF),
                  int(refine_rounds), _lib.ptr(pose), _lib.ptr(n_inl), _lib.ptr(mask), _lib.ptr(status),
                  _lib.stream())
        homo = torch.zeros((B, 4, 4), dtype=torch.float32, device=dev)
        homo[:, :3] = pose
        homo[:, 3, 3] = 1.0
    return {"pose": pose, "pose_homo": homo, "n_inliers": n_inl, "inlier_mask": mask[:M].bool(),
            "state": status.bool()}


def ransac_PnP(K, pts_2d, pts_3d, scale=1, pnp_reprojection_error=5, img_hw=None,
               use_pycolmap_ransac=False):
    """Signature and return values of the reference's ``ransac_PnP`` (metric_utils.py:121-204) for
    one frame, numpy in / numpy out: (pose [3,4], pose_homo [4,4], inlier indices, state)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    p2 = torch.as_tensor(np.ascontiguousarray(pts_2d), dtype=torch.float32, device=dev).reshape(-1, 2)
    p3 = torch.as_tensor(np.ascontiguousarray(pts_3d), dtype=torch.float32, device=dev).reshape(-1, 3)
    Kt = torch.as_tensor(np.asarray(K), dtype=torch.float32, device=dev).reshape(1, 3, 3)
    r = ransac_pnp_batched(torch.zeros(p2.shape[0], dtype=torch.int64, device=dev), p3, p2, Kt, scale=scale,
                           reprojection_error=pnp_reprojection_error)
    if not bool(r["state"][0].item()):
        return np.eye(4)[:3], np.eye(4), np.array([]).astype(bool), False
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
    reference initialises).  The CAD-model ADD / proj2D metrics (LINEMOD evaluation files) are not
    part of this path."""
    unit = configs["model_unit"] if "model_unit" in configs else "m"
    K = data["query_intrinsic"]
    r = ransac_pnp_batched(data["m_bids"], data["mkpts_3d_db"], data["mkpts_query_f"], K.to(data["m_bids"].device),
                           scale=configs.get("point_cloud_rescale", 1.0),
                           reprojection_error=configs["pnp_reprojection_error"])
    poses = r["pose_homo"].double().cpu().numpy()
    state = r["state"].cpu().numpy()
    mask = r["inlier_mask"].cpu().numpy()
    m_bids = data["m_bids"].cpu().numpy()
    gt = data["query_pose_gt"].cpu().numpy()
    data.update({"R_errs": [], "t_errs": [], "inliers": [], "R_errs_c": [], "t_errs_c": [], "inliers_c": []})
    for b in range(K.shape[0]):
        if not state[b]:
            data["R_errs"].append(np.inf)
            data["t_errs"].append(np.inf)
            data["inliers"].append(np.array([]).astype(bool))
            continue
        R_err, t_err = query_pose_error(poses[b][:3], gt[b], unit=unit)
        data["R_errs"].append(R_err)
        data["t_errs"].append(t_err)
        data["inliers"].append(np.nonzero(mask[m_bids == b])[0][:, None].astype(np.int32))
    data["pose_pred"] = poses
