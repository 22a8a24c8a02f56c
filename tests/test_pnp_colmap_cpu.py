"""CPU tests of the pycolmap branch of the pose stage: the oracle's Cauchy refinement
(oracle/pnp_colmap.py) ends at a stationary point of the per-point objective and differs from the
per-component scipy optimum and from least squares, and the host flow of ransac_PnP /
compute_query_pose_errors selects the solver from use_pycolmap_ransac (kernels stubbed)."""
import cv2
import numpy as np
import pytest
import scipy.optimize
import torch

from onepose_plus_plus_b200 import pnp
from oracle import pnp_colmap as opc

GPU_POSE_TOL = 1e-5   # what the GPU test allows between the device pose and the oracle's refinement


def _frames(n):
    b, p3, p2, K, _ = opc.heavy_tailed_frames(n, seed=11)
    for i in range(n):
        m = b == i
        yield K[i].astype(np.float64), p2[m].astype(np.float64), p3[m].astype(np.float64)


def _pose_gap(a, b):
    return np.abs(a[:, :3] - b[:, :3]).max(), np.linalg.norm(a[:, 3] - b[:, 3]) / np.linalg.norm(b[:, 3])


def test_cauchy_refine_is_stationary():
    for K, p2, p3 in _frames(3):
        pose0, mask = opc.ransac(K, p2, p3, 7.0)
        assert mask.sum() > 100
        ref = opc.cauchy_refine(K, p2, p3, pose0, mask)
        g0 = np.abs(opc.cauchy_gradient(K, p2, p3, pose0, mask)).max()
        g1 = np.abs(opc.cauchy_gradient(K, p2, p3, ref, mask)).max()
        assert g1 <= 1e-9 * g0, (g0, g1)
        assert opc.cauchy_cost(K, p2, p3, ref, mask) < opc.cauchy_cost(K, p2, p3, pose0, mask)


def test_per_point_optimum_differs_from_per_component_and_least_squares():
    """scipy's loss="cauchy" applies the loss to u and v separately; Ceres (and the device) per
    point.  On the heavy-tailed workload the two optima, and the least-squares pose, are further
    apart than the GPU test's tolerance, so that test tells them apart."""
    for K, p2, p3 in _frames(3):
        pose0, mask = opc.ransac(K, p2, p3, 7.0)
        ref = opc.cauchy_refine(K, p2, p3, pose0, mask)

        def fun(x):
            pose = np.concatenate([cv2.Rodrigues(x[:3])[0], x[3:, None]], 1)
            return opc.residuals(K, p2[mask], p3[mask], pose)[0].ravel()
        x0 = np.concatenate([cv2.Rodrigues(pose0[:, :3])[0].ravel(), pose0[:, 3]])
        x = scipy.optimize.least_squares(fun, x0, loss="cauchy", f_scale=1.0, xtol=1e-15, ftol=1e-15,
                                         gtol=1e-15).x
        per_component = np.concatenate([cv2.Rodrigues(x[:3])[0], x[3:, None]], 1)
        assert max(_pose_gap(per_component, ref)) > 2 * GPU_POSE_TOL
        assert max(_pose_gap(pose0, ref)) > 2 * GPU_POSE_TOL
        # the per-point objective tells them apart too
        assert opc.cauchy_cost(K, p2, p3, ref, mask) < opc.cauchy_cost(K, p2, p3, per_component, mask)


# ------------------------------------------------------------------------------------------------
# host flow (kernels stubbed)
# ------------------------------------------------------------------------------------------------
def _stub(monkeypatch, B, M):
    calls = []

    def ransac(m_bids, mkpts_3d, mkpts_2d, K, scale=1.0, reprojection_error=5.0, **kw):
        calls.append(kw)
        pose = torch.eye(4)[:3].repeat(B, 1, 1)
        homo = torch.eye(4).repeat(B, 1, 1)
        mask = torch.zeros(M, dtype=torch.bool)
        mask[::2] = True
        return {"pose": pose, "pose_homo": homo, "n_inliers": torch.zeros(B, dtype=torch.int32),
                "inlier_mask": mask, "state": torch.ones(B, dtype=torch.bool)}
    monkeypatch.setattr(pnp, "ransac_pnp_batched", ransac)
    return calls


def test_compute_query_pose_errors_selects_the_solver(monkeypatch):
    B, n = 3, 6
    data0 = {"m_bids": torch.arange(B).repeat_interleave(n), "mkpts_3d_db": torch.zeros(B * n, 3),
             "mkpts_query_f": torch.zeros(B * n, 2), "query_intrinsic": torch.eye(3).repeat(B, 1, 1),
             "query_pose_gt": torch.eye(4).repeat(B, 1, 1)}
    base = {"pnp_reprojection_error": 7, "point_cloud_rescale": 1000}
    for cfg, colmap in ((dict(base, use_pycolmap_ransac=True), True), (dict(base, use_pycolmap_ransac=False), False),
                        (base, False)):
        calls = _stub(monkeypatch, B, B * n)
        data = dict(data0)
        pnp.compute_query_pose_errors(data, cfg)
        assert len(calls) == 1
        assert calls[0] == ({"solver": "colmap"} if colmap else {})
        for inl in data["inliers"]:
            assert inl.tolist() == ([0, 2, 4] if colmap else [[0], [2], [4]])
            assert inl.ndim == (1 if colmap else 2)


def test_bad_arguments_raise_before_any_launch(monkeypatch):
    def no_launch(*a, **k):
        raise AssertionError("launched")
    monkeypatch.setattr(pnp._lib, "call", no_launch)
    K, p2, p3 = np.eye(3), np.zeros((10, 2)), np.zeros((10, 3))
    for hw in (None, [512], [1, 2, 3]):
        with pytest.raises(ValueError, match="img_hw"):
            pnp.ransac_PnP(K, p2, p3, img_hw=hw, use_pycolmap_ransac=True)
    with pytest.raises(ValueError, match="solver"):
        pnp.ransac_pnp_batched(torch.zeros(10, dtype=torch.int64), torch.zeros(10, 3), torch.zeros(10, 2),
                               torch.eye(3)[None], solver="x")
