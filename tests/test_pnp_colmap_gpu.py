"""pytest -m gpu: the pycolmap branch of the pose stage (opp_pnp_ransac_colmap through
pnp.ransac_pnp_batched(solver="colmap"), ransac_PnP(use_pycolmap_ransac=True) and
compute_query_pose_errors) against the CPU oracle oracle/pnp_colmap.py on planted LINEMOD frames
(fx != fy, 30 % outliers, heavy-tailed inlier noise).  Sampling is random in both; what must agree
is the inlier set of the locally optimised RANSAC under the SIMPLE_PINHOLE camera and the
minimiser of the per-point Cauchy cost on it."""
import os

import numpy as np
import pytest
import torch

from onepose_plus_plus_b200 import pnp
from oracle import pnp as opnp
from oracle import pnp_colmap as opc
from oracle import pose_metrics as opm

pytestmark = pytest.mark.gpu

THR = 7.0


def _cuda(b, p3, p2, K):
    return [torch.as_tensor(x, device="cuda") for x in (b, p3, p2, K)]


def _gap(a, b):
    return np.abs(a[:, :3] - b[:, :3]).max(), np.linalg.norm(a[:, 3] - b[:, 3]) / np.linalg.norm(b[:, 3])


@pytest.mark.parametrize("batch", [8, 64])
def test_planted_frames_match_oracle(batch):
    b, p3, p2, K, gt = opc.heavy_tailed_frames(batch, seed=batch)
    r = pnp.ransac_pnp_batched(*_cuda(b, p3, p2, K), reprojection_error=THR, solver="colmap")
    torch.cuda.synchronize()
    assert r["state"].all().item()
    pose = r["pose"].double().cpu().numpy()
    mask = r["inlier_mask"].cpu().numpy()
    n_inl = r["n_inliers"].cpu().numpy()
    worst = [0.0] * 4
    for i in range(batch):
        m = b == i
        Ki, q2, q3 = K[i].astype(np.float64), p2[m].astype(np.float64), p3[m].astype(np.float64)
        # the full oracle: its own RANSAC + LO inlier set, the Cauchy optimum on it
        pose_o, mask_o = opc.ransac(Ki, q2, q3, THR)
        ref = opc.cauchy_refine(Ki, q2, q3, pose_o, mask_o)
        got = mask[m]
        assert int(n_inl[i]) == int(got.sum())
        assert (got ^ mask_o).sum() <= max(2, int(mask_o.sum()) // 100), (i, int(mask_o.sum()), int(got.sum()))
        dR, dt = _gap(pose[i], ref)
        assert dR <= 1e-3 and dt <= 1e-3, (i, dR, dt)
        # on the device's own inlier set: the Cauchy optimum is where the device ended
        ref_d = opc.cauchy_refine(Ki, q2, q3, pose[i], got)
        dR_d, dt_d = _gap(pose[i], ref_d)
        assert dR_d <= 1e-5 and dt_d <= 1e-5, (i, dR_d, dt_d)
        # cost: the fp32 rounding of the output pose alone raises the cost of the optimum by
        # 4e-8 to 7e-8 relative on this workload, so the comparison is made at 1e-6
        c_dev, c_opt = opc.cauchy_cost(Ki, q2, q3, pose[i], got), opc.cauchy_cost(Ki, q2, q3, ref_d, got)
        assert c_dev <= c_opt * (1 + 1e-6), (i, c_dev / c_opt - 1)
        worst = [max(w, x) for w, x in zip(worst, (dR, dt, dR_d, dt_d))]
        assert np.abs(pose[i][:, :3] - gt[i][:, :3]).max() < 5e-3
    print(f"batch {batch}: oracle |dR| {worst[0]:.2e} |dt|/|t| {worst[1]:.2e}; "
          f"own inlier set |dR| {worst[2]:.2e} |dt|/|t| {worst[3]:.2e}")


def test_degenerate_frames_and_determinism():
    b, p3, p2, K, _ = opnp.synthetic_frames(4, n_matches=120, outlier_frac=0.0, seed=5)
    # frame 1 keeps 3 matches (below the minimal sample), frame 2 none, frame 3 exactly 4
    keep = np.ones(len(b), dtype=bool)
    keep[np.nonzero(b == 1)[0][3:]] = False
    keep[b == 2] = False
    keep[np.nonzero(b == 3)[0][4:]] = False
    tb, t3, t2, tK = _cuda(b[keep], p3[keep], p2[keep], K)
    r1 = pnp.ransac_pnp_batched(tb, t3, t2, tK, reprojection_error=THR, seed=7, solver="colmap")
    r2 = pnp.ransac_pnp_batched(tb, t3, t2, tK, reprojection_error=THR, seed=7, solver="colmap")
    torch.cuda.synchronize()
    assert r1["state"].cpu().tolist() == [True, False, False, True]
    eye = torch.eye(4, device="cuda")[:3]
    assert torch.equal(r1["pose"][1], eye) and torch.equal(r1["pose"][2], eye)
    assert r1["n_inliers"].cpu().tolist()[1:] == [0, 0, 4]
    assert not r1["inlier_mask"][tb == 1].any().item()
    for k in ("pose", "n_inliers", "inlier_mask", "state"):
        assert torch.equal(r1[k], r2[k]), f"{k} must not depend on scheduling"
    e = pnp.ransac_pnp_batched(tb[:0], t3[:0], t2[:0], tK, solver="colmap")   # M = 0 does not raise
    assert not e["state"].any().item() and e["inlier_mask"].numel() == 0


def test_reference_signature():
    """The demo's call (demo.py:132): 1-D inlier indices, the pose of the oracle; `scale` unused."""
    b, p3, p2, K, _ = opc.heavy_tailed_frames(2, seed=21)
    m = b == 1
    pose, pose_homo, inliers, state = pnp.ransac_PnP(K[1], p2[m], p3[m], scale=1000, pnp_reprojection_error=7,
                                                     img_hw=[512, 512], use_pycolmap_ransac=True)
    assert state is True and pose.shape == (3, 4) and pose_homo.shape == (4, 4)
    assert inliers.ndim == 1 and inliers.dtype == np.int64 and len(inliers) >= 20
    Ki, q2, q3 = K[1].astype(np.float64), p2[m].astype(np.float64), p3[m].astype(np.float64)
    pose_o, mask_o = opc.ransac(Ki, q2, q3, THR)
    ref = opc.cauchy_refine(Ki, q2, q3, pose_o, mask_o)
    assert len(set(inliers.tolist()) ^ set(np.nonzero(mask_o)[0].tolist())) <= max(2, int(mask_o.sum()) // 100)
    dR, dt = _gap(pose, ref)
    assert dR <= 1e-3 and dt <= 1e-3
    with pytest.raises(ValueError, match="img_hw"):
        pnp.ransac_PnP(K[1], p2[m], p3[m], pnp_reprojection_error=7, use_pycolmap_ransac=True)


def _write_ply(path, verts):
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nend_header\n" % len(verts))
    with open(path, "wb") as f:
        f.write(head.encode() + np.ascontiguousarray(verts, dtype="<f4").tobytes())


def test_linemod_call_end_to_end(tmp_path):
    """compute_query_pose_errors with the LINEMOD evaluation config: the poses are those of
    ransac_pnp_batched(solver="colmap") bit for bit, the inliers 1-D, and ADD / proj2D those of the
    pose-metrics oracle at these poses."""
    objs = {"objA": opm.synthetic_model(3000, 1), "0810-lm10-others": opm.synthetic_model(2001, 3, symmetric180=True)}
    for name, v in objs.items():
        os.makedirs(tmp_path / name / "seq" / "color")
        _write_ply(str(tmp_path / name / "model_eval.ply"), v)
    (tmp_path / "objA" / "diameter.txt").write_text("0.25\n")
    B = 4
    b, p3, p2, K, gt = opc.heavy_tailed_frames(B, seed=33)
    gt_h = np.tile(np.eye(4), (B, 1, 1))
    gt_h[:, :3] = gt
    paths = [str(tmp_path / n / "seq" / "color" / f"{i}.png") for i, n in
             enumerate(["objA", "0810-lm10-others", "objA", "objA"])]
    tb, t3, t2, tK = _cuda(b, p3, p2, K)
    data = {"m_bids": tb, "mkpts_3d_db": t3, "mkpts_query_f": t2, "query_intrinsic": torch.as_tensor(K),
            "query_intrinsic_origin": torch.as_tensor(K), "query_pose_gt": torch.as_tensor(gt_h),
            "query_image_path": paths}
    cfg = {"eval_ADD_metric": True, "pnp_reprojection_error": 7, "point_cloud_rescale": 1000,
           "use_pycolmap_ransac": True, "model_unit": "m"}
    pnp.compute_query_pose_errors(data, cfg)
    r = pnp.ransac_pnp_batched(tb, t3, t2, tK, reprojection_error=7, solver="colmap")
    assert np.array_equal(data["pose_pred"], r["pose_homo"].double().cpu().numpy())
    mask = r["inlier_mask"].cpu().numpy()
    for i in range(B):
        assert np.array_equal(data["inliers"][i], np.nonzero(mask[b == i])[0])
    assert max(data["R_errs"]) < 0.5 and max(data["t_errs"]) < 0.5   # deg, cm
    ref = opm.add_branch(data, data["pose_pred"], cfg)
    assert data["ADD"] == ref["ADD"] == [True] * B
    got, want = np.array(data["proj2D"]), np.array(ref["proj2D"])
    assert (np.abs(got - want) <= 1e-4 + 1e-6 * np.abs(want)).all()
