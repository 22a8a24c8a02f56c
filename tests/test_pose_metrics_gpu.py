"""pytest -m gpu: the LINEMOD pose metrics on the device (opp_pose_metrics through
onepose_plus_plus_b200.pnp) against the CPU oracle (oracle/pose_metrics.py, which
tests/test_pose_metrics_cpu.py pins to the reference's add_metric / projection_2d_error), and the
eval_ADD_metric branch of compute_query_pose_errors end to end on planted frames."""
import os

import numpy as np
import pytest
import torch

from onepose_plus_plus_b200 import _lib, pnp
from oracle import pnp as opnp
from oracle import pose_metrics as opm

pytestmark = pytest.mark.gpu

BAND = 1e-5   # relative band around the threshold inside which the decision may differ


def _cuda(*xs):
    return [torch.as_tensor(np.asarray(x), dtype=torch.float32, device="cuda") for x in xs]


def _device(verts, pred, gt, K, sym, dia):
    r = pnp.pose_metrics_batched(*_cuda(verts, pred, gt, K), sym, dia)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in r.items()}


def _oracle(verts, pred, gt, K, sym):
    dist = np.array([opm.add_mean_distance(verts, p, g, syn=s) for p, g, s in zip(pred, gt, sym)])
    proj = np.array([opm.projection_2d_error(verts, p, g, k) for p, g, k in zip(pred, gt, K)])
    return dist, proj


def _check(got, verts, pred, gt, K, sym, dia):
    dist, proj = _oracle(verts, pred, gt, K, sym)
    assert np.isfinite(dist).all()
    err = np.abs(got["add_dist"] - dist)
    assert (err <= 1e-6 * dia + 1e-5 * dist).all(), (err.max(), dist[err.argmax()])
    fin = np.isfinite(proj)
    assert np.array_equal(np.isfinite(got["proj2d"]), fin)
    perr = np.abs(got["proj2d"][fin] - proj[fin])
    assert (perr <= 1e-4 + 1e-6 * np.abs(proj[fin])).all(), perr.max()
    thr = float(np.asarray(dia)[()] * 0.1)
    assert (np.abs(dist - thr) <= BAND * thr).sum() == 0          # the workload keeps clear of the band
    assert np.array_equal(got["add_pass"], dist < thr)
    return dist, proj


@pytest.mark.parametrize("V", [1, 7, 1000, 5003, 20000])
def test_metrics_match_oracle(V):
    verts = opm.synthetic_model(V, 100 + V)
    dia = max(opm.bbox_diameter(verts), np.float32(0.05))
    B = 64
    pred, gt = opm.metric_frames(verts, dia, B, seed=V, identity_at=5)
    K = np.stack([opm.K_LINEMOD] * B)
    sym = np.arange(B) % 2 == 1
    dist, proj = _check(_device(verts, pred, gt, K, sym, dia), verts, pred, gt, K, sym, dia)
    if V > 1:
        assert np.isinf(proj[5])           # identity pose, a vertex at z = 0: as in numpy
    assert 0 < (dist < 0.1 * dia).sum() < B
    # batch 1, the reference's call pattern: ADD-S, ADD and the identity frame
    for f, s in ((0, True), (1, False), (5, True), (6, False)):
        sl = slice(f, f + 1)
        _check(_device(verts, pred[sl], gt[sl], K[sl], s, dia), verts, pred[sl], gt[sl], K[sl], [s], dia)


def test_symmetric_object_and_determinism():
    verts = opm.synthetic_model(4001, 7, symmetric180=True)
    dia = opm.bbox_diameter(verts)
    rng = np.random.default_rng(8)
    g = opm.gt_pose(rng)
    flipped = opm.as_f32(np.concatenate([g[:, :3] @ np.diag([-1.0, -1.0, 1.0]), g[:, 3:]], 1))
    pred, gt, K = np.stack([flipped] * 2), np.stack([g] * 2), np.stack([opm.K_LINEMOD] * 2)
    got = _device(verts, pred, gt, K, [True, False], dia)
    dist, _ = _oracle(verts, pred, gt, K, [True, False])
    assert got["add_pass"].tolist() == [True, False] == (dist < 0.1 * dia).tolist()   # ADD-S passes, ADD fails
    assert got["add_dist"][0] < 1e-6 * dia and abs(got["add_dist"][1] - dist[1]) <= 1e-6 * dia + 1e-5 * dist[1]
    # two identical calls are bit-identical (the split nearest-neighbour search included)
    verts = opm.synthetic_model(20000, 9)
    pred, gt = opm.metric_frames(verts, opm.bbox_diameter(verts), 64, seed=9, identity_at=3)
    args = _cuda(verts, pred, gt, np.stack([opm.K_LINEMOD] * 64))
    for sym in (np.arange(64) % 3 == 0, [True]):
        n = len(sym)
        a = [pnp.pose_metrics_batched(args[0], args[1][:n], args[2][:n], args[3][:n], sym, 0.1) for _ in range(2)]
        for k in ("add_dist", "proj2d"):
            assert torch.equal(a[0][k].view(torch.int64), a[1][k].view(torch.int64)), k
    # batch 0: empty results, no launch
    before = _lib.LAUNCHES
    e = pnp.pose_metrics_batched(args[0], args[1][:0], args[2][:0], args[3][:0], False, 0.1)
    assert _lib.LAUNCHES == before and all(v.numel() == 0 and v.is_cuda for v in e.values())


def _write_ply(path, verts):
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
            "property float z\nelement face 0\nproperty list uchar int vertex_indices\nend_header\n" % len(verts))
    with open(path, "wb") as f:
        f.write(head.encode() + np.ascontiguousarray(verts, dtype="<f4").tobytes())


def test_compute_query_pose_errors_add_branch(tmp_path):
    """LINEMOD evaluation call on planted frames: objA has model_eval.ply + diameter.txt, objB only
    model.ply, 0810-lm10-others is a symmetric object; frame 3 has too few matches and is scored
    at the identity pose.  ADD / proj2D equal the oracle applied to the returned poses."""
    objs = {"objA": opm.synthetic_model(3000, 1), "objB": opm.synthetic_model(800, 2),
            "0810-lm10-others": opm.synthetic_model(2001, 3, symmetric180=True)}
    for name, v in objs.items():
        os.makedirs(tmp_path / name / "seq" / "color")
        _write_ply(str(tmp_path / name / ("model.ply" if name == "objB" else "model_eval.ply")), v)
    (tmp_path / "objA" / "diameter.txt").write_text("0.25\n")
    b, p3, p2, K, gt = opnp.synthetic_frames(4, seed=3)
    keep = (b != 3) | (np.cumsum(b == 3) <= 3)
    b, p3, p2 = b[keep], p3[keep], p2[keep]
    gt_h = np.tile(np.eye(4), (4, 1, 1))
    gt_h[:, :3] = gt.astype(np.float32)
    paths = [str(tmp_path / n / "seq" / "color" / f"{i}.png") for i, n in
             enumerate(["objA", "objB", "0810-lm10-others", "objA"])]
    dev = torch.device("cuda")
    # point_cloud_rescale 1000: PnP runs on the points in mm and returns t in the bank's metres
    data = {"m_bids": torch.as_tensor(b, device=dev), "mkpts_3d_db": torch.as_tensor(p3, device=dev),
            "mkpts_query_f": torch.as_tensor(p2, device=dev), "query_intrinsic": torch.as_tensor(K),
            "query_intrinsic_origin": torch.as_tensor(K), "query_pose_gt": torch.as_tensor(gt_h),
            "query_image_path": paths}
    cfg = {"eval_ADD_metric": True, "pnp_reprojection_error": 7, "point_cloud_rescale": 1000,
           "use_pycolmap_ransac": True, "model_unit": "m"}
    pnp.compute_query_pose_errors(data, cfg)
    assert len(data["ADD"]) == len(data["proj2D"]) == 4
    ref = opm.add_branch(data, data["pose_pred"], cfg)
    assert data["ADD"] == ref["ADD"] == [True, True, True, False]
    got, want = np.array(data["proj2D"]), np.array(ref["proj2D"])
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin) and not fin[3]
    assert (np.abs(got[fin] - want[fin]) <= 1e-4 + 1e-6 * np.abs(want[fin])).all()
    # what the reference's aggregate_metrics makes of these lists (inference_OnePosePlus.py:109-128)
    assert np.mean(data["ADD"]) == 0.75 and np.mean(np.array(data["proj2D"]) < 5) == 0.75
