"""CPU tests of the LINEMOD pose metrics: the oracle against the unmodified reference's
add_metric / projection_2d_error (tests/golden/reference/pose_metrics.npz), the PLY reader that
stands in for open3d, and the host flow of compute_query_pose_errors' eval_ADD_metric branch with
the kernels replaced by CPU stubs."""
import logging
import os

import numpy as np
import pytest
import torch

from onepose_plus_plus_b200 import cad, pnp
from oracle import pose_metrics as opm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "pose_metrics.npz")


def test_oracle_matches_reference_golden():
    z = np.load(GOLDEN)
    got = {k: [] for k in z.files}
    for _, verts, dia, pred, gt, K in opm.metric_workload():
        for p, g in zip(pred, gt):
            for syn, key in ((False, "add"), (True, "adds")):
                got[key].append(opm.add_metric(verts, dia, p, g, syn=syn))
                got["dist_" + key].append(opm.add_mean_distance(verts, p, g, syn=syn))
            got["proj2d"].append(opm.projection_2d_error(verts, p, g, K))
    assert len(got["add"]) == len(z["add"]) == 22
    for key in ("add", "adds"):
        assert np.array_equal(np.array(got[key]), z[key]), key
    for key in ("dist_add", "dist_adds", "proj2d"):
        ref, val = z[key], np.array(got[key])
        fin = np.isfinite(ref)   # a distance the reference's decision could not pin is stored as NaN
        assert not np.isfinite(val[~fin]).any(), key
        assert np.allclose(val[fin], ref[fin], rtol=1e-12, atol=0), key
    proj, fin = np.array(got["proj2d"]), np.isfinite(z["proj2d"])
    assert np.array_equal(proj[~fin], z["proj2d"][~fin])
    # the workload reaches both decisions of both metrics and the non-finite projection
    assert z["add"].any() and not z["add"].all() and z["adds"].any() and not z["adds"].all()
    assert np.isinf(z["proj2d"]).sum() == 3
    assert z["dist_adds"][-2] == 0.0 and not z["add"][-2] and z["adds"][-2]   # GT composed with the symmetry


# ------------------------------------------------------------------------------------------------
# PLY reader
# ------------------------------------------------------------------------------------------------
def write_ply(path, verts, fmt="binary_little_endian", coord="float", extra=True, faces=True):
    """PLY with x/y/z of type `coord`, optionally normals + colours around them and a face list."""
    V = len(verts)
    props = [("x", coord), ("y", coord), ("z", coord)]
    if extra:
        props = [("nx", "float")] + props[:2] + [("red", "uchar"), ("green", "uchar")] + props[2:] + \
            [("confidence", "double"), ("label", "int")]
    head = ["ply", f"format {fmt} 1.0", "comment written by the test", f"element vertex {V}"]
    head += [f"property {t} {n}" for n, t in props]
    tri = np.array([[0, 1, 2], [2, 1, 0]]) % max(V, 1)
    if faces:
        head += [f"element face {len(tri)}", "property list uchar int vertex_indices"]
    head.append("end_header")
    np_t = {"float": "f4", "double": "f8", "uchar": "u1", "int": "i4"}
    rng = np.random.default_rng(0)
    cols = {"x": verts[:, 0], "y": verts[:, 1], "z": verts[:, 2], "nx": rng.normal(size=V),
            "red": rng.integers(0, 255, V), "green": rng.integers(0, 255, V), "confidence": rng.random(V),
            "label": rng.integers(-5, 5, V)}
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if fmt == "ascii":
            for i in range(V):
                f.write((" ".join(repr(float(cols[n][i])) if np_t[t][0] == "f" else str(int(cols[n][i]))
                                  for n, t in props) + "\n").encode())
            for t in tri if faces else ():
                f.write(("3 " + " ".join(map(str, t)) + "\n").encode())
        else:
            e = "<" if fmt.endswith("little_endian") else ">"
            rec = np.zeros(V, dtype=[(n, e + np_t[t]) for n, t in props])
            for n, _ in props:
                rec[n] = cols[n]
            f.write(rec.tobytes())
            for t in tri if faces else ():
                f.write(np.uint8(3).tobytes() + t.astype(e + "i4").tobytes())


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("coord", ["float", "double"])
def test_ply_reader_formats(tmp_path, fmt, coord):
    rng = np.random.default_rng(1)
    verts = rng.normal(size=(37, 3)) * 0.1
    if coord == "float":
        verts = verts.astype(np.float32).astype(np.float64)
    for extra, faces in ((True, True), (False, False)):
        path = str(tmp_path / f"m_{extra}.ply")
        write_ply(path, verts, fmt, coord, extra, faces)
        got = cad.read_ply_vertices(path)
        assert got.dtype == np.float64 and np.array_equal(got, verts)
        v32, bbox = cad.load_points_from_cad(path)
        assert v32.dtype == np.float32 and np.array_equal(v32, verts.astype(np.float32))
        lo, hi = verts.min(0), verts.max(0)
        assert bbox.shape == (9, 3) and bbox.dtype == np.float32
        assert np.array_equal(bbox[0], lo.astype(np.float32)) and np.array_equal(bbox[7], hi.astype(np.float32))
        assert np.array_equal(bbox[3], np.float32([lo[0], hi[1], hi[2]]))   # x slowest, z fastest
        assert np.array_equal(bbox[4], np.float32([hi[0], lo[1], lo[2]]))
        assert np.array_equal(bbox[8], ((lo + hi) / 2).astype(np.float32))
        assert cad.model_diameter_from_bbox(bbox) == np.linalg.norm(bbox[7] - bbox[0])


def test_ply_reader_rejects_what_it_cannot_read(tmp_path):
    good = str(tmp_path / "good.ply")
    write_ply(good, np.ones((4, 3)), "binary_little_endian")
    raw = open(good, "rb").read()
    cases = {
        "list_on_vertex": raw.replace(b"property float nx", b"property list uchar float nx"),
        "face_first": raw.replace(b"element vertex 4", b"element face 0\nelement vertex 4"),
        "no_z": raw.replace(b"property float z", b"property float w"),
        "truncated": raw[:-40 - 2 * 13],
        "bad_format": raw.replace(b"binary_little_endian", b"binary_middle_endian"),
        "not_ply": b"OFF\n" + raw[4:],
        "bad_type": raw.replace(b"property float nx", b"property float128 nx"),
        "ascii_short": b"ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\n"
                       b"property float z\nend_header\n0 0 0\n1 1 1\n",
        "ascii_columns": b"ply\nformat ascii 1.0\nelement vertex 2\nproperty float x\nproperty float y\n"
                         b"property float z\nend_header\n0 0 0\n1 1\n",
        "empty": b"ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nproperty float y\n"
                 b"property float z\nend_header\n",
    }
    for name, data in cases.items():
        path = str(tmp_path / f"{name}.ply")
        with open(path, "wb") as f:
            f.write(data)
        with pytest.raises(ValueError, match=f"{name}.ply"):
            cad.load_points_from_cad(path)


# ------------------------------------------------------------------------------------------------
# host flow of the eval_ADD_metric branch (kernels stubbed)
# ------------------------------------------------------------------------------------------------
def _stub_kernels(monkeypatch, poses, state):
    """ransac_pnp_batched returns the given poses; pose_metrics_batched computes with the oracle
    on the CPU and records every call.  Also counts CAD reads."""
    calls, reads = [], []

    def ransac(m_bids, mkpts_3d, mkpts_2d, K, scale=1.0, reprojection_error=5.0, **kw):
        pose = torch.as_tensor(poses, dtype=torch.float32)
        homo = torch.zeros(len(poses), 4, 4)
        homo[:, :3], homo[:, 3, 3] = pose, 1.0
        return {"pose": pose, "pose_homo": homo, "n_inliers": torch.zeros(len(poses), dtype=torch.int32),
                "inlier_mask": torch.ones(m_bids.numel(), dtype=torch.bool), "state": torch.as_tensor(state)}

    def metrics(verts, pose_pred, pose_gt, K_origin, symmetric, diameter):
        calls.append({"V": verts.shape[0], "B": pose_pred.shape[0], "sym": list(symmetric),
                      "diameter": diameter})
        v = verts.numpy()
        dist = [opm.add_mean_distance(v, p, g, syn=s) for p, g, s in zip(pose_pred.double().numpy(),
                                                                        pose_gt.double().numpy(), symmetric)]
        proj = [opm.projection_2d_error(v, p, g, k) for p, g, k in zip(pose_pred.double().numpy(),
                                                                       pose_gt.double().numpy(), K_origin.double().numpy())]
        dist = torch.tensor(dist, dtype=torch.float64)
        return {"add_dist": dist, "add_pass": dist < float(np.asarray(diameter)[()] * 0.1),
                "proj2d": torch.tensor(proj, dtype=torch.float64)}

    load = cad.load_points_from_cad

    def counted(path):
        reads.append(path)
        return load(path)
    monkeypatch.setattr(pnp, "ransac_pnp_batched", ransac)
    monkeypatch.setattr(pnp, "pose_metrics_batched", metrics)
    monkeypatch.setattr(cad, "load_points_from_cad", counted)
    return calls, reads


def _object_tree(root):
    """objA: model_eval.ply (binary) + a different model.ply + diameter.txt; objB: model.ply only
    (ascii, diameter from the bbox); 0810-lm10-others: symmetric, model_eval.ply only; objC: no model."""
    models = {"objA": opm.synthetic_model(50, 1), "objB": opm.synthetic_model(30, 2),
              "0810-lm10-others": opm.synthetic_model(40, 3, symmetric180=True)}
    for name, v in models.items():
        os.makedirs(root / name / "seq" / "color")
        write_ply(str(root / name / ("model.ply" if name == "objB" else "model_eval.ply")), v.astype(np.float64),
                  "ascii" if name == "objB" else "binary_little_endian")
    write_ply(str(root / "objA" / "model.ply"), 2 * models["objA"].astype(np.float64))
    (root / "objA" / "diameter.txt").write_text("0.2\n")
    os.makedirs(root / "objC" / "seq" / "color")
    return models, {n: str(root / n / "seq" / "color" / "0.png") for n in list(models) + ["objC"]}


def _data(paths, B, seed=0):
    rng = np.random.default_rng(seed)
    gt = np.tile(np.eye(4), (B, 1, 1))
    gt[:, :3] = np.stack([opm.gt_pose(rng) for _ in range(B)])
    K = torch.as_tensor(np.stack([opm.K_LINEMOD] * B), dtype=torch.float32)
    return {"m_bids": torch.arange(B).repeat_interleave(5), "mkpts_3d_db": torch.zeros(5 * B, 3),
            "mkpts_query_f": torch.zeros(5 * B, 2), "query_intrinsic": K, "query_intrinsic_origin": K * 1.5,
            "query_pose_gt": torch.as_tensor(gt), "query_image_path": paths}


CFG = {"eval_ADD_metric": True, "pnp_reprojection_error": 7, "point_cloud_rescale": 1000,
       "use_pycolmap_ransac": True, "model_unit": "m"}


def test_add_branch_host_flow(monkeypatch, tmp_path, caplog):
    models, img = _object_tree(tmp_path)
    B = 5
    data = _data([img["objA"], img["objB"], img["objA"], img["0810-lm10-others"], img["objA"]], B)
    rng = np.random.default_rng(4)
    poses = np.stack([opm.perturbed_pose(opm.synthetic_model(50, 1), data["query_pose_gt"][b, :3].numpy(),
                                         0.01 * (b + 1), rng) for b in range(B)])
    poses[2] = np.eye(4)[:3]                       # a failed frame is scored at the identity pose
    state = [True, True, False, True, True]
    calls, reads = _stub_kernels(monkeypatch, poses, state)
    pnp.compute_query_pose_errors(data, CFG)
    # the vertex cache: every model file is read once, a second batch reads none
    assert len(reads) == 3 and os.path.basename(reads[0]) == "model_eval.ply"
    pnp.compute_query_pose_errors(dict(data), CFG)
    assert len(reads) == 3
    # one metric call per model file, frames in batch order within it
    calls = calls[:3]
    assert [(c["V"], c["B"], c["sym"]) for c in calls] == [(50, 3, [False] * 3), (30, 1, [False]), (40, 1, [True])]
    assert float(calls[0]["diameter"]) == 0.2                                   # diameter.txt
    vB = models["objB"]
    assert calls[1]["diameter"] == np.linalg.norm(vB.max(0) - vB.min(0))         # bbox of model.ply
    assert len(data["ADD"]) == B and all(type(x) is bool for x in data["ADD"])
    assert len(data["proj2D"]) == B and all(type(x) is float for x in data["proj2D"])
    ref = opm.add_branch(data, data["pose_pred"], CFG)
    assert data["ADD"] == ref["ADD"] and np.allclose(data["proj2D"], ref["proj2D"], rtol=1e-12)
    assert data["ADD"][0] and not data["ADD"][4]
    assert data["R_errs"][2] == np.inf        # unchanged: failed frames keep the inf R/t errors
    # one path for the whole batch (the reference's batch-1 case): one call with every frame
    calls, _ = _stub_kernels(monkeypatch, poses, state)
    d = _data(img["0810-lm10-others"], B)
    pnp.compute_query_pose_errors(d, CFG)
    assert [(c["B"], c["sym"]) for c in calls] == [(B, [True] * B)]
    assert d["ADD"] == opm.add_branch(d, d["pose_pred"], CFG)["ADD"]
    # a missing model: logged, no ADD / proj2D keys, no metric call
    calls.clear()
    d = _data([img["objA"], img["objC"], img["objA"], img["objA"], img["objA"]], B)
    with caplog.at_level(logging.ERROR, logger=pnp.__name__):
        pnp.compute_query_pose_errors(d, CFG)
    assert "ADD" not in d and "proj2D" not in d and calls == []
    assert "objC/model.ply" in caplog.text
    with pytest.raises(ValueError, match="query_image_path"):
        pnp.compute_query_pose_errors(_data([img["objA"]] * 2, B), CFG)


def test_add_branch_off_writes_the_same_keys(monkeypatch, tmp_path):
    _, img = _object_tree(tmp_path)
    B = 2
    calls, reads = _stub_kernels(monkeypatch, np.stack([np.eye(4)[:3]] * B), [True, False])
    keys = []
    for cfg, training in (({k: v for k, v in CFG.items() if k != "eval_ADD_metric"}, False),
                          (dict(CFG, eval_ADD_metric=False), False), (CFG, True)):
        d = _data(img["objA"], B)
        pnp.compute_query_pose_errors(d, cfg, training=training)
        keys.append(set(d))
    assert calls == [] and reads == []
    assert keys[0] == keys[1] == keys[2]
    assert not {"ADD", "proj2D"} & keys[0] and {"R_errs", "t_errs", "inliers", "pose_pred"} <= keys[0]


def test_pose_metrics_batched_validates_before_any_launch():
    v = torch.zeros(10, 3)
    P = torch.zeros(2, 3, 4)
    K = torch.zeros(2, 3, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        pnp.pose_metrics_batched(v, P, P, K, False, 0.1)

    class FakeCuda(torch.Tensor):   # CPU storage that claims to be on a CUDA device (checks only)
        @property
        def is_cuda(self):
            return True

    def fake(t):
        return t.as_subclass(FakeCuda)
    bad = [(torch.zeros(0, 3), P, P, K), (torch.zeros(10, 2), P, P, K), (v, torch.zeros(2, 4, 3), P, K),
           (v, P, torch.zeros(3, 3, 4), K), (v, P, P, torch.zeros(2, 4, 4)), (v, torch.zeros(2, 3, 3), P, K)]
    for args in bad:
        with pytest.raises(ValueError):
            pnp.pose_metrics_batched(*(fake(a) for a in args), False, 0.1)
    with pytest.raises(ValueError, match="symmetric"):
        pnp.pose_metrics_batched(fake(v), fake(P), fake(torch.zeros(2, 4, 4)), fake(K), [True] * 3, 0.1)
