"""CPU oracle for the LINEMOD pose metrics — TEST INFRASTRUCTURE ONLY (see oracle/oracle.py's header).

Restates src/utils/metric_utils.py:31-88 (``projection_2d_error``, ``add_metric`` with ``syn`` =
ADD-S through a scipy cKDTree built on the predicted points and queried with the target points)
and the ``eval_ADD_metric`` branch of ``compute_query_pose_errors`` (:233-289) in numpy, fp64 as
there.  tests/golden/reference/pose_metrics.npz pins it to the unmodified reference on the seeded
``metric_workload``; the GPU tests compare the device metrics against it.  Also builds the synthetic
CAD models and poses those tests use."""
import os.path as osp

import numpy as np
from scipy import spatial

# LINEMOD's published camera (fp32-representable, like everything fed to the fp32 device ABI)
K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]],
                     dtype=np.float32).astype(np.float64)


def _rt(pose):
    pose = np.asarray(pose, dtype=np.float64)
    return pose[:3, :3], pose[:3, 3]


def projection_2d_error(model_3D_pts, pose_pred, pose_targets, K):
    """Mean pixel distance between the model projected with the two poses (z not guarded)."""
    def pixels(pose):
        R, t = _rt(pose)
        cam = model_3D_pts @ R.T + t
        hom = cam @ np.asarray(K, dtype=np.float64).T
        with np.errstate(divide="ignore", invalid="ignore"):
            return hom[:, :2] / hom[:, 2:]
    return np.mean(np.linalg.norm(pixels(pose_pred) - pixels(pose_targets), axis=-1))


def add_mean_distance(model_3D_pts, pose_pred, pose_target, syn=False):
    """ADD: mean distance between corresponding transformed points; ADD-S (syn): mean distance from
    every target point to its nearest predicted point."""
    Rp, tp = _rt(pose_pred)
    Rg, tg = _rt(pose_target)
    pred = model_3D_pts @ Rp.T + tp
    target = model_3D_pts @ Rg.T + tg
    if syn:
        dist, _ = spatial.cKDTree(pred).query(target, k=1)
        return np.mean(dist)
    return np.mean(np.linalg.norm(pred - target, axis=-1))


def add_metric(model_3D_pts, diameter, pose_pred, pose_target, percentage=0.1, syn=False):
    """True when the (symmetric) mean distance is below percentage x diameter (numpy arithmetic:
    a float32 diameter gives a float32 threshold)."""
    return bool(add_mean_distance(model_3D_pts, pose_pred, pose_target, syn) < diameter * percentage)


def add_branch(data, pose_pred, configs, training=False):
    """The eval_ADD_metric branch of compute_query_pose_errors, frame by frame: returns
    {"ADD": [bool], "proj2D": [float]} for the poses pose_pred [B, 4, 4], or {} when the branch is
    off or a model file is missing.  ``query_image_path`` may be one path or one per frame."""
    from onepose_plus_plus_b200 import cad
    if not ("eval_ADD_metric" in configs and configs["eval_ADD_metric"] and not training):
        return {}
    B = len(pose_pred)
    paths = data["query_image_path"]
    paths = [paths] * B if isinstance(paths, str) else list(paths)
    K_origin = np.asarray(data["query_intrinsic_origin"], dtype=np.float64)
    pose_gt = np.asarray(data["query_pose_gt"], dtype=np.float64)
    out = {"ADD": [], "proj2D": []}
    for b, image_path in enumerate(paths):
        root = image_path.rsplit("/", 3)[0]
        model_path = osp.join(root, "model_eval.ply")
        if not osp.exists(model_path):
            model_path = osp.join(root, "model.ply")
        if not osp.exists(model_path):
            return {}
        verts, bbox = cad.load_points_from_cad(model_path)
        diameter_path = osp.join(root, "diameter.txt")
        diameter = np.loadtxt(diameter_path) if osp.exists(diameter_path) else cad.model_diameter_from_bbox(bbox)
        syn = ("0810-" in image_path) or ("0811-" in image_path)
        out["ADD"].append(add_metric(verts, diameter, pose_pred[b], pose_gt[b], syn=syn))
        out["proj2D"].append(float(projection_2d_error(verts, pose_pred[b], pose_gt[b], K_origin[b])))
    return out


# ------------------------------------------------------------------------------------------------
# seeded workload
# ------------------------------------------------------------------------------------------------
def rotation(rvec):
    """Rodrigues: rotation matrix of the axis-angle vector rvec."""
    rvec = np.asarray(rvec, dtype=np.float64)
    th = np.linalg.norm(rvec)
    if th < 1e-300:
        return np.eye(3)
    k = rvec / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def as_f32(pose):
    """[3, 4] pose rounded to fp32 (what the device ABI takes), returned as fp64."""
    return np.asarray(pose, dtype=np.float64)[:3].astype(np.float32).astype(np.float64)


def synthetic_model(n, seed, symmetric180=False):
    """fp32 [n, 3] points in a random ellipsoid of 3-12 cm half-axes around the origin.  Vertex 0 has
    z = 0 exactly (at the identity pose its projection divides by zero).  symmetric180: the point set
    is invariant under the rotation by 180 degrees about z (pairs (x, y, z), (-x, -y, z))."""
    rng = np.random.default_rng(seed)
    axes = rng.uniform(0.03, 0.12, 3)
    m = n // 2 if symmetric180 else n
    p = rng.normal(size=(m, 3))
    p *= (rng.random(m) ** (1 / 3) / np.linalg.norm(p, axis=1))[:, None] * axes
    if n > 1:
        p[0, 2] = 0.0
    if symmetric180:   # mirrored pairs, and an odd point out on the axis
        p = np.concatenate([p, p * np.array([-1.0, -1.0, 1.0])] + [[[0.0, 0.0, axes[2] / 2]]] * (n % 2))
    return p.astype(np.float32)


def bbox_diameter(verts):
    """model_diameter_from_bbox of the model's bounding box (fp32, as load_points_from_cad gives it)."""
    v = verts.astype(np.float64)
    return np.linalg.norm((v.max(0).astype(np.float32) - v.min(0).astype(np.float32)))


def gt_pose(rng):
    """Random rotation, the object 0.5-1.5 m in front of the camera."""
    t = np.array([rng.normal() * 0.05, rng.normal() * 0.05, rng.uniform(0.5, 1.5)])
    return as_f32(np.concatenate([rotation(rng.normal(size=3) * 1.5), t[:, None]], 1))


def perturbed_pose(verts, pose_gt, target, rng):
    """A prediction near pose_gt whose ADD is close to `target` metres: a random rotation and
    translation direction, scaled by the first-order estimate of the step that gives that ADD."""
    w, d = rng.normal(size=3), rng.normal(size=3)
    w *= 0.05 / np.linalg.norm(w)
    d *= 0.01 / np.linalg.norm(d)
    R, t = pose_gt[:, :3], pose_gt[:, 3]

    def pose(s):
        return np.concatenate([rotation(s * w) @ R, (t + s * d)[:, None]], 1)
    s = target / max(add_mean_distance(verts, pose(1.0), pose_gt), 1e-12)
    return as_f32(pose(s))


RATIOS = (0.3, 0.7, 1.5, 3.0)   # prediction ADD / (0.1 x diameter)


def metric_frames(verts, diameter, n_frames, seed, identity_at=None):
    """n_frames (pose_pred, pose_gt) pairs: predictions at RATIOS x the 0.1 x diameter threshold in
    turn; frame `identity_at` predicts the identity (a failed PnP)."""
    rng = np.random.default_rng(seed)
    preds, gts = [], []
    for f in range(n_frames):
        g = gt_pose(rng)
        p = as_f32(np.eye(4)) if f == identity_at else perturbed_pose(verts, g, RATIOS[f % 4] * 0.1 * diameter, rng)
        preds.append(p)
        gts.append(g)
    return np.stack(preds), np.stack(gts)


# the golden workload: (model size, seed); every model gets len(RATIOS) + 1 frames, the last one at
# the identity pose, plus the 180-degree-symmetric model at GT composed with its symmetry
GOLDEN_MODELS = ((1, 11), (7, 12), (300, 13), (2000, 14))


def metric_workload():
    """[(name, verts, diameter, pose_pred [F, 3, 4], pose_gt [F, 3, 4], K [3, 3])], seeded."""
    cases = []
    for n, seed in GOLDEN_MODELS:
        v = synthetic_model(n, seed)
        dia = max(bbox_diameter(v), np.float32(0.05))
        pred, gt = metric_frames(v, dia, len(RATIOS) + 1, seed + 100, identity_at=len(RATIOS))
        cases.append((f"v{n}", v, dia, pred, gt, K_LINEMOD))
    v = synthetic_model(301, 15, symmetric180=True)
    rng = np.random.default_rng(115)
    gt = np.stack([gt_pose(rng), gt_pose(rng)])
    flip = np.diag([-1.0, -1.0, 1.0])
    pred = np.stack([as_f32(np.concatenate([gt[0][:, :3] @ flip, gt[0][:, 3:]], 1)),
                     perturbed_pose(v, gt[1], 0.5 * 0.1 * bbox_diameter(v), rng)])
    cases.append(("sym180", v, bbox_diameter(v), pred, gt, K_LINEMOD))
    return cases
