"""CPU oracle for the pycolmap branch of the pose stage — TEST INFRASTRUCTURE ONLY.

The reference's ``use_pycolmap_ransac`` branch (src/utils/metric_utils.py:137-170) calls
``pycolmap.absolute_pose_estimation`` on a SIMPLE_PINHOLE camera ``[K[0,0], K[0,2], K[1,2]]``:
LO-RANSAC on P3P samples, then a Ceres refinement of the pose on the RANSAC inliers with a Cauchy
loss of scale 1 per residual block (one block = the 2-vector pixel residual of one point).  pycolmap
is not part of this environment, so what is compared is the objective, not bit parity: the inlier
set of a locally optimised RANSAC under that camera, and the minimiser of
``sum_i log(1 + |r_i|^2)`` over it.  Everything here is fp64 numpy / cv2."""
import cv2
import numpy as np

from oracle.pose_metrics import K_LINEMOD


def simple_pinhole(K):
    """The camera pycolmap builds: f = K[0,0] on both axes, principal point (K[0,2], K[1,2]), no skew."""
    K = np.asarray(K, dtype=np.float64)
    return np.array([[K[0, 0], 0.0, K[0, 2]], [0.0, K[0, 0], K[1, 2]], [0.0, 0.0, 1.0]])


def residuals(K, p2, p3, pose):
    """Pixel residuals [n, 2] and depths [n] of the points under `pose` [3, 4] and the SIMPLE_PINHOLE K."""
    Ks = simple_pinhole(K)
    X = np.asarray(p3, np.float64) @ pose[:, :3].T + pose[:, 3]
    uv = X[:, :2] / X[:, 2:] * Ks[0, 0] + Ks[:2, 2]
    return uv - np.asarray(p2, np.float64), X[:, 2]


def inlier_mask(K, p2, p3, pose, thr):
    r, z = residuals(K, p2, p3, pose)
    return ((r ** 2).sum(1) <= thr * thr) & (z > 0)


def least_squares(K, p2, p3, pose, mask):
    """Minimiser of the plain reprojection error over the masked points (cv2 LM, SIMPLE_PINHOLE K)."""
    rvec = cv2.Rodrigues(pose[:, :3])[0]
    tvec = pose[:, 3:].copy()
    rvec, tvec = cv2.solvePnPRefineLM(np.ascontiguousarray(p3[mask], np.float64),
                                      np.ascontiguousarray(p2[mask], np.float64), simple_pinhole(K),
                                      np.zeros((8, 1)), rvec, tvec,
                                      criteria=(cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_COUNT, 200, 1e-14))
    return np.concatenate([cv2.Rodrigues(rvec)[0], tvec], axis=-1)


def ransac(K, p2, p3, thr):
    """RANSAC under the SIMPLE_PINHOLE camera (cv2, many iterations), then local optimisation until
    the inlier set is stable: least squares on the inliers, re-select with error <= thr.  Returns
    (pose [3, 4], inlier mask [n]) or (None, None) when cv2 finds nothing."""
    p2 = np.asarray(p2, np.float64)
    p3 = np.asarray(p3, np.float64)
    ok, rvec, tvec, _ = cv2.solvePnPRansac(np.ascontiguousarray(p3), np.ascontiguousarray(p2), simple_pinhole(K),
                                           np.zeros((8, 1)), reprojectionError=thr, iterationsCount=10000,
                                           confidence=0.9999, flags=cv2.SOLVEPNP_EPNP)
    if not ok:
        return None, None
    pose = np.concatenate([cv2.Rodrigues(rvec)[0], tvec], axis=-1)
    mask = inlier_mask(K, p2, p3, pose, thr)
    for _ in range(50):
        pose = least_squares(K, p2, p3, pose, mask)
        new = inlier_mask(K, p2, p3, pose, thr)
        if np.array_equal(new, mask):
            break
        mask = new
    return pose, mask


def _terms(K, p2, p3, pose, weighted=True):
    """Cost sum log(1 + |r|^2) (or sum |r|^2 unweighted), H = sum w J^T J, g = sum w J^T r over the
    points, J the derivative of r in (w, t) of R <- exp([w]x) R, t <- t + dt."""
    Ks = simple_pinhole(K)
    f = Ks[0, 0]
    Y = p3 @ pose[:, :3].T
    X = Y + pose[:, 3]
    iz = 1.0 / X[:, 2]
    xn, yn = X[:, 0] * iz, X[:, 1] * iz
    r = np.stack([f * xn + Ks[0, 2] - p2[:, 0], f * yn + Ks[1, 2] - p2[:, 1]], 1)
    zero = np.zeros_like(iz)
    gu = np.stack([f * iz, zero, -f * xn * iz], 1)
    gv = np.stack([zero, f * iz, -f * yn * iz], 1)
    J = np.stack([np.concatenate([np.cross(Y, gu), gu], 1), np.concatenate([np.cross(Y, gv), gv], 1)], 1)
    s = (r ** 2).sum(1)
    if weighted:
        w, cost = 1.0 / (1.0 + s), np.log1p(s).sum()
    else:
        w, cost = np.ones_like(s), s.sum()
    H = np.einsum("n,nki,nkj->ij", w, J, J)
    g = np.einsum("n,nki,nk->i", w, J, r)
    return cost, H, g, X[:, 2]


def _step(pose, d):
    R = cv2.Rodrigues(np.asarray(d[:3], np.float64).reshape(3, 1))[0] @ pose[:, :3]
    return np.concatenate([R, (pose[:, 3] + d[3:])[:, None]], 1)


def cauchy_gradient(K, p2, p3, pose, mask):
    """Gradient of sum log(1 + |r_i|^2) over the masked points in (w, t): 2 sum w_i J_i^T r_i."""
    return 2.0 * _terms(K, np.asarray(p2, np.float64)[mask], np.asarray(p3, np.float64)[mask], pose)[2]


def cauchy_cost(K, p2, p3, pose, mask):
    """sum over the masked points of log(1 + |r_i|^2), r_i the pixel residual under SIMPLE_PINHOLE K."""
    r, _ = residuals(K, np.asarray(p2)[mask], np.asarray(p3)[mask], np.asarray(pose, np.float64))
    return float(np.log1p((r ** 2).sum(1)).sum())


def cauchy_refine(K, p2, p3, pose0, mask, max_iter=2000):
    """Minimiser of sum_i log(1 + |r_i|^2) over the masked points from pose0, with the loss applied
    per point as Ceres applies it per residual block: IRLS Levenberg-Marquardt (weights
    1 / (1 + |r_i|^2), analytic Jacobian), run until the gradient vanishes to fp64 precision."""
    p2 = np.asarray(p2, np.float64)[mask]
    p3 = np.asarray(p3, np.float64)[mask]
    pose = np.asarray(pose0, np.float64)[:3].copy()
    cost, H, g, _ = _terms(K, p2, p3, pose)
    g0 = np.abs(g).max()
    lam = 1e-4
    for _ in range(max_iter):
        if np.abs(g).max() <= 1e-13 * g0:
            break
        d = np.linalg.solve(H + lam * np.diag(np.diag(H)), -g)
        trial = _step(pose, d)
        c, Hn, gn, z = _terms(K, p2, p3, trial)
        # near the optimum the cost stops resolving the steps (its fp64 rounding is larger than
        # the decrease); a step that keeps it there and shrinks the gradient is taken
        if (z > 0).all() and (c < cost or (c <= cost + 1e-15 * abs(cost) and np.abs(gn).max() < np.abs(g).max())):
            pose, cost, H, g = trial, c, Hn, gn
            lam = max(lam * 0.1, 1e-14)
        else:
            lam *= 10.0
            if lam > 1e14:
                break
    return pose


def heavy_tailed_frames(batch, seed=0, n_range=(300, 2000), outlier_frac=0.3, hw=(480, 640)):
    """Planted LINEMOD-like workload: per frame a random pose of a ~0.2 m object 0.5-0.9 m away, n in
    n_range points (metres) projected with the FULL LINEMOD K (fx != fy), 0.5 px Gaussian noise,
    10 % of the inliers pushed 3-6 px in a random direction (inside a 7 px threshold), and
    `outlier_frac` of the points replaced by uniformly random pixels.  Returns the matcher-style
    lists (m_bids, mkpts_3d_db, mkpts_query_f), intrinsics [B, 3, 3] and the planted poses."""
    rng = np.random.default_rng(seed)
    h, w = hw
    K = K_LINEMOD.astype(np.float64)
    bids, p3s, p2s, poses = [], [], [], []
    for b in range(batch):
        n = int(rng.integers(n_range[0], n_range[1] + 1))
        R = cv2.Rodrigues(rng.normal(size=3) * 0.6)[0]
        t = np.array([rng.normal() * 0.05, rng.normal() * 0.05, 0.5 + 0.4 * rng.random()])
        P = (rng.random((n, 3)) - 0.5) * 0.2
        X = P @ R.T + t
        uv = X[:, :2] / X[:, 2:] * np.array([K[0, 0], K[1, 1]]) + K[:2, 2]
        noise = rng.normal(size=uv.shape) * 0.5
        heavy = rng.random(n) < 0.1
        ang = rng.random(int(heavy.sum())) * 2 * np.pi
        noise[heavy] = np.stack([np.cos(ang), np.sin(ang)], 1) * rng.uniform(3.0, 6.0, size=(len(ang), 1))
        uv += noise
        out = rng.random(n) < outlier_frac
        uv[out] = rng.random((int(out.sum()), 2)) * np.array([w, h])
        bids.append(np.full(n, b)), p3s.append(P), p2s.append(uv)
        poses.append(np.concatenate([R, t[:, None]], 1))
    return (np.concatenate(bids).astype(np.int64), np.concatenate(p3s).astype(np.float32),
            np.concatenate(p2s).astype(np.float32), np.stack([K] * batch).astype(np.float32), np.stack(poses))
