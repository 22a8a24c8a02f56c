"""Generate tests/golden/reference/pose_metrics.npz (and nothing else): what the UNMODIFIED reference
``src/utils/metric_utils.py`` (imported from /root/reference through oracle/ref_shims.py) computes
on the seeded workload ``oracle.pose_metrics.metric_workload``:

    python -m oracle.make_pose_metrics_golden

Per frame, in workload order: ``add_metric`` with syn = False and True (decisions), the mean
distance behind each decision, and ``projection_2d_error``.  ``add_metric`` returns only the
decision; the distance m is recovered from it exactly: with percentage = 1 the threshold is the
diameter argument t itself, and the smallest double t for which ``m < t`` holds is the successor of
m, found by bisection over the bit patterns of the non-negative doubles.  Where m is not finite
the decision is False for every t and the distance is stored as NaN.

The reference module imports open3d and plyfile (through sample_points_on_cad); neither is
installed here and none of their functions is called, so empty stand-in modules satisfy the import.
"""
import os
import sys
import types

import numpy as np

from . import pose_metrics, ref_shims
from .make_reference_golden import GOLDEN_DIR


def reference_metric_utils():
    for name in ("open3d", "plyfile"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["plyfile"].PlyData = None
    ref_shims.install()
    import importlib
    return importlib.import_module("src.utils.metric_utils")


def recovered_distance(mu, verts, pose_pred, pose_gt, syn):
    def below(bits):   # m < t for the double t with these bits
        t = np.array(bits, dtype=np.int64).view(np.float64)[()]
        return bool(mu.add_metric(verts, t, pose_pred.copy(), pose_gt.copy(), percentage=1.0, syn=syn))
    lo, hi = 0, int(np.array(np.inf).view(np.int64))
    if below(lo) or not below(hi):
        return np.nan
    while hi - lo > 1:   # below(lo) is False, below(hi) is True
        mid = (lo + hi) // 2
        if below(mid):
            hi = mid
        else:
            lo = mid
    return np.array(lo, dtype=np.int64).view(np.float64)[()]   # the predecessor of the smallest t


def main():
    assert ref_shims.available(), "needs /root/reference"
    mu = reference_metric_utils()
    out = {k: [] for k in ("add", "adds", "dist_add", "dist_adds", "proj2d")}
    for name, verts, dia, pred, gt, K in pose_metrics.metric_workload():
        for p, g in zip(pred, gt):
            out["add"].append(mu.add_metric(verts, dia, p.copy(), g.copy(), syn=False))
            out["adds"].append(mu.add_metric(verts, dia, p.copy(), g.copy(), syn=True))
            out["dist_add"].append(recovered_distance(mu, verts, p, g, False))
            out["dist_adds"].append(recovered_distance(mu, verts, p, g, True))
            out["proj2d"].append(mu.projection_2d_error(verts, p.copy(), g.copy(), K.copy()))
        print(f"{name}: {len(pred)} frames")
    arrays = {k: np.array(v, dtype=bool if k in ("add", "adds") else np.float64) for k, v in out.items()}
    path = os.path.join(GOLDEN_DIR, "pose_metrics.npz")
    np.savez_compressed(path, **arrays)
    print(f"pose_metrics -> {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
