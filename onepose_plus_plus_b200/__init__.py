"""onepose_plus_plus_b200 — H100 (sm_90a) implementation of the OnePose++ 2D-3D matcher hot path.

``OnePosePlus_model`` mirrors the reference class of the same name
(src/models/OnePosePlus/OnePosePlusModel.py) and runs on hand-written CUDA kernels through the
C ABI in ``include/opp_b200.h``.
"""
from .model import LazyConfMatrix, OnePosePlus_model, build_backbone  # noqa: F401
from .loftr import LoFTR_for_OnePose_Plus  # noqa: F401  (2D-2D matcher of the SfM / demo stages)
from . import pnp  # noqa: F401  (device-side RANSAC-PnP front end: metric_utils.ransac_PnP)
from . import tracking  # noqa: F401  (demo tracking step: bbox crop on the device, PoseTracker)
from .train_gt import SparseGT, SparseGTDataset, collate_sparse_gt, sparse_gt_sample  # noqa: F401  (training: sparse ground truth)

__version__ = "0.2.0"
