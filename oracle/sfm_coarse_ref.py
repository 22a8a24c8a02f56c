"""Import the UNMODIFIED reference coarse-match stage from /root/reference — TEST INFRASTRUCTURE ONLY
(pins oracle/sfm_coarse.py and generates tests/golden/reference/sfm_coarse.npz).

coarse_match_worker.py imports ray and pytorch_lightning at module level and the package __init__
files pull in the post-optimisation (DeepLM, hydra).  Stand-ins: ``ray.remote`` is an identity
decorator factory, ``pytorch_lightning.seed_everything`` seeds random, numpy and torch, h5py is a
bare module (only the file writers use it), and the packages above the three module files are
registered bare.  /root/reference does not exist on the GPU box: no GPU test may import this.
"""
import importlib
import os
import random
import sys
import types

import numpy as np
import torch

from . import ref_shims


def _module(name):
    m = types.ModuleType(name)
    sys.modules[name] = m
    return m


def load():
    """-> (coarse_match_worker, coarse_match.utils, dataset.loftr_coarse_dataset) reference modules."""
    ref_shims.install()
    if "ray" not in sys.modules:
        ray = _module("ray")

        def remote(*args, **kwargs):
            if len(args) == 1 and callable(args[0]) and not kwargs:
                return args[0]
            return lambda f: f
        ray.remote = remote
    if "pytorch_lightning" not in sys.modules:
        pl = _module("pytorch_lightning")

        def seed_everything(seed):
            random.seed(seed)
            np.random.seed(seed)
            torch.manual_seed(seed)
            return seed
        pl.seed_everything = seed_everything
    try:
        import h5py  # noqa: F401
    except ImportError:
        _module("h5py")
    root = ref_shims.REFERENCE_ROOT
    for name in ("src.KeypointFreeSfM", "src.KeypointFreeSfM.coarse_match", "src.KeypointFreeSfM.dataset",
                 "src.KeypointFreeSfM.loftr_for_sfm"):
        if name not in sys.modules:
            pkg = _module(name)
            pkg.__path__ = [os.path.join(root, *name.split("."))]
    lfs = sys.modules["src.KeypointFreeSfM.loftr_for_sfm"]
    for attr in ("LoFTR_for_OnePose_Plus", "default_cfg"):   # the merge functions use neither
        if not hasattr(lfs, attr):
            setattr(lfs, attr, None)
    worker = importlib.import_module("src.KeypointFreeSfM.coarse_match.coarse_match_worker")
    utils = importlib.import_module("src.KeypointFreeSfM.coarse_match.utils")
    dataset = importlib.import_module("src.KeypointFreeSfM.dataset.loftr_coarse_dataset")
    return worker, utils, dataset


def reference_merge(matches, names):
    """The reference's merge exactly as detector_free_coarse_matching runs it without ray:
    Match2Pts2D -> points2D_worker -> update_matches -> transform_points2D.
    Returns (keypoints, scores, index matches)."""
    worker, utils, _ = load()
    all_kpts = utils.Match2Pts2D(matches, names, name_split=" ")
    keypoints = worker.points2D_worker(all_kpts[0:len(names)], verbose=False)
    updated = worker.update_matches(matches, keypoints, verbose=False, pair_name_split=" ")
    keypoints = {k: v for k, v in keypoints.items() if isinstance(v, dict)}
    kpts, scores = worker.transform_points2D(keypoints, verbose=False)
    return kpts, scores, updated
