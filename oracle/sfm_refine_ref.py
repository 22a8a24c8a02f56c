"""Import the UNMODIFIED reference SfM refinement from /root/reference — TEST INFRASTRUCTURE ONLY
(pins oracle/sfm_refine.py and generates tests/golden/reference/sfm_refine.npz).

feature_aggregation.py imports geometry_utils (pytorch3d, src.utils.colmap.read_write_model) and
h5py at module level, fine_match_worker.py imports pytorch_lightning and ray.  Stand-ins: a bare
``pytorch3d`` with a bare ``transforms``, the reference's own read_write_model.py loaded from the
reference tree (never copied), ``FakeH5`` for h5py (an in-memory file store keyed by path), and
sfm_coarse_ref's ray / pytorch_lightning.  /root/reference does not exist on the GPU box: no GPU
test may import this.
"""
import importlib
import importlib.util
import os
import sys
import types

from . import ref_shims, sfm_coarse_ref
from .sfm_refine import FakeH5, fake_h5py


def _module(name):
    m = types.ModuleType(name)
    sys.modules[name] = m
    return m


def load():
    """-> (feature_aggregation, fine_match_worker, construct_matching_data) reference modules."""
    sfm_coarse_ref.load()
    if "ray.actor" not in sys.modules:
        sys.modules["ray"].actor = _module("ray.actor")
        sys.modules["ray.actor"].ActorHandle = object
    if "pytorch3d" not in sys.modules:
        p3 = _module("pytorch3d")
        p3.transforms = _module("pytorch3d.transforms")
    if "src.utils.colmap.read_write_model" not in sys.modules:
        for name in ("src.utils", "src.utils.colmap"):
            if name not in sys.modules:
                pkg = _module(name)
                pkg.__path__ = [os.path.join(ref_shims.REFERENCE_ROOT, *name.split("."))]
        path = os.path.join(ref_shims.REFERENCE_ROOT, "src", "utils", "colmap", "read_write_model.py")
        spec = importlib.util.spec_from_file_location("src.utils.colmap.read_write_model", path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mod
        spec.loader.exec_module(mod)
    if "h5py" not in sys.modules or not hasattr(sys.modules["h5py"], "File"):
        sys.modules["h5py"] = fake_h5py()
    root = ref_shims.REFERENCE_ROOT
    for name in ("src.KeypointFreeSfM.post_optimization", "src.KeypointFreeSfM.post_optimization.utils",
                 "src.KeypointFreeSfM.post_optimization.matcher_model",
                 "src.KeypointFreeSfM.post_optimization.data_construct"):
        if name not in sys.modules:
            pkg = _module(name)
            pkg.__path__ = [os.path.join(root, *name.split("."))]
    agg = importlib.import_module("src.KeypointFreeSfM.post_optimization.feature_aggregation")
    worker = importlib.import_module("src.KeypointFreeSfM.post_optimization.matcher_model.fine_match_worker")
    cmd = importlib.import_module("src.KeypointFreeSfM.post_optimization.data_construct.construct_matching_data")
    return agg, worker, cmd


def reference_aggregation(ds, results, feats, image_lists, path="/fake/feats.h5"):
    """feature_aggregation_and_update on FakeH5 files: feats (the coarse stage's feature dict) is
    stored as <stem>_coarse.h5; returns (coarse file, fine file) as dicts of dicts of arrays."""
    agg, _, _ = load()
    io = sys.modules["src.KeypointFreeSfM.post_optimization.utils.io_utils"]
    old = io.h5py
    io.h5py = fake_h5py()
    try:
        coarse = path[:-3] + "_coarse.h5"
        FakeH5.store(coarse, feats)
        orig = os.path.exists
        io.osp.exists = lambda p: p in FakeH5.files or orig(p)
        try:
            agg.feature_aggregation_and_update(ds, results, path, image_lists, verbose=False)
        finally:
            io.osp.exists = orig
    finally:
        io.h5py = old
    return ({n: dict(g) for n, g in FakeH5.files[coarse].items()},
            {n: dict(g) for n, g in FakeH5.files[path].items()})
