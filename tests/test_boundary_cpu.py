"""Boundary proof (CPU): the drop-in classes accept what the reference's callers hand them.

INTEGRATION.md §1 changes only import lines in the reference, so its callers keep doing what they
do with the matcher:
  * the inference builder (src/inference/inference_OnePosePlus.py:28-38) constructs the model from
    the config, loads the `matcher.`-prefixed state dict of a Lightning checkpoint with
    strict=True and calls .eval(); Ray then pickles the module for its workers (:86-94);
  * PL_OnePosePlus (src/lightning_model/OnePosePlus_lightning_model.py:20-49) holds the model as
    its `matcher` submodule and loads the whole checkpoint into itself.
The tests below perform those operations on the drop-in with plain PyTorch calls."""
import os
import pickle

import pytest
import torch
import torch.nn as nn

from oracle import oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model


def _pl_checkpoint(tmp_path):
    sd = workload.synthetic_state_dict(0)
    path = str(tmp_path / "pl.ckpt")
    torch.save({"state_dict": {"matcher." + k: v for k, v in sd.items()}}, path)   # PL checkpoint layout
    return sd, path


def test_inference_builder_loads_checkpoint_and_pickles(tmp_path):
    sd, ckpt = _pl_checkpoint(tmp_path)
    model = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    state = torch.load(ckpt, map_location="cpu")["state_dict"]
    model.load_state_dict({k.replace("matcher.", "", 1): v for k, v in state.items()}, strict=True)
    model.eval()
    assert isinstance(model, OnePosePlus_model) and not model.training
    got = model.state_dict()
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    # Ray serialises the module object for its workers
    clone = pickle.loads(pickle.dumps(model))
    assert not clone.training and all(torch.equal(clone.state_dict()[k], sd[k]) for k in sd)
    assert clone._plan is None and clone._ws == {}          # device caches never travel
    # the worker then does match_model.cuda(); match_model(data): without a GPU that must fail loudly
    with pytest.raises(RuntimeError, match="no CPU path"):
        clone(workload.random_workload(64, 64, 50))


def test_lightning_module_holds_the_drop_in_as_matcher(tmp_path):
    sd, ckpt = _pl_checkpoint(tmp_path)

    class Holder(nn.Module):                                # the matcher slot of PL_OnePosePlus
        def __init__(self, config):
            super().__init__()
            self.matcher = OnePosePlus_model(config)

    module = Holder(oracle.DEFAULT_CONFIG)
    module.load_state_dict(torch.load(ckpt, map_location="cpu")["state_dict"], strict=True)
    got = module.matcher.state_dict()
    assert all(torch.equal(got[k], sd[k]) for k in sd)      # the strict full-checkpoint load went through
    module.eval()
    assert not module.matcher.training
    module.train()
    assert module.matcher.training
    assert sum(p.numel() for p in module.parameters()) == 10_226_480


def test_loftr_drop_in_has_the_reference_layout():
    """LoFTR_for_OnePose_Plus (SURVEY §8 f3): same ctor, same state-dict keys / shapes as the reference
    class built from submodules/LoFTR/src/loftr (stored by oracle/make_reference_golden.py; the
    reference loads this layout strictly), non-persistent pos-enc buffer."""
    import numpy as np
    from oracle import loftr_oracle
    from onepose_plus_plus_b200 import LoFTR_for_OnePose_Plus
    from tests import golden_io
    z = np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", "loftr_layout.npz"))
    rs = workload.synthetic_loftr_state_dict(0)
    ours = LoFTR_for_OnePose_Plus(dict(loftr_oracle.DEFAULT_CONFIG), enable_fine_matching=True)
    os_ = ours.state_dict()
    assert sorted(os_) == list(z["keys"])
    assert [str(tuple(os_[k].shape)) for k in sorted(os_)] == list(z["shapes"])
    ours.load_state_dict(rs, strict=True)
    pe = ours.pos_encoding.pe
    assert tuple(pe.shape) == tuple(z["pe_shape"]) and "pos_encoding.pe" not in os_
    assert torch.equal(pe.flatten()[torch.from_numpy(z["pe_idx"])], torch.from_numpy(z["pe"]))
    clone = pickle.loads(pickle.dumps(ours.eval()))
    assert all(torch.equal(clone.state_dict()[k], rs[k]) for k in rs)
    with pytest.raises(RuntimeError, match="no CPU path"):
        clone({"image0": torch.rand(1, 1, 64, 64), "image1": torch.rand(1, 1, 64, 64)})
