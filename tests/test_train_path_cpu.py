"""CPU test of the training-mode forward (onepose_plus_plus_b200/train_path.py) against what the
unmodified reference computes in .train() mode (stored by oracle/make_reference_golden.py): same outputs, same random
ground-truth padding (identical RNG consumption), same gradients, same BatchNorm running-statistic
updates — i.e. PL_OnePosePlus.training_step (OnePosePlus_lightning_model.py:54-60) sees the same
thing from the drop-in as from the reference class."""
import os

import numpy as np
import pytest
import torch

from oracle import make_reference_golden as mrg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model
from tests import golden_io


def _sampled(t, z, name):
    return t.detach().flatten()[torch.from_numpy(z[name + "_idx"])].numpy()


@pytest.fixture
def train_threads():
    threads = torch.get_num_threads()
    torch.set_num_threads(mrg.TRAIN_THREADS)   # the thread count the stored reference was computed with
    yield
    torch.set_num_threads(threads)


@pytest.mark.parametrize("masked", [False, True])
def test_training_forward_and_gradients_match_reference(masked, train_threads):
    z = np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", "train_masked.npz" if masked else "train.npz"))
    sd = workload.synthetic_state_dict(0)
    cfg = mrg.train_config()
    ours = OnePosePlus_model(cfg)
    ours.load_state_dict(sd, strict=True)
    ours.train()
    data = mrg.train_batch(sd, masked)
    do = {k: v.clone() for k, v in data.items()}
    torch.manual_seed(11)
    ours(do)
    loss = mrg.train_loss(do)
    ours.zero_grad()
    loss.backward()
    lo, lr = loss.item(), float(z["loss"])
    assert len(z["b_ids"]) > 50 and z["gt_mask"].any() and not z["gt_mask"].all()   # predictions + gt padding
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "mkpts_3d_db", "mkpts_query_c"):
        assert np.array_equal(do[k].detach().numpy(), z[k]), k
    assert np.allclose(_sampled(do["conf_matrix"], z, "conf_matrix"), z["conf_matrix"], rtol=1e-3, atol=1e-5)
    for k in ("mconf", "mkpts_query_f"):
        assert np.allclose(do[k].detach().numpy(), z[k], rtol=1e-3, atol=1e-5), k
    assert np.allclose(do["expec_f"][:, :2].detach().numpy(), z["expec_f"][:, :2], atol=1e-5)
    assert np.allclose(do["expec_f"][:, 2].detach().numpy(), z["expec_f"][:, 2], atol=5e-3)
    assert do["W"] == 5 and tuple(do["q_hw_c"]) == (12, 16) and abs(lr - lo) <= 1e-4 * abs(lr)
    po = dict(ours.named_parameters())
    checked = 0
    for i, name in enumerate(mrg.TRAIN_GRADS):
        go = po[name].grad
        assert go is not None, name
        assert np.allclose(_sampled(go, z, f"grad{i}"), z[f"grad{i}"], rtol=2e-4,
                           atol=1e-6 + 2e-4 * float(z[f"grad{i}_absmax"])), name
        checked += 1
    assert checked == 8
    # BatchNorm ran on batch statistics and moved its running buffers identically
    bo = dict(ours.named_buffers())
    k = "backbone.layer1.0.bn1.running_mean"
    assert not torch.equal(bo[k], sd[k]) and np.allclose(z["bn_running_mean"], bo[k].numpy(), atol=1e-6)
    assert int(bo["backbone.bn1.num_batches_tracked"]) == 1
    # back in eval mode the CUDA path is the only path (no silent fallback on CPU tensors)
    ours.eval()
    with pytest.raises(RuntimeError, match="no CPU path"):
        ours({k: v.clone() for k, v in data.items() if k != "conf_matrix_gt"})
