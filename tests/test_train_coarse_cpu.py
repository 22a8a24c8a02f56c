"""CPU checks of the coarse training loss: the fp64 oracle (oracle/coarse_loss.py: loss and the
closed-form gradient the opp_coarse_focal kernels implement) against autograd through the
unmodified reference Loss.compute_coarse_loss, and the drop-in losses.Loss against the reference
Loss on a confidence tensor."""
import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import ref_shims
from onepose_plus_plus_b200 import SparseGT, losses

needs_ref = pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")


@needs_ref
@pytest.mark.parametrize("name", cl.CASES)
@pytest.mark.parametrize("gt_dtype", [torch.bool, torch.uint8, torch.int16])
def test_oracle_gradient_matches_reference_autograd(name, gt_dtype):
    a, b, gt, mask = cl.make_case(name)
    if gt_dtype == torch.bool and (name == "no_neg" or name == "random"):
        pytest.skip("bool cannot hold a value that is neither class")
    gt = gt.to(gt_dtype)
    s = cl.scale_of()
    # the reference's settings, then LoFTR's alpha with a non-integer gamma and unequal class weights:
    # at alpha = 0.5 and pos_w = neg_w the two classes' factors cannot be told apart
    for focal in ((0.5, 2.0, 1.0, 1.0), (0.25, 2.5, 2.0, 0.5)):
        config = dict(cl.LOSS_CONFIG, focal_alpha=focal[0], focal_gamma=focal[1], pos_weight=focal[2],
                      neg_weight=focal[3])
        ref_loss, ref_da, ref_db = cl.reference_loss_and_grads(a, b, gt, s, mask, config)
        loss, da, db = cl.focal_loss_and_grads(a, b, gt, s, mask, *focal)
        assert torch.isfinite(loss)
        assert abs(loss.item() - ref_loss.item()) <= 1e-12 * abs(ref_loss.item()), focal
        for got, ref in ((da, ref_da), (db, ref_db)):
            assert ref.abs().max() > 0
            assert torch.allclose(got, ref, rtol=1e-9, atol=1e-12 * float(ref.abs().max())), focal


def test_cases_cover_their_corners():
    s = cl.scale_of()
    for name in cl.CASES:
        a, b, gt, mask = cl.make_case(name)
        _, _, c = cl.dual_softmax(a.double(), b.double(), s, mask)
        npos, nneg = int((gt == 1).sum()), int((gt == 0).sum())
        assert (npos == 0) == (name == "no_pos") and (nneg == 0) == (name == "no_neg")
        if name == "clamp":
            assert (c > cl.HI).any() and (c < cl.LO).any()
        if name == "masked":
            assert (c[~mask[:, None, :].expand_as(c)] == 0).all() and (gt[~mask[:, None, :].expand_as(c)] == 1).any()


def test_no_positives_and_no_negatives_warn_like_the_reference():
    a, b, gt, _ = cl.make_case("planted")
    _, _, conf = cl.dual_softmax(a, b, cl.scale_of())
    loss = losses.Loss(cl.LOSS_CONFIG)
    assert torch.isnan(loss.compute_coarse_loss(conf, torch.full_like(gt, 2)))   # neither class: mean of nothing
    only_neg = loss.compute_coarse_loss(conf, torch.zeros_like(gt))
    assert torch.isfinite(only_neg) and only_neg > 0


@needs_ref
@pytest.mark.parametrize("with_fine", [False, True])
def test_dropin_loss_matches_reference_loss(with_fine):
    ref_shims.install()
    from src.lightning_model.losses import Loss as RefLoss   # type: ignore
    a, b, gt, mask = cl.make_case("masked", 2, 60, 48)
    _, _, conf = cl.dual_softmax(a, b, cl.scale_of(), mask)
    data = {"conf_matrix": conf, "conf_matrix_gt": gt}
    if with_fine:
        g = torch.Generator().manual_seed(4)
        data["expec_f"] = torch.cat([torch.rand(37, 2, generator=g) * 2 - 1, torch.rand(37, 1, generator=g)], 1)
        data["expec_f_gt"] = torch.rand(37, 2, generator=g) * 2.4 - 1.2
    outs = []
    for cls in (RefLoss, losses.Loss):
        d = dict(data)
        m = cls(cl.LOSS_CONFIG).train()
        m(d)
        outs.append(d)
    ref, got = outs
    assert torch.equal(got["loss"], ref["loss"])
    assert sorted(got["loss_scalars"]) == sorted(ref["loss_scalars"])
    for k, v in ref["loss_scalars"].items():
        assert torch.equal(got["loss_scalars"][k], v), k


def test_lazy_handle_rejects_loss_weights():
    class _H(losses.TrainConfHandle):
        def __init__(self):
            self.shape = torch.Size((1, 2, 3))
    with pytest.raises(NotImplementedError):
        losses.Loss(cl.LOSS_CONFIG)({"conf_matrix": _H(), "conf_matrix_gt": torch.zeros(1, 2, 3, dtype=torch.int16),
                                     "mask0": torch.ones(1, 2), "mask1": torch.ones(1, 3)})


def test_gt_dtype_is_checked_on_the_host():
    class _H(losses.TrainConfHandle):
        def __init__(self):
            self.shape = torch.Size((1, 2, 3))
    with pytest.raises(TypeError, match="bool, uint8 or int16"):
        losses.coarse_focal_loss(_H(), torch.zeros(1, 2, 3, dtype=torch.float32), 0.5, 2.0, 1.0, 1.0)


def test_fully_masked_sample_is_rejected():
    """A query mask that keeps no column of a sample leaves its softmax over S without terms: the
    eager path (sim - 1e9 on every column) gives the unmasked or a uniform softmax there, the kernels
    would give c = 0.  coarse_focal_loss refuses such a mask before any launch."""
    class _H(losses.TrainConfHandle):
        def __init__(self, col_mask):
            self.shape = torch.Size((2, 2, 3))
            self.col_mask = col_mask
    gt = torch.zeros(2, 2, 3, dtype=torch.int16)
    mask = torch.tensor([[1, 0, 1], [0, 0, 0]], dtype=torch.uint8)
    for g in (gt, SparseGT(*(torch.zeros(0, dtype=torch.int64),) * 3, torch.zeros(0, 2), (2, 2, 3))):
        with pytest.raises(ValueError, match="keeps no column"):
            losses.coarse_focal_loss(_H(mask), g, 0.5, 2.0, 1.0, 1.0)


def test_skip_mode_cannot_train():
    from oracle import make_reference_golden as mrg, workload
    from onepose_plus_plus_b200 import OnePosePlus_model
    m = OnePosePlus_model(mrg.train_config())
    m.load_state_dict(workload.synthetic_state_dict(0))
    m.train()
    m.conf_matrix_mode = "skip"
    with pytest.raises(ValueError, match="skip"):
        m(mrg.train_batch(workload.synthetic_state_dict(0), False))


def test_golden_matches_oracle():
    """The stored reference numbers (read by the GPU test) are what the fp64 oracle computes."""
    import os
    from tests import golden_io
    z = np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", "coarse_loss.npz"))
    for key, (name, batch, rows, cols) in cl.GOLDEN_CASES.items():
        a, b, gt, mask = cl.make_case(name, batch, rows, cols)
        loss, da, db = cl.focal_loss_and_grads(a, b, gt, cl.scale_of(), mask)
        assert abs(loss.item() - float(z[key + "_loss"])) <= 1e-12 * abs(loss.item())
        for nm, t in (("_da", da), ("_db", db)):
            got = t.flatten()[torch.from_numpy(z[key + nm + "_idx"])].numpy()
            assert np.allclose(got, z[key + nm], rtol=1e-9, atol=1e-12 * float(z[key + nm + "_absmax"]))
