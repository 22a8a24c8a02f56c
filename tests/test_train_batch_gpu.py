"""Training batches on the device: opp_homography_warp_f32 / opp_train_gt_build / opp_train_gt_compact
against the NumPy restatement (oracle/train_batch.py) bit for bit, prepare_batch against the reference
dataset's lists stored in tests/golden/reference/train_batch.npz (128x96 images; the training shape
runs on synthetic batches against the restatement), and a kernel-mode training step
from prepare_batch's batch against the same step with the host-built list."""
import os

import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_batch_golden as mtbg
from oracle import train_batch as otb
from oracle import train_gt as otg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, SparseGT, losses, train_batch, train_gt

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "train_batch.npz")


def golden(name):
    return mtbg.load(GOLDEN, name)


def batch_from(d):
    """the collated ProjectedGTDataset batch the golden was made from (host tensors)"""
    hs = [d["homography"][b] if bool(d["warped"][b]) else None for b in range(len(d["warped"]))]
    src = train_batch.GTSource(d["assign"], d["offsets"], d["kp_offsets"], int(d["kp_offsets"][-1]), d["K_crop"],
                               d["pose_gt"], hs)
    return {"query_image": d["image"].clone(), "keypoints3d": d["keypoints3d"], "query_image_scale": d["scale"],
            "query_intrinsic": d["K_crop"].clone(), "gt_source": src}


def to_cuda(batch):
    return {k: (v.to("cuda") if torch.is_tensor(v) or isinstance(v, train_batch.GTSource) else v)
            for k, v in batch.items()}


def restated(batch):
    """(list, images) of the NumPy restatement on a host batch; the list is the ValueError it raises
    instead, if it does"""
    src = batch["gt_source"]
    img = batch["query_image"]
    h, w = img.shape[-2:]
    packs = [otb.pack_item(src.pose_gt[b], src.K_crop[b], src.homography[b], h, w) for b in range(len(src))]
    assigns = [src.assign[:, src.offsets[b]:src.offsets[b + 1]].numpy() for b in range(len(src))]
    try:
        lst = otb.batch_list(batch["keypoints3d"].numpy(), assigns, packs, batch["query_image_scale"].numpy(),
                             (h, w))
    except ValueError as e:
        lst = e
    return lst, [otb.warp_image(img[b, 0].numpy(), packs[b]) for b in range(len(src))]


def check_against_restatement(batch, expect=None):
    """The device path and the restatement: ids equal, fine_xy and the images bit-equal; or, with
    expect, the ValueError expect names (S = 0: prepare_batch refuses the image up front)."""
    (lst, imgs) = restated(batch)
    if expect == "grid size":
        assert isinstance(lst, ValueError), "the restatement has no cell index at the grid size"
    elif expect is None:
        assert not isinstance(lst, ValueError), lst
    if expect is not None:
        with pytest.raises(ValueError, match=expect):
            train_batch.prepare_batch(to_cuda(batch))
        return None
    lb, li, lj, lxy = lst
    out = train_batch.prepare_batch(to_cuda(batch))
    got = out["gt_sparse"].check()
    assert np.array_equal(got.b_ids.cpu().numpy(), lb) and np.array_equal(got.i_ids.cpu().numpy(), li)
    assert np.array_equal(got.j_ids.cpu().numpy(), lj)
    assert np.array_equal(got.fine_xy.cpu().numpy(), lxy), "fine_xy differs from the restatement"
    for b, want in enumerate(imgs):
        assert np.array_equal(out["query_image"][b, 0].cpu().numpy(), want), f"image {b}"
    return got


@pytest.mark.parametrize("name", ["golden_warp", "golden_exact", "training_shape", "training_shape_scaled",
                                  "no_correspondence", *otb.EDGE_CASES])
def test_kernels_equal_the_restatement(name):
    """Contract 1: ids equal, fine_xy and the images bit-equal; on the edge batches of
    otb.EDGE_CASES (odd sizes, j == S, scales, contention, rounding edges, sign flips, empty items)
    the same list or the same ValueError."""
    if name in otb.EDGE_CASES:
        batch, expect = otb.edge_batch(name)
        got = check_against_restatement(batch, expect)
        print(f"{name}: {'ValueError' if got is None else len(got)}")
        return
    if name.startswith("golden"):
        batch = batch_from(golden(name.split("_")[1]))
    elif name == "no_correspondence":
        batch = otb.synthetic_batch(3, B=2, L=50, n_corr=0, n_2d=10)
    else:
        batch = otb.synthetic_batch(1 if name == "training_shape" else 2,
                                scale=(1.0, 1.0) if name == "training_shape" else (0.9375, 1.25))
    got = check_against_restatement(batch)
    if name.startswith("training_shape"):
        assert got.shape == (4, 7000, 4096) and len(got) > 4 * 1000
        print(f"{name}: {len(got)} correspondences")
    if name == "no_correspondence":
        assert len(got) == 0


@pytest.mark.parametrize("name", ["warp", "exact"])
def test_prepare_batch_gives_the_reference_list(name):
    """Contract 4 against the reference dataset's collated dense tensors (stored as their SparseGT)."""
    d = golden(name)
    out = train_batch.prepare_batch(to_cuda(batch_from(d)))
    got = out["gt_sparse"]
    assert tuple(got.shape) == tuple(d["shape"].tolist())
    for k, r in (("b_ids", "ref_b"), ("i_ids", "ref_i"), ("j_ids", "ref_j")):
        assert torch.equal(getattr(got, k).cpu(), d[r]), k
    if name == "exact":
        assert torch.equal(got.fine_xy.cpu(), d["ref_xy"])
    else:
        assert torch.allclose(got.fine_xy.cpu(), d["ref_xy"], rtol=0, atol=1e-3)
    assert torch.allclose(out["query_image"].cpu(), d["ref_image"], rtol=0, atol=1e-5)
    assert torch.equal(out["query_intrinsic"].cpu(), d["ref_intrinsic"])


def test_cuda_and_cpu_paths_agree():
    batch = batch_from(golden("warp"))
    cpu = train_batch.prepare_batch(batch_from(golden("warp")))
    dev = train_batch.prepare_batch(to_cuda(batch))
    for k in ("b_ids", "i_ids", "j_ids", "fine_xy"):
        assert torch.equal(getattr(dev["gt_sparse"], k).cpu(), getattr(cpu["gt_sparse"], k)), k
    assert torch.equal(dev["query_image"].cpu(), cpu["query_image"])


def test_bad_cell_and_assign_raise():
    from tests.test_train_batch_cpu import handmade_batch
    with pytest.raises(ValueError, match="grid size"):
        train_batch.prepare_batch(to_cuda(handmade_batch([(1.0, 32.0)], [0.5, 0.5])))
    b = handmade_batch([(1.0, 1.0)], [1.0, 1.0])
    b["gt_source"].assign[1, 0] = 8
    with pytest.raises(ValueError, match="3D points"):
        train_batch.prepare_batch(to_cuda(b))


@pytest.mark.parametrize("name", ["exact", "warp"])
def test_training_step_from_prepare_batch(name):
    """model.train(), conf_matrix_mode "lazy", every *_train_mode "kernels": the step on prepare_batch's
    batch and the step on the same batch with the host-built SparseGT of the reference's dense
    tensors give the same gt_mask, ids and RNG state, and the same loss bits where the two lists are
    bit-equal (exact); on the warped batch the fine locations differ by < 1e-3 px, so the loss agrees
    to that."""
    d = golden(name)
    sd = workload.synthetic_state_dict(0)
    h, w = d["image"].shape[-2:]
    base, _ = workload.planted_workload(sd, h, w, int(d["shape"][1]), 150, batch=4, seed=5)
    runs = {}
    for route in ("device", "host"):
        m = OnePosePlus_model(mrg.train_config())
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
        m.conf_matrix_mode = "lazy"
        for k in ("fine_train_mode", "coarse_transformer_train_mode", "backbone_train_mode",
                  "kpt_encoder_train_mode"):
            setattr(m, k, "kernels")
        batch = batch_from(d)
        data = {k: v for k, v in base.items() if k not in ("query_image", "keypoints3d")}
        data.update({k: batch[k] for k in ("query_image", "keypoints3d", "query_image_scale", "query_intrinsic")})
        data["gt_source"] = batch["gt_source"]
        data = to_cuda(data)
        train_batch.prepare_batch(data)
        if route == "host":
            data["gt_sparse"] = SparseGT(d["ref_b"], d["ref_i"], d["ref_j"], d["ref_xy"],
                                         tuple(d["shape"].tolist())).to("cuda")
        torch.manual_seed(11)
        m(data)
        train_gt.fine_supervision(data, otg.config())
        losses.Loss(cl.LOSS_CONFIG).train()(data)
        data["loss"].backward()
        torch.cuda.synchronize()
        runs[route] = (data, torch.cuda.get_rng_state(), torch.get_rng_state())
    (dd, dcr, dhr), (hd, hcr, hhr) = runs["device"], runs["host"]
    for k in ("gt_mask", "b_ids", "i_ids", "j_ids", "m_bids"):
        assert torch.equal(dd[k], hd[k]), k
    assert torch.equal(dcr, hcr) and torch.equal(dhr, hhr)
    if name == "exact":
        assert torch.equal(dd["expec_f_gt"], hd["expec_f_gt"]) and torch.equal(dd["loss"], hd["loss"])
    else:
        assert abs(dd["loss"].item() - hd["loss"].item()) <= 1e-4 * abs(hd["loss"].item()) + 1e-6
