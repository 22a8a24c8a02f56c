"""Training batches with the ground truth projected from the pose (onepose_plus_plus_b200/train_batch.py)
against the live reference dataset (OnePosePlusDataset.read_anno) on seeded on-disk stand-ins: the
same RNG draws, the SparseGT of the reference's dense tensors, the warped images, and the NumPy
restatement bit for bit on the CPU path; the collation of gt_source and the ValueError cases."""
import json

import numpy as np
import pytest
import torch
from torch.utils.data import default_collate

from oracle import ref_shims
from oracle import train_batch as otb
from onepose_plus_plus_b200 import train_batch, train_gt

needs_ref = pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")

CASES = {
    # more 3D points than shape3d (the padding's remap), no warp
    "remap": dict(seed=1, n_items=4, warp=False, shape3d=300, n_3d=420, n_corr=150, collide=6, repeat_2d=4),
    # fewer 3D points than shape3d (random padding), warp on odd indices
    "pad_warp": dict(seed=2, n_items=2, warp=True, shape3d=300, n_3d=200, n_corr=150, collide=6, repeat_2d=4),
    # query_image_scale != 1 and a non-square query image, warped
    "scale": dict(seed=3, n_items=2, warp=True, src_hw=(480, 640), img_resize=(512, 384), shape3d=300, n_3d=350,
                  n_corr=140, collide=4),
    # points behind the camera and outside the image; item 1 has no surviving correspondence
    "behind_outside": dict(seed=4, n_items=2, warp=True, shape3d=300, n_3d=320, n_corr=120, behind=10, outside=20,
                           empty_items=(1,)),
    # exact geometry: the reference's coordinates equal the restatement's bit for bit
    "exact": dict(seed=5, n_items=4, warp=False, src_hw=(480, 640), shape3d=300, n_3d=260, n_corr=150, collide=6,
                  repeat_2d=4, exact=True),
}


def run_items(case, ds, wrapped, n=4):
    refs, items, states = [], [], []
    for idx in range(n):
        seed = case["item_seeds"][idx // 2 if case["warp"] else idx]
        got = []
        for d, out in ((ds, refs), (wrapped, items)):
            np.random.seed(seed)
            torch.manual_seed(seed)
            out.append(d[idx])
            got.append((torch.get_rng_state(), np.random.get_state()))
        states.append(got)
    return refs, items, states


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    if not ref_shims.available():
        pytest.skip("needs the reference tree")
    out = {}
    for name, kw in CASES.items():
        case = otb.make_case(str(tmp_path_factory.mktemp(name)), **kw)
        ds = otb.reference_dataset(case)
        out[name] = (case, ds, *run_items(case, ds, train_batch.ProjectedGTDataset(ds)))
    return out


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_items_follow_the_reference(built, name):
    """Contract 3: the RNG states after each item equal the reference's; the sampled homography is
    the one the reference draws; the item is the reference's without the two dense tensors."""
    case, ds, refs, items, states = built[name]
    for idx, ((r_t, r_n), (m_t, m_n)) in enumerate(states):
        assert torch.equal(r_t, m_t), f"item {idx}: torch RNG state"
        assert r_n[0] == m_n[0] and np.array_equal(r_n[1], m_n[1]) and r_n[2:] == m_n[2:], f"item {idx}: np RNG"
    for idx, (r, m) in enumerate(zip(refs, items)):
        warped = case["warp"] and idx % 2 == 1
        h = m["gt_source"]["homography"]
        assert (h is not None) == warped
        if warped:
            hw = tuple(m["query_image"].shape[1:])
            assert np.array_equal(h.numpy(), otb._sample_homography(case["item_seeds"][idx // 2], *hw))
        assert set(r) - set(m) == {"conf_matrix_gt", "fine_location_matrix_gt"} and set(m) - set(r) == {"gt_source"}
        for k, v in m.items():
            if k in ("gt_source", "query_intrinsic") or (k == "query_image" and warped):
                continue
            assert (torch.equal(v, r[k]) if torch.is_tensor(v) else v == r[k]), k


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_prepare_batch_gives_the_reference_list(built, name):
    """Contracts 2 and 4 on the CPU path: ids equal to SparseGT.from_dense of the reference's collated
    dense tensors, fine_xy within 1e-3 px (bit-equal on the exact case), warped images within 1e-5,
    query_intrinsic = H @ K as the reference sets it."""
    case, ds, refs, items, _ = built[name]
    rb = default_collate(refs)
    want = train_gt.SparseGT.from_dense(rb["conf_matrix_gt"], rb["fine_location_matrix_gt"])
    batch = train_batch.prepare_batch(train_batch.collate(items))
    got = batch["gt_sparse"]
    assert "gt_source" not in batch and got.shape == want.shape
    for k in ("b_ids", "i_ids", "j_ids"):
        assert torch.equal(getattr(got, k), getattr(want, k)), k
    if CASES[name].get("exact"):
        assert torch.equal(got.fine_xy, want.fine_xy)
    else:
        assert torch.allclose(got.fine_xy, want.fine_xy, rtol=0, atol=1e-3)
    assert torch.allclose(batch["query_image"], rb["query_image"], rtol=0, atol=1e-5)
    assert torch.equal(batch["query_intrinsic"], rb["query_intrinsic"].to(batch["query_intrinsic"].dtype))
    if name == "behind_outside":
        # batch item 2 is dataset image 1 unwarped: every point outside (the warp of item 3 may bring
        # some inside)
        assert int((got.b_ids == 2).sum()) == 0 and int((got.b_ids == 0).sum()) > 0
    if name in ("remap", "exact"):
        # the tie rules were exercised: a cell with two correspondences, a repeated 2D keypoint
        assert len(got) < sum(int(it["gt_source"]["assign"].shape[1]) for it in items)


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_cpu_path_equals_the_restatement(built, name):
    """The torch CPU path of prepare_batch and the NumPy restatement: the same list and the same warped
    images bit for bit."""
    case, ds, refs, items, _ = built[name]
    batch = train_batch.collate(items)
    src = batch["gt_source"]
    img = batch["query_image"].clone()
    h, w = img.shape[-2:]
    packs = [otb.pack_item(src.pose_gt[b], src.K_crop[b], src.homography[b], h, w) for b in range(len(src))]
    assigns = [src.assign[:, src.offsets[b]:src.offsets[b + 1]].numpy() for b in range(len(src))]
    want = otb.batch_list(batch["keypoints3d"].numpy(), assigns, packs, batch["query_image_scale"].numpy(), (h, w))
    train_batch.prepare_batch(batch)
    got = batch["gt_sparse"]
    for g, wnt in zip((got.b_ids, got.i_ids, got.j_ids, got.fine_xy), want):
        assert np.array_equal(g.numpy(), wnt)
    for b in range(len(src)):
        assert np.array_equal(batch["query_image"][b, 0].numpy(), otb.warp_image(img[b, 0].numpy(), packs[b]))


@pytest.mark.parametrize("name", list(otb.EDGE_CASES))
def test_cpu_path_on_edge_batches(name):
    """The torch CPU path and the NumPy restatement on the edge batches of otb.EDGE_CASES: the same
    list and images bit for bit, or the same ValueError."""
    batch, expect = otb.edge_batch(name)
    src = batch["gt_source"]
    img = batch["query_image"].clone()
    h, w = img.shape[-2:]
    packs = [otb.pack_item(src.pose_gt[b], src.K_crop[b], src.homography[b], h, w) for b in range(len(src))]
    assigns = [src.assign[:, src.offsets[b]:src.offsets[b + 1]].numpy() for b in range(len(src))]
    args = (batch["keypoints3d"].numpy(), assigns, packs, batch["query_image_scale"].numpy(), (h, w))
    if expect == "grid size":
        with pytest.raises(ValueError, match="cell index == S"):
            otb.batch_list(*args)
    elif expect is None:
        want = otb.batch_list(*args)
    if expect is not None:
        with pytest.raises(ValueError, match=expect):
            train_batch.prepare_batch(batch)
        return
    train_batch.prepare_batch(batch)
    got = batch["gt_sparse"].check()
    for g, wnt in zip((got.b_ids, got.i_ids, got.j_ids, got.fine_xy), want):
        assert np.array_equal(g.numpy(), wnt)
    for b in range(len(src)):
        assert np.array_equal(batch["query_image"][b, 0].numpy(), otb.warp_image(img[b, 0].numpy(), packs[b]))


@needs_ref
def test_collate_and_pin(built, monkeypatch):
    case, ds, refs, items, _ = built["pad_warp"]
    batch = train_batch.collate(items)
    src = batch["gt_source"]
    counts = [it["gt_source"]["assign"].shape[1] for it in items]
    assert src.offsets.tolist() == np.cumsum([0] + counts).tolist()
    assert src.kp_offsets.tolist() == np.cumsum([0] + [it["gt_source"]["n_2d"] for it in items]).tolist()
    assert torch.equal(src.assign, torch.cat([it["gt_source"]["assign"] for it in items], 1))
    assert [h is not None for h in src.homography] == [False, True, False, True]
    pinned = []
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda t: pinned.append(t) or t.clone())
    p = src.pin_memory()
    assert len(pinned) == 3 and torch.equal(p.assign, src.assign) and p.n_kp == src.n_kp
    assert p.K_crop is src.K_crop and p.homography == src.homography
    moved = src.to("cpu")
    assert torch.equal(moved.offsets, src.offsets) and len(moved) == 4
    with pytest.raises(ValueError, match="some items"):
        train_batch.collate([items[0], {k: v for k, v in items[1].items() if k != "gt_source"}])


@needs_ref
@pytest.mark.parametrize("which", [0, 1])
def test_assign_out_of_range_raises(tmp_path, which):
    case = otb.make_case(str(tmp_path), seed=9, n_items=1, shape3d=300, n_3d=320, n_corr=40)
    ds = otb.reference_dataset(case)
    path = ds.coco.loadAnns(ds.coco.getAnnIds(imgIds=0))[0]["anno2d_file"].replace("/anno_loftr/",
                                                                                   "/anno_loftr_coarse/")
    with open(path) as f:
        d = json.load(f)
    d["assign_matrix"][which][3] = len(d["keypoints2d"]) if which == 0 else 320
    with open(path, "w") as f:
        json.dump(d, f)
    with pytest.raises(ValueError, match=f"assign_matrix\\[{which}\\]"):
        train_batch.ProjectedGTDataset(ds)[0]


def handmade_batch(points, scale, hw=(64, 64), L=8):
    """One item, identity pose and K: point (x, y) projects to (x, y) / (1 + 1e-6)."""
    h, w = hw
    kp = torch.zeros(1, L, 3)
    kp[0, :len(points), :2] = torch.tensor(points, dtype=torch.float32)
    kp[0, :, 2] = 1.0
    n = len(points)
    src = train_batch.GTSource(torch.stack([torch.arange(n), torch.arange(n)]), torch.tensor([0, n]),
                               torch.tensor([0, n]), n, torch.eye(3, dtype=torch.float64)[None],
                               torch.eye(4, dtype=torch.float64)[None], [None])
    return {"query_image": torch.zeros(1, 1, h, w), "keypoints3d": kp, "query_intrinsic": torch.eye(3)[None].double(),
            "query_image_scale": torch.tensor([scale], dtype=torch.float32), "gt_source": src}


def test_cell_index_at_the_grid_size_raises():
    """query_image_scale 0.5: the point rounded to (0, 32) gets the cell j = 8 * 8 + 0 = S, which the
    reference's j > S filter keeps and its matrix assignment writes out of bounds."""
    ok = train_batch.prepare_batch(handmade_batch([(9.0, 9.0), (17.0, 9.0)], [0.5, 0.5]))["gt_sparse"]
    assert ok.j_ids.tolist() == [2 * 8 + 2, 2 * 8 + 4] and ok.i_ids.tolist() == [0, 1]
    with pytest.raises(ValueError, match="grid size"):
        train_batch.prepare_batch(handmade_batch([(1.0, 32.0)], [0.5, 0.5]))
    with pytest.raises(ValueError, match="2D keypoints"):
        b = handmade_batch([(1.0, 1.0)], [1.0, 1.0])
        b["gt_source"].assign[0, 0] = 5
        train_batch.prepare_batch(b)


def test_the_later_keypoint_write_and_the_later_cell_write_win():
    """Two correspondences of one 2D keypoint: both read back the location of the one in the later
    np.unique row (the larger rounded x); two of one 3D point in one cell: the later one stays."""
    b = handmade_batch([(41.0, 9.0), (9.0, 17.0), (25.0, 25.0)], [1.0, 1.0])
    b["gt_source"].assign[0] = torch.tensor([0, 0, 1])
    g = train_batch.prepare_batch(b)["gt_sparse"]
    assert g.i_ids.tolist() == [0, 1, 2]
    # keypoint 0 is written by (9, 17) -> row (8, 16) first, then by (41, 9) -> row (40, 8)
    assert g.j_ids.tolist() == [1 * 8 + 5, 1 * 8 + 5, 3 * 8 + 3]
    assert torch.allclose(g.fine_xy[1], g.fine_xy[0]) and abs(float(g.fine_xy[0, 0]) - 41.0) < 1e-3
