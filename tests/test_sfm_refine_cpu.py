"""CPU checks of the SfM refinement drop-ins (onepose_plus_plus_b200.sfm_refine): the NumPy
restatement (oracle/sfm_refine.py) against the live reference's MatchingPairData.__getitem__ (bit
for bit) and sample_feature_from_featuremap (nearest bit for bit, bilinear within four fp32
roundings of the largest tap), the vectorised pair lists and track bookkeeping against the
restatement, and the input errors raised before any launch."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import ref_shims
from oracle import sfm_refine as osr

needs_ref = pytest.mark.skipif(not ref_shims.available(), reason="reference tree not present")
CASES = [dict(seed=0), dict(seed=1, max_track=60, n_images=64, n_points=400, n_kpts=120),
         dict(seed=2, left_f32=False, scale=(1.25, 0.8)), dict(seed=3, n_images=3, n_points=20)]


def _ref_module(rel, name):
    path = os.path.join(ref_shims.REFERENCE_ROOT, rel)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _ImageDataset:
    """The reference MatchingPairData reads colmap_image_dataset[...] for the images; the pair lists do
    not depend on them."""

    def __init__(self, ds):
        self.__dict__.update(ds.__dict__)
        self.colmap_cameras = {}

    def __getitem__(self, i):
        return {"image": torch.zeros(1, 1, 8, 8), "scale": torch.ones(1, 2), "img_path": f"{i}"}


@needs_ref
@pytest.mark.parametrize("case", range(len(CASES)))
def test_pair_lists_equal_reference(case):
    from onepose_plus_plus_b200 import sfm_refine
    ds, _ = osr.seeded_reconstruction(**CASES[case])
    mod = _ref_module("src/KeypointFreeSfM/post_optimization/data_construct/construct_matching_data.py", "_ref_cmd")
    ref_ds = mod.MatchingPairData(_ImageDataset(ds))
    assert ref_ds.all_pairs == ds.all_pairs
    rest = osr.pair_lists(ds)
    pairs, mk0, mk1, idx = sfm_refine.pair_lists(ds)
    assert [list(p) for p in pairs] == ds.all_pairs
    twice = False
    for i in range(len(ref_ds)):
        r = ref_ds[i]
        for got, (a, b, c) in ((r, rest[i]), ({"mkpts0_c": mk0[i], "mkpts1_c": mk1[i], "mkpts0_idx": idx[i]}, rest[i])):
            for k, v in (("mkpts0_c", a), ("mkpts1_c", b), ("mkpts0_idx", c)):
                g = np.asarray(got[k])
                assert g.dtype == v.dtype and np.array_equal(g, v), (i, k)
        twice |= any((ds.colmap_3ds[p].image_ids == ds.all_pairs[i][1]).sum() > 1
                     for p in ds.colmap_frame_dict[ds.all_pairs[i][0]]["all_kpt_status"] if p >= 0)
    assert twice or case == 3


@needs_ref
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nearest", [True, False])
@pytest.mark.parametrize("scale", [(1.0, 1.0), (1.25, 0.8)])
def test_sample_restatement_equals_reference(dtype, nearest, scale):
    ref_shims.install()
    mod = _ref_module("src/KeypointFreeSfM/loftr_for_sfm/utils/sample_feature_from_featuremap.py", "_ref_sff")
    rng = np.random.default_rng(0)
    fmap = rng.standard_normal((32, 12, 16)).astype(np.float32)
    h, w = 96, 128
    k = np.concatenate([[[0, 0], [w - 1, h - 1], [w + 3, 2], [4.5, 7.5], [-2, 5]],
                        np.stack([rng.uniform(-2, w + 2, 400), rng.uniform(-2, h + 2, 400)], 1)]).astype(dtype)
    sc = torch.tensor([scale], dtype=torch.float32)
    imghw = sc.squeeze(0) * torch.tensor((h, w)).to(sc)
    ref = mod.sample_feature_from_featuremap(torch.from_numpy(fmap)[None], torch.from_numpy(k), imghw=imghw,
                                             sample_mode="nearest" if nearest else "bilinear").numpy()
    got = osr.sample(fmap, k, imghw.numpy(), nearest)
    if nearest:
        assert np.array_equal(ref.view(np.int32), got.view(np.int32))
    else:
        # PyTorch's CPU kernel may contract the weighted sum into FMAs; the restatement (and the device
        # kernel) round every product and sum once.  Four roundings of terms bounded by max|map|.
        bound = 4 * np.finfo(np.float32).eps * np.abs(fmap).max()
        assert np.abs(ref - got).max() <= bound


@pytest.mark.parametrize("case", range(len(CASES)))
def test_track_bookkeeping_equals_restatement(case):
    """The host half of feature_aggregation_and_update with the restatement's means in place of the
    device's equals the restatement's loop."""
    from onepose_plus_plus_b200 import sfm_refine
    ds, feats = osr.seeded_reconstruction(**CASES[case])
    res = osr.synthetic_results(ds, case)
    ref_c, ref_f = osr.aggregate(ds, res, feats)
    tm = sfm_refine.track_members(ds, res)
    rowmap = {k: i for i, k in enumerate(tm["row_key"].tolist())}
    rows = np.asarray([rowmap[q] for q in tm["query"].tolist()], np.int64)
    cat = lambda k: np.concatenate([res[n][k] for n in tm["names"]])   # noqa: E731
    c0, c1, f0, f1 = cat("feature_c0"), cat("feature_c1"), cat("feature0"), cat("feature1")
    off = tm["track_off"]
    mean = lambda a: np.stack([np.mean(a[rows[off[t]:off[t + 1]]], axis=0) for t in range(len(off) - 1)])  # noqa: E731
    got_c, got_f = copy.deepcopy(feats), copy.deepcopy(feats)
    sfm_refine.apply_updates(got_c, got_f, ds.colmap_images, tm, mean(c0), mean(f0), c1[rows], f1[rows])
    for ref, got in ((ref_c, got_c), (ref_f, got_f)):
        for n in ref:
            for k in ("descriptors", "keypoints", "scores"):
                assert ref[n][k].dtype == got[n][k].dtype and np.array_equal(ref[n][k], got[n][k]), (n, k)
    n0 = ds.colmap_images[ds.all_pairs[0][0]].name
    assert ref_c[n0]["descriptors"].shape[0] == 256 and ref_f[n0]["descriptors"].shape[0] == 128
    assert ref_f[n0]["descriptors"].dtype == np.float64


def test_cells_round_half_even_and_wrap():
    mk = np.array([[4.0, 12.0], [12.0, 20.0], [125.0, 3.0], [-5.0, 200.0]], np.float64)
    clipped, ids = osr.cells(mk, 96, 128, 12, 16)
    assert clipped[3].tolist() == [0.0, 94.0]
    assert ids[:2].tolist() == [2 * 16 + 0, 2 * 16 + 2]          # 0.5 -> 0, 1.5 -> 2, 2.5 -> 2
    assert ids[2] == 0 * 16 + 16                                  # x rounds to wc: the next row


def test_input_errors():
    from onepose_plus_plus_b200 import sfm_refine
    ds, _ = osr.seeded_reconstruction(0)
    res = osr.synthetic_results(ds, 0)
    first = next(iter(res))
    del res[first]
    with pytest.raises(ValueError, match="not in the fine match results"):
        sfm_refine.track_members(ds, res)
    ds2, _ = osr.seeded_reconstruction(0)
    pid = next(iter(ds2.point_cloud_assigned_imgID_kptID))
    a = ds2.point_cloud_assigned_imgID_kptID[pid][0]
    ds2.colmap_3ds[pid].image_ids[:] = a
    with pytest.raises(ValueError, match="no observation outside"):
        sfm_refine.track_members(ds2, osr.synthetic_results(ds, 0))
    ds3, _ = osr.seeded_reconstruction(0)
    left, right = ds3.all_pairs[0]
    for p in ds3.colmap_3ds.values():
        p.image_ids[p.image_ids == right] = -7
    with pytest.raises(ValueError, match="shares no track"):
        sfm_refine.pair_lists(ds3)
    with pytest.raises(NotImplementedError):
        sfm_refine.feature_aggregation_and_update(ds, res, "/nonexistent/f.h5", [], aggregation_method="max")


@needs_ref
@pytest.mark.parametrize("case", range(len(CASES)))
def test_aggregation_restatement_equals_reference(case):
    """oracle/sfm_refine.py:aggregate against the live feature_aggregation_and_update, through
    in-memory h5 files: both files' keys, shapes, dtypes and values bit for bit (coarse descriptors
    float64 [256, N], fine float64 [128, N] after the re-zero, COLMAP xys as the fine keypoints)."""
    from oracle import sfm_refine_ref
    ds, feats = osr.seeded_reconstruction(**CASES[case])
    res = osr.synthetic_results(ds, case)
    ref_c, ref_f = sfm_refine_ref.reference_aggregation(ds, res, feats, list(feats))
    got_c, got_f = osr.aggregate(ds, res, feats)
    for ref, got in ((ref_c, got_c), (ref_f, got_f)):
        assert list(ref) == list(got)
        for n in ref:
            assert sorted(ref[n]) == sorted(got[n])
            for k in ref[n]:
                assert ref[n][k].dtype == got[n][k].dtype and np.array_equal(ref[n][k], got[n][k]), (n, k)
    touched = {ds.colmap_images[a].name for a, _ in ds.point_cloud_assigned_imgID_kptID.values()}
    for n in touched:
        assert ref_c[n]["descriptors"].dtype == ref_f[n]["descriptors"].dtype == np.float64
        assert ref_c[n]["descriptors"].shape[0] == 256 and ref_f[n]["descriptors"].shape[0] == 128
    for im in ds.colmap_images.values():
        assert ref_f[im.name]["keypoints"] is not None and np.array_equal(ref_f[im.name]["keypoints"], im.xys)


@needs_ref
def test_cells_equal_reference_forward():
    """The clip and the cell ids of the fine-only branch: oracle/sfm_refine.py:cells against the live
    reference forward on CPU (and the stored golden), on points at the clip edge, at .5 cells, at the
    wc wrap, with non-integer scales and fp32 / fp64 keypoints."""
    from oracle import loftr_oracle, make_sfm_refine_golden as mk, workload
    sd, data = workload.planted_loftr(*mk.HW, seed=0)
    ref = ref_shims.build_reference_loftr(sd, loftr_oracle.DEFAULT_CONFIG, enable_fine_matching=False)
    mk0, mk1 = mk.given_matches()
    d = {"image0": data["image0"], "image1": data["image1"],
         "scale0": torch.tensor([mk.FWD_SCALES[0]]), "scale1": torch.tensor([mk.FWD_SCALES[1]]),
         "mkpts0_c": torch.from_numpy(mk0.copy()), "mkpts1_c": torch.from_numpy(mk1.copy())}
    with torch.no_grad():
        ref(d)
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference", "sfm_refine.npz"))
    c0, i_ids = osr.cells(mk0, *mk.HW, 12, 16, mk.FWD_SCALES[0])
    c1, j_ids = osr.cells(mk1, *mk.HW, 12, 16, mk.FWD_SCALES[1])
    for got, want, gold in ((c0, d["mkpts0_c"], "fwd_mkpts0_c"), (c1, d["mkpts1_c"], "fwd_mkpts1_c"),
                            (i_ids, d["i_ids"], "fwd_i_ids"), (j_ids, d["j_ids"], "fwd_j_ids")):
        w = want.numpy()
        assert got.dtype == w.dtype and np.array_equal(got, w) and np.array_equal(got, z[gold])
    assert i_ids[0] == 4 * 16 + 20          # x = 126 / (8 * 0.8) rounds to 20 > wc: it wraps into the next row
