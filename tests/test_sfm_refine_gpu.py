"""pytest -m gpu: the keypoint-free SfM refinement on the device.

  * opp_sample_feature is bit-equal to oracle/sfm_refine.py's sample in nearest and bilinear mode,
    on 256- and 128-channel maps with and without the lo plane, fp32 and fp64 keypoints, points at 0,
    at hw - 1, one ulp past it, outside the map, at .5 and with non-integer scales; outputs prefilled
    with NaN.
  * The lookup and aggregation kernels are bit-equal to the restatement from 1 track to 100 k tracks.
  * The track bookkeeping plus the device means equal oracle/sfm_refine.py's loop restatement of
    feature_aggregation_and_update on seeded reconstructions.
  * fine_matches_for_pairs equals one fine-only forward with both extractions per pair at pair
    batches 1, 7 and 32: ids and sampled features bit-equal, mkpts1_f / expec_f within 1e-4.
  * The fine-only forward with both extractions matches the reference's, stored in
    tests/golden/reference/sfm_refine.npz: ids and clipped keypoints equal, mkpts1_f / expec_f within
    the 2D-2D matcher's tolerances, the sampled features within FEAT_TOL.
  * End to end, fine_matcher equals the stored reference result (the 11 arrays of every pair), and
    feature_aggregation_and_update writes the reference's two files: bit for bit from the reference's
    match results, within FEAT_TOL from ours."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import sfm_refine as osr
from oracle import workload

pytestmark = pytest.mark.gpu


def _store(rng, n, h, w, c, split):
    hi = torch.from_numpy(rng.standard_normal((n, h, w, c)).astype(np.float32)).half()
    if not split:
        return hi.cuda(), hi.float().numpy()
    lo = torch.from_numpy((rng.standard_normal((n, h, w, c)) * 1e-4).astype(np.float32)).half()
    full = (hi.float() + lo.float()).numpy()          # one fp32 rounding, as the kernel adds them
    return torch.cat([hi, lo], -1).contiguous().cuda(), full


def _points(rng, h_img, w_img, n, dtype):
    edge = [[0, 0], [w_img - 1, h_img - 1], [np.nextafter(np.float32(w_img - 1), np.float32(1e9)), 3.0],
            [w_img + 5.0, 2.0], [-3.0, -1.0], [4.5, 7.5], [w_img - 1.5, h_img - 0.5], [2.0, h_img + 0.25]]
    rnd = np.stack([rng.uniform(-2, w_img + 2, n), rng.uniform(-2, h_img + 2, n)], 1)
    half = np.stack([rng.integers(0, w_img // 2, n) + 0.5, rng.integers(0, h_img // 2, n) * 2 + 0.5], 1)
    return np.concatenate([edge, rnd, half]).astype(dtype)


@pytest.mark.parametrize("channels,hm,wm,img", [(256, 12, 16, (96, 128)), (128, 48, 64, (96, 128))])
@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nearest", [True, False])
@pytest.mark.parametrize("scale", [(1.0, 1.0), (1.25, 0.8), (1.0 / 0.75, 1.1)])
def test_sample_feature_bit_equal(channels, hm, wm, img, split, dtype, nearest, scale):
    from onepose_plus_plus_b200 import ops
    rng = np.random.default_rng(channels + hm + int(split) * 7)
    store, full = _store(rng, 2, hm, wm, channels, split)
    imghw = np.stack([np.float32(scale[0]) * np.float32(img[0]), np.float32(scale[1]) * np.float32(img[1])])
    imghw = np.stack([imghw, np.float32([img[0], img[1]])]).astype(np.float32)
    k = _points(rng, img[0], img[1], 300, dtype)
    ids = (np.arange(len(k)) % 2).astype(np.int64)
    out = torch.full((len(k), channels), float("nan"), device="cuda")
    ops.sample_feature(store, channels, split, torch.from_numpy(k).cuda(), torch.from_numpy(imghw).cuda(), nearest,
                       torch.from_numpy(ids).cuda(), out)
    got = out.cpu().numpy()
    for b in (0, 1):
        ref = osr.sample(np.ascontiguousarray(full[b].transpose(2, 0, 1)), k[ids == b], imghw[b], nearest)
        assert np.array_equal(got[ids == b].view(np.int32), ref.view(np.int32))


@pytest.mark.parametrize("tracks,max_len", [(1, 1), (7, 60), (1000, 60), (100_000, 6)])
def test_aggregate_kernels_bit_equal(tracks, max_len):
    from onepose_plus_plus_b200 import ops
    rng = np.random.default_rng(tracks)
    lens = rng.integers(1, max_len + 1, tracks)
    K = int(lens.sum())
    R = K + 17
    rows = rng.permutation(R)[:K].astype(np.int64)     # distinct rows of a results table
    key = rng.permutation(np.arange(R, dtype=np.int64) * 3 + (5 << 32))
    query = key[rows]
    row = ops.sfm_refine_lookup(torch.from_numpy(key).cuda(), torch.from_numpy(query).cuda()).cpu().numpy()
    assert np.array_equal(row, rows)
    miss = ops.sfm_refine_lookup(torch.from_numpy(key).cuda(), torch.tensor([1, int(key[0])], device="cuda"))
    assert miss.tolist() == [-1, int(np.flatnonzero(key == key[0])[0])]
    dup = ops.sfm_refine_lookup(torch.from_numpy(np.r_[key, key[:1]]).cuda(), torch.from_numpy(key[:1]).cuda())
    assert dup.tolist() == [-2]
    c0, c1 = (rng.standard_normal((R, 256)).astype(np.float32) for _ in range(2))
    f0, f1 = (rng.standard_normal((R, 128)).astype(np.float32) for _ in range(2))
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    cu = lambda a: torch.from_numpy(a).cuda()      # noqa: E731
    mc, mf, rc, rf = (o.cpu().numpy() for o in ops.sfm_refine_aggregate(cu(c0), cu(c1), cu(f0), cu(f1), cu(rows),
                                                                        cu(off)))
    assert np.array_equal(rc, c1[rows]) and np.array_equal(rf, f1[rows])
    pick = range(tracks) if tracks <= 1000 else rng.choice(tracks, 2000, replace=False)
    for t in pick:
        seg = rows[off[t]:off[t + 1]]
        assert np.array_equal(mc[t], np.mean(c0[seg], axis=0)), t
        assert np.array_equal(mf[t], np.mean(f0[seg], axis=0)), t


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_aggregation_equals_restatement(seed):
    from onepose_plus_plus_b200 import sfm_refine
    ds, feats = osr.seeded_reconstruction(seed, n_images=10, n_points=300, max_track=10)
    res = osr.synthetic_results(ds, seed)
    ref_c, ref_f = osr.aggregate(ds, res, feats)
    got_c, got_f = copy.deepcopy(feats), copy.deepcopy(feats)
    tm = sfm_refine.track_members(ds, res)
    sfm_refine.apply_updates(got_c, got_f, ds.colmap_images, tm, *sfm_refine._device_means(res, tm))
    for ref, got in ((ref_c, got_c), (ref_f, got_f)):
        assert list(ref) == list(got)
        for n in ref:
            for k in ("descriptors", "keypoints", "scores"):
                assert ref[n][k].dtype == got[n][k].dtype and np.array_equal(ref[n][k], got[n][k]), (n, k)


def _matcher(sd):
    from onepose_plus_plus_b200 import LoFTR_for_OnePose_Plus
    from onepose_plus_plus_b200.sfm_coarse import default_cfg
    m = LoFTR_for_OnePose_Plus(default_cfg, enable_fine_matching=True)
    m.load_state_dict(sd, strict=True)
    return m.eval().cuda()


@pytest.mark.parametrize("pair_batch", [1, 7, 32])
def test_batched_pairs_equal_per_pair_forward(pair_batch):
    sd, data = workload.planted_loftr(96, 128, seed=0)
    m = _matcher(sd)
    ims = torch.cat([data["image0"], data["image1"], data["image1"].flip(-1), data["image0"].flip(-2)], 0)
    u8 = torch.round(ims * 255).clamp(0, 255).to(torch.uint8).cuda()
    rng = np.random.default_rng(pair_batch)
    scales = torch.tensor([[1.0, 1.0], [1.25, 0.8], [1.0 / 0.75, 1.1], [1.0, 1.5]], dtype=torch.float32)
    pairs = np.array([(a, b) for a in range(4) for b in range(4) if a != b] * 3, np.int64)
    counts = rng.integers(1, 60, len(pairs))
    counts[3] = 1
    off = np.concatenate([[0], np.cumsum(counts)])
    M = int(off[-1])
    pair_of = np.repeat(np.arange(len(pairs)), counts)
    sc = scales.numpy().astype(np.float64)

    def inside(img):        # keypoints whose cells lie on the 12 x 16 grid after the clip (some wrap)
        u, v = rng.uniform(-0.3, 15.9, M), rng.uniform(-0.3, 10.4, M)
        return np.stack([u * 8 * sc[img, 1], v * 8 * sc[img, 0]], 1)
    mk0, mk1 = inside(pairs[pair_of, 0]), inside(pairs[pair_of, 1])
    mk0[:4] = [[126, 40], [4.0, 12.0], [127.9, 0.0], [-2.0, 20.0]]     # wrap, .5 cells, clip edge, clip
    mk0 = mk0.astype(np.float32)
    m0, m1 = torch.from_numpy(mk0).cuda(), torch.from_numpy(mk1).cuda()
    res = m.fine_matches_for_pairs(u8, scales, torch.from_numpy(pairs), m0, m1, torch.from_numpy(off),
                                   pair_batch=pair_batch)
    torch.cuda.synchronize()
    worst = 0.0
    for p, (a, b) in enumerate(pairs):
        s, e = off[p], off[p + 1]
        d = {"image0": u8[a:a + 1], "image1": u8[b:b + 1], "scale0": scales[a:a + 1].cuda(),
             "scale1": scales[b:b + 1].cuda(), "mkpts0_c": torch.from_numpy(mk0[s:e]).cuda(),
             "mkpts1_c": torch.from_numpy(mk1[s:e]).cuda()}
        m(d, extract_coarse_feature=True, extract_fine_feature=True)
        assert torch.equal(d["mkpts0_c"], m0[s:e]) and torch.equal(d["mkpts1_c"], m1[s:e])
        assert torch.equal(d["i_ids"], res["i_ids"][s:e]) and torch.equal(d["j_ids"], res["j_ids"][s:e])
        assert d["mconf"].dtype == torch.int64 and d["mkpts1_f"].dtype == torch.float64
        worst = max(worst, (d["mkpts1_f"] - res["mkpts1_f"][s:e]).abs().max().item(),
                    (d["expec_f"] - res["expec_f"][s:e]).abs().max().item())
        for k in ("feat_coarse_b_0", "feat_coarse_b_1", "feat_ext0"):
            assert torch.equal(d[k], res[k][s:e]), k
        # feat_ext1 is sampled at mkpts1_f, which may move within the bound below
        assert (d["feat_ext1"] - res["feat_ext1"][s:e]).abs().max().item() <= 1e-2
    print("pair_batch", pair_batch, "max |mkpts1_f / expec_f diff|", worst)
    assert worst <= 1e-4


def test_given_cells_raise_before_launch():
    """An out-of-grid cell and B > 1 raise before any kernel launch: the C-ABI launch counter and the
    engine's workspace stay untouched and the given keypoints are still clipped as the reference does."""
    from onepose_plus_plus_b200 import _lib
    sd, data = workload.planted_loftr(96, 128, seed=0)
    m = _matcher(sd)
    mk0 = torch.tensor([[200.0, 3.0], [float("nan"), 3.0]], device="cuda")
    d = {"image0": data["image0"].cuda(), "image1": data["image1"].cuda(), "mkpts0_c": mk0,
         "mkpts1_c": torch.zeros(2, 2, device="cuda")}
    launches, ws = _lib.LAUNCHES, dict(m._ws)
    with pytest.raises(ValueError, match="coarse grid"):
        m(d)
    with pytest.raises(NotImplementedError):
        m({"image0": data["image0"].repeat(2, 1, 1, 1).cuda(), "image1": data["image1"].repeat(2, 1, 1, 1).cuda(),
           "mkpts0_c": torch.zeros(1, 2, device="cuda"), "mkpts1_c": torch.zeros(1, 2, device="cuda")})
    assert _lib.LAUNCHES == launches and m._ws.keys() == ws.keys() and "x3_out" not in m._ws
    assert mk0[0].tolist() == [126.0, 3.0]


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "sfm_refine.npz")
# The tolerances of the 2D-2D matcher (tests/test_loftr_gpu.py, tests/parity.py): expec_f x, y 1e-3, its
# std column 5e-3, mkpts1_f 1e-2 px.  Sampled features: the fp16 hi + lo maps carry the fp32 backbone
# to ~1e-5 relative; FEAT_TOL bounds |err| / max(1, |ref|) (measured values are printed).
FEAT_TOL = 1e-3


def _feat_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float((np.abs(got - ref) / np.maximum(1.0, np.abs(ref))).max()) if ref.size else 0.0


def test_forward_given_matches_equals_reference():
    z = np.load(GOLDEN)
    sd, data = workload.planted_loftr(96, 128, seed=0)
    m = _matcher(sd)
    d = {"image0": data["image0"].cuda(), "image1": data["image1"].cuda(),
         "scale0": torch.tensor([[1.25, 0.8]], device="cuda"), "scale1": torch.tensor([[1.0 / 0.75, 1.1]], device="cuda"),
         "mkpts0_c": torch.from_numpy(z["fwd_mk0_in"]).cuda(), "mkpts1_c": torch.from_numpy(z["fwd_mk1_in"]).cuda()}
    m(d, extract_coarse_feature=True, extract_fine_feature=True)
    g = {k: v.cpu().numpy() if torch.is_tensor(v) else v for k, v in d.items()}
    for k in ("i_ids", "j_ids", "mkpts0_c", "mkpts1_c", "mconf"):
        assert g[k].dtype == z["fwd_" + k].dtype and np.array_equal(g[k], z["fwd_" + k]), k
    e_px = np.abs(g["mkpts1_f"] - z["fwd_mkpts1_f"]).max()
    e_xy = np.abs(g["expec_f"][:, :2] - z["fwd_expec_f"][:, :2]).max()
    e_std = np.abs(g["expec_f"][:, 2] - z["fwd_expec_f"][:, 2]).max()
    errs = {k: _feat_err(g[k], z["fwd_" + k]) for k in ("feat_coarse_b_0", "feat_coarse_b_1", "feat_ext0", "feat_ext1")}
    print("mkpts1_f", e_px, "expec xy", e_xy, "std", e_std, errs)
    assert g["mkpts1_f"].dtype == np.float64 and e_px <= 1e-2 and e_xy <= 1e-3 and e_std <= 5e-3
    assert max(errs.values()) <= FEAT_TOL


def _golden_results(z):
    off = z["e2e_offsets"]
    keys = [k[len("e2e_res_"):] for k in z.files if k.startswith("e2e_res_")]
    rows = lambda k, p: slice(p, p + 1) if k.startswith("scale") else slice(off[p], off[p + 1])  # noqa: E731
    return {str(n): {k: z["e2e_res_" + k][rows(k, p)] for k in keys} for p, n in enumerate(z["e2e_pairs"])}


def _golden_files(z, tag):
    out = {}
    for k in z.files:
        if k.startswith(f"e2e_{tag}|"):
            _, n, a = k.split("|")
            out.setdefault(n, {})[a] = z[k]
    return out


def test_end_to_end_equals_reference(monkeypatch):
    import sys
    from onepose_plus_plus_b200 import sfm_refine
    z = np.load(GOLDEN)
    sd, _ = workload.planted_loftr(96, 128, seed=0)
    ds, feats = osr.seeded_reconstruction(**osr.E2E_RECON, images=z["e2e_images"])
    ref = _golden_results(z)
    got = sfm_refine.fine_matcher({"model": None, "extract_feature_method": "fine_match_backbone"}, ds,
                                  verbose=False, matcher=_matcher(sd))
    assert list(got) == list(ref)
    worst = {}
    for n in ref:
        assert list(got[n]) == list(ref[n])
        for k, v in ref[n].items():
            assert got[n][k].dtype == v.dtype and got[n][k].shape == v.shape, (n, k)
            if k in ("mkpts0_c", "mkpts1_c", "mkpts0_f", "mkpts0_idx", "scale0", "scale1"):
                assert np.array_equal(got[n][k], v), (n, k)
            elif k == "mkpts1_f":
                worst[k] = max(worst.get(k, 0.0), float(np.abs(got[n][k] - v).max()))
            else:
                worst[k] = max(worst.get(k, 0.0), _feat_err(got[n][k], v))
    print("end to end", worst)
    assert worst["mkpts1_f"] <= 1e-2 and max(v for k, v in worst.items() if k != "mkpts1_f") <= FEAT_TOL

    monkeypatch.setitem(sys.modules, "h5py", osr.fake_h5py())
    names = list(feats)
    for results, exact in ((ref, True), (got, False)):
        osr.FakeH5.store("/e2e/feats_coarse.h5", feats)
        sfm_refine.feature_aggregation_and_update(ds, results, "/e2e/feats.h5", names, verbose=False)
        for tag, path in (("coarse", "/e2e/feats_coarse.h5"), ("fine", "/e2e/feats.h5")):
            want, have = _golden_files(z, tag), osr.FakeH5.files[path]
            assert list(have) == names
            for n in names:
                assert sorted(have[n]) == sorted(want[n])
                for k, v in want[n].items():
                    h = have[n][k]
                    assert h.dtype == v.dtype and h.shape == v.shape, (tag, n, k)
                    if exact or k != "descriptors":
                        assert np.array_equal(h, v), (tag, n, k)
                    else:
                        assert _feat_err(h, v) <= FEAT_TOL, (tag, n, k)
