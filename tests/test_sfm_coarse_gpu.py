"""pytest -m gpu: the SfM coarse matching on the device (onepose_plus_plus_b200.sfm_coarse).

  * The merge kernels (opp_sfm_points.cu, called through the C ABI with every output and scratch
    buffer prefilled with NaN or a sentinel) are bit-equal to oracle/sfm_coarse.py, from one pair to
    1500 pairs x up to 1500 matches, and two runs give identical bits.
  * The coarse-only image tokens are bit-equal to the tokens forward() computes.
  * The batched pair path gives the per-pair forward's i_ids / j_ids / mkpts*_c and mconf within 1e-5
    at pair batches 1, 7 and 32.
  * End to end, the outputs equal the reference's stored in tests/golden/reference/sfm_coarse.npz."""
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

from oracle import sfm_coarse as osc
from oracle import workload

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference", "sfm_coarse.npz")


def _kernels(matches, offsets, pair_img, images):
    """The opp_sfm_points_* sequence of ops.sfm_points with sentinel-filled buffers."""
    from onepose_plus_plus_b200 import _lib
    from onepose_plus_plus_b200._lib import call, ptr, stream
    dev, i32, i64 = "cuda", torch.int32, torch.int64
    m = torch.from_numpy(matches).to(dev)
    off = torch.from_numpy(offsets).to(dev)
    pimg = torch.from_numpy(pair_img).to(dev)
    M, P = m.shape[0], pimg.shape[0]
    n = 2 * M
    key = torch.full((n,), -7, dtype=i64, device=dev)
    conf = torch.full((n,), float("nan"), device=dev)
    call("opp_sfm_points_emit", ptr(m), M, ptr(off), ptr(pimg), P, ptr(key), ptr(conf), stream())
    sk, perm = torch.sort(key, stable=True)
    scratch = torch.full((_lib.load().opp_sfm_points_segments_scratch(n),), -7, dtype=i32, device=dev)
    start = torch.full((n + 1,), -7, dtype=i32, device=dev)
    groups = torch.full((1,), -7, dtype=i32, device=dev)
    call("opp_sfm_points_segments", ptr(sk), n, ptr(scratch), ptr(start), ptr(groups), stream())
    G = int(groups.item())
    assert int(start[G]) == n and (start[:G] >= 0).all()
    ukey, rank_key = (torch.full((G,), -7, dtype=i64, device=dev) for _ in range(2))
    sums = torch.full((G,), float("nan"), dtype=torch.float64, device=dev)
    img_off = torch.full((images + 1,), -7, dtype=i64, device=dev)
    call("opp_sfm_points_sums", ptr(sk), ptr(perm), ptr(conf), ptr(start), G, images, ptr(ukey), ptr(sums),
         ptr(rank_key), ptr(img_off), stream())
    _, perm1 = torch.sort(rank_key, stable=True)
    img_key = torch.full((G,), -7, dtype=i64, device=dev)
    call("opp_sfm_points_image_key", ptr(ukey), ptr(perm1), G, ptr(img_key), stream())
    _, perm2 = torch.sort(img_key, stable=True)
    kpts = torch.full((G, 2), float("nan"), device=dev)
    scores = torch.full((G,), float("nan"), device=dev)
    id_of = torch.full((G,), -7, dtype=i64, device=dev)
    call("opp_sfm_points_rank", ptr(ukey), ptr(sums), ptr(img_off), ptr(perm1), ptr(perm2), G, ptr(kpts),
         ptr(scores), ptr(id_of), stream())
    idx = torch.full((M, 2), -7, dtype=i64, device=dev)
    status = torch.full((1,), -7, dtype=i32, device=dev)
    call("opp_sfm_points_remap", ptr(m), M, ptr(off), ptr(pimg), P, ptr(ukey), ptr(img_off), ptr(id_of), ptr(idx),
         ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    return {"kpts": kpts.cpu().numpy(), "scores": scores.cpu().numpy(), "img_off": img_off.cpu().numpy(),
            "idx": idx.cpu().numpy(), "sums": sums.cpu().numpy(), "start": start.cpu().numpy()}


def _expected(matches, names):
    kp, sc, idx = osc.merge(matches, names)
    img_off = np.zeros(len(names) + 1, np.int64)
    img_off[1:] = np.cumsum([len(kp[n]) for n in names])
    return (np.concatenate([kp[n] for n in names]), np.concatenate([sc[n] for n in names]), img_off,
            np.concatenate([idx[k] for k in matches]))


def _big(seed, pairs=1500, images=150, max_matches=1500):
    """~1500 pairs of up to 1500 matches on 512^2 images at the scale (1.25, 0.8)."""
    rng = np.random.default_rng(seed)
    names = [f"obj/{i:04d}.png" for i in range(images)]
    out = {}
    for p in range(pairs):
        a = p % images
        b = (a + 1 + p // images) % images
        m = int(rng.integers(0, max_matches + 1)) if p >= images else int(rng.integers(1, max_matches + 1))
        c = rng.integers(0, 64, (m, 4)) * 8 * np.array([1.25, 0.8, 1.25, 0.8])
        out[f"{names[a]} {names[b]}"] = np.concatenate([c, rng.uniform(0.2, 1, (m, 1))], 1).astype(np.float32)
    return out, names


CASES = {
    "one_pair": lambda: osc.seeded_matches(0, n_images=2, n_pairs=1, one_sided=False),
    "self_pair": lambda: osc.seeded_matches(1, n_images=1, n_pairs=1, one_sided=False),
    "hub40": lambda: osc.seeded_matches(2, n_images=45, n_pairs=60, hub=(3, 40)),
    "ties_scaled": lambda: osc.seeded_matches(3, n_images=10, n_pairs=40, scale=(1.0 / 0.75, 1.1), tie_conf=True),
    "many_images": lambda: osc.seeded_matches(4, n_images=300, n_pairs=900, max_matches=40),
    "big": lambda: _big(5),
}


@pytest.mark.parametrize("case", list(CASES))
def test_merge_kernels_equal_the_restatement(case):
    matches, names = CASES[case]()
    flat, offsets, pair_img = osc.flat(matches, names)
    got = _kernels(flat, offsets, pair_img, len(names))
    kp, sc, img_off, idx = _expected(matches, names)
    assert np.array_equal(got["img_off"], img_off)
    assert np.array_equal(got["kpts"], kp) and np.array_equal(got["scores"], sc)
    assert np.array_equal(got["idx"], idx)
    again = _kernels(flat, offsets, pair_img, len(names))
    for k in got:
        assert np.array_equal(got[k].view(np.uint8), again[k].view(np.uint8)), k
    if case == "big":
        assert len(flat) > 1_000_000


@pytest.mark.parametrize("case", ["hub", "scaled_ties"])
def test_merge_equals_the_stored_reference(case):
    z = np.load(GOLDEN)
    p = f"merge_{case}_"
    got = _kernels(z[p + "matches"], z[p + "offsets"], z[p + "pair_img"], len(z[p + "img_off"]) - 1)
    for k in ("kpts", "scores", "img_off", "idx"):
        assert np.array_equal(got[k], z[p + k]), k


def test_ops_wrapper_and_input_guards():
    from onepose_plus_plus_b200 import ops
    matches, names = osc.seeded_matches(6, n_images=8, n_pairs=20, scale=(1.25, 0.8))
    flat, offsets, pair_img = osc.flat(matches, names)
    kp, sc, img_off, idx = _expected(matches, names)
    args = [torch.from_numpy(flat).cuda(), torch.from_numpy(offsets).cuda(), torch.from_numpy(pair_img).cuda()]
    k, s, io, ix, st = ops.sfm_points(*args, len(names))
    assert int(st.item()) == 0 and np.array_equal(io.cpu().numpy(), img_off)
    assert np.array_equal(k.cpu().numpy(), kp) and np.array_equal(s.cpu().numpy(), sc)
    assert np.array_equal(ix.cpu().numpy(), idx)
    for bad in ("neg", "far", "nan", "img"):
        a = [t.clone() for t in args]
        if bad == "neg":
            a[0][3, 1] = -1.0
        elif bad == "far":
            a[0][0, 2] = float(ops.SFM_XY_LIMIT)
        elif bad == "nan":
            a[0][1, 4] = float("nan")
        else:
            a[2][0, 1] = len(names)
        with pytest.raises(ValueError):
            ops.sfm_points(*a, len(names))


def _model(sd):
    from onepose_plus_plus_b200 import LoFTR_for_OnePose_Plus, sfm_coarse
    m = LoFTR_for_OnePose_Plus(sfm_coarse.default_cfg, enable_fine_matching=False)
    m.load_state_dict(sd, strict=True)
    return m.eval().cuda()


def _planted_images(h=256, w=320, n=6):
    """n uint8 crops of the canvas workload.planted_loftr(h, w) draws, at shifts around its (16, 24)."""
    g = torch.Generator().manual_seed(1)
    canvas = torch.rand(1, 1, h + 16, w + 24, generator=g)[0, 0]
    shifts = [(0, 0), (16, 24), (8, 16), (16, 8), (0, 24), (8, 8)][:n]
    return torch.stack([(canvas[dy:dy + h, dx:dx + w] * 255).round().to(torch.uint8) for dy, dx in shifts])[:, None]


@pytest.fixture(scope="module")
def planted():
    sd, _ = workload.planted_loftr(256, 320, seed=0)
    return _model(sd), _planted_images()


def test_image_tokens_equal_forward_tokens(planted):
    m, imgs = planted
    imgs = imgs.cuda()
    tok, _ = m.image_tokens(imgs, image_chunk=4)
    with torch.no_grad():
        for a, b in ((0, 1), (2, 5)):
            m._ensure_plan(imgs.device)
            ref, _, _ = m._backbone(torch.cat([imgs[a:a + 1], imgs[b:b + 1]]).contiguous())
            assert torch.equal(tok[a], ref[0]) and torch.equal(tok[b], ref[1])


@pytest.mark.parametrize("pair_batch", [1, 7, 32])
def test_batched_pairs_equal_per_pair_forward(planted, pair_batch):
    m, imgs = planted
    n = imgs.shape[0]
    pairs = [(a, b) for a in range(n) for b in range(n) if a != b][:20]
    scales = torch.tensor([[1.0 + 0.05 * i, 1.0 - 0.03 * i] for i in range(n)], dtype=torch.float32)
    res = m.coarse_matches_for_pairs(imgs.cuda(), scales, torch.tensor(pairs), pair_batch=pair_batch)
    off = res["offsets"].tolist()
    assert off[-1] == res["mconf"].numel() and off[-1] > 50 * len(pairs)
    for p, (a, b) in enumerate(pairs):
        d = {"image0": imgs[a:a + 1].cuda(), "image1": imgs[b:b + 1].cuda(), "scale0": scales[a:a + 1].cuda(),
             "scale1": scales[b:b + 1].cuda()}
        m(d)
        sl = slice(off[p], off[p + 1])
        assert (res["b_ids"][sl] == p).all()
        for k in ("i_ids", "j_ids", "mkpts0_c", "mkpts1_c"):
            assert torch.equal(res[k][sl], d[k]), (p, k)
        if d["mconf"].numel():
            assert (res["mconf"][sl] - d["mconf"]).abs().max().item() <= 1e-5


class _FakeH5:
    files = {}

    class _Group(dict):
        def create_group(self, name):
            g = self[name] = _FakeH5._Group()
            return g

        def create_dataset(self, name, data):
            self[name] = np.asarray(data)

    def __init__(self, path, mode):
        self.root = _FakeH5.files[path] = _FakeH5._Group()

    def __enter__(self):
        return self.root

    def __exit__(self, *a):
        return False


def test_end_to_end_equals_the_stored_reference(tmp_path, monkeypatch):
    import cv2
    from onepose_plus_plus_b200 import sfm_coarse
    z = np.load(GOLDEN)
    names = []
    for i, im in enumerate(z["e2e_images"]):
        p = str(tmp_path / f"{i:03d}.png")
        cv2.imwrite(p, im)
        names.append(p)
    ref_pairs = [" ".join(str(tmp_path / n) for n in k.split(" ")) for k in z["e2e_pairs"]]
    sd, _ = workload.planted_loftr(136, 176, seed=0)
    model = _model(sd)
    monkeypatch.setitem(sys.modules, "h5py", types.SimpleNamespace(File=_FakeH5))
    # the golden's pair file lists the pairs in this order: (0,1) (1,2) (0,2) (2,3) (3,4) (1,4) (0,4)
    order = [(0, 1), (1, 2), (0, 2), (2, 3), (3, 4), (1, 4), (0, 4)]
    with open(tmp_path / "pairs.txt", "w") as f:
        f.write("\n".join(f"{names[a]} {names[b]}" for a, b in order) + "\n")
    random.seed(int(z["e2e_seed"]))
    out = str(tmp_path / "out")
    kpts, idx = sfm_coarse.detector_free_coarse_matching(names, str(tmp_path / "pairs.txt"), out + "/feats.h5",
                                                         out + "/matches.h5", matcher=model)
    assert list(idx) == ref_pairs                                   # the reference's shuffled order
    raw = _FakeH5.files[out + "/raw_matches.h5"]
    off = z["e2e_offsets"]
    ref_m = z["e2e_matches"]
    for p, key in enumerate(ref_pairs):
        got = raw[key.replace("/", "+")]
        ref = ref_m[off[p]:off[p + 1]]
        assert np.array_equal(got[:, :4], ref[:, :4]), key
        assert np.abs(got[:, 4] - ref[:, 4]).max() <= 5e-3
    # the merge of these matches: bit-equal to the restatement on the device's raw matches, and the
    # reference's keypoints (same coordinates; ids equal where the scores do not nearly tie)
    raw_dict = {k: raw[k.replace("/", "+")] for k in ref_pairs}
    ek, es, ei = osc.merge(raw_dict, names)
    for i, n in enumerate(names):
        assert np.array_equal(kpts[n], ek[n])
        ref_k = z["e2e_kpts"][z["e2e_img_off"][i]:z["e2e_img_off"][i + 1]]
        assert sorted(map(tuple, kpts[n].tolist())) == sorted(map(tuple, ref_k.tolist()))
    for p, key in enumerate(ref_pairs):
        assert np.array_equal(idx[key], ei[key])
        a, b = (names.index(x) for x in key.split(" "))
        ref_ix = z["e2e_idx"][off[p]:off[p + 1]]
        ko = z["e2e_img_off"]
        ref_xy = np.concatenate([z["e2e_kpts"][ko[a] + ref_ix[:, 0]], z["e2e_kpts"][ko[b] + ref_ix[:, 1]]], 1)
        got_xy = np.concatenate([kpts[names[a]][idx[key][:, 0]], kpts[names[b]][idx[key][:, 1]]], 1)
        assert np.array_equal(got_xy, ref_xy)
    feats = _FakeH5.files[out + "/feats.h5"]
    assert list(feats) == names and all(np.array_equal(feats[n]["keypoints"], kpts[n]) for n in names)
