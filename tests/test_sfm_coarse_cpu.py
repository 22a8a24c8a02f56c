"""CPU checks of the SfM coarse-matching drop-in (onepose_plus_plus_b200.sfm_coarse): the NumPy
restatement of the keypoint merge (oracle/sfm_coarse.py) against the live reference functions, the
pair order, the input errors raised before any launch, and the layout of the three files."""
import random
import sys
import types

import numpy as np
import pytest

from oracle import ref_shims
from oracle import sfm_coarse as osc

needs_ref = pytest.mark.skipif(not ref_shims.available(), reason="reference tree not present")

MERGE_CASES = {
    "one_image_self_pair": dict(n_images=1, n_pairs=1, max_matches=50, one_sided=False),
    "small": dict(n_images=3, n_pairs=4, max_matches=20),
    "hub40": dict(n_images=45, n_pairs=60, hub=(3, 40)),
    "ties": dict(n_images=6, n_pairs=20, max_matches=300, tie_conf=True),
    "scaled": dict(n_images=10, n_pairs=30, scale=(1.25, 0.8)),
    "scaled_odd": dict(n_images=10, n_pairs=30, scale=(1.0 / 0.75, 1.1), tie_conf=True),
    "many_images": dict(n_images=300, n_pairs=900, max_matches=40),
}


def _assert_same(got, ref):
    gk, gs, gi = got
    rk, rs, ri = ref
    assert list(gk) == list(rk) or set(gk) == set(rk)
    for n in rk:
        assert gk[n].dtype == rk[n].dtype == np.float32 and np.array_equal(gk[n], rk[n]), n
        assert gs[n].dtype == rs[n].dtype == np.float32 and np.array_equal(gs[n], rs[n]), n
    assert list(gi) == list(ri)
    for k in ri:
        assert gi[k].dtype == ri[k].dtype == np.int64 and gi[k].shape == ri[k].shape and np.array_equal(gi[k], ri[k]), k


@needs_ref
@pytest.mark.parametrize("case", list(MERGE_CASES))
@pytest.mark.parametrize("seed", [0, 1])
def test_restatement_equals_reference_merge(case, seed):
    from oracle import sfm_coarse_ref
    matches, names = osc.seeded_matches(seed, **MERGE_CASES[case])
    ref = sfm_coarse_ref.reference_merge(matches, names)
    _assert_same(osc.merge(matches, names), ref)
    if case == "hub40":
        hits = [k for k in matches if names[3] in k.split(" ") and ((matches[k][:, :2] == (64, 96)).all(1).any()
                                                                  or (matches[k][:, 2:4] == (64, 96)).all(1).any())]
        assert len(hits) >= 40
    if "ties" in case or case == "scaled_odd":
        s = np.concatenate(list(ref[1].values()))
        assert len(np.unique(s)) < len(s)                       # exact ties occur


@needs_ref
def test_one_sided_images_and_empty_pairs():
    matches, names = osc.seeded_matches(5, n_images=8, n_pairs=30)
    only0, only1 = names[-2], names[-1]
    assert all(k.split(" ")[1] != only0 for k in matches) and any(k.split(" ")[0] == only0 for k in matches)
    assert all(k.split(" ")[0] != only1 for k in matches) and any(k.split(" ")[1] == only1 for k in matches)
    assert any(len(v) == 0 for v in matches.values())
    from oracle import sfm_coarse_ref
    _assert_same(osc.merge(matches, names), sfm_coarse_ref.reference_merge(matches, names))


@needs_ref
@pytest.mark.parametrize("seed", [0, 666, 12345])
def test_pair_order_equals_reference_dataset(tmp_path, seed):
    from oracle import sfm_coarse_ref
    from onepose_plus_plus_b200 import sfm_coarse
    _, _, dataset = sfm_coarse_ref.load()
    lines = [f"a/{i}.png b/{(i * 7) % 23}.png" for i in range(40)]
    path = tmp_path / "pairs.txt"
    path.write_text("\n".join(lines) + "\n\n")
    random.seed(seed)
    ref = dataset.LoftrCoarseDataset({"img_resize": None, "df": 8, "shuffle": True}, [], str(path)).pair_list
    random.seed(seed)
    got = sfm_coarse.read_pair_list(str(path))
    assert got == ref == osc.pair_lines(path.read_text(), seed)
    assert sorted(got) == sorted(lines)


def _write_images(tmp_path, n, size=(64, 80)):
    import cv2
    rng = np.random.default_rng(0)
    names = []
    for i in range(n):
        p = str(tmp_path / f"{i}.png")
        cv2.imwrite(p, rng.integers(0, 256, size).astype(np.uint8))
        names.append(p)
    return names


def _write_pairs(tmp_path, lines):
    p = tmp_path / "pairs.txt"
    p.write_text("\n".join(lines) + "\n")
    return str(p)


@pytest.mark.parametrize("bad", ["unknown", "duplicate", "no_pair", "three_names"])
def test_bad_pair_lists_raise_before_any_launch(tmp_path, bad):
    from onepose_plus_plus_b200 import sfm_coarse
    names = _write_images(tmp_path, 3)
    lines = [f"{names[0]} {names[1]}", f"{names[1]} {names[2]}"]
    if bad == "unknown":
        lines.append(f"{names[0]} {tmp_path}/missing.png")
    elif bad == "duplicate":
        lines.append(lines[0])
    elif bad == "no_pair":
        lines = lines[:1]
    else:
        lines.append(f"{names[0]} {names[1]} {names[2]}")

    class NoMatcher:
        def __getattr__(self, k):
            raise AssertionError("the matcher must not be reached")
    with pytest.raises(ValueError):
        sfm_coarse.detector_free_coarse_matching(names, _write_pairs(tmp_path, lines), str(tmp_path / "o/f.h5"),
                                                 str(tmp_path / "o/m.h5"), matcher=NoMatcher())
    assert not (tmp_path / "o").exists()


def test_images_of_different_sizes_raise(tmp_path):
    import cv2
    from onepose_plus_plus_b200 import sfm_coarse
    names = _write_images(tmp_path, 2)
    cv2.imwrite(names[1], np.zeros((72, 80), np.uint8))
    with pytest.raises(NotImplementedError):
        sfm_coarse.read_images(names)


def test_read_images_is_read_grayscale(tmp_path):
    import cv2
    from onepose_plus_plus_b200 import sfm_coarse
    names = _write_images(tmp_path, 2, size=(67, 85))
    frames, scales = sfm_coarse.read_images(names)
    assert frames.dtype.is_floating_point is False and tuple(frames.shape) == (2, 1, 64, 80)
    img = cv2.imread(names[0], cv2.IMREAD_GRAYSCALE)
    assert np.array_equal(frames[0, 0].numpy(), cv2.resize(img, (80, 64)))
    assert np.array_equal(scales.numpy(), np.array([[67 / 64, 85 / 80]] * 2, np.float32))


def test_image_without_keypoint_raises_before_the_merge():
    from onepose_plus_plus_b200 import sfm_coarse
    import torch
    matches, names = osc.seeded_matches(2, n_images=4, n_pairs=6, one_sided=False)
    flat, offsets, pair_img = osc.flat(matches, names)
    dead = pair_img[0, 0]
    keep = np.ones(len(flat), bool)
    for p in range(len(pair_img)):
        if dead in pair_img[p]:
            keep[offsets[p]:offsets[p + 1]] = False
    offsets = np.concatenate([[0], np.cumsum([keep[offsets[p]:offsets[p + 1]].sum() for p in range(len(pair_img))])])
    with pytest.raises(ValueError, match="no keypoint"):
        sfm_coarse._merge(torch.from_numpy(flat[keep]), offsets, pair_img.astype(np.int64), names)
    with pytest.raises(ValueError, match="no keypoint"):
        osc.merge({k: (v if dead not in [names.index(n) for n in k.split(" ")] else v[:0])
                   for k, v in matches.items()}, names)


class _FakeH5:
    """The part of h5py.File the writers use, recording datasets as numpy arrays."""
    files = {}

    class _Group(dict):
        def create_group(self, name):
            assert name not in self
            g = self[name] = _FakeH5._Group()
            return g

        def create_dataset(self, name, data):
            assert name not in self
            self[name] = np.asarray(data)

    def __init__(self, path, mode):
        assert mode == "w"
        self.root = _FakeH5.files[path] = _FakeH5._Group()

    def __enter__(self):
        return self.root

    def __exit__(self, *a):
        return False


def test_h5_layout(monkeypatch, tmp_path):
    from onepose_plus_plus_b200 import sfm_coarse
    monkeypatch.setitem(sys.modules, "h5py", types.SimpleNamespace(File=_FakeH5))
    matches, names = osc.seeded_matches(3, n_images=5, n_pairs=9)
    kpts, _, idx = osc.merge(matches, names)
    f, m, r = (str(tmp_path / x) for x in ("feats.h5", "matches.h5", "raw_matches.h5"))
    sfm_coarse.write_outputs(f, m, r, matches, kpts, idx)
    raw, feats, mt = _FakeH5.files[r], _FakeH5.files[f], _FakeH5.files[m]
    assert list(raw) == [k.replace("/", "+") for k in matches]
    for k, v in matches.items():
        assert np.array_equal(raw[k.replace("/", "+")], v) and raw[k.replace("/", "+")].dtype == np.float32
    assert list(feats) == names
    for n in names:
        g = feats[n]
        K = len(kpts[n])
        assert set(g) == {"keypoints", "descriptors", "scores"}
        assert np.array_equal(g["keypoints"], kpts[n]) and g["keypoints"].dtype == np.float32
        assert g["descriptors"].shape == (256, K) and g["descriptors"].dtype == np.float64 and not g["descriptors"].any()
        assert g["scores"].dtype == np.float64 and (g["scores"] == 1).all() and g["scores"].shape == (K,)
    assert list(mt) == [sfm_coarse.names_to_pair(*k.split(" ")) for k in idx]
    for k, v in idx.items():
        g = mt[sfm_coarse.names_to_pair(*k.split(" "))]
        assert np.array_equal(g["matches"], v) and np.array_equal(g["matches0"], v) and g["matches"].dtype == np.int64
        assert g["matching_scores"].shape == (len(v),) and (g["matching_scores"] == 1).all()


@needs_ref
def test_names_to_pair_and_config_match_reference():
    from oracle import loftr_oracle, sfm_coarse_ref
    from onepose_plus_plus_b200 import sfm_coarse
    worker, _, _ = sfm_coarse_ref.load()
    for a, b in (("x/y/0.png", "x/y/1.png"), ("a", "b")):
        assert sfm_coarse.names_to_pair(a, b) == worker.names_to_pair(a, b)
    assert sfm_coarse.default_cfg == loftr_oracle.DEFAULT_CONFIG


def test_empty_pair_gives_empty_int64_matches():
    matches, names = osc.seeded_matches(4, n_images=6, n_pairs=25)
    _, _, idx = osc.merge(matches, names)
    empty = [k for k, v in matches.items() if len(v) == 0]
    assert empty and all(idx[k].shape == (0, 2) and idx[k].dtype == np.int64 for k in empty)
