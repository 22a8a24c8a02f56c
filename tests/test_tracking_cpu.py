"""CPU tests of the tracking front end (onepose_plus_plus_b200/tracking.py, csrc/opp_image.cu):

* the fixed-point restatement of cv2.warpAffine(INTER_LINEAR) in oracle/warp_fixed.py equals cv2 bit
  for bit on both warps of crop_img_by_bbox, over seeded frames of 64 to 1920 px and boxes inside,
  straddling, wholly outside, 3x the frame, 1 px wide or tall and very non-square;
* the first warp is the zero-padded slice of the frame, and the one-stage warp over the virtual
  source (what the kernel computes) equals the two cv2 calls;
* the host geometry equals the reference's reproj / get_affine_transform / get_K_crop_resize,
  imported live from the reference tree when it is present;
* the kernel parameters equal the inverse cv2 forms from cv2.getAffineTransform;
* bad input raises before anything is launched."""
import sys
import types

import cv2
import numpy as np
import pytest

from onepose_plus_plus_b200 import tracking
from oracle import ref_shims
from oracle import warp_fixed as wf

CROP = 512


def _frame(rng, H, W):
    img = rng.integers(0, 256, (H, W), dtype=np.uint8)
    return cv2.GaussianBlur(img, (0, 0), 1.5)   # smooth content: the bilinear weights all matter


def _box(rng, kind, H, W):
    """(x0, y0, x1, y1) int32 of one category."""
    r = lambda lo, hi: int(rng.integers(lo, max(hi, lo + 1)))   # noqa: E731
    if kind == "inside":
        x0, y0 = r(0, W // 2), r(0, H // 2)
        b = (x0, y0, r(x0 + 2, W + 1), r(y0 + 2, H + 1))
    elif kind == "straddle":
        b = (r(-W // 3, 0), r(-H // 3, 0), r(W // 2, W + W // 3), r(H // 2, H + H // 3))
    elif kind == "outside":
        x0, y0 = r(W + 1, W + 200), r(-H // 2, H // 2)
        b = (x0, y0, x0 + r(8, 300), y0 + r(8, 300))
    elif kind == "triple":
        b = (-W, -H, 2 * W, 2 * H)
    elif kind == "one_px_wide":
        x0, y0 = r(0, W), r(-10, H // 2)
        b = (x0, y0, x0 + 1, y0 + r(1, H))
    elif kind == "one_px_tall":
        x0, y0 = r(-10, W // 2), r(0, H)
        b = (x0, y0, x0 + r(1, W), y0 + 1)
    elif kind == "tall":
        x0, y0 = r(0, W - 8), r(-20, H // 3)
        b = (x0, y0, x0 + r(1, 4), y0 + r(H // 2, H + 40))
    else:   # "wide"
        x0, y0 = r(-20, W // 3), r(0, H - 8)
        b = (x0, y0, x0 + r(W // 2, W + 40), y0 + r(1, 4))
    return np.array(b, dtype=np.int32)


KINDS = ["inside", "straddle", "outside", "triple", "one_px_wide", "one_px_tall", "tall", "wide"]


def _cases(n=48, seed=0):
    """Seeded (frame, box, kind) cases: sizes 64..1920 (odd sizes included), every kind >= 6 times;
    the 3x boxes on frames of at most 480 px (their first warp is 9x the frame)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        hi = 480 if kind == "triple" else 1920
        H, W = int(rng.integers(64, hi + 1)), int(rng.integers(64, hi + 1))
        if i % 3 == 0:
            H |= 1   # odd sides
            W |= 1
        out.append((_frame(rng, H, W), _box(rng, kind, H, W), kind))
    return out


CASES = _cases()


def _two_cv2_warps(frame, box, crop=CROP):
    """crop_img_by_bbox's two cv2.warpAffine calls, matrices from the host geometry."""
    x0, y0, x1, y1 = box
    w, h = int(x1 - x0), int(y1 - y0)
    M1 = tracking._box_map(box, (h, w))
    stage1 = cv2.warpAffine(frame, M1, (w, h), flags=cv2.INTER_LINEAR)
    M2 = tracking._box_map(np.array([0, 0, w, h]), (crop, crop))
    stage2 = cv2.warpAffine(stage1, M2, (crop, crop), flags=cv2.INTER_LINEAR)
    return M1, stage1, M2, stage2


def test_case_coverage():
    sizes = np.array([f.shape for f, _, _ in CASES])
    assert len(CASES) >= 40 and sizes.min() >= 64 and sizes.max() > 1500 and (sizes % 2 == 1).any()
    for kind in KINDS:
        assert sum(k == kind for _, _, k in CASES) >= 6
    for f, b, k in CASES:
        H, W = f.shape
        w, h = b[2] - b[0], b[3] - b[1]
        if k == "outside":
            assert b[0] >= W or b[2] <= 0 or b[1] >= H or b[3] <= 0
        if k == "triple":
            assert w == 3 * W and h == 3 * H
        if k in ("tall", "wide"):
            assert max(w / h, h / w) >= 10


def test_fixed_point_restatement_equals_cv2():
    pixels = 0
    for frame, box, kind in CASES:
        M1, s1, M2, s2 = _two_cv2_warps(frame, box)
        for img, M, ref in ((frame, M1, s1), (s1, M2, s2)):
            got = wf.warp_affine(img, M, (ref.shape[1], ref.shape[0]))
            assert np.array_equal(got, ref), (kind, frame.shape, box.tolist())
            pixels += ref.size
    # generic maps too: rotation, shrink, enlargement (the restatement is not tied to the crop)
    rng = np.random.default_rng(7)
    for _ in range(6):
        f = _frame(rng, int(rng.integers(64, 400)), int(rng.integers(64, 400)))
        c = rng.uniform(0, 300, 2)
        M = tracking.get_affine_transform(c, rng.uniform(20, 500), rng.uniform(-180, 180),
                                          [int(rng.integers(16, 300)), int(rng.integers(16, 300))])
        dsize = (int(rng.integers(16, 300)), int(rng.integers(16, 300)))
        assert np.array_equal(wf.warp_affine(f, M, dsize), cv2.warpAffine(f, M, dsize, flags=cv2.INTER_LINEAR))
    assert pixels > 10_000_000


def test_first_warp_is_the_zero_padded_slice():
    for frame, box, kind in CASES:
        _, s1, _, _ = _two_cv2_warps(frame, box)
        x0, y0, x1, y1 = (int(v) for v in box)
        H, W = frame.shape
        ref = np.zeros((y1 - y0, x1 - x0), np.uint8)
        fx0, fy0, fx1, fy1 = max(x0, 0), max(y0, 0), min(x1, W), min(y1, H)
        if fx1 > fx0 and fy1 > fy0:
            ref[fy0 - y0:fy1 - y0, fx0 - x0:fx1 - x0] = frame[fy0:fy1, fx0:fx1]
        assert np.array_equal(s1, ref), (kind, frame.shape, box.tolist())


def test_one_stage_virtual_source_equals_two_cv2_calls():
    for frame, box, kind in CASES:
        _, _, _, s2 = _two_cv2_warps(frame, box)
        p = tracking.crop_params(box[None], CROP)[0]   # also checks the first warp is an integer shift
        got = wf.warp_virtual(frame, p["m"], CROP, CROP, int(p["x0"]), int(p["y0"]), int(p["w"]), int(p["h"]))
        assert np.array_equal(got, s2), (kind, frame.shape, box.tolist())
        assert (p["x0"], p["y0"], p["x0"] + p["w"], p["y0"] + p["h"]) == tuple(box)
    # a non-square crop side too (the kernel takes any output size)
    frame, box, _ = CASES[1]
    _, _, _, s2 = _two_cv2_warps(frame, box, crop=200)
    p = tracking.crop_params(box[None], 200)[0]
    assert np.array_equal(wf.warp_virtual(frame, p["m"], 200, 200, p["x0"], p["y0"], p["w"], p["h"]), s2)


def test_fixed_point_params_equal_cv2():
    """The inverse handed to the kernel is the one cv2 forms from cv2.getAffineTransform (compared
    with cv2.invertAffineTransform, which uses the same formulas), and so are its fixed-point terms."""
    for frame, box, _ in CASES:
        x0, y0, x1, y1 = box
        w, h = int(x1 - x0), int(y1 - y0)
        p = tracking.crop_params(box[None], CROP)[0]
        M2 = tracking._box_map(np.array([0, 0, w, h]), (CROP, CROP))
        inv = cv2.invertAffineTransform(M2).reshape(-1)
        assert np.array_equal(p["m"], inv)
        for got, ref in zip(tracking._fixed_point_terms(p["m"], CROP, CROP), wf.fixed_point(inv, CROP, CROP)):
            assert np.array_equal(got, ref)


# ------------------------------------------------------------------------------------------------
# host geometry against the reference
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    if not ref_shims.available():
        pytest.skip("reference tree not present")
    # vis_utils imports three packages that its reproj does not use
    for name, attr, val in (("natsort", None, None), ("loguru", "logger", None), ("wis3d", "Wis3D", object)):
        if name not in sys.modules:
            try:
                __import__(name)
            except ImportError:
                m = types.ModuleType(name)
                if attr:
                    setattr(m, attr, val)
                sys.modules[name] = m
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from src.utils import data_utils, vis_utils   # type: ignore
    return types.SimpleNamespace(data=data_utils, vis=vis_utils)


def _poses(rng, n):
    out = []
    for _ in range(n):
        R, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        R *= np.sign(np.linalg.det(R))
        out.append(np.concatenate([R, np.array([[0.1, -0.05, 0.6]]).T + rng.normal(0, 0.05, (3, 1))], 1))
    return out


def test_host_geometry_matches_reference(ref):
    rng = np.random.default_rng(3)
    K = np.array([[572.4, 0, 325.3], [0, 573.6, 242.0], [0, 0, 1]])
    bbox3d = rng.uniform(-0.08, 0.08, (8, 3))
    for pose in _poses(rng, 20):
        for P in (pose, np.concatenate([pose, [[0, 0, 0, 1]]])):
            assert np.array_equal(tracking.reproj(K, P, bbox3d), ref.vis.reproj(K, P, bbox3d))
        uv = ref.vis.reproj(K, pose, bbox3d)
        (x0, y0), (x1, y1) = uv.min(0), uv.max(0)
        want = np.array([x0, y0, x1, y1]).astype(np.int32)   # previous_pose_detect
        got = tracking.bbox_from_pose(K, pose, bbox3d)
        assert got.dtype == np.int32 and np.array_equal(got, want)
    # get_affine_transform: boxes of every kind, plus rotation / shift / inv / scalar scale
    for _, box, _ in CASES:
        c = np.array([(box[0] + box[2]) / 2.0, (box[1] + box[3]) / 2.0])
        s = np.array([box[2] - box[0], box[3] - box[1]])
        for size in ([int(s[0]), int(s[1])], [CROP, CROP]):
            assert np.array_equal(tracking.get_affine_transform(c, s, 0, size),
                                  ref.data.get_affine_transform(c, s, 0, size))
    for _ in range(10):
        c, s, rot = rng.uniform(-100, 900, 2), rng.uniform(5, 800), rng.uniform(-180, 180)
        shift = rng.uniform(-0.2, 0.2, 2).astype(np.float32)
        for inv in (0, 1):
            assert np.array_equal(tracking.get_affine_transform(c, s, rot, [300, 200], shift, inv),
                                  ref.data.get_affine_transform(c, s, rot, [300, 200], shift, inv))
    # K_crop: get_K_crop_resize alone and composed twice as crop_img_by_bbox does
    for _, box, _ in CASES:
        x0, y0, x1, y1 = box
        shape = np.array([y1 - y0, x1 - x0])
        for Ko in (K, np.concatenate([K, np.zeros((3, 1))], 1)):
            g, gh = tracking.get_K_crop_resize(box, Ko, shape)
            r, rh = ref.data.get_K_crop_resize(box, Ko, shape)
            assert np.allclose(g, r, rtol=1e-12, atol=0) and np.allclose(gh, rh, rtol=1e-12, atol=0)
        K1, _ = ref.data.get_K_crop_resize(box, K, shape)
        K2, _ = ref.data.get_K_crop_resize(np.array([0, 0, x1 - x0, y1 - y0]), K1, np.array([CROP, CROP]))
        got = tracking.crop_K(box, K, CROP)
        assert np.allclose(got, K2, rtol=1e-12, atol=0) and np.array_equal(got == 0, K2 == 0)
    # the reference's image warp with its own matrices equals the restatement
    for frame, box, _ in CASES[:8]:
        x0, y0, x1, y1 = box
        s1, T1 = ref.data.get_image_crop_resize(frame, box, np.array([y1 - y0, x1 - x0]))
        _, m1, _, _ = _two_cv2_warps(frame, box)
        assert np.array_equal(s1, m1) and np.array_equal(T1[:2], tracking._box_map(box, (y1 - y0, x1 - x0)))


# ------------------------------------------------------------------------------------------------
# input errors
# ------------------------------------------------------------------------------------------------
def test_input_errors_raise():
    ok = np.array([[10, 10, 50, 60]], dtype=np.int32)
    assert tracking.crop_params(ok).shape == (1,)
    bad = {
        "zero width": [[10, 10, 10, 60]], "negative height": [[10, 60, 50, 10]],
        "far": [[1 << 20, 0, (1 << 20) + 5, 5]], "far negative": [[-(1 << 20), 0, 5, 5]],
        "too wide": [[0, 0, 32767, 5]],
    }
    for name, b in bad.items():
        with pytest.raises(ValueError):
            tracking.crop_params(np.array(b, dtype=np.int64))
        with pytest.raises(ValueError):   # before any upload or launch
            tracking.crop_resize_batched(np.zeros((1, 64, 64), np.uint8), np.array(b))
    with pytest.raises(ValueError, match="integers"):
        tracking.crop_params(ok.astype(np.float64))
    with pytest.raises(ValueError, match=r"\[B, 4\]"):
        tracking.crop_params(ok[0])
    for crop in (0, 40000, 12.5):
        with pytest.raises(ValueError, match="crop_size"):
            tracking.crop_params(ok, crop)
    with pytest.raises(TypeError, match="uint8"):
        tracking._frames(np.zeros((1, 64, 64), np.float32))
    with pytest.raises(ValueError, match="frame width"):
        tracking._frames(np.zeros((1, 8, 40000), np.uint8))
    with pytest.raises(ValueError):
        tracking._frames(np.zeros((2, 3, 8, 8), np.uint8))
    with pytest.raises(ValueError, match="K"):
        tracking.reproj(np.eye(4), np.eye(4)[:3], np.zeros((8, 3)))

    class NoBank:
        _bank = None
    with pytest.raises(ValueError, match="set_bank"):
        tracking.PoseTracker(NoBank(), np.eye(3), np.zeros((8, 3)))

    class Bank:
        _bank = object()
    with pytest.raises(ValueError, match="multiple of 8"):
        tracking.PoseTracker(Bank(), np.eye(3), np.zeros((8, 3)), crop_size=100)
    with pytest.raises(ValueError, match="K must"):
        tracking.PoseTracker(Bank(), np.eye(4), np.zeros((8, 3)))
