"""The training batch's kernels one entry point at a time (opp_homography_warp_f32, opp_train_gt_build,
opp_train_gt_compact), called through the C ABI with every output and scratch buffer poisoned (NaN
for floats, a sentinel for ints), so an entry that is never written cannot pass:
  - the warp at sizes its 32 x 8 tile does not divide: every pixel written, unwarped items copied,
    bit-equal to the NumPy restatement (oracle/train_batch.py), and within a first-order bound of an
    fp64 kornia warp derived from the kernel's fp32 roundings (U = 2^-24);
  - the build's scratch arrays (rank_of, cell_owner, kp_owner, fine, key, key_xy) and status bits
    against their restatement on the edge batches of otb.EDGE_CASES, and run to run;
  - the compaction at its 1024-key chunk edges against a NumPy "keep the last of each (b, i, j)";
  - the list at the training shape against the same steps in fp64, fine_xy within a derived bound;
  - the host guards, which raise before any launch.
The largest err / bound of each fp64 comparison is printed."""
import numpy as np
import pytest
import torch

from oracle import train_batch as otb
from onepose_plus_plus_b200 import _lib, ops, train_batch

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
SENT = -777                              # int sentinel: neither a fill of the kernels nor an index
SIZES = [(2, 2), (7, 33), (97, 131), (100, 100), (511, 509), (8, 1000), (512, 512)]
SZ_BAND = 1e-6                           # |sz| below this is excluded from the fp64 bound (see warp_bound)


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _sent(*shape, dtype=torch.int32):
    return torch.full(shape, SENT, dtype=dtype, device=DEV)


def _bits(t):
    """bit patterns of a float32 array, so NaN poison compares equal to itself"""
    return np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else t).view(np.int32)


def pack_size():
    return _lib.load().opp_train_batch_pack_size()


# ---- the entry points with poisoned outputs (the calls of ops.homography_warp / ops.train_gt) ----

def run_warp(img, pack):
    B, _, h, w = img.shape
    out = _nan(B, 1, h, w)
    ops.call("opp_homography_warp_f32", ops.ptr(img), ops.ptr(pack), B, h, w, ops.ptr(out), ops.stream())
    torch.cuda.synchronize()
    return out


def host_args(batch):
    src = batch["gt_source"]
    h, w = batch["query_image"].shape[-2:]
    packs = [otb.pack_item(src.pose_gt[b], src.K_crop[b], src.homography[b], h, w) for b in range(len(src))]
    return src, (h, w), packs


def run_build(batch, scale=None):
    """opp_train_gt_build on a host batch: the scratch arrays and status as NumPy"""
    src, (h, w), packs = host_args(batch)
    kp3d = batch["keypoints3d"].to(DEV, torch.float32).contiguous()
    B, L, _ = kp3d.shape
    n = src.assign.shape[1]
    R = ((w - 1) // 8 + 1) * ((h - 1) // 8 + 1)
    w_c, S = int(w / 8), int(h / 8) * int(w / 8)
    scale = batch["query_image_scale"] if scale is None else scale
    bufs = {"cell_owner": _sent(B * R), "kp_owner": _sent(max(src.n_kp, 1)), "rank_of": _sent(n),
            "fine": _nan(n, 2), "key": _sent(n, dtype=torch.int64), "key_xy": _nan(n, 2), "status": _sent(2)}
    args = [src.assign.to(DEV).contiguous(), src.offsets.to(DEV), src.kp_offsets.to(DEV),
            torch.from_numpy(np.stack(packs)).to(DEV), scale.to(DEV, torch.float32).contiguous()]
    ops.call("opp_train_gt_build", ops.ptr(kp3d), ops.ptr(args[0]), n, ops.ptr(args[1]), ops.ptr(args[2]),
             int(src.n_kp), ops.ptr(args[3]), ops.ptr(args[4]), B, L, h, w, w_c, S,
             *(ops.ptr(bufs[k]) for k in ("cell_owner", "kp_owner", "rank_of", "fine", "key", "key_xy", "status")),
             ops.stream())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in bufs.items()}


def run_compact(sorted_key, perm, key_xy, L, S, R):
    n = len(sorted_key)
    outs = [_sent(max(n, 1), dtype=torch.int64) for _ in range(3)] + [_nan(max(n, 1), 2), _sent(2)]
    ins = [torch.from_numpy(sorted_key).to(DEV), torch.from_numpy(perm).to(DEV), torch.from_numpy(key_xy).to(DEV)]
    ops.call("opp_train_gt_compact", ops.ptr(ins[0]), ops.ptr(ins[1]), n, ops.ptr(ins[2]), L, S, R,
             *(ops.ptr(t) for t in outs), ops.stream())
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in outs]


def restated_scratch(batch, scale=None):
    src, hw, packs = host_args(batch)
    scale = (batch["query_image_scale"] if scale is None else scale).numpy()
    return otb.batch_scratch(batch["keypoints3d"].numpy(), src.assign.numpy(), src.offsets.numpy(),
                             src.kp_offsets.numpy(), packs, scale, hw)


# ---- the warp --------------------------------------------------------------------------------------

def warp_packs(h, w, seed):
    """four items: unwarped, a random homography, a warp whose z changes sign at gx = 1 / 1.6, and one
    that maps the image far outside itself"""
    g = np.random.default_rng(seed)
    eye = np.eye(4)
    far = np.array([[1, 0, 40.0 * w], [0, 1, -30.0 * h], [0, 0, 1]])
    hs = [None, otb.random_homography(g, h, w), otb._perspective_flip(h, w, 1.6), far]
    return np.stack([otb.pack_item(eye, np.eye(3), H, h, w) for H in hs])


def warp_bound(img, pack, h, w):
    """(fp64 kornia warp, first-order bound on the kernel's error, mask of the pixels bounded).
    The kernel computes the grid, sx / sy / sz (mad3: 3 roundings each), 1 / sz, ix and iy (3
    roundings each) in fp32; its coordinate error is propagated in fp64 from the operand magnitudes,
    plus the grid's own difference from torch.linspace's (the kernel follows linspace's scalar
    formula; torch's vectorised CPU linspace rounds a few points differently), times the largest tap
    difference of the zero-padded image around the sample, plus 8 U max|tap| for the four-tap sum.
    The warp is continuous across tap switches and the zero border, so the bound holds wherever the
    coordinate error is first order: everywhere except |sz| < SZ_BAND, where 1 / sz blows up (and
    the kernel's |sz| > 1e-8 switch sits)."""
    p = pack.astype(np.float64)
    A = p[34:43]
    ref = otb.homography_warp(torch.from_numpy(img.astype(np.float64))[None, None],
                              torch.from_numpy(A.reshape(1, 3, 3)), (h, w))[0, 0].numpy()
    gx = otb.linspace_pm1(w).astype(np.float64)[None, :]
    gy = otb.linspace_pm1(h).astype(np.float64)[:, None]
    dgx = np.abs(gx - torch.linspace(-1, 1, w, dtype=torch.float).double().numpy()[None, :])
    dgy = np.abs(gy - torch.linspace(-1, 1, h, dtype=torch.float).double().numpy()[:, None])
    rows = [(A[3 * r] * gx, A[3 * r + 1] * gy, A[3 * r + 2] + 0 * gx * gy) for r in range(3)]
    sx, sy, sz = (a + b + c for a, b, c in rows)
    e_sx, e_sy, e_sz = (3 * U * (np.abs(a) + np.abs(b) + np.abs(c)) for a, b, c in rows)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = 1 / sz
        e_s = e_sz * s * s + U * np.abs(s)
        out = []
        for v, e_v, n, k in ((sx, e_sx, w, 0), (sy, e_sy, h, 3)):
            X = s * v
            e_X = np.abs(s) * e_v + np.abs(v) * e_s + U * np.abs(X)
            i = (X + 1) * (n / 2) - 0.5
            e_i = (e_X + U * np.abs(X + 1)) * (n / 2) + U * np.abs((X + 1) * n / 2) + U * np.abs(i)
            # the grid's difference from torch.linspace, through d i / d g = (n / 2) (A_k sz - A_6 v) / sz^2
            e_i += (n / 2) * (np.abs(A[k] * sz - A[6] * v) * dgx + np.abs(A[k + 1] * sz - A[7] * v) * dgy) * s * s
            out.append((i, e_i))
    (ix, e_ix), (iy, e_iy) = out
    P = np.pad(img.astype(np.float64), 3)
    dX, dY = np.abs(np.diff(P, axis=1)), np.abs(np.diff(P, axis=0))
    x0 = np.clip(np.floor(np.nan_to_num(ix, nan=-3, posinf=w + 2, neginf=-3)), -3, w + 1).astype(np.int64) + 3
    y0 = np.clip(np.floor(np.nan_to_num(iy, nan=-3, posinf=h + 2, neginf=-3)), -3, h + 1).astype(np.int64) + 3
    gxm = np.zeros_like(ix)
    gym = np.zeros_like(ix)
    vmax = np.zeros_like(ix)
    for dy in (-1, 0, 1, 2):
        for dx in (-1, 0, 1, 2):
            yy, xx = np.clip(y0 + dy, 0, h + 5), np.clip(x0 + dx, 0, w + 5)
            gxm = np.maximum(gxm, dX[yy, np.clip(xx, 0, w + 4)])
            gym = np.maximum(gym, dY[np.clip(yy, 0, h + 4), xx])
            if dy in (0, 1) and dx in (0, 1):
                vmax = np.maximum(vmax, np.abs(P[yy, xx]))
    with np.errstate(invalid="ignore"):
        bound = 2 * (gxm * e_ix + gym * e_iy) + 8 * U * vmax
    mask = np.abs(sz) >= SZ_BAND
    return ref, np.where(mask, bound, np.inf), mask


@pytest.mark.parametrize("hw", SIZES)
def test_warp_every_pixel_bit_equal_and_fp64_bound(hw):
    h, w = hw
    g = np.random.default_rng(h * 1000 + w)
    packs = warp_packs(h, w, h + w)
    img = g.random((len(packs), 1, h, w), dtype=np.float32)
    got = run_warp(torch.from_numpy(img).to(DEV), torch.from_numpy(packs).to(DEV)).cpu().numpy()
    assert not np.isnan(got).any(), "a pixel was not written"
    assert np.array_equal(got[0, 0], img[0, 0]), "the unwarped item is not an exact copy"
    worst, excluded = 0.0, 0
    for b in range(1, len(packs)):
        want = otb.warp_image(img[b, 0], packs[b])
        assert np.array_equal(_bits(got[b, 0]), _bits(want)), f"item {b}: not bit-equal to the restatement"
        ref, bound, mask = warp_bound(img[b, 0], packs[b], h, w)
        err = np.abs(got[b, 0].astype(np.float64) - ref)
        ratio = np.where(mask, err / np.maximum(bound, 1e-300), 0)
        excluded += int((~mask).sum())
        worst = max(worst, float(ratio.max()))
        assert (ratio <= 1).all(), f"item {b}: err / bound {ratio.max():.3g} at {np.unravel_index(ratio.argmax(), ratio.shape)}"
    print(f"warp {h}x{w}: largest err / bound vs fp64 {worst:.3g} ({excluded} px in the |sz| < {SZ_BAND} band)")


# ---- the build -------------------------------------------------------------------------------------

def check_scratch(got, want, n):
    assert got["status"][0] == want["bits"], f"status bits {got['status'][0]} != {want['bits']}"
    if n == 0:
        return
    assert np.array_equal(got["rank_of"], want["rank_of"]), "rank_of"
    assert np.array_equal(got["cell_owner"], want["cell_owner"]), "cell_owner"
    if len(want["kp_owner"]):
        assert np.array_equal(got["kp_owner"][:len(want["kp_owner"])], want["kp_owner"]), "kp_owner"
    has = want["rank_of"] >= 0
    assert np.array_equal(_bits(got["fine"][has]), _bits(want["fine"][has])), "fine"
    assert np.array_equal(got["key"], want["key"]), "key"
    emitted = want["key"] != otb.KEY_DROPPED
    assert np.array_equal(_bits(got["key_xy"][emitted]), _bits(want["key_xy"][emitted])), "key_xy"


@pytest.mark.parametrize("name", ["training_shape", *otb.EDGE_CASES])
def test_build_scratch_equals_the_restatement(name):
    """rank_of, cell_owner (with its 0x7f7f7f7f fill), kp_owner (-1 fill), fine, key (INT64_MAX where
    dropped), key_xy and the status bits; two runs bit-identical"""
    batch = otb.synthetic_batch(1) if name == "training_shape" else otb.edge_batch(name)[0]
    n = batch["gt_source"].assign.shape[1]
    h, w = batch["query_image"].shape[-2:]
    if h < 8 or w < 8:
        # no coarse cell (w_c or S = 0): the build refuses the shape before it writes anything
        with pytest.raises(RuntimeError, match="bad shape"):
            run_build(batch)
        torch.cuda.synchronize()
        return
    want = restated_scratch(batch)
    first, second = run_build(batch), run_build(batch)
    check_scratch(first, want, n)
    for k in first:
        assert np.array_equal(_bits(first[k]) if first[k].dtype == np.float32 else first[k],
                              _bits(second[k]) if second[k].dtype == np.float32 else second[k]), f"{k}: run to run"
    if n:
        # the compaction of these keys (the sort ops.train_gt runs) against keep-last in NumPy
        key = first["key"]
        perm = np.argsort(key, kind="stable")
        src, (h, w), _ = host_args(batch)
        L = batch["keypoints3d"].shape[1]
        R, S = ((w - 1) // 8 + 1) * ((h - 1) // 8 + 1), int(h / 8) * int(w / 8)
        check_compact(key[perm], perm.astype(np.int64), first["key_xy"], L, S, R)
    print(f"{name}: n {n}, {int((want['key'] != otb.KEY_DROPPED).sum())} keys, bits {want['bits']}")


def _error_batch(kind):
    """(batch, scale or None): one item of the cell_S_avoid batch broken as kind says"""
    batch, _ = otb.edge_batch("cell_S_avoid")
    src = batch["gt_source"]
    scale = None
    n2d = int(src.kp_offsets[1])
    L = batch["keypoints3d"].shape[1]
    if kind == "a0_high":
        src.assign[0, 5] = n2d
    elif kind == "a0_negative":
        src.assign[0, 5] = -1
    elif kind == "a1_high":
        src.assign[1, 7] = L
    elif kind == "a1_negative":
        src.assign[1, 7] = -3
    elif kind == "cell_S":
        batch, _ = otb.edge_batch("cell_S_hit")
    elif kind in ("scale_0", "scale_nan"):
        scale = batch["query_image_scale"].clone()
        scale[1] = 0.0 if kind == "scale_0" else float("nan")
    elif kind == "mix":
        # item 0: a bad 2D keypoint and (ignored there) a bad 3D point on one correspondence, a bad
        # 3D point on another; item 1: NaN scale
        src.assign[0, 2], src.assign[1, 2] = n2d, L
        src.assign[1, 9] = L + 5
        scale = batch["query_image_scale"].clone()
        scale[1, 0] = float("nan")
    return batch, scale


@pytest.mark.parametrize("kind", ["a0_high", "a0_negative", "a1_high", "a1_negative", "cell_S", "scale_0",
                                  "scale_nan", "mix"])
def test_status_bits(kind):
    batch, scale = _error_batch(kind)
    want = restated_scratch(batch, scale)
    expect = {"a0_high": 2, "a0_negative": 2, "a1_high": 4, "a1_negative": 4, "cell_S": 1, "scale_0": 1,
              "scale_nan": 1, "mix": 7}[kind]
    assert want["bits"] == expect
    check_scratch(run_build(batch, scale), want, batch["gt_source"].assign.shape[1])


# ---- the compaction --------------------------------------------------------------------------------

def check_compact(sorted_key, perm, key_xy, L, S, R):
    n = len(sorted_key)
    b_ids, i_ids, j_ids, fxy, status = run_compact(sorted_key, perm, key_xy, L, S, R)
    drop = sorted_key == otb.KEY_DROPPED
    cell = sorted_key // R
    last = ~drop
    last[:-1] &= (cell[1:] != cell[:-1]) | drop[1:]
    keep = np.nonzero(last)[0]
    m = len(keep)
    assert status[0] == SENT and status[1] == m, f"status {status.tolist()}, {m} kept"
    c = cell[keep]
    assert np.array_equal(b_ids[:m], c // (S * L)) and np.array_equal(i_ids[:m], (c // S) % L)
    assert np.array_equal(j_ids[:m], c % S)
    assert np.array_equal(_bits(fxy[:m]), _bits(key_xy[perm[keep]]))
    for t in (b_ids, i_ids, j_ids):
        assert (t[m:] == SENT).all(), "written past status[1]"
    assert np.isnan(fxy[m:]).all(), "fine_xy written past status[1]"
    return m


def compact_keys(n, kind, seed, L=50, S=40, R=64):
    """sorted keys cell * R + rank: runs of one (b, i, j) up to 60 long that straddle every multiple
    of 1024 (mixed), or every cell distinct (kept), or all INT64_MAX (dropped); mixed ends in dropped"""
    g = np.random.default_rng(seed)
    if kind == "dropped" or n == 0:
        key = np.full(n, otb.KEY_DROPPED, np.int64)
    else:
        step = np.ones(n, np.int64) if kind == "kept" else (g.random(n) < 0.4).astype(np.int64)
        if kind == "mixed":
            p = np.arange(n)
            step[(p % 1024 >= 1024 - 5) | (p % 1024 <= 5)] = 0      # a run across each chunk edge
            step[::57] = 1                                          # runs shorter than R
        step[0] = 0
        cell = np.cumsum(step) + g.integers(0, 3)
        run_start = np.maximum.accumulate(np.where(np.r_[True, cell[1:] != cell[:-1]], np.arange(n), 0))
        key = cell * R + (np.arange(n) - run_start)
        if kind == "mixed":
            key[n - n // 5:] = otb.KEY_DROPPED
    perm = g.permutation(n).astype(np.int64)
    return key, perm, g.standard_normal((n, 2)).astype(np.float32), (L, S, R)


@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 2047, 2048, 2049, 28000])
@pytest.mark.parametrize("kind", ["mixed", "kept", "dropped"])
def test_compaction_at_chunk_edges(n, kind):
    key, perm, xy, (L, S, R) = compact_keys(n, kind, n + len(kind))
    live = key[key != otb.KEY_DROPPED]
    assert (np.diff(key) >= 0).all() and (live % R < 60).all() and (live // R).max(initial=0) < 16 * L * S
    m = check_compact(key, perm, xy, L, S, R)
    if kind == "mixed" and n > 1:
        assert 0 < m < n - n // 5


# ---- fp64 at the training shape --------------------------------------------------------------------

def coord_bound(X, p):
    """first-order bound on |fp32 - fp64| of the kernel's projected (x, y) for points X fp64 [k, 3] and
    the fp64-promoted pack p: each product, sum and quotient one rounding of U |value|, propagated"""
    R, t, K = p[0:9].reshape(3, 3), p[9:12], p[12:21].reshape(3, 3)
    cam = X @ R.T + t
    e_cam = 4 * U * (np.abs(X) @ np.abs(R).T + np.abs(t))
    q = cam @ K.T
    e_q = e_cam @ np.abs(K).T + 3 * U * (np.abs(cam) @ np.abs(K).T)
    zd = q[:, 2] + float(np.float32(1e-6))
    e_zd = e_q[:, 2] + U * np.abs(zd)
    x, y = q[:, 0] / zd, q[:, 1] / zd
    e_x = (e_q[:, 0] + np.abs(x) * e_zd) / np.abs(zd) + U * np.abs(x)
    e_y = (e_q[:, 1] + np.abs(y) * e_zd) / np.abs(zd) + U * np.abs(y)
    if p[43]:
        M = p[21:30].reshape(3, 3)
        xn, yn = p[30] * x + p[31], p[32] * y + p[33]
        e_xn = abs(p[30]) * e_x + 2 * U * (np.abs(p[30] * x) + abs(p[31]))
        e_yn = abs(p[32]) * e_y + 2 * U * (np.abs(p[32] * y) + abs(p[33]))
        v = np.stack([xn, yn, np.ones_like(xn)], 1)
        wv = v @ M.T
        e_w = np.stack([e_xn, e_yn, 0 * e_xn], 1) @ np.abs(M).T + 3 * U * (np.abs(v) @ np.abs(M).T)
        x, y = wv[:, 0] / wv[:, 2], wv[:, 1] / wv[:, 2]
        e_x = (e_w[:, 0] + np.abs(x) * e_w[:, 2]) / np.abs(wv[:, 2]) + U * np.abs(x)
        e_y = (e_w[:, 1] + np.abs(y) * e_w[:, 2]) / np.abs(wv[:, 2]) + U * np.abs(y)
    return 2 * e_x, 2 * e_y


def test_training_shape_against_fp64():
    """B = 4, 512², L = 7000, 3000 correspondences per item, odd items warped, every point planted
    MARGIN px from the rounding boundaries: the device list's ids equal the fp64 list's, fine_xy is
    within coord_bound of it."""
    batch = otb.planted_batch(7)
    src, hw, packs = host_args(batch)
    kp3d = batch["keypoints3d"].numpy()
    assigns = [src.assign[:, src.offsets[b]:src.offsets[b + 1]].numpy() for b in range(len(src))]
    scale = batch["query_image_scale"].numpy()
    lb, li, lj, lxy = otb.batch_list(kp3d, assigns, packs, scale, hw, dt=np.float64)
    out = train_batch.prepare_batch({k: (v.to(DEV) if torch.is_tensor(v) or isinstance(v, train_batch.GTSource)
                                         else v) for k, v in batch.items()})
    got = out["gt_sparse"].check()
    assert len(got) > 4 * 1000
    for t, want in zip((got.b_ids, got.i_ids, got.j_ids), (lb, li, lj)):
        assert np.array_equal(t.cpu().numpy(), want)
    gxy = got.fine_xy.cpu().numpy().astype(np.float64)
    # the bound of each entry's location: the fp64 coordinates of every correspondence, matched to the
    # list by the survivor the entry carries (the fp32 restatement's fine of the same correspondence)
    ratio = 0.0
    for b in range(len(src)):
        sel = lb == b
        a = assigns[b]
        x32, y32, _ = otb.project(kp3d[b], a, packs[b], hw)
        ex, ey = coord_bound(kp3d[b].astype(np.float64)[a[1]], packs[b].astype(np.float64))
        where = {(float(x), float(y)): k for k, (x, y) in enumerate(zip(x32, y32))}
        k = np.array([where[(float(x), float(y))] for x, y in got.fine_xy.cpu().numpy()[sel]])
        err = np.abs(gxy[sel] - lxy[sel])
        r = np.maximum(err[:, 0] / ex[k], err[:, 1] / ey[k])
        assert (r <= 1).all(), f"item {b}: fine_xy err / bound {r.max():.3g}"
        ratio = max(ratio, float(r.max()))
    print(f"training shape: {len(got)} correspondences, fine_xy largest err / bound vs fp64 {ratio:.3g}")


# ---- host guards -----------------------------------------------------------------------------------

@pytest.mark.parametrize("hw", [(1, 8), (8, 1), (1, 1)])
def test_warp_rejects_a_single_row_or_column(hw):
    h, w = hw
    img = torch.zeros(1, 1, h, w, device=DEV)
    pack = torch.from_numpy(warp_packs(4, 4, 0)[1:2]).to(DEV)
    out = _nan(1, 1, h, w)
    with pytest.raises(RuntimeError, match="bad shape"):
        ops.call("opp_homography_warp_f32", ops.ptr(img), ops.ptr(pack), 1, h, w, ops.ptr(out), ops.stream())
    torch.cuda.synchronize()
    assert torch.isnan(out).all()


def test_key_overflow_and_bad_pack_raise_before_a_launch():
    dev = DEV
    one = torch.zeros(2, 1, dtype=torch.int64, device=dev)
    offs = torch.tensor([0, 1], dtype=torch.int64, device=dev)
    kp3d = torch.ones(1, 1, 3, device=dev)
    pack = torch.zeros(1, pack_size(), device=dev)
    scale = torch.ones(1, 2, device=dev)
    status = _sent(2)
    small = [_sent(4), _sent(4), _sent(4), _nan(4), _sent(4, dtype=torch.int64), _nan(4), status]
    # B L S R = 1 * 2^20 * 4096^2 * 4096^2 overflows the int64 key
    with pytest.raises(RuntimeError, match="overflows"):
        ops.call("opp_train_gt_build", ops.ptr(kp3d), ops.ptr(one), 1, ops.ptr(offs), ops.ptr(offs), 1,
                 ops.ptr(pack), ops.ptr(scale), 1, 1 << 20, 32768, 32768, 4096, 4096 * 4096,
                 *(ops.ptr(t) for t in small), ops.stream())
    torch.cuda.synchronize()
    assert (status.cpu() == SENT).all() and (small[0].cpu() == SENT).all(), "written before the guard"
    img = torch.zeros(1, 1, 16, 16, device=dev)
    with pytest.raises(ValueError, match="pack"):
        ops.homography_warp(img, torch.zeros(1, pack_size() - 1, device=dev))
    with pytest.raises(ValueError, match="pack"):
        ops.train_gt(kp3d, one, offs, offs, 1, torch.zeros(1, pack_size() - 1, device=dev), scale, (16, 16), 2, 4)
