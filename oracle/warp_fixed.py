"""CPU restatement of cv2.warpAffine(INTER_LINEAR) on uint8 single-channel images — the fixed-point
scheme of OpenCV's warpAffine + remapBilinear (BORDER_CONSTANT 0) — and of the one-stage form of
the demo's two-warp bbox crop that opp_crop_resize_u8 computes (csrc/opp_image.cu).

    m = the inverse of M as warpAffine forms it (fp64)
    adelta[x] = rint(m0 x 1024), bdelta[x] = rint(m3 x 1024)
    X0[y] = rint((m1 y + m2) 1024) + 16, Y0[y] = rint((m4 y + m5) 1024) + 16
    X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5
    taps at (X >> 5, Y >> 5) + {0, 1}^2, fractions a = X & 31, b = Y & 31,
    out = (sum v w + 2^14) >> 15, w = 32 (32 - a)(32 - b), ..., v = 0 outside the source

numpy's fp64 products and sums are single IEEE operations (no contraction), and np.rint rounds
half to even like cvRound.  TEST INFRASTRUCTURE: used by tests/test_tracking_*.py.
"""
import numpy as np

AB_BITS, INTER_BITS = 10, 5
AB_SCALE, TAB = 1 << AB_BITS, 1 << INTER_BITS


def invert_affine(M):
    """The 2x3 inverse warpAffine computes from M when WARP_INVERSE_MAP is not set (fp64 [6])."""
    M = np.asarray(M, dtype=np.float64).reshape(-1).copy()
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0], M[4] = A11, A22
    M[1] *= -D
    M[3] *= -D
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return M


def fixed_point(m, out_w, out_h):
    """(adelta [out_w], bdelta [out_w], X0 [out_h], Y0 [out_h]) as int64 — cv2's per-column and
    per-row fixed-point terms of the inverse map m."""
    xs = np.arange(out_w, dtype=np.float64)
    ys = np.arange(out_h, dtype=np.float64)
    adelta = np.rint(m[0] * xs * AB_SCALE).astype(np.int64)
    bdelta = np.rint(m[3] * xs * AB_SCALE).astype(np.int64)
    rd = AB_SCALE // TAB // 2
    X0 = np.rint((m[1] * ys + m[2]) * AB_SCALE).astype(np.int64) + rd
    Y0 = np.rint((m[4] * ys + m[5]) * AB_SCALE).astype(np.int64) + rd
    return adelta, bdelta, X0, Y0


def warp_virtual(frame, m, out_w, out_h, x0=0, y0=0, w=None, h=None):
    """The fixed-point warp with inverse map m over the virtual source (frame shifted by (x0, y0),
    zero outside the frame and outside [0, w) x [0, h)); w, h default to the frame (a plain
    cv2.warpAffine of `frame`)."""
    frame = np.asarray(frame)
    H, W = frame.shape
    w = W if w is None else w
    h = H if h is None else h
    adelta, bdelta, X0, Y0 = fixed_point(m, out_w, out_h)
    X = (X0[:, None] + adelta[None]) >> (AB_BITS - INTER_BITS)
    Y = (Y0[:, None] + bdelta[None]) >> (AB_BITS - INTER_BITS)
    sx = np.clip(X >> INTER_BITS, -32768, 32767)
    sy = np.clip(Y >> INTER_BITS, -32768, 32767)
    ax, ay = X & (TAB - 1), Y & (TAB - 1)
    src = frame.astype(np.int64)

    def tap(u, v):
        fx, fy = u + x0, v + y0
        ok = (u >= 0) & (u < w) & (v >= 0) & (v < h) & (fx >= 0) & (fx < W) & (fy >= 0) & (fy < H)
        return np.where(ok, src[np.clip(fy, 0, H - 1), np.clip(fx, 0, W - 1)], 0)

    acc = (tap(sx, sy) * ((TAB - ax) * (TAB - ay)) + tap(sx + 1, sy) * (ax * (TAB - ay)) +
           tap(sx, sy + 1) * ((TAB - ax) * ay) + tap(sx + 1, sy + 1) * (ax * ay)) * 32
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def warp_affine(img, M, dsize):
    """cv2.warpAffine(img, M, dsize, flags=INTER_LINEAR) for uint8 [H, W]; dsize = (w, h)."""
    return warp_virtual(img, invert_affine(M), int(dsize[0]), int(dsize[1]))
