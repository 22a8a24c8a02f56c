"""The opp_coarse_focal_* kernels one pass at a time (statistics, forward, backward, the scalar and R/C
finalisers, the sparse ground truth) against plain fp64 statements of the same quantities
(oracle/coarse_loss.py), at the tile edges of their launches and at loss settings other than the
reference's (alpha = 0.5 and pos_w = neg_w would hide a swapped class factor).

Techniques:
  - exact sim: features are multiples of 2^-4 in [-1/2, 1/2] and the scale is a power of two, so
    every fp32 sim (K = 256) is exact.  The maxima must equal fp64; everything else carries only the
    roundings of expf / logf / expm1f / powf and of the fp32 sums, and is held to a first-order bound
    derived from them in fp64 (U = 2^-24; expf 2 ulp, logf / expm1f 1 ulp, powf 4 ulp);
  - poisoned outputs: every output of the entry points starts as NaN (int64: a negative sentinel),
    so a value that is never written cannot pass;
  - random features at the training shape and at the golden shapes: the statistics within the same
    bound plus the fp32 rounding of sim, the loss and gradients within the 2e-4 rule of
    test_train_coarse_gpu (there sim rounding at |sim| ~ 260 dominates).
The largest err / bound of each quantity is printed."""
import types

import pytest
import torch

from oracle import coarse_loss as cl
from oracle import train_gt as otg
from onepose_plus_plus_b200 import SparseGT, _lib, losses, ops, train_gt, train_path

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
K = 256
T = 64                                 # own rows per CTA = streamed rows per tile
RTOL = 2e-4
SENTINEL = -777
LO = cl.LO
DEFAULT = (0.5, 2.0, 1.0, 1.0)
FOCALS = [(a, g, pw, nw) for a in (0.25, 0.5, 0.8) for g in (0.0, 1.0, 2.0, 2.5) for pw, nw in ((1.0, 1.0), (2.0, 0.5))]
OTHER = (0.25, 2.5, 2.0, 0.5)          # LoFTR's alpha, a non-integer gamma, unequal class weights
CM = types.SimpleNamespace(temperature=cl.TEMPERATURE)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _blocks(n):
    return _lib.load().opp_coarse_focal_blocks(n)


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _sentinel(*shape):
    return torch.full(shape, SENTINEL, dtype=torch.int64, device=DEV)


# ------------------------------------------------------------------------------------------------
# The entry points with poisoned outputs (the same C ABI calls as ops.coarse_focal_*)
# ------------------------------------------------------------------------------------------------
def run_stats(a, b, mask, scale):
    B, L, _ = a.shape
    S = b.shape[1]
    st_rows, st_cols = _nan(B, L, 2), _nan(B, S, 2)
    ops.call("opp_coarse_focal_stats", ops.ptr(a), ops.ptr(b), ops.ptr(mask), B, L, S, K, float(scale),
             ops.ptr(_nan(B, _blocks(L), S, 2)), ops.ptr(st_rows), ops.ptr(st_cols), ops.stream())
    return st_rows, st_cols


def run_fwd(a, b, st, gt, mask, scale, focal, index=None):
    """(loss, counts, wts, r, c); index = (row_ptr, j_ids, ...) runs the sparse entry point."""
    B, L, _ = a.shape
    S = b.shape[1]
    nb = _blocks(L)
    parts = (_nan(B * nb, 2, dtype=torch.float64), _sentinel(B * nb, 2), _nan(B, L, 2, dtype=torch.float64),
             _nan(B, nb, S, 2, dtype=torch.float64))
    outs = (_nan(1), _sentinel(2), _nan(2), _nan(B, L, dtype=torch.float64), _nan(B, S, dtype=torch.float64))
    head = (ops.ptr(a), ops.ptr(b), ops.ptr(st[0]), ops.ptr(st[1]))
    if index is None:
        head += (ops.ptr(gt), ops.GT_BYTES[gt.dtype])
        name = "opp_coarse_focal_fwd"
    else:
        head += (ops.ptr(index[0]), ops.ptr(index[1]))
        name = "opp_coarse_focal_fwd_sparse"
    ops.call(name, *head, ops.ptr(mask), B, L, S, K, float(scale), *(float(x) for x in focal),
             *(ops.ptr(t) for t in parts + outs), ops.stream())
    return outs


def run_bwd(a, b, st, fwd, grad, gt, mask, scale, focal, index=None):
    """(dA, dB) for the incoming gradient grad (a Python float)."""
    B, L, _ = a.shape
    S = b.shape[1]
    da, db = _nan(B, L, K), _nan(B, S, K)
    go = torch.tensor([grad], dtype=torch.float32, device=DEV)
    head = (ops.ptr(a), ops.ptr(b), ops.ptr(st[0]), ops.ptr(st[1]), ops.ptr(fwd[3]), ops.ptr(fwd[4]),
            ops.ptr(fwd[2]), ops.ptr(go))
    if index is None:
        head += (ops.ptr(gt), ops.GT_BYTES[gt.dtype])
        name = "opp_coarse_focal_bwd"
    else:
        head += tuple(ops.ptr(t) for t in index)
        name = "opp_coarse_focal_bwd_sparse"
    ops.call(name, *head, ops.ptr(mask), B, L, S, K, float(scale), float(focal[0]), float(focal[1]),
             ops.ptr(da), ops.ptr(db), ops.stream())
    return da, db


def run_all(a, b, gt, mask, scale, focal, grads, index=None):
    st = run_stats(a, b, mask, scale)
    fwd = run_fwd(a, b, st, gt, mask, scale, focal, index)
    return st, fwd, [run_bwd(a, b, st, fwd, g, gt, mask, scale, focal, index) for g in grads]


# ------------------------------------------------------------------------------------------------
# Inputs
# ------------------------------------------------------------------------------------------------
def _grid(shape, g):
    """Multiples of 2^-4 in [-1/2, 1/2]: K = 256 products and their sums are exact in fp32."""
    return torch.randint(-8, 9, shape, generator=g, device=DEV).float() / 16


def _signs(shape, g):
    return (torch.randint(0, 2, shape, generator=g, device=DEV).float() - 0.5)


def exact_case(B, L, S, seed, kind="planted", gt_dtype=torch.int16, pos=0.03):
    """(a, b, gt, scale) with exact fp32 sim.
      planted: scale 2^-2, half of min(L, S) columns of b copy a row of a (c up to ~0.7);
      clamp:   scale 1, the planted rows are +-1/2 (sim 64 against |sim| < ~25 elsewhere), so c
               passes both clamp bounds.
    Every sample's last row matches its column 0 with the largest sim of that column (the column's
    maximum lies in the last, partial CTA); gt: the plants, `pos` random positives, 1 % neither (2)."""
    g = _gen(seed)
    a, b = _grid((B, L, K), g), _grid((B, S, K), g)
    gt = (torch.rand((B, L, S), generator=g, device=DEV) < pos).to(torch.int16)
    if gt_dtype != torch.bool:
        gt[torch.rand((B, L, S), generator=g, device=DEV) < 0.01] = 2
    n = max(1, min(L, S) // 2)
    for bi in range(B):
        ri = torch.randperm(L, generator=g, device=DEV)[:n]
        cj = torch.randperm(S, generator=g, device=DEV)[:n]
        if kind == "clamp":
            b[bi, cj] = _signs((n, K), g)
            a[bi, ri] = b[bi, cj]
        else:
            b[bi, cj] = a[bi, ri]
        gt[bi, ri, cj] = 1
        b[bi, 0] = _signs((K,), g)
        a[bi, L - 1] = b[bi, 0]
        gt[bi, L - 1, 0] = 1
    return a.contiguous(), b.contiguous(), gt.to(gt_dtype), (1.0 if kind == "clamp" else 0.25)


def edge_mask(B, S, seed):
    """uint8 [B, S]: sample 3k keeps a random 70 %, 3k + 1 exactly one column (S // 2), 3k + 2 only
    the columns of the last 64-column tile."""
    g = _gen(seed)
    m = (torch.rand((B, S), generator=g, device=DEV) < 0.7)
    for bi in range(B):
        if bi % 3 == 0:
            m[bi, S // 2] = True
        elif bi % 3 == 1:
            m[bi] = False
            m[bi, S // 2] = True
        else:
            m[bi] = False
            m[bi, T * ((S - 1) // T):] = True
    return m.to(torch.uint8).contiguous()


# ------------------------------------------------------------------------------------------------
# fp64 references and first-order fp32 bounds
# ------------------------------------------------------------------------------------------------
# Rounding steps of the statistics pass, counted along its reduction tree (coarse_focal_kernel with
# kStats, then coarse_focal_colstats_kernel).  Row: a thread folds its 4 columns of every 64-column
# tile one at a time (a rescale or an add, <= 6 U each), then the 16 threads' partials are merged
# (<= 10 U each).  Column: a thread folds 4 rows, 16 partials merge per CTA, and the colstats kernel
# merges the CTAs' partials in order.  These counts must follow that tree if it changes.
def _stat_steps(L, S):
    return 6 * 4 * -(-S // T) + 10 * 16 + 4, 6 * 4 + 10 * (16 + _blocks(L)) + 4


def _stats_bounds(sim, keep, rm, rl, cm, cl_, e_sim):
    """Bounds on |(m + log s) - lse| per row (kept columns) and per column (every row) of sim
    [b, L, S], and on the maxima (0 for exact sim, e_sim None): the chain steps above, logf 1 ulp,
    x - m rounded by U |x - m| (weighted by the softmax), and a sim error moves a max or a
    log-sum-exp by at most its largest value."""
    k_row, k_col = _stat_steps(*sim.shape[1:])
    simk = sim.masked_fill(~keep, float("-inf"))
    q, p = torch.softmax(simk, 2), torch.softmax(sim, 1)
    tol_rl = (k_row * U + U * (q * (rm[..., None] - simk)).nan_to_num(0.0, 0.0, 0.0).sum(2)
              + 2 * U * (rl - rm).abs())
    tol_cl = k_col * U + U * (p * (cm[:, None] - sim)).sum(1) + 2 * U * (cl_ - cm).abs()
    if e_sim is None:
        return tol_rl, tol_cl, 0.0, 0.0
    e_r, e_c = e_sim.masked_fill(~keep, 0.0).amax(2), e_sim.amax(1)
    return tol_rl + e_r, tol_cl + e_c, e_r, e_c


class Reference:
    """fp64 statistics, loss, counts, weights, R, C, dA and dB of one case, with the bounds the
    kernels' fp32 roundings allow (exact: sim is exact in fp32; otherwise its (K + 2) U |a||b| s
    rounding bound enters every exponent).  The statistics and their bounds are taken one sample at
    a time, so at the training shape only the oracle's loss and gradients hold [B, L, S] fp64 terms."""

    def __init__(self, a, b, gt, mask, scale, focal, exact):
        alpha, gamma, pw, nw = focal
        B = a.shape[0]
        a64, b64 = a.double(), b.double()
        stats, tols = [], []
        for bi in range(B):
            sl = slice(bi, bi + 1)
            ms = mask[sl] if mask is not None else None
            st = cl.softmax_stats(a64[sl], b64[sl], scale, ms)
            sim = scale * torch.einsum("blk,bsk->bls", a64[sl], b64[sl])
            keep = torch.ones_like(sim, dtype=torch.bool) if ms is None else ms.bool()[:, None, :].expand_as(sim)
            e_sim = None if exact else (K + 2) * U * scale * torch.einsum("blk,bsk->bls", a64[sl].abs(),
                                                                          b64[sl].abs())
            stats.append(st)
            tols.append(_stats_bounds(sim, keep, *st, e_sim))
            del sim, keep, e_sim
        self.rm, self.rl, self.cm, self.cl = (torch.cat(t) for t in zip(*stats))
        self.tol_rl, self.tol_cl = torch.cat([t[0] for t in tols]), torch.cat([t[1] for t in tols])
        self.tol_rm = 0.0 if exact else torch.cat([t[2] for t in tols])
        self.tol_cm = 0.0 if exact else torch.cat([t[3] for t in tols])
        del stats, tols
        self.loss, self.da, self.db, self.R, self.C = cl.focal_loss_and_grads(
            a64, b64, gt, scale, mask, alpha, gamma, pw, nw, with_rc=True)
        self.npos, self.nneg = int((gt == 1).sum()), int((gt == 0).sum())
        self.wts = torch.tensor([pw / self.npos if self.npos else 0.0, nw / self.nneg if self.nneg else 0.0],
                                dtype=torch.float64).float()
        self.tol_loss = None
        if not exact:
            return
        sim = scale * torch.einsum("blk,bsk->bls", a64, b64)
        keep = torch.ones_like(sim, dtype=torch.bool) if mask is None else mask.bool()[:, None, :].expand_as(sim)
        # per element: log q (softmax over S, kept columns) and log p (over L) as the kernels form them
        lq = (sim - self.rl[..., None]).masked_fill(~keep, 0.0)
        lp = (sim - self.cl[:, None]).masked_fill(~keep, 0.0)
        e_lq = (self.tol_rl[..., None] + U * (sim - self.rm[..., None]).abs() + U * lq.abs()).masked_fill(~keep, 0.0)
        e_lp = (self.tol_cl[:, None] + U * (sim - self.cm[:, None]).abs() + U * lp.abs()).masked_fill(~keep, 0.0)
        P, Q = lp.exp() * keep, lq.exp() * keep
        c = P * Q
        om = torch.where(keep, -torch.expm1(lp + lq), torch.ones_like(c))
        dP, dQ = P * (e_lp + 4 * U), Q * (e_lq + 4 * U)
        dc = c * (e_lp + e_lq + 9 * U)
        dom = c * (e_lp + e_lq + U * (lp + lq).abs()) + 2 * U * om
        del lq, lp, e_lq, e_lp, sim
        passes = keep & (c >= LO) & (om >= LO)
        amb = keep & (((c - LO).abs() <= dc + LO * U) | ((om - LO).abs() <= dom + LO * U))
        sens = (passes | amb).double()
        ct, omt = c.clamp(LO, 1 - LO), om.clamp(LO, 1 - LO)
        lc, lom = ct.log().abs(), omt.log().abs()
        pos, neg = gt == 1, gt == 0
        # loss terms and their first-order error (c and 1 - c are formed independently)
        l_pos = alpha * omt ** gamma * lc
        l_neg = (1 - alpha) * ct ** gamma * lom
        dl_pos = sens * (alpha * omt ** gamma / ct * dc + alpha * gamma * omt ** (gamma - 1) * lc * dom) + 16 * U * l_pos
        dl_neg = sens * ((1 - alpha) * gamma * ct ** (gamma - 1) * lom * dc + (1 - alpha) * ct ** gamma / omt * dom) \
            + 16 * U * l_neg
        self.tol_loss = ((pw / self.npos * dl_pos[pos].sum() if self.npos else 0.0)
                         + (nw / self.nneg * dl_neg[neg].sum() if self.nneg else 0.0)
                         + 2 * U * abs(float(self.loss)))
        del l_pos, l_neg, dl_pos, dl_neg
        # c dl/dc per class (unweighted, as focal_term), its error, then weighted
        h_pos = alpha * (gamma * ct * omt ** (gamma - 1) * lc + omt ** gamma)
        dh_pos = (alpha * gamma * omt ** (gamma - 1) * (lc + 1) * dc
                  + alpha * (gamma * abs(gamma - 1) * ct * omt ** (gamma - 2) * lc + gamma * omt ** (gamma - 1)) * dom
                  + 24 * U * h_pos)
        h_neg = (1 - alpha) * (gamma * ct ** gamma * lom + ct ** (gamma + 1) / omt)
        dh_neg = ((1 - alpha) * (gamma ** 2 * ct ** (gamma - 1) * lom + (gamma + 1) * ct ** gamma / omt) * dc
                  + (1 - alpha) * (gamma * ct ** gamma / omt + ct ** (gamma + 1) / omt ** 2) * dom
                  + 24 * U * h_neg)
        wp, wn = float(self.wts[0]), float(self.wts[1])
        w = torch.where(pos, wp, torch.where(neg, wn, 0.0)).double()
        h = torch.where(pos, h_pos, h_neg)
        dh = torch.where(pos, dh_pos, dh_neg)
        del h_pos, dh_pos, h_neg, dh_neg, ct, omt, lc, lom
        # h above bounds |c dl/dc|; so g, |R - g|, |C - g| and |dsim| below are magnitudes
        g = w * h * passes
        dg = w * ((dh + U * h) * passes + 2 * h * amb)
        self.tol_R, self.tol_C = dg.sum(2), dg.sum(1)
        Rg = self.R.abs()[..., None] + g
        Cg = self.C.abs()[:, None] + g
        # dsim = g (1 - p) + g (1 - q) - p (C - g) - q (R - g); the same matrix in both launches
        d = 2 * g + P * Cg + Q * Rg
        self.dd = (2 * dg + g * (dP + dQ + 2 * U) + dP * Cg + P * self.tol_C[:, None] + dQ * Rg
                   + Q * self.tol_R[..., None] + 2 * U * d) * keep
        self.d = d * keep
        self.a_abs, self.b_abs, self.scale = a64.abs(), b64.abs(), scale
        self.amb = int(amb.sum())

    def grad_bounds(self, grad):
        """Bounds on dA and dB at the incoming gradient `grad`: dsim's error, the fp32 FMA chain over
        the S (L) streamed rows and the final scale multiply."""
        go = abs(grad)
        L, S = self.a_abs.shape[1], self.b_abs.shape[1]
        dd, ad = go * self.dd, go * self.d
        tda = self.scale * (torch.einsum("bls,bsk->blk", dd, self.b_abs)
                            + (S + 1) * U * torch.einsum("bls,bsk->blk", ad, self.b_abs)) + U * go * self.da.abs()
        tdb = self.scale * (torch.einsum("bls,blk->bsk", dd, self.a_abs)
                            + (L + 1) * U * torch.einsum("bls,blk->bsk", ad, self.a_abs)) + U * go * self.db.abs()
        return tda, tdb


def _ratio(err, tol):
    if not torch.is_tensor(err):
        return float(err / max(tol, 1e-300))
    return float((err / torch.as_tensor(tol).clamp_min(1e-300)).max()) if err.numel() else 0.0


class Report:
    def __init__(self, label):
        self.label, self.worst = label, {}

    def check(self, name, got, ref, tol):
        err = (got.double() - ref).abs() if torch.is_tensor(got) else abs(got - ref)
        ok = bool((err <= tol).all()) if torch.is_tensor(err) else err <= tol
        ratio = _ratio(err, tol)
        assert ok, f"{self.label}: {name} max err / bound {ratio:.3g}"
        self.worst[name] = max(self.worst.get(name, 0.0), ratio)

    def print(self):
        print(f"{self.label}: max |err| / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in self.worst.items()))


def check_stats(rep, ref, st, exact):
    st_rows, st_cols = st
    assert not torch.isnan(st_rows).any() and not torch.isnan(st_cols).any()
    if exact:
        assert torch.equal(st_rows[..., 0].double(), ref.rm), "row max"
        assert torch.equal(st_cols[..., 0].double(), ref.cm), "column max"
    else:
        rep.check("row max", st_rows[..., 0], ref.rm, ref.tol_rm)
        rep.check("col max", st_cols[..., 0], ref.cm, ref.tol_cm)
    rep.check("row lse", st_rows[..., 0].double() + st_rows[..., 1].double(), ref.rl, ref.tol_rl)
    rep.check("col lse", st_cols[..., 0].double() + st_cols[..., 1].double(), ref.cl, ref.tol_cl)


def check_fwd(rep, ref, fwd, exact):
    loss, counts, wts, r, c = fwd
    assert counts.tolist() == [ref.npos, ref.nneg]
    assert torch.equal(wts.cpu(), ref.wts)
    assert not torch.isnan(r).any() and not torch.isnan(c).any()
    rl = float(ref.loss)
    if exact:
        rep.check("loss", float(loss), rl, ref.tol_loss)
        rep.check("R", r, ref.R, ref.tol_R)
        rep.check("C", c, ref.C, ref.tol_C)
    else:
        rep.check("loss", float(loss), rl, RTOL * abs(rl))
        rep.check("R", r, ref.R, RTOL * ref.R.abs() + 1e-6 + RTOL * float(ref.R.abs().max()))
        rep.check("C", c, ref.C, RTOL * ref.C.abs() + 1e-6 + RTOL * float(ref.C.abs().max()))


def check_bwd(rep, ref, grad, dab, exact):
    da, db = dab
    assert not torch.isnan(da).any() and not torch.isnan(db).any()
    if exact:
        tda, tdb = ref.grad_bounds(grad)
    else:
        tda = RTOL * (grad * ref.da).abs() + 1e-6 + RTOL * abs(grad) * float(ref.da.abs().max())
        tdb = RTOL * (grad * ref.db).abs() + 1e-6 + RTOL * abs(grad) * float(ref.db.abs().max())
    rep.check("dA", da, grad * ref.da, tda)
    rep.check("dB", db, grad * ref.db, tdb)


def check_case(label, a, b, gt, mask, scale, focal, grads, exact=True):
    st, fwd, bwds = run_all(a, b, gt, mask, scale, focal, grads)
    ref = Reference(a, b, gt, mask, scale, focal, exact)
    rep = Report(label)
    check_stats(rep, ref, st, exact)
    check_fwd(rep, ref, fwd, exact)
    for g, dab in zip(grads, bwds):
        check_bwd(rep, ref, g, dab, exact)
    rep.print()
    return st, fwd, bwds, ref


# ------------------------------------------------------------------------------------------------
# Every pass at the tile edges: L in {1, 63, 64, 65, 7000}, S in {1, 63, 64, 65, 4095, 4096, 4097}
# ------------------------------------------------------------------------------------------------
SHAPES = [(1, 1, 4097), (3, 63, 65), (1, 64, 4095), (3, 65, 63), (1, 7000, 4096), (3, 7000, 1), (3, 64, 64),
          (1, 65, 1)]


@pytest.mark.parametrize("B,L,S", SHAPES)
@pytest.mark.parametrize("masked", [False, True])
def test_passes_at_tile_edges(B, L, S, masked):
    """Statistics, forward and backward (grad 1 and -3) on exact sim at OTHER's loss settings; the
    gt dtype cycles through int16, uint8 and bool.  Determinism: a second run gives the same bits."""
    seed = 1000 * L + S + 7 * B + masked
    dt = (torch.int16, torch.uint8, torch.bool)[seed % 3]
    a, b, gt, scale = exact_case(B, L, S, seed, gt_dtype=dt)
    mask = edge_mask(B, S, seed) if masked else None
    label = f"B={B} L={L} S={S} masked={masked} gt={str(dt)[6:]}"
    st, fwd, bwds, ref = check_case(label, a, b, gt, mask, scale, OTHER, (1.0, -3.0))
    if L > T:
        # the column maximum of column 0 sits in the last CTA: its rows are part of the statistics
        assert bool((ref.cm[:, 0] == scale * 64).all())
    st2, fwd2, bwds2 = run_all(a, b, gt, mask, scale, OTHER, (1.0, -3.0))
    for x, y in zip(st + fwd + sum(bwds, ()), st2 + fwd2 + sum(bwds2, ())):
        assert torch.equal(x, y), "two runs differ"


# ------------------------------------------------------------------------------------------------
# Loss settings: alpha, gamma and the class weights
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("focal", FOCALS, ids=lambda f: "a{}-g{}-w{}-{}".format(*f))
def test_focal_settings(focal):
    """Every alpha / gamma / (pos_w, neg_w) of the grid on the planted and the clamp cases (B = 3,
    L = 65, S = 130: partial last CTA and tile, the edge mask), grad 1, 0.7 and -3."""
    for kind in ("planted", "clamp"):
        a, b, gt, scale = exact_case(3, 65, 130, 11 if kind == "planted" else 12, kind)
        mask = edge_mask(3, 130, 13)
        check_case(f"{kind} {focal}", a, b, gt, mask, scale, focal, (1.0, 0.7, -3.0))
        if kind == "clamp":
            _, _, c = cl.dual_softmax(a.double(), b.double(), scale, mask)
            assert bool((c > cl.HI).any()) and bool(((c < cl.LO) & (c > 0)).any())


# ------------------------------------------------------------------------------------------------
# Finalisers: more than 256 per-CTA partials
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [257, 513])
def test_finalisers_over_many_parts(B):
    """B * ceil(L / 64) = 257 and 513 parts: the scalar kernel's strided loop over its 256 threads."""
    a, b, gt, scale = exact_case(B, 64, 5, B)
    check_case(f"B={B} L=64 S=5", a, b, gt, None, scale, OTHER, (-3.0,))


# ------------------------------------------------------------------------------------------------
# Random features: training shape and golden shapes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["training"] + list(cl.GOLDEN_CASES))
def test_random_features(key):
    """make_case features (sim rounding dominates): statistics within the derived bound with the
    rounding of sim, loss / R / C / dA / dB within 2e-4, counts and weights exact."""
    if key == "training":
        a, b, gt, mask = cl.make_case("planted", 4, 7000, 4096, seed=1)
        gt[torch.rand(gt.shape, generator=torch.Generator().manual_seed(2)) < 2e-4] = 1
        focal, grads = (0.25, 2.0, 2.0, 0.5), (-3.0,)
    else:
        name, batch, rows, cols = cl.GOLDEN_CASES[key]
        a, b, gt, mask = cl.make_case(name, batch, rows, cols)
        focal, grads = (0.8, 1.0, 2.0, 0.5), (0.7,)
    mask = mask.to(torch.uint8).cuda() if mask is not None else None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    check_case(f"random {key}", a.cuda(), b.cuda(), gt.cuda(), mask, cl.scale_of(), focal, grads, exact=False)
    peak = torch.cuda.max_memory_allocated() - base
    print(f"random {key}: peak device memory above the start {peak / 2**30:.1f} GiB")


# ------------------------------------------------------------------------------------------------
# Sparse ground truth: the bucket walk at tile boundaries
# ------------------------------------------------------------------------------------------------
def boundary_gt(B, L, S):
    """bool [B, L, S]: sample 0: row 5 holds j = 0, 63, 64, 127, S - 1 with empty neighbours, row 9
    fills the tile [64, 128) and continues to 140, column 70 holds every row but the first and the
    last few, first and last rows empty; sample 1 empty; samples 2 .. B - 1 random 4 % with empty
    first and last rows."""
    conf = torch.zeros(B, L, S, dtype=torch.bool)
    conf[0, 5, [0, 63, 64, 127, S - 1]] = True
    conf[0, 9, 64:141] = True
    conf[0, 3:L - 3, 70] = True
    conf[2:] = torch.rand(B - 2, L, S, generator=torch.Generator().manual_seed(3)) < 0.04
    conf[2:, 0] = False
    conf[2:, L - 1] = False
    return conf


@pytest.mark.parametrize("masked", [False, True])
def test_sparse_walk_at_tile_boundaries(masked):
    """B = 4, L = 450, S = 300 (neither on the 64 grid; B S + 1 = 1201 column pointers, two rounds of
    gt_index's scan): the sparse forward and backward equal the dense ones bit for bit (statistics
    shared), the dense ones meet the fp64 bounds, and the column side's bucket of column 70 spans
    every tile of L."""
    B, L, S = 4, 450, 300
    a, b, _, scale = exact_case(B, L, S, 21)
    conf = boundary_gt(B, L, S).cuda()
    assert int(conf[1].sum()) == 0 and int(conf[0, :, 70].sum()) == L - 6
    mask = edge_mask(B, S, 22) if masked else None
    if mask is not None:
        mask[0] = 1                               # sample 0 keeps every column
    grads = (0.7, -3.0)
    _, fwd_d, bwd_d, _ = check_case(f"sparse boundaries masked={masked}", a, b, conf.to(torch.int16), mask, scale,
                                    OTHER, grads)
    bi, ii, jj = torch.where(conf)
    gt = SparseGT(bi, ii, jj, torch.zeros(len(bi), 2, device=DEV), (B, L, S)).check()
    row_ptr, col_ptr, col_rows = ops.gt_index(gt.b_ids, gt.i_ids, gt.j_ids, gt.shape)
    st = run_stats(a, b, mask, scale)
    fwd_s = run_fwd(a, b, st, None, mask, scale, OTHER, (row_ptr, gt.j_ids))
    bwd_s = [run_bwd(a, b, st, fwd_s, g, None, mask, scale, OTHER, (row_ptr, gt.j_ids, col_ptr, col_rows))
             for g in grads]
    names = ("loss", "counts", "wts", "r", "c")
    for name, d, s in zip(names, fwd_d, fwd_s):
        assert torch.equal(d, s), f"{name}: sparse differs from dense"
    for g, (da, db), (sa, sb) in zip(grads, bwd_d, bwd_s):
        assert torch.equal(da, sa) and torch.equal(db, sb), f"grad {g}: sparse differs from dense"


# ------------------------------------------------------------------------------------------------
# A query mask that keeps no column of a sample
# ------------------------------------------------------------------------------------------------
def test_fully_masked_sample_is_rejected():
    """The eager path gives such a sample the unmasked (fp64) or a uniform (fp32) softmax over S; the
    lazy loss refuses it, dense and sparse, before any launch."""
    B, L, S = 2, 70, 90
    a, b, gt, _ = cl.make_case("planted", B, L, S)
    mask = torch.ones(B, S, dtype=torch.bool)
    mask[1] = False
    h = train_path.TrainConfHandle(CM, a.cuda(), b.cuda(), mask.cuda())
    bi, ii, jj = torch.where(gt.cuda() == 1)
    sparse = SparseGT(bi, ii, jj, torch.zeros(len(bi), 2, device=DEV), (B, L, S))
    for g in (gt.cuda(), sparse):
        with pytest.raises(ValueError, match="keeps no column"):
            losses.coarse_focal_loss(h, g, *DEFAULT)
    mask[1, -1] = True                            # one kept column is enough
    h = train_path.TrainConfHandle(CM, a.cuda(), b.cuda(), mask.cuda())
    loss, _ = losses.coarse_focal_loss(h, gt.cuda(), *DEFAULT)
    assert torch.isfinite(loss)


# ------------------------------------------------------------------------------------------------
# fine_supervision edges
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["empty_list", "outside_keys"])
def test_fine_supervision_edges(case):
    """An empty list with matches (every output from the -50 fill), and matches whose key sorts
    before the first or after the last entry, with query_image_scale on sample 1: bit-equal to the
    PyTorch formula on the dense tensor."""
    B, L, hc, wc = 2, 40, 6, 8
    S = hc * wc
    if case == "empty_list":
        ids, xy = [[], [], []], torch.zeros(0, 2)
    else:
        ids = [[0, 0, 1, 1], [3, 3, 7, 20], [5, 40, 0, 30]]
        xy = torch.tensor([[11.5, 3.25], [2.0, 40.5], [-3.0, 7.75], [60.25, 33.0]])
    m = [[0, 0, 1, 1, 1, 0], [0, 3, 7, L - 1, 20, 3], [0, 40, 0, S - 1, 30, 5]]
    keys = set(zip(*ids))
    # outside_keys: (0, 0, 0) sorts before the first entry, (1, L - 1, S - 1) after the last
    assert sum(k in keys for k in zip(*m)) == (0 if case == "empty_list" else 4)
    lng = [torch.tensor(t, dtype=torch.int64, device=DEV) for t in ids + m]
    gt = SparseGT(*lng[:3], xy.to(DEV), (B, L, S)).check()
    outs = []
    for sparse in (True, False):
        data = {"b_ids": lng[3], "i_ids": lng[4], "j_ids": lng[5], "q_hw_c": (hc, wc),
                "query_image_scale": torch.tensor([[1.0, 1.0], [1.25, 0.75]], device=DEV)}
        if sparse:
            data["gt_sparse"] = gt                            # opp_fine_supervision
        else:
            data["fine_location_matrix_gt"] = gt.to_dense()[1]   # the reference formula, by PyTorch
        train_gt.fine_supervision(data, otg.config())
        outs.append(data["expec_f_gt"])
    assert outs[0].shape == (6, 2) and torch.equal(outs[0], outs[1])
