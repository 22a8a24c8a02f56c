"""The opp_fine_train_* kernels one at a time, at the launch shapes of train_fine's _layer_fwd /
_layer_bwd, against plain fp64 PyTorch statements of the same operations (F.unfold / F.fold, x @ W.T,
F.layer_norm, train_path._linear_attention and train_path.fine_matching with autograd).

Three techniques:
  - exact cases: inputs are multiples of 2^-4 (or small integers) of small range, so every product
    and partial sum is exact in fp32 and the kernel must equal the fp64 reference bit for bit; a
    dropped, doubled or misplaced row, column, tile or group shows up whatever its size;
  - poisoned outputs: every output starts as NaN and must be fully written; the columns and rows of
    a wider buffer that a strided view does not cover hold a sentinel and must stay untouched;
  - random cases at realistic magnitudes, within a bound derived from fp32 rounding of the same sums
    (U = 2^-24 times the number of roundings along the sum times the sum of absolute terms, computed
    in fp64); the largest err / bound is printed per kernel.
Row counts: 26·m for m in {1, 3, 115, 192} (one match, a few, the tail chunk at M = 4915, a full
chunk of 192) and 255, 256, 257, 511 (around the 64-row tiles and the 256-row groups)."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from oracle import make_train_fine_golden as mtf
from oracle import workload
from onepose_plus_plus_b200 import ops, train_fine, train_path

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24                       # unit roundoff of fp32
D, TOK, WIN = 128, 26, 25
SENTINEL = 12345.5
ROWS = (26, 78, 2990, 4992, 255, 256, 257, 511)

# (name, n, k, epilogue) of each fine_train_linear call in _layer_fwd (trans_w) and _layer_bwd
FWD_SHAPES = (("qkv", 384, 128), ("merge", 128, 128), ("mlp0", 256, 256), ("mlp2", 128, 256))
BWD_SHAPES = (("dh1", 256, 128), ("dxm", 256, 256), ("da", 128, 128), ("dx", 128, 384))
# (name, dW shape, ld of the x operand) of each fine_train_wgrad call: the qkv one reads x = xm[:, :128]
WGRAD_SHAPES = (("qkv", 384, 128, 256), ("merge", 128, 128, 128), ("mlp0", 256, 256, 256), ("mlp2", 128, 256, 256))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _grid16(shape, g, span=16):
    """Multiples of 2^-4 in [-span/16, span/16], fp32 on the device."""
    return torch.randint(-span, span + 1, shape, generator=g, device=DEV).float() / 16


def _randn(shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device=DEV) * scale


def _framed(rows, cols, ld=None, extra_rows=8):
    """(buffer, view): view = buffer[:rows, :cols] is NaN, the rest of the buffer (row stride ld,
    extra_rows more rows) holds SENTINEL."""
    ld = cols if ld is None else ld
    buf = torch.full((rows + extra_rows, ld), SENTINEL, device=DEV)
    view = buf[:rows, :cols]
    view.fill_(float("nan"))
    return buf, view


def _assert_framed(buf, rows, cols, what):
    """The view of _framed is fully written (no NaN) and nothing around it moved."""
    view = buf[:rows, :cols]
    assert not torch.isnan(view).any(), f"{what}: {int(torch.isnan(view).sum())} outputs not written"
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:rows, :cols] = False
    assert bool((buf[outside] == SENTINEL).all()), f"{what}: written outside its view"


def _placed(values, ld):
    """values [rows, cols] copied into the first columns of a [rows, ld] NaN buffer: the view."""
    buf = torch.full((values.shape[0], ld), float("nan"), device=DEV)
    buf[:, :values.shape[1]] = values
    return buf[:, :values.shape[1]]


def _ratio(err, tol):
    return float((err / tol.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _report(name, ratio):
    print(f"{name}: max |err| / bound = {ratio:.3g}")


# ------------------------------------------------------------------------------------------------
# Gather and its backward
# ------------------------------------------------------------------------------------------------
def _ids(B, hc, wc, n3d, m_random, g, crowd=0):
    """b, i, j: the four corner cells of every image, m_random random cells, two repeats of the
    first random match and, with crowd > 0, crowd matches in one interior cell."""
    corners = torch.tensor([0, wc - 1, (hc - 1) * wc, hc * wc - 1])
    b = [torch.arange(B).repeat_interleave(4), torch.randint(0, B, (m_random,), generator=g)]
    j = [corners.repeat(B), torch.randint(0, hc * wc, (m_random,), generator=g)]
    b.append(b[1][:1].repeat(2))
    j.append(j[1][:1].repeat(2))
    if crowd:
        b.append(torch.full((crowd,), B - 1))
        j.append(torch.full((crowd,), (hc // 2) * wc + wc // 2))
    b, j = torch.cat(b), torch.cat(j)
    i = torch.randint(0, n3d, (len(b),), generator=g)
    perm = torch.randperm(len(b), generator=g)
    return [t[perm].to(DEV) for t in (b, i, j)]


def fold_reference(dx, b_ids, j_ids, B, hc, wc, stride, hf, wf):
    """d feat_f of fine_preprocess's window rows: the window gradients dx [M, 25, 128] put at their
    (b, j) cell (index_put_ with accumulate) and folded back onto the map (F.fold, padding 2)."""
    dunf = torch.zeros(B, hc * wc, WIN, D, dtype=dx.dtype, device=dx.device)
    dunf.index_put_((b_ids, j_ids), dx, accumulate=True)
    return F.fold(dunf.permute(0, 3, 2, 1).reshape(B, D * WIN, hc * wc), (hf, wf), kernel_size=5, stride=stride,
                  padding=2)


@pytest.mark.parametrize("stride", [2, 4, 8])
def test_gather_exact_against_unfold(stride):
    """x[m·26 + t] = F.unfold's window row t of (b, j) and x[m·26 + 25] = descriptors3d_db[b, :, i],
    written into xm[:, :128] (row stride 256) with xm[:, 128:] untouched."""
    g = torch.Generator().manual_seed(10 + stride)
    B, hc, wc, n3d = 3, 5, 7, 30
    hf, wf = hc * stride, wc * stride
    feat = torch.randn(B, D, hf, wf, generator=g).to(DEV)
    desc = torch.randn(B, D, n3d, generator=g).to(DEV)
    b, i, j = _ids(B, hc, wc, n3d, 40, g)
    M = len(b)
    buf, x = _framed(M * TOK, D, ld=2 * D)
    ops.fine_train_gather(feat, desc, b, i, j, hc, wc, stride, x)
    _assert_framed(buf, M * TOK, D, "gather")
    data = {"b_ids": b, "i_ids": i, "j_ids": j, "q_hw_c": (hc, wc), "q_hw_f": (hf, wf)}
    f3d, f2d = train_path.fine_preprocess(5, D, data, desc.double(), feat.double())
    ref = torch.cat([f2d, f3d.transpose(1, 2)], 1).reshape(M * TOK, D)
    assert torch.equal(x.double(), ref)


@pytest.mark.parametrize("stride", [2, 4, 8])
def test_gather_backward_exact_against_fold(stride):
    """d feat_f from integer window gradients (every sum exact), with one cell holding 50 matches
    and the column index built by ops.gt_index as FineStage.backward builds it; dx is read from a
    row stride of 256 whose other columns are NaN.  At stride 8 the pixels no window covers are 0."""
    g = torch.Generator().manual_seed(20 + stride)
    B, hc, wc = 3, 5, 7
    hf, wf = hc * stride, wc * stride
    b, _, j = _ids(B, hc, wc, 1, 40, g, crowd=50)
    M = len(b)
    dxv = torch.randint(-4, 5, (M, TOK, D), generator=g).float().to(DEV)
    dx = _placed(dxv.reshape(M * TOK, D), 2 * D)
    cells = (b * (hc * wc) + j).contiguous()
    _, col_ptr, col_rows = ops.gt_index(torch.zeros_like(b), torch.arange(M, device=DEV), cells, (1, M, B * hc * wc))
    dfeat = torch.full((B, D, hf, wf), float("nan"), device=DEV)
    ops.fine_train_gather_bwd(dx, col_ptr, col_rows, hc, wc, stride, dfeat)
    ref = fold_reference(dxv[:, :WIN].double(), b, j, B, hc, wc, stride, hf, wf)
    assert not torch.isnan(dfeat).any()
    assert torch.equal(dfeat.double(), ref)
    crowd = dfeat[B - 1, :, (hc // 2) * stride, (wc // 2) * stride]
    assert crowd.abs().sum() > 0
    if stride == 8:
        covered = torch.zeros(hf, wf, dtype=torch.bool)
        for cy in range(hc):
            for cx in range(wc):
                covered[max(0, cy * 8 - 2):cy * 8 + 3, max(0, cx * 8 - 2):cx * 8 + 3] = True
        assert (~covered).any()
        assert bool((dfeat[:, :, ~covered.to(DEV)] == 0).all())


# ------------------------------------------------------------------------------------------------
# Token-row GEMM
# ------------------------------------------------------------------------------------------------
def _relu_backward(grad, out):
    """ReLU's backward by autograd at the ReLU output `out` (passes grad where out > 0)."""
    h = out.detach().double().requires_grad_(True)
    (d,) = torch.autograd.grad(F.relu(h), h, grad)
    return d


def _linear_case(rows, n, k, trans_w, epi, aux_on, aux2_on, exact, seed):
    """Runs one fine_train_linear call laid out as the stage lays it out (the qkv forward reads
    xm[:, :128] with row stride 256, the dx call reads aux = dxm[:, :128] with row stride 256) and
    returns (out buffer, out fp64, reference fp64, bound or None)."""
    g = _gen(seed)
    draw = (lambda s: _grid16(s, g)) if exact else (lambda s: _randn(s, g, 0.5))
    a = _placed(draw((rows, k)), 256 if (trans_w and n == 384) else k)
    w = draw((n, k) if trans_w else (k, n)).contiguous()
    aux = aux2 = None
    if epi == ops.EPI_MASK:
        r = F.relu(draw((rows, n)))
        r[::7, ::5] = -0.0                     # -0.0 is not > 0: masked
        aux = r
    elif epi == ops.EPI_ADD:
        if aux_on:
            aux = _placed(draw((rows, n)), n + 128)
        if aux2_on:
            aux2 = draw((rows, n))
    buf, out = _framed(rows, n, ld=n + 64)
    ops.fine_train_linear(a, w, trans_w, out, epi, aux=aux, aux2=aux2)
    a64, w64 = a.double(), w.double()
    wt = w64.T if trans_w else w64
    y = a64 @ wt
    mag = a64.abs() @ wt.abs()
    if epi == ops.EPI_RELU:
        y = F.relu(y)
    elif epi == ops.EPI_MASK:
        y = _relu_backward(y, aux)
    elif epi == ops.EPI_ADD:
        for t in (aux, aux2):
            if t is not None:
                y = y + t.double()
                mag = mag + t.double().abs()
    bound = None if exact else (k + 2) * U * mag
    return buf, out.double(), y, bound


@pytest.mark.parametrize("name,n,k", FWD_SHAPES)
@pytest.mark.parametrize("epi", [ops.EPI_STORE, ops.EPI_RELU])
def test_linear_forward(name, n, k, epi):
    worst = 0.0
    for rows in ROWS:
        buf, out, ref, _ = _linear_case(rows, n, k, True, epi, False, False, True, rows)
        _assert_framed(buf, rows, n, f"{name} rows={rows}")
        assert torch.equal(out, ref), (name, rows)
        _, out, ref, tol = _linear_case(rows, n, k, True, epi, False, False, False, rows + 1)
        err = (out - ref).abs()
        assert bool((err <= tol).all()), (name, rows, _ratio(err, tol))
        worst = max(worst, _ratio(err, tol))
    _report(f"linear {name} trans_w epi={epi}", worst)


BWD_EPIS = [(ops.EPI_STORE, False, False), (ops.EPI_MASK, True, False), (ops.EPI_ADD, True, True),
            (ops.EPI_ADD, True, False), (ops.EPI_ADD, False, True), (ops.EPI_ADD, False, False)]


@pytest.mark.parametrize("name,n,k", BWD_SHAPES)
@pytest.mark.parametrize("epi,aux_on,aux2_on", BWD_EPIS)
def test_linear_data_gradient(name, n, k, epi, aux_on, aux2_on):
    worst = 0.0
    for rows in ROWS:
        buf, out, ref, _ = _linear_case(rows, n, k, False, epi, aux_on, aux2_on, True, rows)
        _assert_framed(buf, rows, n, f"{name} rows={rows}")
        assert torch.equal(out, ref), (name, rows)
        _, out, ref, tol = _linear_case(rows, n, k, False, epi, aux_on, aux2_on, False, rows + 1)
        err = (out - ref).abs()
        assert bool((err <= tol).all()), (name, rows, _ratio(err, tol))
        worst = max(worst, _ratio(err, tol))
    _report(f"linear {name} epi={epi} aux={aux_on} aux2={aux2_on}", worst)


def test_linear_mask_zero_is_masked():
    """EPI_MASK passes the gradient where aux > 0 only: aux = +0.0 and -0.0 give exactly 0."""
    rows, n, k = 64, 256, 128
    g = _gen(5)
    a, w = _grid16((rows, k), g), _grid16((k, n), g)
    aux = torch.zeros(rows, n, device=DEV)
    aux[1::2] = -0.0
    aux[:, ::3] = 0.5
    out = torch.full((rows, n), float("nan"), device=DEV)
    ops.fine_train_linear(a, w, False, out, ops.EPI_MASK, aux=aux)
    y = a.double() @ w.double()
    assert bool((y[:, 1::3] != 0).any())
    assert bool((out[:, 1::3] == 0).all()) and bool((out[:, 2::3] == 0).all())
    assert torch.equal(out.double(), _relu_backward(y, aux))


def test_linear_host_rejections():
    """Shapes and layouts the kernel is not built for raise RuntimeError before any launch: the
    output keeps its poison."""
    rows = 64
    a = torch.ones(rows, 128, device=DEV)
    w = torch.ones(128, 128, device=DEV)
    out = torch.full((rows, 128), float("nan"), device=DEV)
    cases = [
        (a, torch.ones(96, 128, device=DEV), True, out[:, :96], ops.EPI_STORE, None, "shape"),   # n = 96
        (a[:, :120], torch.ones(128, 120, device=DEV), True, out, ops.EPI_STORE, None, "shape"),  # k = 120
        (a, w, False, out, ops.EPI_RELU, None, "not built"),                                      # RELU, trans_w 0
        (a, w, True, out, ops.EPI_MASK, None, "not built|aux"),                                   # MASK, trans_w 1
        (a, w, False, out, ops.EPI_MASK, None, "aux"),                                            # MASK without aux
        (torch.ones(rows, 130, device=DEV)[:, :128], w, True, out, ops.EPI_STORE, None, "misaligned"),  # lda 130
        (torch.ones(rows, 132, device=DEV)[:, 1:129], w, True, out, ops.EPI_STORE, None, "misaligned"),  # base + 4 B
    ]
    for a_, w_, tw, o, epi, aux, match in cases:
        with pytest.raises(RuntimeError, match=match):
            ops.fine_train_linear(a_, w_, tw, o, epi, aux=aux)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out).all())


# ------------------------------------------------------------------------------------------------
# Weight gradient
# ------------------------------------------------------------------------------------------------
WGRAD_ROWS = (26, 255, 256, 257, 2990, 4992)


def _wgrad(gm, am, n, k, dw0, accumulate):
    groups = ops.fine_train_groups(gm.shape[0])
    assert groups == -(-gm.shape[0] // 256)
    part = torch.full((groups * n * k,), float("nan"), device=DEV)
    dw = dw0.clone()
    ops.fine_train_wgrad(gm, am, part, dw, accumulate)
    return dw


@pytest.mark.parametrize("name,n,k,lda", WGRAD_SHAPES)
@pytest.mark.parametrize("accumulate", [0, 1])
def test_wgrad(name, n, k, lda, accumulate):
    """dW (+)= G^T A over the token rows: exact on a 2^-4 grid; on random rows within
    (rows + groups + 2)·U·|G|^T|A| (one rounding per row of a group, per group in the ordered reduce
    and for the accumulate); accumulate = 1 onto a nonzero dW, accumulate = 0 over a NaN dW."""
    worst = 0.0
    for rows in WGRAD_ROWS:
        K = rows + ops.fine_train_groups(rows) + 2
        g = _gen(rows + 7 * accumulate)
        for exact in (True, False):
            draw = (lambda s: _grid16(s, g)) if exact else (lambda s: _randn(s, g))
            gm, am = draw((rows, n)), _placed(draw((rows, k)), lda)
            dw0 = draw((n, k)) if accumulate else torch.full((n, k), float("nan"), device=DEV)
            dw = _wgrad(gm, am, n, k, dw0, accumulate)
            ref = gm.double().T @ am.double()
            mag = gm.double().abs().T @ am.double().abs()
            if accumulate:
                ref, mag = ref + dw0.double(), mag + dw0.double().abs()
            if exact:
                assert torch.equal(dw.double(), ref), (name, rows)
            else:
                err, tol = (dw.double() - ref).abs(), K * U * mag
                assert bool((err <= tol).all()), (name, rows, _ratio(err, tol))
                worst = max(worst, _ratio(err, tol))
    _report(f"wgrad {name} accumulate={accumulate}", worst)


@pytest.mark.parametrize("rows", [300, 512, 4992])
def test_wgrad_group_edge_rows(rows):
    """Only rows 0, 255, 256 and rows - 1 are nonzero, each with its own power of two: dW tells
    which rows were summed, and how often.  rows - 1 ends a ragged group (300, 4992) or a full one
    (512)."""
    n, k = 128, 128
    gm = torch.zeros(rows, n, device=DEV)
    am = torch.zeros(rows, k, device=DEV)
    for idx, r in enumerate((0, 255, 256, rows - 1)):
        gm[r] = 2.0 ** idx
        am[r] = 1.0
    dw = _wgrad(gm, am, n, k, torch.full((n, k), float("nan"), device=DEV), 0)
    assert torch.equal(dw.double(), gm.double().T @ am.double())
    assert float(dw[0, 0]) == 15.0


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def _ln_inputs(rows, g):
    """Rows of N(0, 1) with gamma / beta of realistic size; row 0 and the last row constant
    (var = 0), every 5th row 1000 + N(0, 1) (the variance must not cancel)."""
    x = _randn((rows, D), g)
    x[0] = 3.25
    x[-1] = -0.75
    x[1:-1:5] += 1000.0
    gamma = 1.0 + 0.2 * _randn((D,), g)
    beta = 0.1 * _randn((D,), g)
    return x, gamma, beta


def _ln_fwd_bounds(x64, gamma64, beta64, resid64, y64):
    """Per-element bounds on y and per-row bounds on mean and rstd of the one-warp LayerNorm: the
    mean's sum runs through 8 roundings (4 channels per lane, then 5 shuffle levels), the variance's
    through 10, rsqrtf adds 2 ulp."""
    mean, var = x64.mean(1, keepdim=True), x64.var(1, unbiased=False, keepdim=True)
    rstd = 1 / torch.sqrt(var + 1e-5)
    e_mu = 9 * U * x64.abs().mean(1, keepdim=True)
    e_rs = rstd * (16 * U + e_mu ** 2 / (var + 1e-5))
    xh = (x64 - mean) * rstd
    tol_y = gamma64.abs() * (rstd * e_mu + xh.abs() * (e_rs / rstd + 4 * U)) + 2 * U * (beta64.abs() + y64.abs())
    if resid64 is not None:
        tol_y = tol_y + U * resid64.abs()
    return mean, rstd, e_mu, e_rs, tol_y


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("with_resid", [False, True])
def test_layer_norm_forward(rows, with_resid):
    """y = LayerNorm(x) (+ resid) with x, resid and y strided (row stride 256, as xm's halves);
    stats = (mean, rstd) against fp64."""
    g = _gen(rows + with_resid)
    x, gamma, beta = _ln_inputs(rows, g)
    xv = _placed(x, 2 * D)
    resid = _placed(_randn((rows, D), g), 2 * D) if with_resid else None
    buf, y = _framed(rows, D, ld=2 * D)
    stats = torch.full((rows, 2), float("nan"), device=DEV)
    ops.fine_train_ln(xv, gamma, beta, resid, y, stats)
    _assert_framed(buf, rows, D, "ln y")
    x64 = x.double()
    ref = F.layer_norm(x64, (D,), gamma.double(), beta.double(), 1e-5)
    r64 = resid.double() if with_resid else None
    if with_resid:
        ref = ref + r64
    mean, rstd, e_mu, e_rs, tol = _ln_fwd_bounds(x64, gamma.double(), beta.double(), r64, ref)
    assert not torch.isnan(stats).any()
    err_mu, err_rs, err_y = (stats[:, :1].double() - mean).abs(), (stats[:, 1:].double() - rstd).abs(), (y.double() - ref).abs()
    assert bool((err_mu <= e_mu).all()), _ratio(err_mu, e_mu)
    assert bool((err_rs <= e_rs).all()), _ratio(err_rs, e_rs)
    assert bool((err_y <= tol).all()), _ratio(err_y, tol)
    # the constant rows: y = beta (+ resid) exactly, mean exact
    const = [0, rows - 1]
    exp = beta.expand(2, D) + (resid[const] if with_resid else 0)
    assert torch.equal(y[const], exp)
    assert torch.equal(stats[const, 0], x[const, 0])
    _report(f"ln rows={rows} resid={with_resid}: mean {_ratio(err_mu, e_mu):.3g}, rstd {_ratio(err_rs, e_rs):.3g}, y",
            _ratio(err_y, tol))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("strided", [False, True])
def test_layer_norm_backward(rows, strided):
    """dx, dgamma and dbeta against fp64 autograd of F.layer_norm, from the kernel's own forward
    stats (as the stage runs it); dy on a 2^-4 grid, so dbeta (a sum of dy over the rows) is exact.
    accumulate 0 over NaN and 1 onto a nonzero [dgamma; dbeta]."""
    g = _gen(100 + rows + strided)
    x, gamma, beta = _ln_inputs(rows, g)
    dyv = _grid16((rows, D), g)
    ld = 2 * D if strided else D
    xv, dy = _placed(x, ld), _placed(dyv, ld)
    stats = torch.empty(rows, 2, device=DEV)
    ops.fine_train_ln(xv, gamma, beta, None, torch.empty(rows, D, device=DEV), stats)
    x64 = x.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    dy64 = dyv.double()
    rx, rg, rb = torch.autograd.grad(F.layer_norm(x64, (D,), g64, b64, 1e-5), [x64, g64, b64], dy64)
    x64 = x64.detach()
    # bounds: xh carries the stats' error (e_mu, e_rs); the two row means of dx run through 8
    # roundings, dgamma / dbeta through one per row
    mean, rstd, e_mu, e_rs, _ = _ln_fwd_bounds(x64, gamma.double(), beta.double(), None, x64)
    xh = (x64 - mean) * rstd
    e_xh = rstd * e_mu + xh.abs() * (e_rs / rstd + 2 * U)
    dxh = (dy64 * gamma.double()).abs()
    m2 = (dy64 * gamma.double() * xh).mean(1, keepdim=True).abs()
    tol_dx = (rstd * (12 * U * (dxh + dxh.mean(1, keepdim=True) + xh.abs() * (dxh * xh.abs()).mean(1, keepdim=True))
                      + m2 * e_xh + xh.abs() * (dxh * e_xh).mean(1, keepdim=True))
              + rx.abs() * (e_rs / rstd + 2 * U))
    tol_dg = (rows + 2) * U * (dy64 * xh).abs().sum(0) + (dy64.abs() * e_xh).sum(0)
    worst = [0.0, 0.0]
    for accumulate in (0, 1):
        dbuf, dx = _framed(rows, D, ld=ld)
        groups = ops.fine_train_groups(rows)
        part = torch.full((groups * 2 * D,), float("nan"), device=DEV)
        dgb0 = _grid16((2, D), g) if accumulate else torch.full((2, D), float("nan"), device=DEV)
        dgb = dgb0.clone()
        ops.fine_train_ln_bwd(xv, gamma, stats, dy, dx, part, dgb, accumulate)
        _assert_framed(dbuf, rows, D, "ln dx")
        base = dgb0.double() if accumulate else torch.zeros(2, D, dtype=torch.float64, device=DEV)
        assert torch.equal(dgb[1].double(), base[1] + rb), ("dbeta", accumulate)
        err_dx, err_dg = (dx.double() - rx).abs(), (dgb[0].double() - base[0] - rg).abs()
        tdg = tol_dg + U * (base[0] + rg).abs()
        assert bool((err_dx <= tol_dx).all()), ("dx", accumulate, _ratio(err_dx, tol_dx))
        assert bool((err_dg <= tdg).all()), ("dgamma", accumulate, _ratio(err_dg, tdg))
        worst = [max(worst[0], _ratio(err_dx, tol_dx)), max(worst[1], _ratio(err_dg, tdg))]
    _report(f"ln_bwd rows={rows} strided={strided}: dx {worst[0]:.3g}, dgamma", worst[1])


# ------------------------------------------------------------------------------------------------
# Linear attention
# ------------------------------------------------------------------------------------------------
def _heads(t):
    return t.reshape(*t.shape[:-1], 8, 16)


def attention_reference(qkv, cross, eps=1e-6):
    """The attention messages of one fine layer on the 26-row layout: qkv [m, 26, 384] rows
    [q | k | v], window tokens 0..24, 3D token 25.  Self: each sequence attends to itself; cross:
    the window to the 3D token and the 3D token to the window (train_path.transformer's calls of
    train_path._linear_attention).  Returns [m, 26, 128]."""
    q, k, v = _heads(qkv[..., :D]), _heads(qkv[..., D:2 * D]), _heads(qkv[..., 2 * D:])
    win, d3 = slice(0, WIN), slice(WIN, TOK)
    src_win, src_3d = (d3, win) if cross else (win, d3)
    out_win = train_path._linear_attention(q[:, win], k[:, src_win], v[:, src_win], eps=eps)
    out_3d = train_path._linear_attention(q[:, d3], k[:, src_3d], v[:, src_3d], eps=eps)
    return torch.cat([out_win, out_3d], 1).reshape(qkv.shape[0], TOK, D)


def _attention_bounds(qkv, dout, cross, eps=1e-6):
    """fp32 rounding bounds of the attention forward and backward: K·U times the same sums taken
    over absolute values (every ELU+1 feature, ksum and Z is positive), K = the roundings along the
    longest chain (16-channel dots, up to 25 source rows, up to 25 query rows, ELU and divisions)."""
    m = qkv.shape[0]
    Qf, Kf = F.elu(_heads(qkv[..., :D])) + 1, F.elu(_heads(qkv[..., D:2 * D])) + 1
    V, G = _heads(qkv[..., 2 * D:]).abs(), _heads(dout).abs()
    out_b = torch.zeros(m, TOK, 8, 16, dtype=qkv.dtype, device=qkv.device)
    dq_b, dk_b, dv_b = torch.zeros_like(out_b), torch.zeros_like(out_b), torch.zeros_like(out_b)
    win, d3 = slice(0, WIN), slice(WIN, TOK)
    for ql, sl in ((win, d3 if cross else win), (d3, win if cross else d3)):
        qf, kf, vs, gl = Qf[:, ql], Kf[:, sl], V[:, sl] / Kf[:, sl].shape[1], G[:, ql]
        n = kf.shape[1]
        kv = torch.einsum("nshd,nshv->nhdv", kf, vs)
        ks = kf.sum(1)
        z = 1 / (torch.einsum("nlhd,nhd->nlh", qf, ks) + eps)
        a = torch.einsum("nlhd,nhdv->nlhv", qf, kv)
        out_b[:, ql] = a * z[..., None] * n
        da = n * z[..., None] * gl
        dden = z ** 2 * n * (gl * a).sum(-1)
        dqf = torch.einsum("nhdv,nlhv->nlhd", kv, da) + dden[..., None] * ks[:, None]
        dkv = torch.einsum("nlhd,nlhv->nhdv", qf, da)
        dks = torch.einsum("nlh,nlhd->nhd", dden, qf)
        dkf = torch.einsum("nhdv,nshv->nshd", dkv, vs) + dks[:, None]
        dv_b[:, sl] = torch.einsum("nshd,nhdv->nshv", kf, dkv) / n
        dq_b[:, ql] = dqf * torch.where(qkv[..., :D].reshape(m, TOK, 8, 16)[:, ql] > 0, 1.0, qf)
        dk_b[:, sl] = dkf * torch.where(qkv[..., D:2 * D].reshape(m, TOK, 8, 16)[:, sl] > 0, 1.0, kf)
    k_fwd = 2 * WIN + 48              # KV and ksum over the sources, two 16-channel dots, Z, ELU+1
    k_bwd = 4 * WIN + 112             # dden carries Z twice and A once, then the sums over queries
    rows = [t.reshape(m, TOK, D) for t in (out_b, dq_b, dk_b, dv_b)]
    return k_fwd * U * rows[0], k_bwd * U * torch.cat(rows[1:], -1)


def _attention_inputs(m, g):
    """q, k, v of N(0, 1), with entries exactly 0 and +-1e-8 scattered, and in every match one head
    whose q are about -20, one whose k are about -20 and one with both (ELU+1 underflows toward 0, Z
    grows large)."""
    qkv = _randn((m, TOK, 3 * D), g)
    pick = torch.rand((m, TOK, 2 * D), generator=g, device=DEV)
    qk = qkv[..., :2 * D]
    qk[pick < 0.05] = 0.0
    qk[(pick >= 0.05) & (pick < 0.08)] = 1e-8
    qk[(pick >= 0.08) & (pick < 0.11)] = -1e-8
    low = -20.0 + 0.5 * _randn((m, TOK, 16), g)
    qkv[..., 0:16] = low                            # head 0: q
    qkv[..., D + 16:D + 32] = low                   # head 1: k
    qkv[..., 32:48] = low                           # head 2: q and k
    qkv[..., D + 32:D + 48] = low
    return qkv


@pytest.mark.parametrize("m", [1, 193])
@pytest.mark.parametrize("cross", [0, 1])
def test_attention_forward_and_backward(m, cross):
    """fine_train_attention / _bwd against fp64 autograd of train_path._linear_attention on the
    25 + 1 token split; out and dqkv start as NaN, so every row and column must be written."""
    g = _gen(300 + m + cross)
    qkv = _attention_inputs(m, g)
    dout = _randn((m, TOK, D), g)
    out = torch.full((m * TOK, D), float("nan"), device=DEV)
    dqkv = torch.full((m * TOK, 3 * D), float("nan"), device=DEV)
    q2 = qkv.reshape(m * TOK, 3 * D)
    ops.fine_train_attention(q2, out, m, cross)
    ops.fine_train_attention_bwd(q2, dout.reshape(m * TOK, D), dqkv, m, cross)
    q64 = qkv.double().requires_grad_(True)
    ref = attention_reference(q64, cross)
    (dref,) = torch.autograd.grad(ref, q64, dout.double())
    tol_out, tol_d = _attention_bounds(qkv.double(), dout.double(), cross)
    assert not torch.isnan(out).any() and not torch.isnan(dqkv).any()
    err_o = (out.double().reshape(m, TOK, D) - ref.detach()).abs()
    err_d = (dqkv.double().reshape(m, TOK, 3 * D) - dref).abs()
    assert bool((err_o <= tol_out).all()), _ratio(err_o, tol_out)
    assert bool((err_d <= tol_d).all()), _ratio(err_d, tol_d)
    _report(f"attention m={m} cross={cross}: out {_ratio(err_o, tol_out):.3g}, dqkv", _ratio(err_d, tol_d))


# ------------------------------------------------------------------------------------------------
# Heatmap expectation
# ------------------------------------------------------------------------------------------------
def _match_inputs(m, g):
    """x [m, 26, 128]: f0 = row 25, window rows 0..24.  Matches cycle through: random rows (sim of
    order 1), a uniform heatmap (window rows 0), a one-hot heatmap (the clamp of var is active),
    saturated correlations of +-80 with one top (one-hot) and with two tops (a split heatmap)."""
    x = _randn((m, TOK, D), g)
    f0 = x[:, WIN]
    unit = f0 / (f0 * f0).sum(-1, keepdim=True) * D ** 0.5       # f0 . unit / sqrt(128) = 1
    for idx in range(m):
        kind = idx % 5
        if kind == 1:
            x[idx, :WIN] = 0.0
        elif kind == 2:
            x[idx, 7] = 40.0 * f0[idx]
        elif kind in (3, 4):
            sims = torch.full((WIN,), -80.0, device=DEV) + _randn((WIN,), g)
            sims[3] = 80.0
            if kind == 4:
                sims[16] = 80.0
            x[idx, :WIN] = sims[:, None] * unit[idx] + 1e-3 * _randn((WIN, D), g)
    return x


def _match_reference(x64, w64):
    """train_path.fine_matching with autograd in fp64: expec_f and d(sum(expec_f * w)) / dx."""
    m = x64.shape[0]
    xr = x64.clone().requires_grad_(True)
    data = {"q_hw_i": (64, 64), "q_hw_f": (32, 32), "mkpts_query_c": torch.zeros(m, 2, dtype=x64.dtype, device=DEV),
            "b_ids": torch.zeros(m, dtype=torch.long, device=DEV)}
    with mtf.default_dtype(torch.float64):
        train_path.fine_matching(xr[:, WIN:], xr[:, :WIN], data, True)
    (dx,) = torch.autograd.grad(data["expec_f"], xr, w64)
    return data["expec_f"].detach(), dx


def _match_bounds(x64, w64):
    """First-order fp32 bounds of the expectation and its backward.  The 25 correlations are
    128-term dot products (8 roundings per lane, 5 shuffle levels: e_r = 16·U·sum |f0||v_r| /
    sqrt(128)); a softmax probability then moves by p_r (e_r + sum_s p_s e_s + 64 U), or by 2^-126
    where fp32 exp underflows to 0; the expectation, the variance and the backward's sums add their
    own roundings."""
    f0, v = x64[:, WIN], x64[:, :WIN]
    sims = torch.einsum("mc,mrc->mr", f0, v) / D ** 0.5
    p = torch.softmax(sims, 1)
    e = 16 * U * torch.einsum("mc,mrc->mr", f0.abs(), v.abs()) / D ** 0.5
    e = e + U * (sims.max(1, keepdim=True).values - sims)                     # sim - max rounded
    dp = p * (e + (p * e).sum(1, keepdim=True) + 64 * U) + 2.0 ** -126
    lin = torch.linspace(-1, 1, 5, dtype=x64.dtype, device=DEV)
    grid = torch.stack([lin.repeat(5), lin.repeat_interleave(5)], 1)          # [25, 2]
    c = p @ grid
    tol_c = dp @ grid.abs() + 32 * U * (p @ grid.abs())
    var = p @ grid ** 2 - c ** 2
    dvar = dp @ grid ** 2 + 2 * c.abs() * tol_c + 32 * U * (p @ grid ** 2 + c ** 2)
    vc = var.clamp_min(1e-10)
    tol_std = (torch.minimum(dvar.sqrt(), dvar / vc.sqrt()) + 4 * U * vc.sqrt()).sum(1)
    # backward, from d expec = w = (gx, gy, gs)
    gxy, gs = w64[:, :2], w64[:, 2:]
    dv = torch.where(var >= 1e-10, gs / (2 * vc.sqrt()), torch.zeros_like(var))
    ddv = dv.abs() * (dvar / (2 * vc) + 4 * U)
    dc = gxy - 2 * c * dv
    ddc = 2 * c.abs() * ddv + 2 * dv.abs() * tol_c + 4 * U * (gxy.abs() + 2 * (c * dv).abs())
    dh = dc @ grid.T + dv @ (grid ** 2).T                                     # [m, 25]
    dh_mag = dc.abs() @ grid.abs().T + dv.abs() @ (grid ** 2).T
    ddh = ddc @ grid.abs().T + ddv @ (grid ** 2).T + 8 * U * dh_mag
    dot = (p * dh).sum(1, keepdim=True)
    ddot = (dp * dh.abs() + p * ddh).sum(1, keepdim=True) + 32 * U * (p * dh_mag).sum(1, keepdim=True)
    ds = p * (dh - dot) / D ** 0.5
    dds = (dp * (dh - dot).abs() + p * (ddh + ddot) + 8 * U * p * (dh_mag + dot.abs())) / D ** 0.5
    tol_rows = dds[..., None] * f0.abs()[:, None] + U * (ds[..., None] * f0[:, None]).abs()
    tol_f0 = torch.einsum("mr,mrc->mc", dds, v.abs()) + 32 * U * torch.einsum("mr,mrc->mc", ds.abs(), v.abs())
    return torch.cat([tol_c, tol_std[:, None]], 1), torch.cat([tol_rows, tol_f0[:, None]], 1)


@pytest.mark.parametrize("m", [1, 5, 115])
def test_match_forward_and_backward(m):
    """fine_train_match / _bwd against fp64 autograd of train_path.fine_matching, with a nonzero
    gradient on every column (std included); m is not a multiple of the 4 matches per CTA."""
    g = _gen(400 + m)
    x = _match_inputs(m, g)
    w = _randn((m, 3), g)
    xd = x.reshape(m * TOK, D)
    expec = torch.full((m, 3), float("nan"), device=DEV)
    dx = torch.full((m * TOK, D), float("nan"), device=DEV)
    ops.fine_train_match(xd, m, expec)
    ops.fine_train_match_bwd(xd, w, m, dx)
    ref, dref = _match_reference(x.double(), w.double())
    tol_e, tol_dx = _match_bounds(x.double(), w.double())
    assert not torch.isnan(expec).any() and not torch.isnan(dx).any()
    err_e = (expec.double() - ref).abs()
    err_d = (dx.double().reshape(m, TOK, D) - dref).abs()
    assert bool((err_e <= tol_e).all()), _ratio(err_e, tol_e)
    assert bool((err_d <= tol_dx).all()), _ratio(err_d, tol_dx)
    if m >= 5:
        assert float(ref[2, 2]) == pytest.approx(2e-5)                        # one-hot: the clamp is active
        assert float(ref[3, 2]) == pytest.approx(2e-5)
        assert float(ref[4, 2]) > 0.5                                         # two saturated tops
    _report(f"match m={m}: expec {_ratio(err_e, tol_e):.3g}, dx", _ratio(err_d, tol_dx))


# ------------------------------------------------------------------------------------------------
# FineStage across chunk boundaries
# ------------------------------------------------------------------------------------------------
def _case(M, seed):
    """mtf.make_case's case (corner cells first, repeated cells) cut to M matches."""
    case = mtf.make_case(seed, B=2, hc=4, wc=5, stride=4, n3d=24, M=max(M, 11))
    for k in ("b_ids", "i_ids", "j_ids", "expec_f_gt"):
        case[k] = case[k][:M]
    return case


@pytest.mark.parametrize("M", [1, 191, 192, 193, 385])
def test_fine_stage_chunks_against_fp64(M):
    """FineStage at one match, around one chunk (192) and past two, against the fp64 train_path
    run: the fp64-distance rule of test_train_fine_gpu, with a gradient on the std column."""
    from tests.test_train_fine_gpu import _assert_fp64_distance, _runs
    case = _case(M, 30 + M)
    w = torch.randn(M, 3, generator=torch.Generator().manual_seed(M), dtype=torch.float64)
    report = []
    _assert_fp64_distance(*_runs(case, w), report)
    print(f"M={M}:\n" + "\n".join(report))


def test_fine_stage_without_matches():
    """M = 0: expec_f is empty, d feat_f is zero and every parameter gradient is zero."""
    case = _case(0, 1)
    fine = mtf.fine_module(workload.synthetic_state_dict(0), torch.float32, DEV)
    feat = case["feat_f"].to(DEV, torch.float32).requires_grad_(True)
    desc = case["desc3d"].to(DEV, torch.float32).contiguous()
    ids = [case[k].to(DEV) for k in ("b_ids", "i_ids", "j_ids")]
    params = [p for layer in fine.layers for p in train_fine.layer_params(layer)]
    expec = train_fine.FineStage.apply(feat, desc, *ids, (4, 5, 4), *params)
    assert expec.shape == (0, 3)
    grads = torch.autograd.grad(expec.sum(), [feat] + params)
    assert all(bool((t == 0).all()) for t in grads)
    assert grads[0].shape == feat.shape
