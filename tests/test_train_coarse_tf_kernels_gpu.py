"""Each opp_coarse_tf_* kernel on its own against fp64 PyTorch (oracle/coarse_tf.py, itself checked
against autograd on the CPU), at the coarse transformer's launch shapes and edges:
  - exact cases: inputs on a 2^-4 grid with k > 0 and power-of-two lengths, so every fp32 sum is exact
    and the kernel must equal fp64 bit for bit (the state, the source pass, dbeta);
  - random cases within bounds derived from fp32 rounding of the same sums (c * 2^-24 * sum |terms|,
    computed in fp64);
  - NaN-poisoned outputs, and strided row views framed by a sentinel that must stay untouched;
  - rows per batch element around the chunk (1, 127, 128, 129, 7000), B = 1 and 4, no mask and
    all-ones, partial and all-zero masks;
  - LayerNorm over 256 channels at the stage's row counts."""
import pytest
import torch

from oracle import coarse_tf
from onepose_plus_plus_b200 import ops

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
SENTINEL = 12345.0
H, DH, D = 8, 32, 256


def _rows(rows, cols, g, grid=False, positive=False, lo=-3.0, hi=3.0):
    if grid:
        t = torch.randint(0 if positive else -32, 33, (rows, cols), generator=g).double() / 16
        if positive:
            t = t + 1 / 16
    else:
        t = torch.rand(rows, cols, generator=g, dtype=torch.float64) * (hi - lo) + lo
    return t.float().double()                                           # what the kernels read


def _framed(t, extra=32):
    """A CUDA fp32 row view of t with row stride cols + extra; the frame holds SENTINEL."""
    rows, cols = t.shape
    buf = torch.full((rows, cols + extra), SENTINEL, dtype=torch.float32, device="cuda")
    buf[:, :cols] = t.float().cuda()
    return buf, buf[:, :cols]


def _mask(B, n, kind):
    if kind == "none":
        return None
    m = torch.ones(B, n, dtype=torch.uint8)
    if kind == "partial":
        m[:, n - n // 3:] = 0
        m[0, ::3] = 0
    if kind == "zero":
        m.zero_()
    return m


def _heads(t, B, n):
    """[B*n, 256] -> [B, n, 8, 32]."""
    return t.reshape(B, n, H, DH)


def _fm(m):
    return None if m is None else m.double()


LENS = [1, 127, 128, 129, 7000]
MASKS = ["none", "ones", "partial", "zero"]


def _qkv(B, n, g, grid=False):
    q = _rows(B * n, D, g, grid)
    k = _rows(B * n, D, g, grid, positive=grid)
    v = _rows(B * n, D, g, grid)
    return torch.cat([q, k, v], 1)


def _state(qkv, mask, B, n):
    buf, view = _framed(qkv)
    mk = None if mask is None else mask.reshape(-1).cuda()
    part = ops.coarse_tf_part(B, n, "cuda")
    kv = torch.full((B, H, DH, DH), float("nan"), device="cuda")
    ks = torch.full((B, H, DH), float("nan"), device="cuda")
    ops.coarse_tf_kv(view, mk, B, part, kv, ks)
    assert bool((buf[:, 3 * D:] == SENTINEL).all())
    return kv, ks


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("n", LENS)
@pytest.mark.parametrize("kind", MASKS)
def test_kv_state(B, n, kind):
    g = torch.Generator().manual_seed(n * 10 + B)
    qkv = _qkv(B, n, g)
    mask = _mask(B, n, kind)
    kv, ks = _state(qkv, mask, B, n)
    k, v = _heads(qkv[:, D:2 * D], B, n), _heads(qkv[:, 2 * D:], B, n)
    rkv, rks = coarse_tf.state(k, v, _fm(mask))
    m = torch.ones(B, n, 1, 1, dtype=torch.float64) if mask is None else mask.double()[:, :, None, None]
    K = torch.where(k > 0, k + 1, k.clamp(max=0).exp()) * m
    terms = torch.einsum("nshd,nshv->nhdv", K.abs(), (v * m / n).abs())
    c = n // 128 + 128 + 8
    assert ((kv.double().cpu() - rkv).abs() <= c * U * terms + 1e-30).all()
    assert ((ks.double().cpu() - rks).abs() <= c * U * K.abs().sum(1) + 1e-30).all()
    if kind == "zero":
        assert float(kv.abs().max()) == 0 and float(ks.abs().max()) == 0


@pytest.mark.parametrize("B,n", [(1, 1), (4, 128), (2, 512), (3, 1024)])
def test_kv_state_exact_on_grid(B, n):
    g = torch.Generator().manual_seed(n + B)
    qkv = _qkv(B, n, g, grid=True)
    mask = _mask(B, n, "partial")
    kv, ks = _state(qkv, mask, B, n)
    rkv, rks = coarse_tf.state(_heads(qkv[:, D:2 * D], B, n), _heads(qkv[:, 2 * D:], B, n), _fm(mask))
    assert torch.equal(kv.double().cpu(), rkv) and torch.equal(ks.double().cpu(), rks)


def _attn_inputs(B, L, S, g, kind):
    q = _rows(B * L, D, g)
    KV = torch.randn(B, H, DH, DH, generator=g, dtype=torch.float64).float().double()
    ksum = (torch.rand(B, H, DH, generator=g, dtype=torch.float64) * S).float().double()
    if kind == "zero":
        KV.zero_(), ksum.zero_()
    return q, KV, ksum


def _attn_ref(q, KV, ksum, S, mask, B, L):
    qh = _heads(q, B, L)
    m = torch.ones(B, L, 1, 1, dtype=torch.float64) if mask is None else mask.double()[:, :, None, None]
    Q = torch.where(qh > 0, qh + 1, qh.clamp(max=0).exp()) * m
    A = torch.einsum("nlhd,nhdv->nlhv", Q, KV)
    Aabs = torch.einsum("nlhd,nhdv->nlhv", Q.abs(), KV.abs())
    den = torch.einsum("nlhd,nhd->nlh", Q, ksum) + 1e-6
    Z = 1 / den
    return Q, A, Aabs, Z


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("L", LENS)
@pytest.mark.parametrize("kind", MASKS)
def test_attn(B, L, kind):
    g = torch.Generator().manual_seed(L * 7 + B)
    S = 301
    q, KV, ksum = _attn_inputs(B, L, S, g, kind)
    mask = _mask(B, L, kind)
    qkv = torch.cat([q, torch.zeros(B * L, 2 * D, dtype=torch.float64)], 1)
    _, qv = _framed(qkv)
    obuf, out = _framed(torch.full((B * L, D), float("nan")))
    ops.coarse_tf_attn(qv, None if mask is None else mask.reshape(-1).cuda(), B, KV.float().cuda(),
                       ksum.float().cuda(), S, out)
    assert bool((obuf[:, D:] == SENTINEL).all())
    Q, A, Aabs, Z = _attn_ref(q, KV, ksum, S, mask, B, L)
    ref = (A * Z[..., None] * S).reshape(B * L, D)
    bound = (40 * U * (Aabs * Z[..., None].abs() * S)).reshape(B * L, D) + \
        (ref.abs() * (40 * U * torch.einsum("nlhd,nhd->nlh", Q.abs(), ksum.abs()) * Z.abs() + 8 * U)[..., None]
         .expand(B, L, H, DH).reshape(B * L, D))
    err = (out.double().cpu() - ref).abs()
    assert bool(torch.isfinite(out).all())
    assert bool((err <= bound + 1e-30).all()), float((err / (bound + 1e-30)).max())
    if kind == "zero":
        assert float(out.abs().max()) == 0


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("L", LENS)
@pytest.mark.parametrize("kind", MASKS)
def test_attn_bwd_q(B, L, kind):
    g = torch.Generator().manual_seed(L * 11 + B)
    S = 301
    q, KV, ksum = _attn_inputs(B, L, S, g, kind)
    dout = _rows(B * L, D, g)
    mask = _mask(B, L, kind)
    qkv = torch.cat([q, torch.full((B * L, 2 * D), float("nan"), dtype=torch.float64)], 1)
    _, qv = _framed(qkv)
    _, dv = _framed(dout)
    dbuf, dqkv = _framed(torch.full((B * L, 3 * D), float("nan")))
    dkv = torch.full((B, H, DH, DH), float("nan"), device="cuda")
    dks = torch.full((B, H, DH), float("nan"), device="cuda")
    ops.coarse_tf_attn_bwd_q(qv, None if mask is None else mask.reshape(-1).cuda(), B, KV.float().cuda(),
                             ksum.float().cuda(), S, dv, dqkv, ops.coarse_tf_part(B, L, "cuda"), dkv, dks)
    assert bool((dbuf[:, 3 * D:] == SENTINEL).all())
    assert bool(torch.isnan(dqkv[:, D:]).all())                       # k / v columns untouched
    rq, rdkv, rdks = coarse_tf.backward_q(_heads(q, B, L), KV, ksum, S, _heads(dout, B, L), _fm(mask))
    Q, A, Aabs, Z = _attn_ref(q, KV, ksum, S, mask, B, L)
    gh = _heads(dout, B, L)
    cond = 1 + torch.einsum("nlhd,nhd->nlh", Q.abs(), ksum.abs()) * Z.abs()          # relative error of Z / U
    dU_abs = gh.abs() * Z.abs()[..., None] * S
    dden_abs = S * Z ** 2 * (gh.abs() * Aabs).sum(-1)
    dq_abs = torch.einsum("nhdv,nlhv->nlhd", KV.abs(), dU_abs) + ksum.abs()[:, None] * dden_abs[..., None]
    bound_q = (80 * U * dq_abs * cond[..., None]).reshape(B * L, D)                # elu' <= 1
    err = (dqkv[:, :D].double().cpu() - rq.reshape(B * L, D)).abs()
    assert bool((err <= bound_q + 1e-30).all()), float((err / (bound_q + 1e-30)).max())
    c = 80 + L // 128 + 128
    bkv = c * U * torch.einsum("nlhd,nlhv->nhdv", Q.abs(), dU_abs * cond[..., None])
    bks = c * U * torch.einsum("nlhd,nlh->nhd", Q.abs(), dden_abs * cond)
    assert bool(((dkv.double().cpu() - rdkv).abs() <= bkv + 1e-30).all())
    assert bool(((dks.double().cpu() - rdks).abs() <= bks + 1e-30).all())


def _bwd_kv(qkv, mask, B, n, dKV, dks):
    _, qv = _framed(qkv)
    dbuf, dqkv = _framed(torch.full((B * n, 3 * D), float("nan")))
    ops.coarse_tf_attn_bwd_kv(qv, None if mask is None else mask.reshape(-1).cuda(), B, dKV.float().cuda(),
                              dks.float().cuda(), dqkv)
    assert bool((dbuf[:, 3 * D:] == SENTINEL).all())
    assert bool(torch.isnan(dqkv[:, :D]).all())                       # q columns untouched
    return dqkv


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("n", LENS)
@pytest.mark.parametrize("kind", MASKS)
def test_attn_bwd_kv(B, n, kind):
    g = torch.Generator().manual_seed(n * 13 + B)
    qkv = _qkv(B, n, g)
    dKV = torch.randn(B, H, DH, DH, generator=g, dtype=torch.float64).float().double()
    dks = torch.randn(B, H, DH, generator=g, dtype=torch.float64).float().double()
    mask = _mask(B, n, kind)
    dqkv = _bwd_kv(qkv, mask, B, n, dKV, dks)
    k, v = _heads(qkv[:, D:2 * D], B, n), _heads(qkv[:, 2 * D:], B, n)
    rk, rv = coarse_tf.backward_kv(k, v, dKV, dks, _fm(mask))
    K = torch.where(k > 0, k + 1, k.clamp(max=0).exp())
    ep = torch.where(k > 0, torch.ones_like(k), K)
    bk = 40 * U * (torch.einsum("nhdv,nshv->nshd", dKV.abs(), v.abs()) / n + dks.abs()[:, None]) * ep
    bv = 40 * U * torch.einsum("nhdv,nshd->nshv", dKV.abs(), K.abs()) / n
    ek = (dqkv[:, D:2 * D].double().cpu() - rk.reshape(B * n, D)).abs()
    ev = (dqkv[:, 2 * D:].double().cpu() - rv.reshape(B * n, D)).abs()
    assert bool((ek <= bk.reshape(B * n, D) + 1e-30).all())
    assert bool((ev <= bv.reshape(B * n, D) + 1e-30).all())
    if kind == "zero":
        assert float(dqkv[:, D:].abs().max()) == 0


@pytest.mark.parametrize("B,n", [(1, 1), (4, 128), (2, 512)])
def test_attn_bwd_kv_exact_on_grid(B, n):
    g = torch.Generator().manual_seed(n + 3 * B)
    qkv = _qkv(B, n, g, grid=True)
    dKV = torch.randint(-16, 17, (B, H, DH, DH), generator=g).double() / 16
    dks = torch.randint(-16, 17, (B, H, DH), generator=g).double() / 16
    mask = _mask(B, n, "partial")
    dqkv = _bwd_kv(qkv, mask, B, n, dKV, dks)
    rk, rv = coarse_tf.backward_kv(_heads(qkv[:, D:2 * D], B, n), _heads(qkv[:, 2 * D:], B, n), dKV, dks, _fm(mask))
    assert torch.equal(dqkv[:, D:2 * D].double().cpu(), rk.reshape(B * n, D))
    assert torch.equal(dqkv[:, 2 * D:].double().cpu(), rv.reshape(B * n, D))


def test_chunks_and_bad_arguments():
    assert [ops.coarse_tf_chunks(n) for n in (1, 127, 128, 129, 7000)] == [1, 1, 1, 2, 55]
    qkv = torch.zeros(10, 3 * D, device="cuda")
    with pytest.raises(ValueError, match="batch"):
        ops.coarse_tf_kv(qkv, None, 3, ops.coarse_tf_part(3, 3, "cuda"), torch.empty(3, H, DH, DH, device="cuda"),
                         torch.empty(3, H, DH, device="cuda"))
    with pytest.raises(ValueError, match="mask"):
        ops.coarse_tf_kv(qkv, torch.ones(9, dtype=torch.uint8, device="cuda"), 2, ops.coarse_tf_part(2, 5, "cuda"),
                         torch.empty(2, H, DH, DH, device="cuda"), torch.empty(2, H, DH, device="cuda"))
    with pytest.raises(RuntimeError, match="opp_coarse_tf_attn"):
        ops.coarse_tf_attn(torch.zeros(10, 2 * D, device="cuda"), None, 2, torch.zeros(2, H, DH, DH, device="cuda"),
                           torch.zeros(2, H, DH, device="cuda"), 5, torch.empty(10, D, device="cuda"))


def _ln_bounds(x32, gamma, beta, dy):
    """fp64 LayerNorm of the fp32 rows x32 and its backward, with error bounds of the fp32 kernels
    (8 summation levels of the warp reduction, rsqrtf, and the propagation of the mean's error)."""
    mean, var = x32.mean(1, keepdim=True), x32.var(1, unbiased=False, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    d = x32 - mean
    xh = d * rstd
    dm = 16 * U * x32.abs().mean(1, keepdim=True)                       # |error of the mean|
    rel = (2 * d.abs().mean(1, keepdim=True) * dm + 16 * U * var) / (var + 1e-5) + 4 * U   # of rstd
    e_xh = (dm + U * d.abs()) * rstd + xh.abs() * rel
    y = xh * gamma + beta
    by = gamma.abs() * e_xh + 8 * U * (xh.abs() * gamma.abs() + beta.abs())
    dxh = dy * gamma
    m1, m2 = dxh.mean(1, keepdim=True), (dxh * xh).mean(1, keepdim=True)
    dx = rstd * (dxh - m1 - xh * m2)
    dm2 = (dxh.abs() * e_xh).mean(1, keepdim=True) + 16 * U * (dxh * xh).abs().mean(1, keepdim=True)
    bdx = dx.abs() * rel + rstd * (e_xh * m2.abs() + xh.abs() * dm2 + 16 * U * dxh.abs().mean(1, keepdim=True)
                                   + 8 * U * (dxh.abs() + m1.abs() + (xh * m2).abs()))
    c = x32.shape[0] // 256 + 16
    bdg = (dy.abs() * e_xh).sum(0) + c * U * (dy * xh).abs().sum(0)
    return (mean[:, 0], rstd[:, 0], dm[:, 0], rel[:, 0]), (y, by), (dx, bdx), ((dy * xh).sum(0), bdg)


@pytest.mark.parametrize("rows", [1, 255, 256, 257, 4 * (4096 + 7000)])
@pytest.mark.parametrize("resid", [False, True])
def test_layernorm_256(rows, resid):
    g = torch.Generator().manual_seed(rows + resid)
    x = _rows(rows, D, g)
    x[0] = 1.5                                                          # a constant row
    if rows > 3:
        x[1] = 1000 + _rows(1, D, g) * 0.01
    gamma, beta = _rows(1, D, g)[0], _rows(1, D, g)[0]
    r = _rows(rows, D, g) if resid else None
    xb, xv = _framed(x)
    yb, yv = _framed(torch.full((rows, D), float("nan")))
    st = torch.full((rows, 2), float("nan"), device="cuda")
    rv = _framed(r)[1] if resid else None
    ops.coarse_tf_ln(xv, gamma.float().cuda(), beta.float().cuda(), rv, yv, st)
    assert bool((yb[:, D:] == SENTINEL).all())
    x32 = x.float().double()
    dy = _rows(rows, D, g)
    (mean, rstd, dm, rel), (ref, by), (rdx, bdx), (rdg, bdg) = _ln_bounds(
        x32, gamma.float().double(), beta.float().double(), dy.float().double())
    if resid:
        ref = ref + r.float().double()
        by = by + 4 * U * ref.abs()
    assert bool(((st[:, 0].double().cpu() - mean).abs() <= dm + 1e-30).all())
    assert bool(((st[:, 1].double().cpu() - rstd).abs() <= rel * rstd).all())
    assert bool(((yv.double().cpu() - ref).abs() <= 2 * by + 1e-30).all())
    _, dyv = _framed(dy)
    dxb, dxv = _framed(torch.full((rows, D), float("nan")))
    groups = ops.fine_train_groups(rows)
    part = torch.empty(groups * 2 * D, device="cuda")
    dgb = torch.full((2, D), 7.0, device="cuda")
    ops.coarse_tf_ln_bwd(xv, gamma.float().cuda(), st, dyv, dxv, part, dgb, True)
    assert bool((dxb[:, D:] == SENTINEL).all())
    assert bool(((dxv.double().cpu() - rdx).abs() <= 2 * bdx + 1e-30).all())
    assert bool(((dgb[0].double().cpu() - 7 - rdg).abs() <= 2 * bdg + 8 * U * 7 + 1e-30).all())
    assert float((dgb[1].double().cpu() - 7 - dy.float().double().sum(0)).abs().max()) <= \
        float((rows // 256 + 16) * U * dy.abs().sum(0).max()) + 8 * U * 7
    if rows <= 4096:                                                    # dbeta is a sum of dy: exact on the grid
        dyg = torch.randint(-32, 33, (rows, D), generator=g).double() / 16
        _, dyv = _framed(dyg)
        ops.coarse_tf_ln_bwd(xv, gamma.float().cuda(), st, dyv, dxv, part, dgb, False)
        assert torch.equal(dgb[1].double().cpu(), dyg.sum(0))
