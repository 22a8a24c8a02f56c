"""The opp_kpt_train_* entry points (and the opp_kpt_stats statistics they read) one at a time against
fp64 PyTorch statements of the same operations (oracle/kpt_enc.py, train_path.normalize_3d_keypoints).

  - poisoned outputs: out, the partials and the parameter gradient start as NaN and must be written;
  - bounds derived from fp32 rounding of the same sums: first-order propagation, in fp64, of
    U = 2^-24 times the number of roundings along each sum times the sum of absolute terms, through
    the layers (the ReLU is 1-Lipschitz; a ReLU mask that the input error can flip adds |dz|); the
    largest err / bound is printed per entry point;
  - group edges: an upstream gradient that is non-zero only on the first and last row of each
    32-row group, in one call and in slices, so a dropped, doubled or misplaced row or partial shows up.
Sizes: N = 1, 255, 256, 257, 7000, 20000 with B = 1 and 4 (rows of one tile span batch elements)."""
import copy

import pytest
import torch

from oracle import kpt_enc, oracle, workload
from onepose_plus_plus_b200 import OnePosePlus_model, ops, train_kpt, train_path

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
SIZES = [(b, n) for n in (1, 255, 256, 257, 7000, 20000) for b in (1, 4)]


def _params():
    m = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    m.load_state_dict(workload.synthetic_state_dict(0), strict=True)
    return [p.detach().to(DEV).float().contiguous() for p in train_kpt.params(m.kpt_3d_pos_encoding)]


def _case(B, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kpts = torch.rand(B, N, 3, generator=g, device=DEV) * torch.tensor([0.12, 0.08, 0.1], device=DEV) + \
        torch.tensor([0.3, -0.2, 0.9], device=DEV)
    desc = torch.randn(B, 256, N, generator=g, device=DEV)
    up = torch.randn(B, N, 256, generator=g, device=DEV)
    return kpts, desc, up


def _stats(kpts):
    st = torch.full((kpts.shape[0], 4), float("nan"), device=DEV)
    ops.kpt_stats(kpts, st)
    return st


def _mlp_stats(kpts):
    """The statistics the MLP entry points are checked with: opp_kpt_stats', except that a single point
    has extent 0 and normalize_3d_keypoints divides by it (NaN, as in the reference), so N = 1 gets a
    finite scale."""
    st = _stats(kpts)
    if kpts.shape[1] == 1:
        st[:, 3] = 0.06
    return st


def _x0(kpts, st):
    """The normalised keypoints in fp64 from the kernel's statistics, and their bound (subtraction and
    division each round once)."""
    x0 = (kpts.double() - st[:, None, :3].double()) / st[:, None, 3:].double()
    return x0, 2 * U * x0.abs() + 1e-300


def _gamma(k):
    return k * U / (1 - k * U)


def _fwd_bounds(p, x0, ex0):
    """fp64 forward of the hidden layers with the first-order error bound of each value."""
    z, ez, layers = x0, ex0, []
    for i in range(3):
        W, b = p[2 * i].double(), p[2 * i + 1].double()
        C, K = W.shape
        a = z @ W.T + b
        ea = ez @ W.abs().T + _gamma(K + 1) * (z.abs() @ W.abs().T + b.abs())
        mu = a.mean(-1, keepdim=True)
        r = 1.0 / torch.sqrt(((a - mu) ** 2).mean(-1, keepdim=True) + 1e-5)
        y = (a - mu) * r
        er_rel = r * (y.abs() * ea).mean(-1, keepdim=True) + _gamma(C + 6)
        ey = r * (ea + ea.mean(-1, keepdim=True)) + y.abs() * er_rel + \
            _gamma(C + 6) * (y.abs() + r * a.abs().mean(-1, keepdim=True))
        layers.append((z, ez, y, ey, r, er_rel))
        z, ez = torch.clamp(y, min=0), ey
    return layers, z, ez


def _bounds(p, x0, ex0, desc, up, groups):
    """(out, eout, grads, egrads) in fp64: forward output [B, N, 256] and the eight parameter gradients
    for the upstream gradient up [B, N, 256], each with its bound; groups = partials summed per weight."""
    layers, z3, ez3 = _fwd_bounds(p, x0, ex0)
    W4, b4 = p[6].double(), p[7].double()
    mlp = z3 @ W4.T + b4
    d = desc.double().transpose(1, 2)
    out = mlp + d
    eout = ez3 @ W4.abs().T + _gamma(129) * (z3.abs() @ W4.abs().T + b4.abs()) + U * (mlp.abs() + out.abs())
    g = up.double()
    ns = _gamma(32 + groups + 1)          # products + the in-tile sum + the partial sum

    def wsum(da, eda, zin, ezin):
        dW = torch.einsum("bnc,bnk->ck", da, zin)
        edW = torch.einsum("bnc,bnk->ck", eda, zin.abs()) + torch.einsum("bnc,bnk->ck", da.abs(), ezin) + \
            ns * torch.einsum("bnc,bnk->ck", da.abs(), zin.abs())
        db = da.sum((0, 1))
        edb = eda.sum((0, 1)) + ns * da.abs().sum((0, 1))
        return dW, edW, db, edb

    grads, egrads = [None] * 8, [None] * 8
    grads[6], egrads[6], grads[7], egrads[7] = wsum(g, torch.zeros_like(g), z3, ez3)
    dz, edz = g @ W4, _gamma(256) * (g.abs() @ W4.abs())
    for i in (2, 1, 0):
        zin, ezin, y, ey, r, er_rel = layers[i]
        C = y.shape[-1]
        m = y > 0
        dy = torch.where(m, dz, torch.zeros_like(dz))
        edy = torch.where(m, edz, torch.zeros_like(edz)) + torch.where(y.abs() <= ey, dz.abs(), torch.zeros_like(dz))
        m1, m2 = dy.mean(-1, keepdim=True), (dy * y).mean(-1, keepdim=True)
        da = r * (dy - m1 - y * m2)
        eda = r * (edy + edy.mean(-1, keepdim=True) + y.abs() * (y.abs() * edy + dy.abs() * ey).mean(-1, keepdim=True)
                   + ey * m2.abs()) + da.abs() * er_rel + \
            _gamma(C + 6) * r * (dy.abs() + dy.abs().mean(-1, keepdim=True) +
                                 y.abs() * (dy * y).abs().mean(-1, keepdim=True))
        grads[2 * i], egrads[2 * i], grads[2 * i + 1], egrads[2 * i + 1] = wsum(da, eda, zin, ezin)
        if i:
            W = p[2 * i].double()
            dz, edz = da @ W, eda @ W.abs() + _gamma(W.shape[0]) * (da.abs() @ W.abs())
    return out, eout, grads, egrads


def _ratio(err, bound):
    return float((err / bound).max())


@pytest.mark.parametrize("B,N", SIZES)
def test_stats_against_normalize_3d_keypoints(B, N):
    kpts, _, _ = _case(B, N, seed=N + B)
    st = _stats(kpts)
    k64 = kpts.double()
    mean = k64.mean(1)
    ext = (k64[0].max(0).values - k64[0].min(0).values).max() * 0.6
    emean = _gamma(-(-N // 256) + 9) * k64.abs().mean(1)
    assert bool(((st[:, :3].double() - mean).abs() <= emean).all()), (st[:, :3], mean)
    assert abs(float(st[0, 3]) - float(ext)) <= _gamma(3) * float(ext)
    assert bool((st[:, 3] == st[0, 3]).all())
    # the fp32 statistics against train_path.normalize_3d_keypoints in fp64: the normalised keypoints
    x0, _ = _x0(kpts, st)
    ref = train_path.normalize_3d_keypoints(k64)
    if N == 1:                    # extent 0: both divide 0 by 0
        assert float(st[0, 3]) == 0.0 and bool(x0.isnan().all()) and bool(ref.isnan().all())
        return
    assert float((x0 - ref).abs().max()) <= 64 * _gamma(-(-N // 256) + 12) * float(ref.abs().max() + 1)


@pytest.mark.parametrize("B,N", SIZES)
def test_forward_against_fp64(B, N):
    p = _params()
    kpts, desc, up = _case(B, N, seed=10 * N + B)
    st = _mlp_stats(kpts)
    out = torch.full((B * N, 256), float("nan"), device=DEV)
    ops.kpt_train_fwd(kpts, st, desc, train_kpt.pack(p), out)
    assert not torch.isnan(out).any()
    x0, ex0 = _x0(kpts, st)
    ref, eref, _, _ = _bounds(p, x0, ex0, desc, up, 1)
    err = (out.view(B, N, 256).double() - ref).abs()
    r = _ratio(err, eref)
    print(f"kpt_train_fwd B={B} N={N}: largest err / bound {r:.3g}")
    assert r <= 1.0
    ref_o, _ = kpt_enc.forward([t.double() for t in p], x0, desc.double())
    torch.testing.assert_close(ref_o.transpose(1, 2), ref, rtol=0, atol=1e-12)


def _bwd(kpts, st, up, p, slices=None):
    B, N, _ = kpts.shape
    rows, group, nparams = B * N, ops.kpt_train_group(), ops.kpt_train_params()
    step = rows if slices is None else slices * group
    part = torch.full((-(-min(rows, step) // group) * nparams,), float("nan"), device=DEV)
    flat = torch.full((nparams,), float("nan"), device=DEV)
    for r0 in range(0, rows, step):
        ops.kpt_train_bwd(kpts, st, up, train_kpt.pack(p), r0, min(step, rows - r0), part, flat, r0 > 0)
    assert not torch.isnan(flat).any()
    return flat


def _check_grads(flat, p, grads, egrads, label):
    worst, off = 0.0, 0
    for i, (t, g, e) in enumerate(zip(p, grads, egrads)):
        got = flat[off:off + t.numel()].view(t.shape).double()
        off += t.numel()
        r = _ratio((got - g).abs(), e + 1e-300)
        worst = max(worst, r)
        assert r <= 1.0, (label, i, r)
    print(f"kpt_train_bwd {label}: largest err / bound {worst:.3g}")


@pytest.mark.parametrize("B,N", SIZES)
def test_backward_against_fp64(B, N):
    p = _params()
    kpts, desc, up = _case(B, N, seed=20 * N + B)
    st = _mlp_stats(kpts)
    flat = _bwd(kpts, st, up, p)
    groups = -(-(B * N) // ops.kpt_train_group())
    x0, ex0 = _x0(kpts, st)
    _, _, grads, egrads = _bounds(p, x0, ex0, desc, up, groups)
    _check_grads(flat, p, grads, egrads, f"B={B} N={N}")
    ref = kpt_enc.backward([t.double() for t in p], x0, up.double().transpose(1, 2))
    for a, b in zip(ref, grads):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("slices", [None, 1, 3])
def test_backward_group_edges(slices):
    """Only the first and last row of each 32-row group carry a gradient; one call and sliced calls."""
    p = _params()
    B, N = 4, 257
    kpts, desc, up = _case(B, N, seed=77)
    group = ops.kpt_train_group()
    rows = torch.arange(B * N, device=DEV)
    edge = (rows % group == 0) | (rows % group == group - 1) | (rows == B * N - 1)
    up = (up.view(B * N, 256) * edge[:, None]).view(B, N, 256).contiguous()
    st = _stats(kpts)
    flat = _bwd(kpts, st, up, p, slices)
    x0, ex0 = _x0(kpts, st)
    _, _, grads, egrads = _bounds(p, x0, ex0, desc, up, -(-(B * N) // group))
    _check_grads(flat, p, grads, egrads, f"group edges, slices of {slices} groups")
    # every row's contribution counted once: dropping or doubling an edge row moves db4 by at least
    # that row's gradient, far beyond the bound
    one = up.clone().view(B * N, 256)
    one[group - 1] = 0
    flat2 = _bwd(kpts, st, one.view(B, N, 256), p, slices)
    db4 = slice(flat.numel() - 256, flat.numel())
    torch.testing.assert_close((flat[db4] - flat2[db4]).double(), up.view(B * N, 256)[group - 1].double(),
                               rtol=0, atol=float(egrads[7].max()) * 4)


def test_backward_is_bit_reproducible_and_slices_agree():
    p = _params()
    kpts, desc, up = _case(4, 7000, seed=5)
    st = _stats(kpts)
    a, b = _bwd(kpts, st, up, p), _bwd(kpts, st, up, p)
    assert torch.equal(a, b)
    c = _bwd(kpts, st, up, p, slices=128)
    assert torch.equal(c, _bwd(kpts, st, up, p, slices=128))
    x0, ex0 = _x0(kpts, st)
    _, _, grads, egrads = _bounds(p, x0, ex0, desc, up, -(-28000 // ops.kpt_train_group()))
    _check_grads(c, p, grads, egrads, "B=4 N=7000 in slices of 128 groups")


def test_bad_slices_raise():
    p = _params()
    kpts, _, up = _case(1, 100, seed=1)
    st = _stats(kpts)
    part = torch.empty(4 * ops.kpt_train_params(), device=DEV)
    flat = torch.empty(ops.kpt_train_params(), device=DEV)
    for r0, n in ((3, 10), (0, 101), (96, 5), (0, 0)):
        with pytest.raises(RuntimeError, match="opp_kpt_train_bwd"):
            ops.kpt_train_bwd(kpts, st, up, train_kpt.pack(p), r0, n, part, flat, False)
