"""Each opp_backbone_train_* kernel on its own against fp64 PyTorch: every convolution configuration the
backbone launches (enumerated from the module), at the small shape and at B = 4, 512 x 512, and edges (a
1 x 1 coarse map, widths that are not multiples of the tile, B = 1).  Inputs on a 2^-4 grid are exact
wherever every partial sum fits in 24 bits; elsewhere the bound is derived from fp32 rounding of the
same sums (K·2^-24·sum|terms|, in fp64).  Outputs start NaN-poisoned."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import oracle
from onepose_plus_plus_b200 import OnePosePlus_model, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24


def _grid(*shape, seed, lo=-8, hi=8):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi + 1, shape, generator=g).float() / 16).to(DEV)


def _rand(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _configs():
    """(name, c_in, c_out, k, stride, input divisor of the image size) of every backbone convolution."""
    bb = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG)).backbone
    out = []
    scale = {"conv1": 1, "layer1": 2, "layer2.0.conv1": 2, "layer2.0.downsample": 2, "layer2": 4,
             "layer3.0.conv1": 4, "layer3.0.downsample": 4, "layer3": 8, "layer3_outconv": 8,
             "layer2_outconv": 4, "layer1_outconv": 2}
    for n, m in bb.named_modules():
        if isinstance(m, torch.nn.Conv2d):
            key = max((k for k in scale if n.startswith(k)), key=len)
            out.append((n, m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0], scale[key]))
    assert len(out) == 22
    return out


CONFIGS = _configs()
UNIQUE = sorted({c[1:] for c in CONFIGS})


def _bound(terms_abs_sum, k):
    return k * U * terms_abs_sum + 1e-30


def _check_conv(ci, co, k, s, B, H, W, exact, seed):
    gen = _grid if exact else _rand
    x = gen(B, ci, H, W, seed=seed)
    w = gen(co, ci, k, k, seed=seed + 1) if exact else _rand(co, ci, k, k, seed=seed + 1) * (2.0 / (ci * k * k)) ** 0.5
    ho, wo = ops.conv_out_hw(H, W, k, s)
    dy = gen(B, co, ho, wo, seed=seed + 2)
    x64, w64, dy64 = x.double().requires_grad_(True), w.double().requires_grad_(True), dy.double()
    y64 = F.conv2d(x64, w64, stride=s, padding=k // 2)
    dx64, dw64 = torch.autograd.grad(y64, (x64, w64), dy64)
    y = _nan(B, co, ho, wo)
    ops.backbone_conv(x, w, s, y)
    dx = _nan(B, ci, H, W)
    ops.backbone_conv_dgrad(dy, w, s, dx, False)
    dw = _nan(co, ci, k, k)
    pixels = B * ho * wo
    group = ops.backbone_wgrad_group()
    step = 3 * group                                   # slices with accumulate, as the stage calls it
    part = torch.empty(3 * dw.numel(), device=DEV)
    dw.zero_()
    for p0 in range(0, pixels, step):
        ops.backbone_conv_wgrad(x, dy, s, dw, part, p0, min(step, pixels - p0), True)
    with torch.no_grad():
        ya = F.conv2d(x64.abs(), w64.abs(), stride=s, padding=k // 2)
    ratios = []
    for name, got, ref, absum, K in (("y", y, y64, ya, ci * k * k), ("dx", dx, dx64, None, co * k * k),
                                     ("dw", dw, dw64, None, pixels)):
        assert not torch.isnan(got).any(), name
        err = (got.double() - ref).abs()
        if exact:
            assert float(err.max()) == 0.0, (name, float(err.max()))
        else:
            ref_abs = float(ref.abs().max())
            bound = (absum if absum is not None else ref.abs() + ref_abs) * K * U + 1e-6 * ref_abs
            ratios.append(float((err / bound).max()))
            assert float((err - bound).max()) <= 0, (name, float(err.max()))
    return ratios


@pytest.mark.parametrize("cfg", UNIQUE, ids=lambda c: f"{c[0]}-{c[1]}-k{c[2]}s{c[3]}")
def test_conv_configs_small_exact_and_random(cfg):
    ci, co, k, s, div = cfg
    H, W = 96 // div, 128 // div
    _check_conv(ci, co, k, s, 2, H, W, exact=True, seed=1)
    print(cfg, _check_conv(ci, co, k, s, 2, H, W, exact=False, seed=5))


@pytest.mark.parametrize("cfg", UNIQUE, ids=lambda c: f"{c[0]}-{c[1]}-k{c[2]}s{c[3]}")
def test_conv_configs_training_shape(cfg):
    ci, co, k, s, div = cfg
    print(cfg, _check_conv(ci, co, k, s, 4, 512 // div, 512 // div, exact=False, seed=9))


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 3, 5, 3), (1, 2, 2, 1), (2, 37, 23, 1), (1, 17, 9, 2)])
@pytest.mark.parametrize("ks", [(1, 1), (1, 2), (3, 1), (3, 2), (7, 2)])
def test_conv_edges(shape, ks):
    B, H, W, _ = shape
    k, s = ks
    _check_conv(5, 70, k, s, B, H, W, exact=True, seed=3)
    _check_conv(70, 5, k, s, B, H, W, exact=True, seed=4)


@pytest.mark.parametrize("shape", [(1, 3, 1, 1), (2, 5, 1, 1), (4, 128, 256, 256), (3, 7, 33, 17), (1, 2, 4097, 1)])
@pytest.mark.parametrize("act", ["none", "relu", "leaky"])
def test_batchnorm_forward_and_backward(shape, act):
    B, C, H, W = shape
    x = _rand(*shape, seed=1) * 3 + 1
    res = _rand(*shape, seed=2)
    gamma, beta = _rand(C, seed=3), _rand(C, seed=4)
    dy = _rand(*shape, seed=5)
    rm, rv = _rand(C, seed=6), _rand(C, seed=7).abs() + 0.5
    n = B * H * W
    mean, invstd = _nan(C), _nan(C)
    rm_k, rv_k = rm.clone(), rv.clone()
    part = ops.backbone_bn_part(B, C, H * W, DEV)
    ops.backbone_bn_stats(x, 1e-5, part, mean, invstd, *((rm_k, rv_k, 0.1) if n > 1 else ()))
    x64 = x.double()
    m64 = x64.mean((0, 2, 3))
    v64 = x64.var((0, 2, 3), unbiased=False)
    assert float((mean.double() - m64).abs().max()) <= 4 * U * float(m64.abs().max() + x64.std())
    torch.testing.assert_close(invstd.double(), torch.rsqrt(v64 + 1e-5), rtol=4 * U, atol=0)
    if n > 1:
        torch.testing.assert_close(rm_k.double(), 0.9 * rm.double() + 0.1 * m64, rtol=4 * U, atol=4 * U)
        torch.testing.assert_close(rv_k.double(), 0.9 * rv.double() + 0.1 * v64 * n / (n - 1), rtol=4 * U, atol=4 * U)
    for batch in (True, False):
        if n == 1 and batch:
            continue                                     # F.batch_norm refuses a 1-value batch
        mu, r = (mean, invstd) if batch else (rm, torch.rsqrt(rv + 1e-5))
        xr = x64.clone().requires_grad_(True)
        gr, br, rr = (t.double().requires_grad_(True) for t in (gamma, beta, res))
        z = F.batch_norm(xr, mu.double(), (1.0 / r.double() ** 2 - 1e-5), gr, br, training=False, eps=1e-5) \
            if not batch else (xr - mu.double()[None, :, None, None]) * r.double()[None, :, None, None] * \
            gr[None, :, None, None] + br[None, :, None, None]
        z = z + rr
        y64 = {"none": z, "relu": F.relu(z), "leaky": F.leaky_relu(z, 0.01)}[act]
        y = _nan(*shape)
        ops.backbone_bn_act(x, mu, r, gamma, beta, res, act, y)
        scale = float(y64.abs().max()) + 1
        assert float((y.double() - y64).abs().max()) <= 16 * U * scale
        # the activation's derivative from the kernel's own output (a z within rounding of 0 may sit on
        # either side of the kink), then the BatchNorm backward in fp64
        slope = {"none": 1.0, "relu": 0.0, "leaky": 0.01}[act]
        dz64 = dy.double() * (torch.where(y > 0, 1.0, slope).double() if act != "none" else 1.0)
        if batch:
            xb = x64.clone().requires_grad_(True)
            zb = F.batch_norm(xb, None, None, gr, br, training=True, eps=1e-5) + rr
            gx, gg, gb, grs = torch.autograd.grad(zb, (xb, gr, br, rr), dz64)
        else:
            gx, gg, gb, grs = torch.autograd.grad(z, (xr, gr, br, rr), dz64)
        dx, dres, dgb = _nan(*shape), _nan(*shape), _nan(2, C)
        ops.backbone_bn_act_bwd(x, None if act == "none" else y, dy, mu, r, gamma, act, batch, part, dx, dres, dgb)
        # per-element bound on dx from the size of its terms: gamma r (|dz| + |sum dz| / n + |xhat| |sum dz xhat| / n)
        dz = dz64.abs()
        xhat = ((x64 - mu.double()[None, :, None, None]) * r.double()[None, :, None, None]).abs()
        gr_ = (gamma.double() * r.double()).abs()[None, :, None, None]
        term = gr_ * (dz + (gb.abs() / n)[None, :, None, None] + xhat * (gg.abs() / n)[None, :, None, None])
        for name, got, ref, tol in (("dx", dx, gx, 64 * U * term + 1e-7), ("dres", dres, grs, U * grs.abs()),
                                    ("dgamma", dgb[0], gg, 16 * U * float((dz * xhat).sum((0, 2, 3)).max()) + 1e-6),
                                    ("dbeta", dgb[1], gb, 16 * U * float(dz.sum((0, 2, 3)).max()) + 1e-6)):
            err = (got.double() - ref).abs()
            assert bool((err <= tol).all()), (name, batch, float(err.max()))


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (2, 3, 1, 3), (1, 4, 2, 2), (2, 5, 12, 16), (4, 256, 64, 64),
                                   (1, 3, 7, 5)])
def test_upsample_add_and_backward(shape):
    B, C, h, w = shape
    x = _grid(B, C, h, w, seed=1)
    lat = _grid(B, C, 2 * h, 2 * w, seed=2)
    dout = _grid(B, C, 2 * h, 2 * w, seed=3)
    xr = x.double().requires_grad_(True)
    y64 = lat.double() + F.interpolate(xr.float(), scale_factor=2.0, mode="bilinear", align_corners=True).double()
    out = _nan(B, C, 2 * h, 2 * w)
    ops.backbone_up2x_add(x, lat, out)
    assert float((out.double() - y64).abs().max()) <= 4 * U * (float(y64.abs().max()) + 1)
    xf = x.clone().requires_grad_(True)
    (ref,) = torch.autograd.grad(F.interpolate(xf, scale_factor=2.0, mode="bilinear", align_corners=True), xf, dout)
    din = _nan(B, C, h, w)
    ops.backbone_up2x_bwd(dout, din, False)
    tol = 64 * U * (float(ref.abs().max()) + 1)
    assert float((din - ref).abs().max()) <= tol
    base = _grid(B, C, h, w, seed=4)
    acc = base.clone()
    ops.backbone_up2x_bwd(dout, acc, True)
    assert float((acc - base - din).abs().max()) <= tol
    ops.backbone_up2x_add(x, lat, lat)                   # in place on the lateral
    assert torch.equal(lat, out)
