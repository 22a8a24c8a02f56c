"""Each opp_backbone_train_* kernel on its own against fp64 PyTorch: the convolutions (3xTF32 on the
tensor cores) at every configuration the backbone launches (enumerated from the module), at the small
shape and at B = 4, 512 x 512, and edges (1 x 1 maps, widths that are not multiples of the tile, B = 1,
5 and 70 channels); BatchNorm and the upsample.  Outputs start NaN-poisoned.

Exact: inputs on the 2^-4 grid are tf32 values (lo = 0), so y, dx and dw equal fp64 bit for bit wherever
every partial sum fits in 24 bits.

Random (randn inputs): with a = hi_a + lo_a, hi_a = rna_tf32(a), the kernel forms lo_a' = rna_tf32(a - hi_a)
and sums hi_a hi_b + hi_a lo_b' + lo_a' hi_b in fp32.  Per term, with u = 2^-11 (the tf32 unit roundoff):
  - |a - hi_a| <= u |a|, and lo_a' differs from lo_a by <= u |lo_a| <= u^2 |a|;
  - the dropped lo_a lo_b is <= u^2 |a b|, the two roundings of lo add <= 2 u^2 |a b| (+ higher order);
so each term is within 3.01 u^2 |a b| = 7.2e-7 |a b| of a·b.  The fp32 accumulation over K terms (the
tensor core's sums, the partials of wgrad and their reduce) adds at most K 2^-24 sum|a b| in the usual
worst-case form.  The bound is therefore (3.01 u^2 + K 2^-24) sum|a b| (fp64) + 1e-6 absmax(ref).

The lo terms matter: each check also computes the error of 1xTF32 products (hi_a hi_b summed in fp64) on
the same inputs and asserts that it exceeds the kernel's own error by at least 10x, so a kernel without
the hi·lo / lo·hi MMAs could not pass.  It is compared with the measured 3xTF32 error, not with the
bound above: the bound's accumulation term grows like K while the 1xTF32 rounding errors cancel like
sqrt(K) (random signs), so from K of a few thousand on (every dw at the training shape) the worst-case
bound is larger than the 1xTF32 error itself and cannot tell the two kernels apart."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import oracle
from onepose_plus_plus_b200 import OnePosePlus_model, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
UT = 2.0 ** -11                      # tf32 unit roundoff (10 stored mantissa bits, round to nearest)
TERM = 3.01 * UT * UT


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


def _tf32(t):
    """Round fp32 to tf32, to nearest with ties away from zero (cvt.rna.tf32.f32), as fp64."""
    # sign-magnitude: rounding the magnitude half away from zero is adding half an ulp to the bit pattern
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


def _calls(x, w, dy, s, B, ci, co, k, H, W, slice_groups=3):
    ho, wo = ops.conv_out_hw(H, W, k, s)
    y = _nan(B, co, ho, wo)
    ops.backbone_conv(x, w, s, y)
    dx = _nan(B, ci, H, W)
    ops.backbone_conv_dgrad(dy, w, s, dx, False)
    dw = _nan(co, ci, k, k)
    pixels = B * ho * wo
    group = ops.backbone_wgrad_group()
    step = slice_groups * group                        # slices with accumulate, as the stage calls it
    part = torch.empty(slice_groups * dw.numel(), device=DEV)
    dw.zero_()
    for p0 in range(0, pixels, step):
        ops.backbone_conv_wgrad(x, dy, s, dw, part, p0, min(step, pixels - p0), True)
    return y, dx, dw


def _refs(x, w, dy, s, k):
    """fp64 (y, dx, dw) and the same of |x|, |w|, |dy| (sum|a b| of every output)."""
    def grads(xx, ww, gg):
        x64, w64 = xx.double().requires_grad_(True), ww.double().requires_grad_(True)
        y64 = F.conv2d(x64, w64, stride=s, padding=k // 2)
        dx64, dw64 = torch.autograd.grad(y64, (x64, w64), gg.double())
        return y64.detach(), dx64, dw64
    return grads(x, w, dy), grads(x.abs(), w.abs(), dy.abs())


def _check_conv(ci, co, k, s, B, H, W, exact, seed):
    gen = _grid if exact else _rand
    x = gen(B, ci, H, W, seed=seed)
    w = gen(co, ci, k, k, seed=seed + 1) if exact else _rand(co, ci, k, k, seed=seed + 1) * (2.0 / (ci * k * k)) ** 0.5
    ho, wo = ops.conv_out_hw(H, W, k, s)
    dy = gen(B, co, ho, wo, seed=seed + 2)
    got = _calls(x, w, dy, s, B, ci, co, k, H, W)
    again = _calls(x, w, dy, s, B, ci, co, k, H, W)
    for name, a, b in zip(("y", "dx", "dw"), got, again):
        assert torch.equal(a, b), f"{name}: two calls differ"
    ref, absum = _refs(x, w, dy, s, k)
    if not exact:
        ref1, _ = _refs(_tf32(x).float(), _tf32(w).float(), _tf32(dy).float(), s, k)       # 1xTF32 products
    ratios = []
    for i, (name, K) in enumerate((("y", ci * k * k), ("dx", co * k * k), ("dw", B * ho * wo))):
        assert not torch.isnan(got[i]).any(), name
        err = (got[i].double() - ref[i]).abs()
        if exact:
            assert float(err.max()) == 0.0, (name, float(err.max()))
            continue
        ref_abs = float(ref[i].abs().max())
        bound = (TERM + K * U) * absum[i] + 1e-6 * ref_abs
        assert float((err - bound).max()) <= 0, (name, float((err / bound).max()))
        err1, err3 = float((ref1[i] - ref[i]).abs().max()), float(err.max())
        ratios.append((name, f"err/bound {float((err / bound).max()):.3f}", f"3xTF32 {err3:.2e}", f"1xTF32 {err1:.2e}"))
        assert err1 >= 10 * err3, (name, err1, err3)
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


@pytest.mark.parametrize("ks", [(1, 1), (3, 1), (3, 2), (7, 2)])
def test_conv_edges_random(ks):
    """Random inputs at edge shapes: a K that is not a multiple of the 32-wide chunk, a partial M tile."""
    k, s = ks
    print(ks, _check_conv(5, 70, k, s, 2, 37, 23, exact=False, seed=6))
    print(ks, _check_conv(70, 5, k, s, 1, 17, 9, exact=False, seed=7))


def test_configs_cover_the_backbone():
    assert len(CONFIGS) == 22 and len(UNIQUE) >= 10


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
