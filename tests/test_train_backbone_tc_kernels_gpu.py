"""Each opp_backbone_train_conv*_tf32x3 entry point (3xTF32 on the tensor cores) on its own against fp64
PyTorch: every convolution configuration the backbone launches (enumerated from the module, as in
test_train_backbone_kernels_gpu.py), at the small shape and at B = 4, 512 x 512, and edges (1 x 1 maps,
widths that are not multiples of the tile, B = 1, 5 and 70 channels).  Outputs start NaN-poisoned.

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
import pytest
import torch
import torch.nn.functional as F

from onepose_plus_plus_b200 import ops
from tests.test_train_backbone_kernels_gpu import CONFIGS, UNIQUE

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


def _tf32(t):
    """Round fp32 to tf32, to nearest with ties away from zero (cvt.rna.tf32.f32), as fp64."""
    # sign-magnitude: rounding the magnitude half away from zero is adding half an ulp to the bit pattern
    b = t.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32).double()


def _calls(x, w, dy, s, B, ci, co, k, H, W, slice_groups=3):
    ho, wo = ops.conv_out_hw(H, W, k, s)
    y = _nan(B, co, ho, wo)
    ops.backbone_conv(x, w, s, y, tf32x3=True)
    dx = _nan(B, ci, H, W)
    ops.backbone_conv_dgrad(dy, w, s, dx, False, tf32x3=True)
    dw = _nan(co, ci, k, k)
    pixels = B * ho * wo
    group = ops.backbone_wgrad_group()
    step = slice_groups * group                        # slices with accumulate, as the stage calls it
    part = torch.empty(slice_groups * dw.numel(), device=DEV)
    dw.zero_()
    for p0 in range(0, pixels, step):
        ops.backbone_conv_wgrad(x, dy, s, dw, part, p0, min(step, pixels - p0), True, tf32x3=True)
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
def test_tc_conv_configs_small_exact_and_random(cfg):
    ci, co, k, s, div = cfg
    H, W = 96 // div, 128 // div
    _check_conv(ci, co, k, s, 2, H, W, exact=True, seed=1)
    print(cfg, _check_conv(ci, co, k, s, 2, H, W, exact=False, seed=5))


@pytest.mark.parametrize("cfg", UNIQUE, ids=lambda c: f"{c[0]}-{c[1]}-k{c[2]}s{c[3]}")
def test_tc_conv_configs_training_shape(cfg):
    ci, co, k, s, div = cfg
    print(cfg, _check_conv(ci, co, k, s, 4, 512 // div, 512 // div, exact=False, seed=9))


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 3, 5, 3), (1, 2, 2, 1), (2, 37, 23, 1), (1, 17, 9, 2)])
@pytest.mark.parametrize("ks", [(1, 1), (1, 2), (3, 1), (3, 2), (7, 2)])
def test_tc_conv_edges(shape, ks):
    B, H, W, _ = shape
    k, s = ks
    _check_conv(5, 70, k, s, B, H, W, exact=True, seed=3)
    _check_conv(70, 5, k, s, B, H, W, exact=True, seed=4)


@pytest.mark.parametrize("ks", [(1, 1), (3, 1), (3, 2), (7, 2)])
def test_tc_conv_edges_random(ks):
    """Random inputs at edge shapes: a K that is not a multiple of the 32-wide chunk, a partial M tile."""
    k, s = ks
    print(ks, _check_conv(5, 70, k, s, 2, 37, 23, exact=False, seed=6))
    print(ks, _check_conv(70, 5, k, s, 1, 17, 9, exact=False, seed=7))


def test_tc_default_keyword_is_the_fp32_kernel():
    """tf32x3=False (the default) calls the CUDA-core entry point: on randn inputs the two differ, and the
    default matches an explicit tf32x3=False bit for bit."""
    x, w = _rand(2, 64, 24, 32, seed=1), _rand(128, 64, 3, 3, seed=2) * 0.06
    y0, y1, y2 = _nan(2, 128, 24, 32), _nan(2, 128, 24, 32), _nan(2, 128, 24, 32)
    ops.backbone_conv(x, w, 1, y0)
    ops.backbone_conv(x, w, 1, y1, tf32x3=False)
    ops.backbone_conv(x, w, 1, y2, tf32x3=True)
    assert torch.equal(y0, y1)
    assert not torch.equal(y0, y2)


def test_configs_cover_the_backbone():
    assert len(CONFIGS) == 22 and len(UNIQUE) >= 10
