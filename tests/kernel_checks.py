"""Per-kernel numerics checks of libopp_b200.so against plain fp32 torch math on the same
(fp16-rounded) inputs.  Used by tests/test_kernels_gpu.py (pytest -m gpu) and runnable as a script
(`python tests/kernel_checks.py [name ...]`), where every check runs in its own subprocess so that
a device-side trap in one kernel cannot poison the others.
"""
import contextlib
import functools
import math
import subprocess
import sys
import os
import tempfile

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_plus_plus_b200 import _lib, ops  # noqa: E402

DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


class _Tally:
    """|got - ref| <= atol + rtol |ref| over one tensor compared in chunks; a NaN in `got` (an
    element the kernel never wrote into a NaN-prefilled output) counts as out of tolerance."""

    def __init__(self, name, rtol, atol):
        self.name, self.rtol, self.atol = name, rtol, atol
        self.n = self.bad = 0
        self.max_err = self.worst = 0.0

    def add(self, got, ref, slack=0.0):
        """slack: a per-element term added to the tolerance"""
        got, ref = got.float(), ref.float()
        err = (got - ref).abs()
        tol = self.atol + self.rtol * ref.abs() + slack
        self.bad += (~(err <= tol)).sum().item()
        self.n += err.numel()
        if err.numel():
            self.max_err = max(self.max_err, err.max().item())
            self.worst = max(self.worst, (err / tol).max().item())

    def check(self):
        print(f"  {self.name}: max_abs_err={self.max_err:.3e} worst/tol={self.worst:.3f} bad={self.bad}/{self.n}")
        assert self.bad == 0, f"{self.name}: {self.bad} elements out of tolerance (worst {self.worst:.2f}x)"


def _close(name, got, ref, rtol, atol):
    t = _Tally(name, rtol, atol)
    t.add(got, ref)
    t.check()


def _chunk(per_image):
    """images per chunk of a reference computation: about 2^24 elements per tensor (128 MB in fp64)"""
    return max(1, (1 << 24) // per_image)


def _bits_equal(a, b):
    """bit-identical fp16 tensors (torch.equal alone takes -0 for +0)"""
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _elu1(x):
    return F.elu(x) + 1


# ------------------------------------------------------------------------------------------ GEMMs
# tolerances: split=1 (hi|lo planes, 3 MMAs) must be fp32-grade; split=0 is plain fp16 operands
def _tol(split, loose, tight):
    return tight if split else loose


def _planes(x, split):
    return ops.to_planes(x, split)


def _unplanes(t, split):
    return ops.from_planes(t, split)


def _q(x, split):
    """what the kernel sees: the value represented by the stored planes"""
    return _unplanes(_planes(x, split), split)


def check_linear_act():
    for split in (0, 1):
        for (rows, k0, k1, n, act, act_cols) in [(1000, 256, 0, 512, 2, 256), (777, 128, 128, 256, 1, 256),
                                                 (300, 128, 0, 384, 2, 256), (128 * 150 + 5, 256, 256, 512, 1, 512)]:
            a0f = _rand(rows, k0, seed=1)
            a1f = _rand(rows, k1, seed=2) if k1 else None
            wf = _rand(n, k0 + k1, scale=0.05, seed=3)
            a0 = _planes(a0f, split)
            a1 = _planes(a1f, split) if k1 else None
            w = _planes(wf, split)
            pl = 2 if split else 1
            out = torch.full((rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
            _lib.call("opp_linear_act_f16", _lib.ptr(a0), k0, _lib.ptr(a1), k1, _lib.ptr(w),
                      _lib.ptr(out), rows, n, act, act_cols, split, _lib.stream())
            torch.cuda.synchronize()
            a = _q(a0f, split) if a1 is None else torch.cat([_q(a0f, split), _q(a1f, split)], 1)
            ref = (a.double() @ _q(wf, split).double().t()).float()
            fn = torch.relu if act == 1 else _elu1
            ref[:, :act_cols] = fn(ref[:, :act_cols])
            _close(f"linear_act split={split} rows={rows} k={k0}+{k1} n={n}", _unplanes(out, split), ref,
                   *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))


def check_linear_ln():
    for split in (0, 1):
        for (B, rows, k0, n, batched, resid, want32, rshared) in [(2, 1000, 256, 256, True, False, False, False),
                                                                  (1, 2600, 128, 128, False, False, True, False),
                                                                  (3, 500, 512, 256, False, True, False, False),
                                                                  (3, 700, 512, 256, False, True, False, True),
                                                                  (1, 26 * 70, 256, 128, False, True, True, False),
                                                                  # N = 256 at a small grid = N-split cluster
                                                                  # (DSMEM statistics exchange), fp32 output too
                                                                  (1, 600, 256, 256, False, True, True, False),
                                                                  # > 66 M tiles: whole-row tiles, accumulator over the operand ring
                                                                  (1, 12000, 256, 256, False, True, False, False)]:
            a0f = _rand(B * rows, k0, seed=1)
            wf = _rand(B if batched else 1, n, k0, scale=0.05, seed=3)
            gamma = 1 + 0.1 * _rand(n, seed=4)
            beta = 0.1 * _rand(n, seed=5)
            resf = _rand((1 if rshared else B) * rows, n, seed=6) if resid else None
            pl = 2 if split else 1
            out16 = torch.full((B * rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
            out32 = torch.full((B * rows, n), float("nan"), device=DEV) if want32 else None
            a0, w = _planes(a0f, split), _planes(wf, split)
            res = _planes(resf, split) if resid else None
            _lib.call("opp_linear_ln", _lib.ptr(a0), k0, None, 0, _lib.ptr(w), int(batched),
                      _lib.ptr(gamma), _lib.ptr(beta), 1e-5, _lib.ptr(res), int(rshared), _lib.ptr(out16),
                      _lib.ptr(out32), B, rows, n, split, _lib.stream())
            torch.cuda.synchronize()
            a = _q(a0f, split).view(B, rows, k0).double()
            y = torch.einsum("brk,bnk->brn", a, _q(wf, split).double().expand(B, n, k0)).reshape(B * rows, n)
            ref = F.layer_norm(y, (n,), gamma.double(), beta.double(), 1e-5)
            if resid:
                r = _q(resf, split).double()
                ref = ref + (r.repeat(B, 1) if rshared else r)
            ref = ref.float()
            name = f"linear_ln split={split} B={B} rows={rows} k={k0} n={n} resid_shared={rshared}"
            _close(name + " out16", _unplanes(out16, split), ref, *_tol(split, (2e-3, 3e-3), (2e-5, 2e-5)))
            if want32:
                _close(name + " out32", out32, ref, *_tol(split, (1e-3, 2e-3), (2e-5, 2e-5)))


def check_linear_q():
    for split in (0, 1):
        for shared in (False, True):
            B, rows, d = 2, 1111, 256
            xf = _rand((1 if shared else B) * rows, d, seed=1)
            wf = _rand(d, d, scale=0.06, seed=2)
            ksum = _rand(B, d, seed=3).abs() * 100 + 50
            pl = 2 if split else 1
            out = torch.full((B * rows, pl * d), float("nan"), device=DEV, dtype=torch.half)
            x, wq = _planes(xf, split), _planes(wf, split)
            _lib.call("opp_linear_q_f16", _lib.ptr(x), _lib.ptr(wq), _lib.ptr(ksum), _lib.ptr(out), B, rows,
                      d, 4096.0, 1e-6, split, int(shared), None, _lib.stream())
            torch.cuda.synchronize()
            xq = _q(xf, split).double()
            if shared:
                xq = xq.repeat(B, 1)
            q = _elu1((xq @ _q(wf, split).double().t())).view(B, rows, 8, 32)
            z = 1.0 / (torch.einsum("blhd,bhd->blh", q, ksum.double().view(B, 8, 32)) + 1e-6)
            ref = (q * z[..., None] * 4096.0).reshape(B * rows, d).float()
            _close(f"linear_q split={split} x_shared={shared}", _unplanes(out, split), ref,
                   *_tol(split, (2e-3, 1e-4), (2e-5, 1e-6)))


def check_linear_act_shared():
    """batched opp_linear_act_f16_b with the first operand shared by every batch element"""
    for split in (0, 1):
        B, rows, k0, k1, n = 3, 700, 256, 256, 512
        a0f, a1f = _rand(rows, k0, seed=1), _rand(B * rows, k1, seed=2)
        wf = _rand(n, k0 + k1, scale=0.05, seed=3)
        pl = 2 if split else 1
        out = torch.full((B * rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
        ops.linear_act(_planes(a0f, split), _planes(a1f, split), _planes(wf, split), out, rows, 1, n, split,
                       batches=B, a0_shared=True)
        torch.cuda.synchronize()
        a = torch.cat([_q(a0f, split).repeat(B, 1), _q(a1f, split)], 1)
        ref = torch.relu(a.double() @ _q(wf, split).double().t()).float()
        _close(f"linear_act_b split={split} a0_shared", _unplanes(out, split), ref,
               *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))


def _pad16(c):
    return (c + 15) // 16 * 16


def _nhwc_planes(B, H, W, c, c_pad, split, seed, scale=1.0):
    """fp16 planes [B, H, W, planes * c_pad] of N(0, scale^2) values in channels [0, c) and zeros in
    the padding channels, drawn on the device a few images at a time (a batch-64 map of the bench
    shape is 2 GiB; no fp32 copy of it is made)"""
    pl = 2 if split else 1
    out = torch.empty(B, H, W, pl * c_pad, device=DEV, dtype=torch.half)
    g = torch.Generator(device=DEV).manual_seed(seed)
    step = _chunk(H * W * c_pad)
    for b0 in range(0, B, step):
        n = min(step, B - b0)
        xf = torch.zeros(n, H, W, c_pad, device=DEV)
        xf[..., :c] = torch.randn(n, H, W, c, device=DEV, generator=g) * scale
        out[b0:b0 + n] = _planes(xf, split)
    return out


def _up2x_ref(u, oh, ow):
    """Bilinear x2 upsample (align_corners=True) of the NHWC map u [n, h, w, C] to oh x ow, sampled where
    F.interpolate samples an fp32 map (scale (in-1)/(out-1) and scale * dst in fp32; the kernel's
    epilogue does the same) and blended in fp64.  At a 256-wide output an fp32 position near 127 is
    off by up to 7.6e-6, which times the difference of two neighbours is a few 1e-5 - as much as the
    fp16x3 tolerance, although the kernel samples exactly where the model does."""
    def axis(n_in, n_out):
        f = torch.arange(n_out, dtype=torch.float32) * (torch.tensor(n_in - 1.0) / torch.tensor(n_out - 1.0))
        i0 = f.long()
        return i0.to(DEV), (i0 + 1).clamp(max=n_in - 1).to(DEV), (f - i0.float()).double().to(DEV)
    y0, y1, wy = axis(u.shape[1], oh)
    x0, x1, wx = axis(u.shape[2], ow)
    wy, wx = wy.view(1, -1, 1, 1), wx.view(1, 1, -1, 1)
    top, bot = u[:, y0], u[:, y1]
    return ((top[:, :, x0] * (1 - wx) + top[:, :, x1] * wx) * (1 - wy)
            + (bot[:, :, x0] * (1 - wx) + bot[:, :, x1] * wx) * wy)


def _conv_params(cin, cin_pad, cout, cout_pad, k, split):
    """filter planes [cout_pad, planes * k*k*cin_pad] (zero in the padding rows / channels) and bias"""
    wf = torch.zeros(cout_pad, k, k, cin_pad, device=DEV)
    wf[:cout, :, :, :cin] = _rand(cout, k, k, cin, scale=1.0 / math.sqrt(k * k * cin), seed=2)
    bias = torch.zeros(cout_pad, device=DEV)
    bias[:cout] = _rand(cout, seed=3) * 0.1
    return _planes(wf.reshape(cout_pad, -1), split), bias


def _accum_slack(k, cin):
    """Tolerance term per unit |convolution sum| for fp16x3 convolutions at production K.  The wgmma
    accumulator is rounded toward zero once per instruction: on the H100 the convolution sum shrinks
    by about 1.7e-8 of itself per accumulating wgmma (regression of the error on the sum: R^2 0.75,
    spread evenly over columns, images and tile rows; 3x3 convs at K = 1152, 1764, 2304).  The error
    therefore grows with K and with the running sum, not with the output (the residual and the
    upsampled map are added afterwards in fp32), and at K >= 1764 it exceeds 2e-5 + 2e-5 |out| in
    about 1e-5 of the elements.  Bound: less than one ulp (2^-23) per wgmma, 3 per 16-channel K step
    (hi.hi, hi.lo, lo.hi), of the running sum, taken as |sum| + the rms of the sums (a sum that ends
    near zero has run through values of the usual size)."""
    return 3 * k * k * -(-cin // 16) * 2.0 ** -23


def _conv_case(split, B, H, W, cin, cin_pad, cout, cout_pad, k, stride, act, resid, tokens, up=False,
               resid_is_input=False, check=True, accum_tol=False):
    """One opp_conv2d_nhwc launch into NaN-prefilled outputs, checked against F.conv2d in fp64 on the
    values the stored planes represent, + bias, bilinear x2 upsample-add, residual, activation and
    (tokens) + pe, computed a few images at a time so that production batches stay within a few GB.
    resid_is_input: the input map itself is the residual (the stride-1 BasicBlock's shortcut is the
    block input, model.py:459-462).  check=False: launch only.  accum_tol: see _accum_slack.
    Returns (out, tok)."""
    pad = k // 2
    oh, ow = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    pl = 2 if split else 1
    x16 = _nhwc_planes(B, H, W, cin, cin_pad, split, seed=1)
    w16, bias = _conv_params(cin, cin_pad, cout, cout_pad, k, split)
    res = None
    if resid_is_input:
        assert resid and stride == 1 and (cin, cin_pad) == (cout, cout_pad)
        res = x16
    elif resid:
        res = _nhwc_planes(B, oh, ow, cout, cout_pad, split, seed=4)
    out = torch.full((B, oh, ow, pl * cout_pad), float("nan"), device=DEV, dtype=torch.half)
    tok = pe = None
    if tokens:
        tok = torch.full((B, oh * ow, pl * cout_pad), float("nan"), device=DEV, dtype=torch.half)
        pe = _rand(oh * ow, cout_pad, seed=5)
    # FPN top-down merge: + bilinear x2 (align_corners=True) of a coarser map, fused in the epilogue
    up16 = _nhwc_planes(B, oh // 2, ow // 2, cout, cout_pad, split, seed=6) if up else None
    _lib.call("opp_conv2d_nhwc", _lib.ptr(x16), _lib.ptr(w16), _lib.ptr(bias), _lib.ptr(res),
              _lib.ptr(out), B, H, W, cin_pad, cout_pad, k, stride, act, 0.01, _lib.ptr(tok),
              _lib.ptr(pe), _lib.ptr(up16), split, _lib.stream())
    torch.cuda.synchronize()
    if not check:
        return out, tok
    name = (f"conv split={split} B={B} k={k} s={stride} {cin}->{cout} {H}x{W} act={act} resid={resid}"
            f"{' (input)' if resid_is_input else ''} tokens={tokens} up={up}")
    tol = _tol(split, (2e-3, 3e-3), (2e-5, 2e-5))
    t_out, t_tok = _Tally(name, *tol), _Tally(name + " tok", *tol)
    g = _accum_slack(k, cin) if (accum_tol and split) else 0.0
    w64 = _unplanes(w16, split).view(cout_pad, k, k, cin_pad)[..., :cin].double().permute(0, 3, 1, 2)
    step = _chunk(max(H * W * cin, oh * ow * cout_pad))
    for b0 in range(0, B, step):
        sl = slice(b0, b0 + step)
        xin = _unplanes(x16[sl], split)[..., :cin].double().permute(0, 3, 1, 2)
        acc = F.conv2d(xin, w64, None, stride=stride, padding=pad)
        ref = (acc + bias.double().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
        if up:
            ref = ref + _up2x_ref(_unplanes(up16[sl], split).double(), oh, ow)
        if resid:
            ref = ref + _unplanes(res[sl], split).double()
        if act == 1:
            ref = torch.relu(ref)
        elif act == 2:
            ref = F.leaky_relu(ref, 0.01)
        got = _unplanes(out[sl], split)
        slack = g * (acc.abs() + acc.square().mean().sqrt()).permute(0, 2, 3, 1) if g else 0.0
        t_out.add(got, ref, slack)
        if cout_pad > cout:
            assert got[..., cout:].abs().max().item() == 0.0, "padding channels must stay zero"
        if tokens:
            t_tok.add(_unplanes(tok[sl], split), ref.reshape(-1, oh * ow, cout_pad) + pe.double(),
                      slack.reshape(-1, oh * ow, cout_pad) if g else 0.0)
    t_out.check()
    if tokens:
        t_tok.check()
    return out, tok


# ------------------------------------------------------------------ engine tile log ($OPP_LOG_TILES=1)
TILE_PREFIX = "opp gemm tile: "
_TILES_SEEN = []   # every tile configuration this process has printed, as dicts


@contextlib.contextmanager
def _tile_log():
    """Collects the tile configurations the engine prints while the block runs ($OPP_LOG_TILES=1):
    the yielded list holds them, as dicts ("mode", "n", "block_n", "mma_n", "stages", "cluster", ...),
    when the block ends.  The engine writes them to file descriptor 2, which is redirected meanwhile;
    everything else written there is passed on."""
    new = []
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            yield new
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            f.seek(0)
            for line in f.read().decode(errors="replace").splitlines():
                if line.startswith(TILE_PREFIX):
                    fl = line[len(TILE_PREFIX):].split()
                    new.append({fl[i]: int(fl[i + 1]) if fl[i] != "epi" else fl[i + 1]
                                for i in range(0, len(fl) - 1, 2)})
                else:
                    sys.stderr.write(line + "\n")
            _TILES_SEEN.extend(new)


def _launch_tile(new, mode, n, k, conv_c, epi=None):
    """Tile configuration of the one GEMM launch that ran under _tile_log (`new`).  The engine prints a
    configuration once per process ($OPP_LOG_TILES=1): a launch that printed nothing has the
    configuration of an earlier one with the same (mode, n, k, conv_c), which must then be unique.
    epi: the epilogue name the engine adds to every launch's line at $OPP_LOG_TILES=2 (None: any)."""
    same = lambda t: ((t["mode"], t["n"], t["k"], t["conv_c"]) == (mode, n, k, conv_c)   # noqa: E731
                      and epi in (None, t.get("epi")))
    mine = [t for t in new if same(t)] or [t for t in _TILES_SEEN if same(t)]
    mine = list({tuple((f, v) for f, v in t.items() if epi or f != "epi"): t for t in mine}.values())
    assert len(mine) == 1, f"no unique tile line for mode {mode} n {n} k {k} conv_c {conv_c} epi {epi}: {mine}"
    return mine[0]


def _cluster_tiles(t, batches, m_tiles, grid_m_tiles=None):
    """(fewest, most) tiles one cluster of the persistent grid walks: super tiles of `cluster` adjacent
    M tiles per N tile, dealt round-robin to min(super tiles, SMs / cluster) clusters.  grid_m_tiles:
    the M tiles the grid was sized for when the kernel reads a smaller row count from the device."""
    def sup(m):
        return batches * -(-m // t["cluster"]) * -(-t["n"] // t["block_n"])
    clusters = min(sup(grid_m_tiles or m_tiles), _lib.load().opp_num_sms() // t["cluster"])
    return sup(m_tiles) // clusters, -(-sup(m_tiles) // clusters)


def _conv_tile(new, cin_pad, cout_pad, k, mode=1):
    return _launch_tile(new, mode, cout_pad, k * k * -(-cin_pad // 64) * 64, cin_pad)


def _run_child(name, timeout=900, **env):
    """CHECKS/CHILD_CHECKS entry `name` in a child process with `env` added: the engine reads its knobs
    ($OPP_CLUSTER, $OPP_STAGES, $OPP_NSPLIT, $OPP_LOG_TILES) once per process"""
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", name], env=dict(os.environ, **env),
                       timeout=timeout)
    assert r.returncode == 0, f"{name} failed in a child process with {env}"


def check_conv():
    for split in (0, 1):
        _conv_case(split, 2, 64, 64, 128, 128, 128, 128, 3, 1, 1, True, False)
        _conv_case(split, 1, 64, 96, 128, 128, 196, 208, 3, 2, 1, False, False)
        _conv_case(split, 2, 32, 48, 196, 208, 196, 208, 3, 1, 2, False, False)
        _conv_case(split, 1, 64, 64, 128, 128, 196, 208, 1, 2, 0, False, False)
        _conv_case(split, 2, 30, 40, 256, 256, 256, 256, 1, 1, 0, False, True)
        _conv_case(split, 1, 60, 80, 196, 208, 256, 256, 3, 2, 1, False, False)
        _conv_case(split, 1, 24, 40, 256, 256, 196, 208, 3, 1, 0, False, False)
        # lateral 1x1 convs with the fused upsample-add (resnet.py:149-157), incl. ragged 8x16 tiles
        _conv_case(split, 2, 60, 80, 196, 208, 256, 256, 1, 1, 0, False, False, up=True)
        _conv_case(split, 1, 100, 72, 128, 128, 196, 208, 1, 1, 0, False, False, up=True)
        _conv_case(split, 1, 8, 16, 128, 128, 196, 208, 1, 1, 0, False, False, up=True)


def _conv_up_cases():
    for split in (0, 1):
        _conv_case(split, 2, 60, 80, 196, 208, 256, 256, 1, 1, 0, False, False, up=True)
        _conv_case(split, 1, 100, 72, 128, 128, 196, 208, 1, 1, 0, False, False, up=True)


def check_conv_up_odd_clusters():
    """The fused-upsample convs with an odd number of clusters in the persistent grid.  In fp16x3
    the N = 256 tile does not fit next to its fp32 accumulator and runs as 2 x 128 columns; with an
    odd cluster count a CTA then visits tiles of both column halves, and each tile must use its own
    bias.  The cluster size is read once per process ($OPP_CLUSTER), hence the child process."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    cluster = next((c for c in (4, 2) if (sms // c) % 2 == 1), 4)
    print(f"  OPP_CLUSTER={cluster} ({sms} SMs)")
    _run_child("conv_up", timeout=600, OPP_CLUSTER=str(cluster))


# Every opp_conv2d_nhwc launch of the backbone (model.py _backbone and _fine_head_dense) for 512x512
# images: feature maps of 256^2, 128^2 and 64^2 pixels, batch 8 at the first two output sizes and 32 at
# the last, so that each cluster of the persistent grid walks several tiles (as at bench.py's batch 64:
# the bias staged once per CTA, the ring phase carried from tile to tile, the two warpgroups apart).
# extra: "resid" (a residual map), "resid=input" (the input map is the residual), "tokens" (+ pe into
# the token rows), "up" (+ bilinear x2 of a coarser map).  The expected tile configuration of the
# fp16x3 mode (mma_n, N tiles, ring stages, cluster) is the one bench.py's batch 64 runs with; the
# fp16 mode has deeper rings, so only (mma_n, N tiles) is pinned there.
#  name                  batch  in  cin  cout k  s act extra          fp16x3            fp16
BACKBONE_CONVS = [
    ("layer1 conv1",         8, 256, 128, 128, 3, 1, 1, "",            (128, 1, 3, 2), (128, 1)),
    ("layer1 conv2",         8, 256, 128, 128, 3, 1, 1, "resid=input", (128, 1, 3, 2), (128, 1)),
    ("layer2.0 conv1",       8, 256, 128, 196, 3, 2, 1, "",            (208, 1, 2, 2), (208, 1)),
    ("layer2.0 down",        8, 256, 128, 196, 1, 2, 0, "",            (208, 1, 2, 2), (208, 1)),
    ("layer2 conv2",         8, 128, 196, 196, 3, 1, 1, "resid=input", (208, 1, 2, 2), (208, 1)),
    ("layer3.0 conv1",      32, 128, 196, 256, 3, 2, 1, "",            (256, 1, 2, 2), (256, 1)),
    ("layer3.0 down",       32, 128, 196, 256, 1, 2, 0, "",            (256, 1, 2, 2), (256, 1)),
    ("layer3 conv2",        32,  64, 256, 256, 3, 1, 1, "resid",       (256, 1, 2, 2), (256, 1)),
    ("layer3_outconv",      32,  64, 256, 256, 1, 1, 0, "tokens",      (256, 1, 2, 2), (256, 1)),
    ("layer2_outconv",       8, 128, 196, 256, 1, 1, 0, "up",          (128, 2, 2, 2), (256, 1)),
    ("layer2_outconv2.0",    8, 128, 256, 256, 3, 1, 2, "",            (256, 1, 2, 2), (256, 1)),
    ("layer2_outconv2.3",    8, 128, 256, 196, 3, 1, 0, "",            (208, 1, 2, 2), (208, 1)),
    ("layer1_outconv",       8, 256, 128, 196, 1, 1, 0, "up",          (208, 1, 2, 2), (208, 1)),
    ("layer1_outconv2.0",    8, 256, 196, 196, 3, 1, 2, "",            (208, 1, 2, 2), (208, 1)),
    ("layer1_outconv2.3",    8, 256, 196, 128, 3, 1, 0, "",            (128, 1, 3, 2), (128, 1)),
]


def _backbone_conv(split, name, check=True):
    """one BACKBONE_CONVS launch through _conv_case -> (out, tok, tile line, (fewest, most) tiles per cluster)"""
    (_, B, hw, cin, cout, k, stride, act, extra, _, _) = next(c for c in BACKBONE_CONVS if c[0] == name)
    with _tile_log() as new:
        out, tok = _conv_case(split, B, hw, hw, cin, _pad16(cin), cout, _pad16(cout), k, stride, act,
                              extra.startswith("resid"), extra == "tokens", up=extra == "up",
                              resid_is_input=extra == "resid=input", check=check, accum_tol=True)
    t = _conv_tile(new, _pad16(cin), _pad16(cout), k)
    oh = (hw - 1) // stride + 1
    return out, tok, t, _cluster_tiles(t, B, -(-oh // 16) * -(-oh // 8))


def _conv_layers(split):
    failed = []
    for (name, B, hw, cin, cout, k, stride, act, extra, want1, want0) in BACKBONE_CONVS:
        try:
            _, _, t, (lo, hi) = _backbone_conv(split, name)
            got = (t["mma_n"], -(-t["n"] // t["block_n"]), t["stages"], t["cluster"])
            print(f"  {name}: mma_n {got[0]} N tiles {got[1]} stages {got[2]} alias {t['alias']} cluster {got[3]} "
                  f"tiles per cluster {lo}-{hi}")
            if split:
                assert got == want1, f"{name}: tile (mma_n, N tiles, stages, cluster) = {got}, expected {want1}"
            else:
                assert got[:2] == want0, f"{name}: tile (mma_n, N tiles) = {got[:2]}, expected {want0}"
            assert hi >= 8, f"{name}: only {hi} tiles per cluster at batch {B}"
        except AssertionError as e:   # go on: which launches fail locates a defect
            print(f"  {name}: FAILED: {e}")
            failed.append(name)
    assert not failed, f"split={split}: {failed}"


def check_conv_layers():
    """The backbone's convolutions at production widths and tile configurations against fp64
    (BACKBONE_CONVS), in both operand modes; the tile log shows which configuration each one ran."""
    for split in (1, 0):
        _run_child(f"conv_layers_split{split}", OPP_LOG_TILES="1")


# conv_launch_invariance: per output element the K order, the MMA sequence and the epilogue order do
# not depend on the grid, so which CTA computes a pixel must not change it.  Launch configurations
# forced through the engine's knobs, and the tile fields each must show in the log.
INVARIANCE_VARIANTS = {
    "default": ({}, {"layer1 conv2": {"cluster": 2, "stages": 3}, "layer2 conv2": {"cluster": 2},
                     "layer3_outconv": {"cluster": 2}, "layer3 conv2 batch 1": {"mma_n": 64, "block_n": 64}}),
    # pick_cluster takes 4 where the W slices stay whole swizzle groups (N = 128, 256), not at 208
    "cluster4": ({"OPP_CLUSTER": "4"}, {"layer1 conv2": {"cluster": 4}, "layer2 conv2": {"cluster": 2},
                                        "layer3_outconv": {"cluster": 4}}),
    "stages2": ({"OPP_STAGES": "2"}, {"layer1 conv2": {"stages": 2}}),
    # batch 1 at 64^2: the latency split runs 4 N tiles of 64 columns; without it, one of 256
    "nsplit0": ({"OPP_NSPLIT": "0"}, {"layer3 conv2 batch 1": {"mma_n": 256, "block_n": 256}}),
}


def _conv_variant(tag):
    """The INVARIANCE_VARIANTS[tag] launches (fp16x3) under this process's knobs; outputs saved to
    $KERNEL_CHECK_DIR/<tag>.pt.  The default configuration is also checked against fp64."""
    _, launches = INVARIANCE_VARIANTS[tag]
    saved = {}
    for name, want in launches.items():
        if name == "layer3 conv2 batch 1":
            with _tile_log() as new:
                out, tok = _conv_case(1, 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, True, False, check=tag == "default",
                                      accum_tol=True)
            t = _conv_tile(new, 256, 256, 3)
        else:
            out, tok, t, _ = _backbone_conv(1, name, check=tag == "default")
        print(f"  [{tag}] {name}: mma_n {t['mma_n']} block_n {t['block_n']} stages {t['stages']} cluster {t['cluster']}")
        assert all(t[f] == v for f, v in want.items()), f"[{tag}] {name}: tile {t}, expected {want}"
        saved[name] = (out.cpu(), tok.cpu() if tok is not None else None)
    torch.save(saved, os.path.join(os.environ["KERNEL_CHECK_DIR"], f"{tag}.pt"))


def _conv_batch_slices():
    """The dominant launch as bench.py runs it: layer1.x conv2 (3x3 128->128 + the block input, ReLU)
    over batch 64 of 512x512 images in the fp16x3 mode, with the conv input, the block input and the
    output 2 GiB each.  NaN-free, and every 8-image slice bit-identical to a batch-8 launch on the same
    images (the configuration conv_layers checks against fp64) - every tile of the batch-64 launch is
    checked without an fp64 reference at batch 64.  Likewise at N = 208, where no knob changes the
    launch: each image of the batch-8 layer2 conv2 (7-8 tiles per cluster) against a batch-1 launch
    of that image (one tile per cluster)."""
    B, hw, c = 64, 256, 128
    t64 = _nhwc_planes(B, hw, hw, c, c, 1, seed=1)     # t: the output of the block's conv1
    x64 = _nhwc_planes(B, hw, hw, c, c, 1, seed=4)     # the block input, added as the residual
    w16, bias = _conv_params(c, c, c, c, 3, 1)
    out64 = torch.full((B, hw, hw, 2 * c), float("nan"), device=DEV, dtype=torch.half)
    with _tile_log() as new:
        ops.conv2d_nhwc(t64, w16, bias, out64, 3, 1, 1, act=1, resid=x64)
    t_big = _conv_tile(new, c, c, 3)
    lo, hi = _cluster_tiles(t_big, B, (hw // 16) * (hw // 8))
    print(f"  batch 64: mma_n {t_big['mma_n']} stages {t_big['stages']} cluster {t_big['cluster']} "
          f"tiles per cluster {lo}-{hi}")
    out8 = torch.empty(8, hw, hw, 2 * c, device=DEV, dtype=torch.half)
    differ = []
    for b0 in range(0, B, 8):
        sl = slice(b0, b0 + 8)
        assert not torch.isnan(out64[sl]).any(), f"batch 64: NaN (unwritten) outputs in images {b0}-{b0 + 7}"
        out8.fill_(float("nan"))
        with _tile_log() as new:
            ops.conv2d_nhwc(t64[sl], w16, bias, out8, 3, 1, 1, act=1, resid=x64[sl])
        t8 = _conv_tile(new, c, c, 3)
        assert all(t8[f] == t_big[f] for f in ("mma_n", "stages", "cluster")), (t8, t_big)
        if not _bits_equal(out8, out64[sl]):
            differ.append(f"images {b0}-{b0 + 7}: {int((out8 != out64[sl]).sum())} elements")
    assert not differ, f"batch-64 launch differs from batch-8 launches of the same images: {differ}"
    print("  batch 64: NaN-free, every 8-image slice bit-identical to its batch-8 launch")
    del t64, x64, out64, out8
    B, hw, c, c_pad = 8, 128, 196, 208
    x8 = _nhwc_planes(B, hw, hw, c, c_pad, 1, seed=1)
    w16, bias = _conv_params(c, c_pad, c, c_pad, 3, 1)
    out8 = torch.full((B, hw, hw, 2 * c_pad), float("nan"), device=DEV, dtype=torch.half)
    with _tile_log() as new:
        ops.conv2d_nhwc(x8, w16, bias, out8, 3, 1, 1, act=1, resid=x8)
    t8 = _conv_tile(new, c_pad, c_pad, 3)
    lo8 = _cluster_tiles(t8, B, (hw // 16) * (hw // 8))[0]
    assert t8["mma_n"] == 208 and lo8 > 1, t8
    assert not torch.isnan(out8).any(), "N = 208: NaN (unwritten) outputs in the batch-8 launch"
    out1 = torch.empty(1, hw, hw, 2 * c_pad, device=DEV, dtype=torch.half)
    for b in range(B):
        out1.fill_(float("nan"))
        with _tile_log() as new:
            ops.conv2d_nhwc(x8[b:b + 1], w16, bias, out1, 3, 1, 1, act=1, resid=x8[b:b + 1])
        t1 = _conv_tile(new, c_pad, c_pad, 3)
        assert t1["mma_n"] == 208 and _cluster_tiles(t1, 1, (hw // 16) * (hw // 8))[1] < lo8, t1
        if not _bits_equal(out1, out8[b:b + 1]):
            differ.append(f"image {b}: {int((out1 != out8[b:b + 1]).sum())} elements")
    assert not differ, f"N = 208: batch-8 launch differs from batch-1 launches of the same images: {differ}"
    print("  N = 208: every image of the batch-8 launch bit-identical to its batch-1 launch")


def check_conv_launch_invariance():
    """INVARIANCE_VARIANTS against the default configuration, bit for bit, and _conv_batch_slices."""
    with tempfile.TemporaryDirectory() as d:
        for tag, (env, _) in INVARIANCE_VARIANTS.items():
            _run_child(f"conv_variant_{tag}", OPP_LOG_TILES="1", KERNEL_CHECK_DIR=d, **env)
        base = torch.load(os.path.join(d, "default.pt"))
        differ = []
        for tag in INVARIANCE_VARIANTS:
            if tag == "default":
                continue
            for name, tensors in torch.load(os.path.join(d, f"{tag}.pt")).items():
                for what, a, b in zip(("out", "tok"), tensors, base[name]):
                    if a is None:
                        continue
                    if _bits_equal(a, b):
                        print(f"  {tag} vs default, {name} {what}: bit-identical")
                        continue
                    diff = (_unplanes(a, 1) - _unplanes(b, 1)).abs().max().item()
                    print(f"  {tag} vs default, {name} {what}: {int((a != b).sum())} fp16 elements differ, "
                          f"max |diff| of the represented values {diff:.3e}")
                    differ.append(f"{tag}: {name} {what}")
    _run_child("conv_batch_slices", OPP_LOG_TILES="1")
    assert not differ, f"outputs depend on the launch configuration: {differ}"


def _win_mismatches(got, dense, b_ids, j_ids, wc, win, org, outside_zero, stride=4):
    """Window positions (match, ly, lx) of opp_conv_win's compact output `got` [>= M, win, pitch, C]
    whose fp16 bits differ from the dense map `dense` [B, H, W, C] at image position
    (stride * cell + org + (ly, lx)), for the M = len(j_ids) matches.  Positions outside the image
    must be zero when outside_zero (conv A's 7x7 windows: they are conv B's zero padding), else they
    are not compared (conv B's 5x5 windows: the gather never reads them)."""
    M = j_ids.numel()
    _, H, W, _ = dense.shape
    r = torch.arange(win, device=DEV)
    y = (stride * (j_ids // wc) + org).view(M, 1, 1) + r.view(1, win, 1)
    x = (stride * (j_ids % wc) + org).view(M, 1, 1) + r.view(1, 1, win)
    inside = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    want = dense[b_ids.view(M, 1, 1), y.clamp(0, H - 1), x.clamp(0, W - 1)]
    want = torch.where(inside[..., None], want, torch.zeros_like(want))
    differs = (got[:M, :, :win].view(torch.int16) != want.view(torch.int16)).any(-1)
    if not outside_zero:
        differs &= inside
    return int(differs.sum())


def check_conv_win():
    """opp_conv_win (3x3 convolutions on per-match windows, the sparse form of layer1_outconv2)
    against the dense convolutions of the same engine (bit-equal at the window positions: same K
    order, same MMA sequence) and against fp64 torch; matches on the image border (zero padding of
    both convolutions, windows reaching outside the map) and ragged tile counts included."""
    from onepose_plus_plus_b200 import ops
    for split in (0, 1):
        pl = 2 if split else 1
        for (B, H, W, M, dyn) in [(2, 64, 96, 37, False), (1, 32, 32, 64, True), (3, 40, 72, 1, False),
                                  (1, 64, 64, 200, True)]:
            hc, wc = H // 4, W // 4
            cin, cin_pad, cmid, cmid_pad, cout = 196, 208, 196, 208, 128
            xf = torch.zeros(B, H, W, cin_pad, device=DEV)
            xf[..., :cin] = _rand(B, H, W, cin, seed=1)
            w0f = torch.zeros(cmid_pad, 3, 3, cin_pad, device=DEV)
            w0f[:cmid, :, :, :cin] = _rand(cmid, 3, 3, cin, scale=1.0 / math.sqrt(9 * cin), seed=2)
            b0 = torch.zeros(cmid_pad, device=DEV)
            b0[:cmid] = _rand(cmid, seed=3) * 0.1
            w1f = torch.zeros(cout, 3, 3, cmid_pad, device=DEV)
            w1f[:, :, :, :cmid] = _rand(cout, 3, 3, cmid, scale=1.0 / math.sqrt(9 * cmid), seed=4)
            b1 = _rand(cout, seed=5) * 0.1
            x16 = _planes(xf, split)
            w0, w1 = _planes(w0f.reshape(cmid_pad, -1), split), _planes(w1f.reshape(cout, -1), split)
            g = torch.Generator().manual_seed(7)
            b_ids = torch.randint(0, B, (M,), generator=g).sort().values
            j_ids = torch.randint(0, hc * wc, (M,), generator=g)
            j_ids[: min(M, 4)] = torch.tensor([0, wc - 1, (hc - 1) * wc, hc * wc - 1])[: min(M, 4)]   # corners
            b_ids, j_ids = b_ids.to(DEV), j_ids.to(DEV)
            # dense reference on the same engine
            t_d = torch.empty(B, H, W, pl * cmid_pad, device=DEV, dtype=torch.half)
            o_d = torch.empty(B, H, W, pl * cout, device=DEV, dtype=torch.half)
            ops.conv2d_nhwc(x16, w0, b0, t_d, 3, 1, split, 2)
            ops.conv2d_nhwc(t_d, w1, b1, o_d, 3, 1, split, 0)
            cap = M + 5 if dyn else M
            count = torch.tensor([M], dtype=torch.int32, device=DEV) if dyn else None
            bi = torch.cat([b_ids, b_ids.new_zeros(cap - M)]) if dyn else b_ids
            ji = torch.cat([j_ids, j_ids.new_zeros(cap - M)]) if dyn else j_ids
            t_w = torch.full((cap, 7, 8, pl * cmid_pad), float("nan"), device=DEV, dtype=torch.half)
            o_w = torch.full((cap, 5, ops.conv_win_pitch(5), pl * cout), float("nan"), device=DEV, dtype=torch.half)
            ops.conv_win(x16, w0, b0, t_w, 7, split, cap, act=2, b_ids=bi, j_ids=ji, wc=wc, stride=4, org=-3,
                         count=count)
            ops.conv_win(t_w, w1, b1, o_w, 5, split, cap, count=count)
            torch.cuda.synchronize()
            bad_t = _win_mismatches(t_w, t_d, b_ids, j_ids, wc, 7, -3, True)
            bad_o = _win_mismatches(o_w, o_d, b_ids, j_ids, wc, 5, -2, False)
            assert bad_t == 0 and bad_o == 0, (f"conv_win split={split} B={B} {H}x{W} M={M} dyn={dyn}: {bad_t} window "
                                               f"positions of conv A and {bad_o} of conv B differ from the dense conv")
            if dyn:
                assert torch.isnan(o_w[M:].float()).all(), "rows past the device-side match count were written"
            # and the dense engine result itself against fp64 torch (layer1_outconv2 shape)
            ref = F.leaky_relu(F.conv2d(_q(xf, split).double().permute(0, 3, 1, 2),
                                        _q(w0f, split).double().permute(0, 3, 1, 2), b0.double(), padding=1), 0.01)
            _close(f"conv_win dense-ref split={split}", _unplanes(t_d, split), ref.permute(0, 2, 3, 1).float(),
                   *_tol(split, (2e-3, 3e-3), (2e-5, 2e-5)))
            print(f"conv_win split={split} B={B} {H}x{W} M={M} dyn={dyn}: windows bit-equal to the dense conv")


def _conv_win_production():
    """The window head (layer1_outconv2 on the match windows, model.py _fine_head_windows) at what a
    batch of 512x512 images produces: 3000 matches over four 256x256 half-resolution maps, a
    device-side match count below the capacity, windows on all four image borders.  Both window convs
    must equal the dense convolutions of the same engine bit for bit (conv_layers checks those against
    fp64 at this configuration), rows past the count must stay NaN, and every cluster of the
    persistent grid must walk more than one tile."""
    B, H, W, M, cap, stride = 4, 256, 256, 3000, 3100, 4
    hc, wc = H // stride, W // stride
    cin, cmid, cout = 196, 196, 128
    for split in (0, 1):
        pl = 2 if split else 1
        x16 = _nhwc_planes(B, H, W, cin, _pad16(cin), split, seed=1)
        w0, b0 = _conv_params(cin, _pad16(cin), cmid, _pad16(cmid), 3, split)
        w1, b1 = _conv_params(cmid, _pad16(cmid), cout, cout, 3, split)
        t_d = torch.empty(B, H, W, pl * _pad16(cmid), device=DEV, dtype=torch.half)
        o_d = torch.empty(B, H, W, pl * cout, device=DEV, dtype=torch.half)
        ops.conv2d_nhwc(x16, w0, b0, t_d, 3, 1, split, 2)
        ops.conv2d_nhwc(t_d, w1, b1, o_d, 3, 1, split, 0)
        g = torch.Generator().manual_seed(11)
        b_ids = torch.randint(0, B, (M,), generator=g).sort().values
        cy, cx = torch.randint(0, hc, (M,), generator=g), torch.randint(0, wc, (M,), generator=g)
        # every 7th match on an image border: top, bottom, left, right in turn (the corners among them)
        side = torch.arange(0, M, 7) // 7 % 4
        cy[::7] = torch.where(side == 0, 0, torch.where(side == 1, hc - 1, cy[::7]))
        cx[::7] = torch.where(side == 2, 0, torch.where(side == 3, wc - 1, cx[::7]))
        cy[:4], cx[:4] = torch.tensor([0, 0, hc - 1, hc - 1]), torch.tensor([0, wc - 1, 0, wc - 1])
        b_ids, j_ids = b_ids.to(DEV), (cy * wc + cx).to(DEV)
        count = torch.tensor([M], dtype=torch.int32, device=DEV)
        bi, ji = torch.cat([b_ids, b_ids.new_zeros(cap - M)]), torch.cat([j_ids, j_ids.new_zeros(cap - M)])
        t_w = torch.full((cap, 7, 8, pl * _pad16(cmid)), float("nan"), device=DEV, dtype=torch.half)
        o_w = torch.full((cap, 5, ops.conv_win_pitch(5), pl * cout), float("nan"), device=DEV, dtype=torch.half)
        with _tile_log() as new_a:
            ops.conv_win(x16, w0, b0, t_w, 7, split, cap, act=2, b_ids=bi, j_ids=ji, wc=wc, stride=stride, org=-3,
                         count=count)
        with _tile_log() as new_b:
            ops.conv_win(t_w, w1, b1, o_w, 5, split, cap, count=count)
        torch.cuda.synchronize()
        name = f"conv_win_production split={split} B={B} {H}x{W} M={M} of {cap}"
        for (new, win, c_in, c_out) in ((new_a, 7, _pad16(cin), _pad16(cmid)), (new_b, 5, _pad16(cmid), cout)):
            t = _conv_tile(new, c_in, c_out, 3, mode=2)
            per_tile = 128 // (ops.conv_win_pitch(win) * win)
            lo, hi = _cluster_tiles(t, 1, -(-M // per_tile), grid_m_tiles=-(-cap // per_tile))
            print(f"  {name} {win}x{win} windows: mma_n {t['mma_n']} stages {t['stages']} cluster {t['cluster']} "
                  f"tiles per cluster {lo}-{hi}")
            assert lo > 1, f"{name}: a cluster walks only {lo} tile(s) of the {win}x{win} window conv"
        bad_t = _win_mismatches(t_w, t_d, b_ids, j_ids, wc, 7, -3, True, stride)
        bad_o = _win_mismatches(o_w, o_d, b_ids, j_ids, wc, 5, -2, False, stride)
        assert bad_t == 0 and bad_o == 0, (f"{name}: {bad_t} window positions of conv A and {bad_o} of conv B "
                                           f"differ from the dense conv")
        assert torch.isnan(t_w[M:].float()).all() and torch.isnan(o_w[M:].float()).all(), \
            f"{name}: rows past the device-side match count were written"
        print(f"  {name}: windows bit-equal to the dense conv, rows past the count untouched")


def check_conv_win_production():
    _run_child("conv_win_production_tiles", OPP_LOG_TILES="1")


# ------------------------------------------------------------------------------------------ SIMT
def _conv1_gemm_case(split, B, H, W, C, u8):
    """conv1 as im2col + one 64-wide wgmma K chunk (bias in K column 49), fp32 and uint8 images"""
    if u8:
        img = torch.randint(0, 256, (B, 1, H, W), device=DEV, dtype=torch.uint8)
        imgf = img.float() / 255.0
    else:
        img = imgf = torch.rand(B, 1, H, W, device=DEV)
    w = _rand(C, 1, 7, 7, scale=0.15, seed=2)
    bias = _rand(C, seed=3) * 0.1
    w64 = torch.zeros(C, 64, device=DEV)
    w64[:, :49] = w.view(C, 49)
    w64[:, 49] = bias
    w16 = _planes(w64, split)
    pl = 2 if split else 1
    a_buf = torch.full((B * (H // 2) * (W // 2), pl * 64), float("nan"), device=DEV, dtype=torch.half)
    out = torch.full((B, H // 2, W // 2, pl * C), float("nan"), device=DEV, dtype=torch.half)
    ops.conv1_gemm(img, w16, a_buf, out, split)
    torch.cuda.synchronize()
    wq = _q(w64, split).double()
    tally = _Tally(f"conv1_gemm split={split} u8={u8} B={B} {H}x{W}", *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))
    step = _chunk(H * W * C // 4)
    for b0 in range(0, B, step):
        sl = slice(b0, b0 + step)
        ref = torch.relu(F.conv2d(imgf[sl].double(), wq[:, :49].reshape(C, 1, 7, 7), wq[:, 49], stride=2, padding=3))
        tally.add(_unplanes(out[sl], split), ref.permute(0, 2, 3, 1))
    tally.check()


def check_conv1_gemm():
    for split in (0, 1):
        _conv1_gemm_case(split, 2, 96, 128, 128, False)
        _conv1_gemm_case(split, 1, 72, 200, 128, True)     # ragged 16x16 im2col tiles, uint8 image
        # bench.py's image size: 524288 im2col rows per batch of 8
        _conv1_gemm_case(split, 8, 512, 512, 128, False)
        _conv1_gemm_case(split, 8, 512, 512, 128, True)


def check_kpt_encode():
    for split in (0, 1):
        B, N = 2, 1003
        kpts = torch.rand(B, N, 3, device=DEV) - 0.5
        desc = _rand(B, 256, N, seed=1)
        dims = [3, 32, 64, 128, 256]
        ws = [_rand(dims[i + 1], dims[i], scale=1 / math.sqrt(dims[i]), seed=10 + i) for i in range(4)]
        bs = [_rand(dims[i + 1], seed=20 + i) * 0.1 for i in range(4)]
        stats = torch.empty(B, 4, device=DEV)
        pl = 2 if split else 1
        tok = torch.empty(B, N, pl * 256, device=DEV, dtype=torch.half)
        _lib.call("opp_kpt_stats", _lib.ptr(kpts), _lib.ptr(stats), B, N, _lib.stream())
        wts = [w.t().contiguous() for w in ws]
        _lib.call("opp_kpt_encode", _lib.ptr(kpts), _lib.ptr(stats), _lib.ptr(desc), _lib.ptr(wts[0]),
                  _lib.ptr(bs[0]), _lib.ptr(wts[1]), _lib.ptr(bs[1]), _lib.ptr(wts[2]), _lib.ptr(bs[2]),
                  _lib.ptr(wts[3]), _lib.ptr(bs[3]), _lib.ptr(tok), B, N, split, _lib.stream())
        torch.cuda.synchronize()
        ext = (kpts[0].max(0).values - kpts[0].min(0).values).max() * 0.6
        x = (kpts - kpts.mean(1, keepdim=True)) / ext
        for i in range(4):
            x = x @ ws[i].t() + bs[i]
            if i < 3:
                m = x.mean(-1, keepdim=True)
                v = x.var(-1, unbiased=False, keepdim=True)
                x = torch.relu((x - m) / torch.sqrt(v + 1e-5))
        ref = desc.transpose(1, 2) + x
        _close(f"kpt_encode split={split}", _unplanes(tok, split), ref, *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))


def check_kv_state():
    """single-plane K'/V rows (what the forward writes in both operand modes) -> KV state, with the
    mt output in both plane modes"""
    for split in (0, 1):
        B, S, d = 2, 1000, 256
        kvf = torch.cat([_rand(B, S, d, seed=1).abs() + 0.1, _rand(B, S, d, seed=2)], 2)
        kv = _planes(kvf, 0)
        mw = _rand(d, d, scale=0.06, seed=3)
        chunks = _lib.load().opp_kv_chunks_b(S, B)
        pl = 2 if split else 1
        part = torch.empty(B, chunks, 8, 33, 32, device=DEV)
        mt = torch.empty(B, d, pl * d, device=DEV, dtype=torch.half)
        ksum = torch.empty(B, d, device=DEV)
        _lib.call("opp_kv_partial", _lib.ptr(kv), _lib.ptr(part), B, S, d, _lib.stream())
        _lib.call("opp_kv_finalize", _lib.ptr(part), _lib.ptr(mw), _lib.ptr(mt), _lib.ptr(ksum), B,
                  chunks, d, float(S), split, _lib.stream())
        torch.cuda.synchronize()
        kvq = _q(kvf, 0).double()
        K = kvq[..., :d].view(B, S, 8, 32)
        V = kvq[..., d:].view(B, S, 8, 32)
        KV = torch.einsum("bshd,bshv->bhdv", K, V) / S
        ref_ksum = K.sum(1).reshape(B, d).float()
        # mt[b][c][h*32+dd] = sum_v mw[c][h*32+v] KV[b][h][dd][v]
        ref_mt = torch.einsum("chv,bhdv->bchd", mw.double().view(d, 8, 32), KV).reshape(B, d, d).float()
        _close(f"kv ksum split={split}", ksum, ref_ksum, 1e-5, 1e-3)
        _close("kv mt", _unplanes(mt, split), ref_mt, *_tol(split, (2e-3, 1e-4), (2e-5, 1e-6)))


def check_fine():
    for split in (0, 1):
        B, hf, wf, N, wc = 2, 64, 80, 500, 20
        M = 333
        pl = 2 if split else 1
        finef = _rand(B, hf, wf, 128, seed=1)
        fine = _planes(finef, split)
        desc = _rand(B, 128, N, seed=2)
        g = torch.Generator().manual_seed(1)
        b_ids = torch.randint(0, B, (M,), generator=g).sort().values.to(DEV)
        i_ids = torch.randint(0, N, (M,), generator=g).to(DEV)
        j_ids = torch.randint(0, (hf // 4) * wc, (M,), generator=g).to(DEV)
        x32 = torch.empty(M * 26, 128, device=DEV)
        x16 = torch.empty(M * 26, pl * 128, device=DEV, dtype=torch.half)
        _lib.call("opp_fine_gather", _lib.ptr(fine), _lib.ptr(desc), _lib.ptr(b_ids), _lib.ptr(i_ids),
                  _lib.ptr(j_ids), _lib.ptr(x32), _lib.ptr(x16), M, hf, wf, wc, 4, N, split, 0, 0, None, _lib.stream())
        torch.cuda.synchronize()
        unf = F.unfold(_q(finef, split).permute(0, 3, 1, 2), kernel_size=5, stride=4, padding=2)
        unf = unf.view(B, 128, 25, -1).permute(0, 3, 2, 1)  # n l ww c
        ref = torch.cat([desc.permute(0, 2, 1)[b_ids, i_ids][:, None], unf[b_ids, j_ids]], 1)
        assert torch.equal(x32.view(M, 26, 128), ref), "fine_gather mismatch"
        _close(f"fine_gather planes split={split}", _unplanes(x16, split), x32, *_tol(split, (1e-3, 1e-3), (1e-6, 1e-6)))

        # attention
        qkvf = torch.cat([_rand(M * 26, 256, seed=3).abs() + 0.05, _rand(M * 26, 128, seed=4)], 1)
        qkv = _planes(qkvf, split)
        for cross in (0, 1):
            msg = torch.empty(M * 26, pl * 128, device=DEV, dtype=torch.half)
            _lib.call("opp_fine_attention", _lib.ptr(qkv), _lib.ptr(msg), M, cross, 1e-6, split, None, _lib.stream())
            torch.cuda.synchronize()
            t = _q(qkvf, split).double().view(M, 26, 3, 8, 16)
            Q, K, V = t[:, :, 0], t[:, :, 1], t[:, :, 2]

            def attn(q, k, v):
                vl = v.size(1)
                kvm = torch.einsum("nshd,nshv->nhdv", k, v / vl)
                z = 1 / (torch.einsum("nlhd,nhd->nlh", q, k.sum(1)) + 1e-6)
                return torch.einsum("nlhd,nhdv,nlh->nlhv", q, kvm, z) * vl

            if cross == 0:
                m3 = attn(Q[:, :1], K[:, :1], V[:, :1])
                m2 = attn(Q[:, 1:], K[:, 1:], V[:, 1:])
            else:
                m3 = attn(Q[:, :1], K[:, 1:], V[:, 1:])
                m2 = attn(Q[:, 1:], K[:, :1], V[:, :1])
            ref = torch.cat([m3, m2], 1).reshape(M * 26, 128).float()
            _close(f"fine_attention split={split} cross={cross}", _unplanes(msg, split), ref,
                   *_tol(split, (2e-3, 1e-3), (2e-5, 2e-6)))

    # matching
    B, M = 2, 333
    g = torch.Generator().manual_seed(1)
    b_ids = torch.randint(0, B, (M,), generator=g).sort().values.to(DEV)
    xf = _rand(M * 26, 128, seed=5)
    mkc = torch.rand(M, 2, device=DEV) * 300
    scale = torch.rand(B, 2, device=DEV) + 0.5
    ef = torch.empty(M, 3, device=DEV)
    mf = torch.empty(M, 2, device=DEV)
    _lib.call("opp_fine_match", _lib.ptr(xf), _lib.ptr(mkc), _lib.ptr(b_ids), _lib.ptr(scale),
              _lib.ptr(ef), _lib.ptr(mf), M, 2.0, None, _lib.stream())
    torch.cuda.synchronize()
    x = xf.view(M, 26, 128)
    sim = torch.einsum("mc,mrc->mr", x[:, 0], x[:, 1:]) / math.sqrt(128)
    hm = torch.softmax(sim, 1)
    lin = torch.linspace(-1, 1, 5, device=DEV)
    gx = lin.repeat(5)
    gy = lin.repeat_interleave(5)
    grid = torch.stack([gx, gy], 1)
    co = hm @ grid
    var = hm @ grid ** 2 - co ** 2
    std = torch.sqrt(var.clamp(min=1e-10)).sum(-1)
    _close("fine_match expec_f", ef, torch.cat([co, std[:, None]], 1), 1e-4, 1e-5)
    _close("fine_match mkpts_f", mf, mkc + co * 2 * (2.0 * scale[b_ids][:, [1, 0]]), 1e-5, 1e-4)


def check_full_attention():
    """opp_full_attention against softmax(QK^T/sqrt(D))V in fp64 (linear_attention.py:64-95)"""
    for split in (0, 1):
        for (B, L, S, H, D) in [(2, 300, 517, 8, 32), (1, 130, 64, 8, 32), (3, 26, 25, 8, 16)]:
            dm = H * D
            qf = _rand(B * L, dm, seed=1)
            kvf = torch.cat([_rand(B * S, dm, seed=2), _rand(B * S, dm, seed=3)], 1)
            pl = 2 if split else 1
            out = torch.full((B * L, pl * dm), float("nan"), device=DEV, dtype=torch.half)
            ops.full_attention(_planes(qf, split), _planes(kvf, split), out, B, L, S, H, D, split)
            torch.cuda.synchronize()
            q = _q(qf, split).double().view(B, L, H, D)
            k = _q(kvf[:, :dm], split).double().view(B, S, H, D)
            v = _q(kvf[:, dm:], split).double().view(B, S, H, D)
            a = torch.softmax(torch.einsum("nlhd,nshd->nlsh", q, k) / D ** 0.5, dim=2)
            ref = torch.einsum("nlsh,nshd->nlhd", a, v).reshape(B * L, dm).float()
            _close(f"full_attention split={split} B={B} L={L} S={S} D={D}", _unplanes(out, split), ref,
                   *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))


# ------------------------------------------------------------------------------ LoFTR 2D-2D kernels
def check_loftr_kernels():
    """opp_seq_attention / opp_fine_gather_2d / opp_fine_match_2d / opp_match_select_2d against torch
    restatements of submodules/LoFTR/src/loftr (linear_attention.py, fine_preprocess.py:41-49,
    fine_matching.py:46-70, coarse_matching.py:9-28,197-253)."""
    g = torch.Generator().manual_seed(3)
    for split in (0, 1):
        pl = 2 if split else 1
        # linear attention between token groups
        for (G, L, S) in [(37, 81, 81), (5, 25, 25), (3, 81, 30)]:
            qf = _rand(G * L, 128, seed=1).abs() + 0.05
            kvf = torch.cat([_rand(G * S, 128, seed=2).abs() + 0.05, _rand(G * S, 128, seed=3)], 1)
            out = torch.full((G * L, pl * 128), float("nan"), device=DEV, dtype=torch.half)
            ops.seq_attention(_planes(qf, split), _planes(kvf, split), out, G, L, S, split)
            torch.cuda.synchronize()
            Q = _q(qf, split).double().view(G, L, 8, 16)
            K = _q(kvf[:, :128], split).double().view(G, S, 8, 16)
            V = _q(kvf[:, 128:], split).double().view(G, S, 8, 16)
            kvm = torch.einsum("nshd,nshv->nhdv", K, V / S)
            z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, K.sum(1)) + 1e-6)
            ref = (torch.einsum("nlhd,nhdv,nlh->nlhv", Q, kvm, z) * S).reshape(G * L, 128).float()
            _close(f"seq_attention split={split} G={G} L={L} S={S}", _unplanes(out, split), ref,
                   *_tol(split, (2e-3, 1e-3), (2e-5, 2e-6)))
        # W x W windows of both fine maps, sequence-major
        B, hf, wf, wc, W, M = 2, 48, 64, 16, 9, 150
        f0f, f1f = _rand(B, hf, wf, 128, seed=4), _rand(B, hf, wf, 128, seed=5)
        b_ids = torch.randint(0, B, (M,), generator=g).sort().values.to(DEV)
        i_ids = torch.randint(0, (hf // 4) * wc, (M,), generator=g).to(DEV)
        j_ids = torch.randint(0, (hf // 4) * wc, (M,), generator=g).to(DEV)
        x16 = torch.full((2 * M * W * W, pl * 128), float("nan"), device=DEV, dtype=torch.half)
        ops.fine_gather_2d(_planes(f0f, split), _planes(f1f, split), b_ids, i_ids, j_ids, x16, M, hf, wf, wc, hf, wf,
                           wc, 4, W, split)
        torch.cuda.synchronize()

        def unfold(f):
            u = F.unfold(_q(f, split).permute(0, 3, 1, 2), kernel_size=W, stride=4, padding=W // 2)
            return u.view(B, 128, W * W, -1).permute(0, 3, 2, 1)

        ref = torch.cat([unfold(f0f)[b_ids, i_ids], unfold(f1f)[b_ids, j_ids]], 0).reshape(2 * M * W * W, 128)
        _close(f"fine_gather_2d split={split}", _unplanes(x16, split), ref, *_tol(split, (1e-3, 1e-3), (1e-6, 1e-6)))
    # fine matching, W = 9 and 5
    for W in (9, 5):
        M, B = 211, 2
        WW = W * W
        xf = _rand(2 * M * WW, 128, seed=6)
        mk1c = torch.rand(M, 2, device=DEV) * 300
        b_ids = torch.randint(0, B, (M,), generator=g).sort().values.to(DEV)
        scale1 = torch.rand(B, 2, device=DEV) + 0.5
        ef, mf = torch.empty(M, 3, device=DEV), torch.empty(M, 2, device=DEV)
        ops.fine_match_2d(xf, mk1c, b_ids, scale1, ef, mf, M, W, 2.0)
        torch.cuda.synchronize()
        x = xf.view(2, M, WW, 128)
        hm = torch.softmax(torch.einsum("mc,mrc->mr", x[0][:, WW // 2], x[1]) / math.sqrt(128), 1)
        lin = torch.linspace(-1, 1, W, device=DEV)
        grid = torch.stack([lin.repeat(W), lin.repeat_interleave(W)], 1)
        co = hm @ grid
        std = torch.sqrt((hm @ grid ** 2 - co ** 2).clamp(min=1e-10)).sum(-1)
        _close(f"fine_match_2d W={W} expec_f", ef, torch.cat([co, std[:, None]], 1), 1e-4, 2e-5)
        _close(f"fine_match_2d W={W} mkpts1_f", mf, mk1c + co * (W // 2) * (2.0 * scale1[b_ids]), 1e-5, 2e-4)
    # match selection on two image grids
    B, h0, w0, h1, w1 = 2, 12, 16, 10, 20
    L, S = h0 * w0, h1 * w1
    conf = torch.rand(B, L, S, device=DEV) * 0.3
    idx = torch.randperm(L, generator=g)[:90]
    conf[0, idx, torch.randperm(S, generator=g)[:90]] = 0.5 + 0.4 * torch.rand(90, device=DEV)
    conf[1, idx[:60], torch.randperm(S, generator=g)[:60]] = 0.5 + 0.4 * torch.rand(60, device=DEV)
    pt_val, pt_idx = conf.max(2)
    colmax = conf.max(1).values.contiguous().view(torch.int32)
    cap = B * L
    outs = [torch.empty(cap, dtype=torch.int64, device=DEV) for _ in range(3)]
    mconf, mk0, mk1 = torch.empty(cap, device=DEV), torch.empty(cap, 2, device=DEV), torch.empty(cap, 2, device=DEV)
    cnt = torch.zeros(1, device=DEV, dtype=torch.int32)
    s0, s1 = torch.rand(B, 2, device=DEV) + 0.5, torch.rand(B, 2, device=DEV) + 0.5
    ops.match_select_2d(pt_val.contiguous(), pt_idx.int().contiguous(), colmax, s0, s1, B, h0, w0, h1, w1, 0.2, 2, 8.0,
                        torch.empty((cap + 1023) // 1024 + 2, device=DEV, dtype=torch.int32), *outs, mconf, mk0, mk1, cnt)
    torch.cuda.synchronize()
    M = int(cnt.item())
    mask = (conf > 0.2).view(B, h0, w0, h1, w1).clone()
    for d in (1, 2, 3, 4):
        sl = [slice(None)] * 5
        sl[d] = slice(0, 2)
        mask[tuple(sl)] = False
        sl[d] = slice(-2, None)
        mask[tuple(sl)] = False
    mask = mask.view(B, L, S) * (conf == conf.max(2, keepdim=True)[0]) * (conf == conf.max(1, keepdim=True)[0])
    mv, aj = mask.max(2)
    rb, ri = torch.where(mv)
    rj = aj[rb, ri]
    assert M == len(rb) and M > 40, (M, len(rb))
    assert torch.equal(outs[0][:M], rb) and torch.equal(outs[1][:M], ri) and torch.equal(outs[2][:M], rj)
    assert torch.equal(mconf[:M], conf[rb, ri, rj])
    _close("match_select_2d mkpts0_c", mk0[:M], torch.stack([ri % w0, ri // w0], 1) * 8.0 * s0[rb], 1e-6, 1e-4)
    _close("match_select_2d mkpts1_c", mk1[:M], torch.stack([rj % w1, rj // w1], 1) * 8.0 * s1[rb], 1e-6, 1e-4)


# ------------------------------------------------------------------------------ one-pass dual softmax
def check_sim_colmax():
    for split in (0, 1):
        for (B, L, S, K) in [(2, 700, 520, 256), (1, 300, 100, 256), (1, 5000, 4096, 256)]:
            af = _rand(B, L, K, scale=0.9, seed=1)
            bf = _rand(B, S, K, scale=0.9, seed=2)
            a, b = _planes(af, split), _planes(bf, split)
            scale = 1.0 / (256 * 0.0801)
            sim = (torch.einsum("blk,bsk->bls", _q(af, split).double(), _q(bf, split).double()) * scale)
            ts, groups = _lib.load().opp_sim_tiles(S), (L + 31) // 32
            lse_pt, lse_px = torch.empty(B, L, device=DEV), torch.empty(B, S, device=DEV)
            ops.sim_lse_cols(a, b, B, L, S, K, scale, torch.empty(B * L, ts, device=DEV),
                             torch.empty(B * L, ts, device=DEV), lse_pt, torch.empty(B, groups, S, device=DEV),
                             torch.empty(B, groups, S, device=DEV), lse_px, split)
            conf = torch.full((B, L, S), float("nan"), device=DEV)
            pv = torch.empty(B * L, ts, device=DEV)
            pi = torch.empty(B * L, ts, device=DEV, dtype=torch.int32)
            bv = torch.empty(B, L, device=DEV)
            bi = torch.empty(B, L, device=DEV, dtype=torch.int32)
            colmax = torch.full((B, S), -1, device=DEV, dtype=torch.int32)   # the call must zero it
            ops.sim_conf_colmax(a, b, lse_pt, lse_px, conf, B, L, S, K, scale, pv, pi, bv, bi, colmax, split)
            torch.cuda.synchronize()
            conf_ref = (torch.softmax(sim, 1) * torch.softmax(sim, 2)).float()
            _close(f"sim_colmax conf split={split} B={B} L={L} S={S}", conf, conf_ref, 5e-4, 1e-7)
            v, i = conf.max(2)
            assert torch.equal(bi.long(), i) and torch.equal(bv, v), "row max / argmax mismatch"
            cm = conf.max(1).values
            assert torch.equal(colmax, cm.view(torch.int32)), "column maxima are not the bits of conf.max(1)"
            # the value-based mutual test selects exactly the cells that are row- and column-maximal
            mutual = (conf == conf.max(2, keepdim=True).values) & (conf == conf.max(1, keepdim=True).values)
            sel = torch.gather(colmax, 1, bi.long()) == bv.view(torch.int32)
            assert torch.equal(sel, mutual.any(2)), "mutual-nearest selection differs"


def check_sim_lse_cols():
    for split in (0, 1):
        for (B, L, S, K) in [(2, 700, 520, 256), (1, 300, 100, 256), (1, 5000, 4096, 256)]:
            af = _rand(B, L, K, scale=0.9, seed=1)
            bf = _rand(B, S, K, scale=0.9, seed=2)
            a, b = _planes(af, split), _planes(bf, split)
            scale = 1.0 / (256 * 0.0801)
            sim = (torch.einsum("blk,bsk->bls", _q(af, split).double(), _q(bf, split).double()) * scale)
            ts = _lib.load().opp_sim_tiles(S)
            groups = (L + 31) // 32
            lse_rows = torch.full((B, L), float("nan"), device=DEV)
            lse_cols = torch.full((B, S), float("nan"), device=DEV)
            col_m = torch.full((B, groups, S), float("nan"), device=DEV)
            col_s = torch.full((B, groups, S), float("nan"), device=DEV)
            ops.sim_lse_cols(a, b, B, L, S, K, scale, torch.empty(B * L, ts, device=DEV),
                             torch.empty(B * L, ts, device=DEV), lse_rows, col_m, col_s, lse_cols, split)
            torch.cuda.synchronize()
            assert not torch.isnan(col_m).any() and not torch.isnan(col_s).any(), "unwritten column partials"
            _close(f"sim_lse_cols split={split} rows B={B} L={L} S={S}", lse_rows,
                   torch.logsumexp(sim, 2).float(), 1e-5, 1e-4)
            _close("sim_lse_cols cols", lse_cols, torch.logsumexp(sim, 1).float(), 1e-5, 1e-4)


def check_kv_single_plane():
    """split operands -> single-plane K'/V rows -> KV state: opp_linear_act_f16_out1 + opp_kv_partial
    (plain rows) + opp_kv_finalize (split mt).  Tolerances: one fp16 rounding of the rows (5e-4)
    for the GEMM, and its average over S rows for the state."""
    B, S, d = 2, 1000, 256
    xf = _rand(B * S, d, seed=1)
    wf = _rand(2 * d, d, scale=0.05, seed=2)
    x, w = _planes(xf, 1), _planes(wf, 1)
    kv = torch.full((B * S, 2 * d), float("nan"), device=DEV, dtype=torch.half)
    ops.linear_act(x, None, w, kv, B * S, 2, d, True, out_split=False)
    torch.cuda.synchronize()
    ref = (_q(xf, 1).double() @ _q(wf, 1).double().t()).float()
    ref[:, :d] = _elu1(ref[:, :d])
    _close("linear_act_out1", kv, ref, 6e-4, 1e-4)
    mw = _rand(d, d, scale=0.06, seed=3)
    chunks = _lib.load().opp_kv_chunks_b(S, B)
    part = torch.empty(B, chunks, 8, 33, 32, device=DEV)
    mt = torch.empty(B, d, 2 * d, device=DEV, dtype=torch.half)
    ksum = torch.empty(B, d, device=DEV)
    ops.kv_state(kv, part, mw, mt, ksum, B, S, d, float(S), True)
    torch.cuda.synchronize()
    kvq = kv.double().view(B, S, 2 * d)
    K, V = kvq[..., :d].view(B, S, 8, 32), kvq[..., d:].view(B, S, 8, 32)
    KV = torch.einsum("bshd,bshv->bhdv", K, V) / S
    ref_mt = torch.einsum("chv,bhdv->bchd", mw.double().view(d, 8, 32), KV).reshape(B, d, d).float()
    _close("kv1 ksum", ksum, K.sum(1).reshape(B, d).float(), 1e-5, 1e-3)
    _close("kv1 mt", _unplanes(mt, 1), ref_mt, 2e-5, 1e-6)


# ------------------------------------------------------------ token-row GEMMs at the forward's launches
# Every token-row GEMM launch of one forward (model.py _src_state / _encoder_layer on the 2D side,
# S = 4096 cells of a 512x512 image, and on the 3D side, N = 5000 points, incl. the resident-bank forms
# of layer 1; _fine at ROW_MATCHES matches per image, 26 rows each, with the row count on the host or
# on the device), run at bench.py's batch 64 and at batch 1.  epi: "act" (EpiStoreF16), "q" (EpiQ),
# "ln" (EpiLN); rows per image: "S", "N" or "F" (26 per match).  Options: flat (one launch over
# batch * rows, as the forward passes B * len), out1 (the K'/V rows: split operands, one fp16 output
# plane), a0_shared, w_batched (one weight per image: the attention state mt), resid, resid_shared,
# out32 (fp32 output only: the last fine layer), dyn (row count read on the device, = the capacity).
ROW_S, ROW_N, ROW_MATCHES = 4096, 5000, 1000
_FINE_GEMMS = [
    ("fine wqkv",          "act", "F", 128, 0, 384, dict(flat=1, act=2, act_cols=256)),
    ("fine merge LN",      "ln",  "F", 128, 0, 128, dict(flat=1)),
    ("fine mlp0",          "act", "F", 128, 128, 256, dict(flat=1, act=1, act_cols=256)),
    ("fine mlp2 LN",       "ln",  "F", 256, 0, 128, dict(flat=1, resid=1)),
    ("fine mlp2 LN out32", "ln",  "F", 256, 0, 128, dict(flat=1, resid=1, out32=1)),
]
ROW_GEMMS = [
    # name                     epi    rows k0   k1   n    options
    ("wkv 2D",                 "act", "S", 256, 0,   512, dict(flat=1, act=2, act_cols=256, out1=1)),
    ("wkv 3D",                 "act", "N", 256, 0,   512, dict(flat=1, act=2, act_cols=256, out1=1)),
    ("linear_q 2D",            "q",   "S", 256, 0,   256, {}),
    ("linear_q 3D",            "q",   "N", 256, 0,   256, {}),
    ("linear_q 3D x_shared",   "q",   "N", 256, 0,   256, dict(a0_shared=1)),
    ("merge LN mt 2D",         "ln",  "S", 256, 0,   256, dict(w_batched=1)),
    ("merge LN mt 3D",         "ln",  "N", 256, 0,   256, dict(w_batched=1)),
    ("merge LN bank state 2D", "ln",  "S", 256, 0,   256, {}),
    ("mlp0 2D",                "act", "S", 256, 256, 512, dict(flat=1, act=1, act_cols=512)),
    ("mlp0 3D",                "act", "N", 256, 256, 512, dict(flat=1, act=1, act_cols=512)),
    ("mlp0 3D a0_shared",      "act", "N", 256, 256, 512, dict(act=1, act_cols=512, a0_shared=1)),
    ("mlp2 2D",                "ln",  "S", 512, 0,   256, dict(flat=1, resid=1)),
    ("mlp2 3D",                "ln",  "N", 512, 0,   256, dict(flat=1, resid=1)),
    ("mlp2 3D resid_shared",   "ln",  "N", 512, 0,   256, dict(resid=1, resid_shared=1)),
] + _FINE_GEMMS + [(name + " dyn", e, r, k0, k1, n, dict(o, dyn=1)) for (name, e, r, k0, k1, n, o) in _FINE_GEMMS]
_EPI_LOG = {"act": "store_f16", "q": "q", "ln": "ln"}

# The tile configuration each launch runs, (block_n, mma_n, cluster, pair, stages), in the fp16x3
# mode at batch 64 and batch 1 (fp16: block_n, mma_n, cluster and pair are pinned, the ring is deeper).
# At batch 1 the 2D side (32 M tiles) takes the latency forms: N tiles halved (split_n_for_latency)
# and the LayerNorm N-split pair cluster; the 3D side (40 M tiles) halves linear_q only, its
# N = 512 GEMMs already have 80 super tiles.  The fine GEMMs have no latency forms (the device-count
# launches are sized at capacity, and the host-count ones have hundreds of M tiles).
_W256, _W128, _Q64, _PAIR = (256, 256, 2, 0, 2), (128, 128, 2, 0, 3), (64, 64, 2, 0, 4), (128, 128, 2, 2, 3)
ROW_TILES = {
    **{(name, 64): _W256 for name in ("wkv 2D", "wkv 3D", "linear_q 2D", "linear_q 3D", "linear_q 3D x_shared",
                                      "merge LN mt 2D", "merge LN mt 3D", "merge LN bank state 2D", "mlp0 2D",
                                      "mlp0 3D", "mlp0 3D a0_shared", "mlp2 2D", "mlp2 3D", "mlp2 3D resid_shared")},
    ("wkv 2D", 1): _W128, ("wkv 3D", 1): _W256,
    ("linear_q 2D", 1): _Q64, ("linear_q 3D", 1): _W128, ("linear_q 3D x_shared", 1): _W128,
    ("merge LN mt 2D", 1): _PAIR, ("merge LN mt 3D", 1): _PAIR, ("merge LN bank state 2D", 1): _PAIR,
    ("mlp0 2D", 1): _W128, ("mlp0 3D", 1): _W256, ("mlp0 3D a0_shared", 1): _W256,
    ("mlp2 2D", 1): _PAIR, ("mlp2 3D", 1): _PAIR, ("mlp2 3D resid_shared", 1): _PAIR,
    **{(name + dyn, B): (_W256 if name == "fine mlp0" else _W128)
       for (name, *_) in _FINE_GEMMS for dyn in ("", " dyn") for B in (64, 1)},
}


def _drand(rows, cols, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(rows, cols, device=DEV, generator=g) * scale


def _row_inputs(split, spec, B):
    """operand planes of one ROW_GEMMS launch at batch B (drawn on the device from fixed seeds)"""
    _, epi, rk, k0, k1, n, o = spec
    rows = {"S": ROW_S, "N": ROW_N, "F": 26 * ROW_MATCHES}[rk]
    inp = {"rows": rows,
           "a0": _planes(_drand((1 if o.get("a0_shared") else B) * rows, k0, 1), split),
           "a1": _planes(_drand(B * rows, k1, 2), split) if k1 else None,
           "w": _planes(_drand((B if o.get("w_batched") else 1) * n, k0 + k1, 3, 0.06 if epi == "q" else 0.05),
                        split)}
    if epi == "q":
        inp["ksum"] = _drand(B, 256, 4).abs() * 100 + 50
    if epi == "ln":
        inp["gamma"], inp["beta"] = 1 + 0.1 * _drand(1, n, 5)[0], 0.1 * _drand(1, n, 6)[0]
        if o.get("resid"):
            inp["res"] = _planes(_drand((1 if o.get("resid_shared") else B) * rows, n, 7), split)
    return inp


def _row_launch(split, spec, B, inp, out, out32=None, count=None, row_mask=None):
    """the launch of ROW_GEMMS entry `spec` as the forward makes it; count: device row count in
    matches (26 rows each); the host row count is the capacity then"""
    _, epi, _, k0, k1, n, o = spec
    rows = inp["rows"]
    nb, lr = (1, B * rows) if o.get("flat") else (B, rows)
    dyn = {} if count is None else {"count": count, "rows_per_count": 26}
    if epi == "act":
        ops.linear_act(inp["a0"], inp["a1"], inp["w"], out, lr, o["act"], o["act_cols"], split,
                       out_split=False if (split and o.get("out1")) else None, batches=nb,
                       a0_shared=bool(o.get("a0_shared")), row_mask=row_mask, **dyn)
    elif epi == "q":
        ops.linear_q(inp["a0"], inp["w"], inp["ksum"], out, B, rows, ROW_S, split,
                     x_shared=bool(o.get("a0_shared")), row_mask=row_mask)
    else:
        w = inp["w"].view(B if o.get("w_batched") else 1, n, -1)
        ops.linear_ln(inp["a0"], inp["a1"], w, bool(o.get("w_batched")), inp["gamma"], inp["beta"], nb, lr, split,
                      resid=inp.get("res"), out16=out, out32=out32, resid_shared=bool(o.get("resid_shared")), **dyn)
    return nb, lr


def _row_outputs(split, spec, B, rows):
    _, _, _, _, _, n, o = spec
    pl = 1 if (o.get("out1") or not split) else 2
    out = None if o.get("out32") else torch.full((B * rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
    out32 = torch.full((B * rows, n), float("nan"), device=DEV) if o.get("out32") else None
    return out, out32


def _row_check(split, spec, B, inp, out, out32, valid_rows=None):
    """outputs of one ROW_GEMMS launch against fp64 on the values the stored planes represent, a few
    images at a time; rows from valid_rows on (a device-side count) must still be NaN"""
    name, epi, _, k0, k1, n, o = spec
    rows = inp["rows"]
    K = k0 + k1
    out1 = split and o.get("out1")
    if epi == "act":
        tol = (6e-4, 1e-4) if out1 else _tol(split, (2e-3, 2e-3), (2e-5, 2e-5))
    elif epi == "q":
        tol = _tol(split, (2e-3, 1e-4), (2e-5, 1e-6))
    else:
        tol = (_tol(split, (1e-3, 2e-3), (2e-5, 2e-5)) if out32 is not None else
               _tol(split, (2e-3, 3e-3), (2e-5, 2e-5)))
    t = _Tally(f"{name} split={split} batch {B}", *tol)
    W = _unplanes(inp["w"], split).double().view(-1, n, K)
    total = B * rows if valid_rows is None else valid_rows
    step = _chunk(rows * max(n, K))
    for b0 in range(0, B, step):
        b1 = min(B, b0 + step)
        sl = slice(b0 * rows, b1 * rows)
        A = _unplanes(inp["a0"] if o.get("a0_shared") else inp["a0"][sl], split).double()
        if o.get("a0_shared"):
            A = A.repeat(b1 - b0, 1)
        if k1:
            A = torch.cat([A, _unplanes(inp["a1"][sl], split).double()], 1)
        Wb = W[b0:b1] if o.get("w_batched") else W.expand(b1 - b0, n, K)
        y = torch.bmm(A.view(b1 - b0, rows, K), Wb.transpose(1, 2)).reshape(-1, n)
        if epi == "act":
            y[:, :o["act_cols"]] = (torch.relu if o["act"] == 1 else _elu1)(y[:, :o["act_cols"]])
            ref = y
        elif epi == "q":
            q = _elu1(y).view(b1 - b0, rows, 8, 32)
            z = 1.0 / (torch.einsum("blhd,bhd->blh", q, inp["ksum"][b0:b1].double().view(-1, 8, 32)) + 1e-6)
            ref = (q * z[..., None] * ROW_S).reshape(-1, n)
        else:
            ref = F.layer_norm(y, (n,), inp["gamma"].double(), inp["beta"].double(), 1e-5)
            if o.get("resid"):
                r = _unplanes(inp["res"] if o.get("resid_shared") else inp["res"][sl], split).double()
                ref = ref + (r.repeat(b1 - b0, 1) if o.get("resid_shared") else r)
        got = out32[sl] if out32 is not None else (out[sl].float() if out1 else _unplanes(out[sl], split))
        r0, r1 = b0 * rows, b1 * rows
        if r0 < total:
            v = min(r1, total) - r0
            t.add(got[:v], ref[:v])
        if r1 > total:
            assert torch.isnan(got[max(total - r0, 0):]).all(), f"{name}: rows past the device-side count written"
    t.check()


def _row_cluster_tiles(t, batches, m_tiles):
    if t["pair"]:     # N-split LayerNorm: one 2-CTA cluster per M tile, both column halves
        sup = batches * m_tiles
        clusters = min(sup, _lib.load().opp_num_sms() // 2)
        return sup // clusters, -(-sup // clusters)
    return _cluster_tiles(t, batches, m_tiles)


def _row_gemm(split, spec, B):
    """one ROW_GEMMS launch at batch B under the tile log: checked against fp64, returns the tile
    line and (fewest, most) tiles per cluster"""
    inp = _row_inputs(split, spec, B)
    out, out32 = _row_outputs(split, spec, B, inp["rows"])
    count = None
    if spec[6].get("dyn"):
        count = torch.tensor([B * ROW_MATCHES], dtype=torch.int32, device=DEV)
    with _tile_log() as new:
        nb, lr = _row_launch(split, spec, B, inp, out, out32, count=count)
        torch.cuda.synchronize()
    t = _launch_tile(new, 0, spec[5], spec[3] + spec[4], 0, _EPI_LOG[spec[1]])
    _row_check(split, spec, B, inp, out, out32)
    return t, _row_cluster_tiles(t, nb, -(-lr // 128))


def _row_layers(split):
    failed = []
    for spec in ROW_GEMMS:
        name = spec[0]
        for B in (64, 1):
            try:
                t, (lo, hi) = _row_gemm(split, spec, B)
                got = (t["block_n"], t["mma_n"], t["cluster"], t["pair"], t["stages"])
                print(f"  {name} batch {B}: block_n {got[0]} mma_n {got[1]} cluster {got[2]} pair {got[3]} "
                      f"stages {got[4]} tiles per cluster {lo}-{hi}")
                want = ROW_TILES.get((name, B))
                assert want is not None, f"{name} batch {B}: no pinned tile configuration"
                if split:
                    assert got == want, f"{name} batch {B}: tile {got}, expected {want}"
                else:
                    assert got[:4] == want[:4], f"{name} batch {B}: tile {got[:4]}, expected {want[:4]}"
                if B == 64:
                    assert hi >= 8, f"{name}: only {hi} tiles per cluster at batch 64"
            except AssertionError as e:   # go on: which launches fail locates a defect
                print(f"  {name} batch {B}: FAILED: {e}")
                failed.append(f"{name} batch {B}")
            torch.cuda.empty_cache()
    assert not failed, f"split={split}: {failed}"


def check_row_gemms():
    """The token-row GEMMs at the forward's launch configurations against fp64 (ROW_GEMMS), in both
    operand modes; the tile log shows which configuration each one ran."""
    for split in (1, 0):
        _run_child(f"row_gemms_split{split}", OPP_LOG_TILES="2")


# row_launch_invariance: EpiStoreF16 and EpiQ compute an element from its own accumulator and (EpiQ)
# the 32-column head it lies in, so the N tile width (64, 128, 256 columns: the latency split and
# $OPP_NSPLIT=0) and the batch of the launch must not change its bits.  EpiLN merges the statistics
# of a row across the two CTAs of the N-split cluster in another order than within one CTA: the pair
# form is compared with fp64 only (row_gemms at batch 1).
ROW_VARIANTS = {"default": {}, "nsplit0": {"OPP_NSPLIT": "0"}}


def _row_variant(tag):
    """fixed launches under this process's knobs; image-0 rows saved to $KERNEL_CHECK_DIR/<tag>.pt with
    the N tile width each ran"""
    saved = {}
    q_spec, kv_spec = ROW_GEMMS[2], ("kv", "act", "S", 256, 0, 512, dict(flat=1, act=2, act_cols=256))
    for split in (1, 0):
        # EpiQ: image 0 alone and inside a batch of 2 (default: 64- and 128-column tiles)
        inp2 = _row_inputs(split, q_spec, 2)    # drawn once at batch 2: image 0 is the same in both launches
        for B in ((1, 2) if tag == "default" else (1,)):
            inp = dict(inp2, a0=inp2["a0"][:B * ROW_S].contiguous(), ksum=inp2["ksum"][:B].contiguous())
            out, _ = _row_outputs(split, q_spec, B, ROW_S)
            with _tile_log() as new:
                _row_launch(split, q_spec, B, inp, out)
                torch.cuda.synchronize()
            t = _launch_tile(new, 0, 256, 256, 0, "q")
            saved[f"q split={split} batch {B}"] = (t["block_n"], out[:ROW_S].cpu())
        # EpiStoreF16 (K'/V rows with both planes): 4096 rows, and their first 1024 alone
        for rows in ((ROW_S, 1024) if tag == "default" else (ROW_S,)):
            inp = _row_inputs(split, kv_spec, 1)
            inp["rows"] = rows
            inp["a0"] = inp["a0"][:rows].contiguous()
            out, _ = _row_outputs(split, kv_spec, 1, rows)
            with _tile_log() as new:
                _row_launch(split, kv_spec, 1, inp, out)
                torch.cuda.synchronize()
            t = _launch_tile(new, 0, 512, 256, 0, "store_f16")
            saved[f"kv split={split} rows {rows}"] = (t["block_n"], out[:1024].cpu())
    for k, (bn, _) in saved.items():
        print(f"  [{tag}] {k}: block_n {bn}")
    torch.save(saved, os.path.join(os.environ["KERNEL_CHECK_DIR"], f"{tag}.pt"))


def _row_batch_slices():
    """Each image of a batch-64 linear_q against a batch-1 launch of the same image, both with
    256-column tiles ($OPP_NSPLIT=0 keeps the batch-1 tile whole), and each 4-image slice of a batch-64
    merge LayerNorm with one state mt per image (w_batched) against a batch-4 launch of those images
    (whole-row tiles in both; batch 1 would take the N-split cluster)."""
    differ = []
    for split in (1, 0):
        for spec, step, tag in ((ROW_GEMMS[2], 1, "q"), (ROW_GEMMS[5], 4, "ln")):
            B = 64
            inp = _row_inputs(split, spec, B)
            out, _ = _row_outputs(split, spec, B, ROW_S)
            with _tile_log() as new:
                _row_launch(split, spec, B, inp, out)
                torch.cuda.synchronize()
            t64 = _launch_tile(new, 0, 256, 256, 0, tag)
            assert not torch.isnan(out.float()).any(), f"{spec[0]} batch 64: NaN (unwritten) outputs"
            pl = out.shape[1] // 256
            for b0 in range(0, B, step):
                sl = slice(b0 * ROW_S, (b0 + step) * ROW_S)
                part = {"rows": ROW_S, "a0": inp["a0"][sl].contiguous(), "a1": None,
                        "w": inp["w"].view(B, 256, -1)[b0:b0 + step].contiguous() if tag == "ln" else inp["w"]}
                for k in ("ksum", "gamma", "beta"):
                    if k in inp:
                        part[k] = inp[k][b0:b0 + step].contiguous() if k == "ksum" else inp[k]
                o = torch.full((step * ROW_S, pl * 256), float("nan"), device=DEV, dtype=torch.half)
                with _tile_log() as new:
                    _row_launch(split, spec, step, part, o)
                    torch.cuda.synchronize()
                t = _launch_tile(new, 0, 256, 256, 0, tag)
                assert (t["block_n"], t["pair"]) == (t64["block_n"], t64["pair"]) == (256, 0), (t, t64)
                if not _bits_equal(o, out[sl]):
                    differ.append(f"{spec[0]} split={split} images {b0}-{b0 + step - 1}: "
                                  f"{int((o != out[sl]).sum())} elements")
            print(f"  {spec[0]} split={split}: batch 64 (block_n {t64['block_n']}) against batch-{step} launches")
    assert not differ, f"batch-64 launches differ from smaller launches of the same images: {differ}"


def check_row_launch_invariance():
    with tempfile.TemporaryDirectory() as d:
        for tag, env in ROW_VARIANTS.items():
            _run_child(f"row_variant_{tag}", OPP_LOG_TILES="2", KERNEL_CHECK_DIR=d, **env)
        saved = {tag: torch.load(os.path.join(d, f"{tag}.pt")) for tag in ROW_VARIANTS}
    differ = []
    for kind in ("q split=1", "q split=0", "kv split=1", "kv split=0"):
        runs = [(f"{tag} {k}", bn, t) for tag, s in saved.items() for k, (bn, t) in s.items() if k.startswith(kind)]
        widths = sorted({bn for _, bn, _ in runs})
        print(f"  {kind}: N tile widths {widths}")
        assert widths == [64, 128, 256], f"{kind}: the variants ran N tiles of {widths}, expected 64, 128 and 256"
        for what, bn, t in runs[1:]:
            if not _bits_equal(t, runs[0][2]):
                differ.append(f"{what} (block_n {bn}) vs {runs[0][0]}: {int((t != runs[0][2]).sum())} elements")
    _run_child("row_batch_slices", OPP_LOG_TILES="2", OPP_NSPLIT="0")
    assert not differ, f"token-row outputs depend on the N tile width: {differ}"


# ------------------------------------------------------------------ device-side row counts (fine stage)
def check_row_dyn():
    """The fine stage launched at capacity with the match count on the device (CUDA-graph path):
    opp_linear_act_f16_dyn / opp_linear_ln_dyn (26 rows per match) and fine_gather / fine_attention /
    fine_match, at counts 0, 1, a ragged last 128-row tile, the capacity and past it (clamped).  Rows
    below count * 26 against fp64 (GEMMs) and bit-identical to the launch with the row count on the
    host; rows past it untouched (NaN)."""
    cap = 150
    for split in (1, 0):
        pl = 2 if split else 1
        for spec in _FINE_GEMMS:
            inp = _row_inputs(split, spec, 1)
            inp["rows"] = 26 * cap
            for k in ("a0", "a1", "res"):
                if inp.get(k) is not None:
                    inp[k] = inp[k][:26 * cap].contiguous()
            for c in (0, 1, 37, cap, cap + 5):
                m = min(c, cap)
                out, out32 = _row_outputs(split, spec, 1, 26 * cap)
                _row_launch(split, spec, 1, inp, out, out32, count=torch.tensor([c], dtype=torch.int32, device=DEV))
                torch.cuda.synchronize()
                _row_check(split, spec, 1, inp, out, out32, valid_rows=26 * m)
                if m:
                    host = {"rows": 26 * m, **{k: (v[:26 * m].contiguous() if k in ("a0", "a1", "res") and
                                                   v is not None else v) for k, v in inp.items() if k != "rows"}}
                    ho, ho32 = _row_outputs(split, spec, 1, 26 * m)
                    _row_launch(split, spec, 1, host, ho, ho32)
                    torch.cuda.synchronize()
                    got, want = (out32[:26 * m], ho32) if out32 is not None else (out[:26 * m], ho)
                    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
                        f"{spec[0]} split={split} count {c}: device-count launch differs from the host-count launch"
        # fine_gather / fine_attention / fine_match
        B, hf, wf, N, wc = 2, 64, 80, 500, 20
        fine = _planes(_rand(B, hf, wf, 128, seed=1), split)
        desc = _rand(B, 128, N, seed=2)
        g = torch.Generator().manual_seed(1)
        b_ids = torch.randint(0, B, (cap,), generator=g).sort().values.to(DEV)
        i_ids = torch.randint(0, N, (cap,), generator=g).to(DEV)
        j_ids = torch.randint(0, (hf // 4) * wc, (cap,), generator=g).to(DEV)
        qkv = _planes(torch.cat([_rand(cap * 26, 256, seed=3).abs() + 0.05, _rand(cap * 26, 128, seed=4)], 1), split)
        xf = _rand(cap * 26, 128, seed=5)
        mkc = torch.rand(cap, 2, device=DEV) * 300
        scale = torch.rand(B, 2, device=DEV) + 0.5

        def run(m, count):
            o = {"x32": torch.full((m * 26, 128), float("nan"), device=DEV),
                 "x16": torch.full((m * 26, pl * 128), float("nan"), device=DEV, dtype=torch.half),
                 "msg": torch.full((m * 26, pl * 128), float("nan"), device=DEV, dtype=torch.half),
                 "ef": torch.full((m, 3), float("nan"), device=DEV),
                 "mf": torch.full((m, 2), float("nan"), device=DEV)}
            ops.fine_gather(fine, desc, b_ids, i_ids, j_ids, o["x32"], o["x16"], m, hf, wf, wc, 4, N, split,
                            count=count)
            ops.fine_attention(qkv, o["msg"], m, 1, split, count=count)
            ops.fine_match(xf, mkc, b_ids, scale, o["ef"], o["mf"], m, 2.0, count=count)
            torch.cuda.synchronize()
            return o

        for c in (0, 1, 37, cap, cap + 5):
            m = min(c, cap)
            got = run(cap, torch.tensor([c], dtype=torch.int32, device=DEV))
            host = run(m, None) if m else None
            for k, v in got.items():
                per = 26 if v.shape[0] == 26 * cap else 1
                assert torch.isnan(v[per * m:].float()).all(), f"fine {k} split={split} count {c}: rows past the count"
                if m:
                    assert torch.equal(v[:per * m].view(torch.int16) if v.dtype == torch.half else v[:per * m],
                                       host[k].view(torch.int16) if v.dtype == torch.half else host[k]), \
                        f"fine {k} split={split} count {c}: device-count launch differs from the host-count launch"
        print(f"  fine_gather / fine_attention / fine_match split={split}: counts 0, 1, 37, {cap}, {cap + 5}")


# --------------------------------------------------------------------------------- masks, colmax selection
def check_row_masks():
    """row_mask (query_image_mask) on the K'/V rows (opp_linear_act_f16_b, _out1) and on linear_q (also
    with the 3D tokens shared): masked rows exactly zero, every other row bit-identical to the launch
    without a mask."""
    B = 3
    g = torch.Generator().manual_seed(9)
    mask = (torch.rand(B * ROW_S, generator=g) > 0.3).to(torch.uint8).to(DEV)
    mask[ROW_S:2 * ROW_S] = 0          # one image fully padded
    kv_spec = ("kv", "act", "S", 256, 0, 512, dict(flat=1, act=2, act_cols=256))
    for split in (1, 0):
        cases = [("linear_act_b", kv_spec), ("linear_q", ROW_GEMMS[2]), ("linear_q x_shared", ROW_GEMMS[4])]
        if split:
            cases.insert(1, ("linear_act_out1", ROW_GEMMS[0]))
        for what, spec in cases:
            spec = (spec[0], spec[1], "S") + spec[3:]
            inp = _row_inputs(split, spec, B)
            outs = []
            for rm in (None, mask):
                out, _ = _row_outputs(split, spec, B, ROW_S)
                if spec[1] == "act":     # the forward's masked form: batches = 1 over B * S rows
                    ops.linear_act(inp["a0"], None, inp["w"], out, B * ROW_S, 2, 256, split,
                                   out_split=False if what == "linear_act_out1" else None, row_mask=rm)
                else:
                    _row_launch(split, spec, B, inp, out, row_mask=rm)
                outs.append(out)
            torch.cuda.synchronize()
            keep = mask.bool()
            assert not torch.isnan(outs[1].float()).any(), f"{what} split={split}: unwritten rows"
            assert (outs[1][~keep].view(torch.int16) == 0).all(), f"{what} split={split}: masked rows not zero"
            assert _bits_equal(outs[1][keep], outs[0][keep]), f"{what} split={split}: unmasked rows changed"
            print(f"  {what} split={split}: {int((~keep).sum())} masked rows zero, the others unchanged")


SCALE_COARSE = 1.0 / (256 * 0.0801)


def check_sim_col_mask():
    """col_mask (query_image_mask) in sim_lse_cols / lse_col_finalize and the conf pass against
    softmax(sim - 1e9 [masked columns], 1) * softmax(., 2) in fp64 (coarse_matching.py:108-115):
    lse_cols = +inf and conf exactly 0 in masked columns.  Image 0: a random mask with a whole
    256-column tile masked; image 1: a single valid column; L = 1000 (a ragged last 32-row group)."""
    B, L, S, K = 2, 1000, 700, 256
    for split in (1, 0):
        af, bf = _rand(B, L, K, scale=0.9, seed=1), _rand(B, S, K, scale=0.9, seed=2)
        a, b = _planes(af, split), _planes(bf, split)
        g = torch.Generator().manual_seed(4)
        cm = (torch.rand(B, S, generator=g) > 0.4).to(torch.uint8)
        cm[0, 256:512] = 0
        cm[1] = 0
        cm[1, 333] = 1
        cm = cm.to(DEV)
        ts, groups = ops.sim_tiles(S), (L + 31) // 32
        lse_rows, lse_cols = torch.full((B, L), float("nan"), device=DEV), torch.full((B, S), float("nan"), device=DEV)
        ops.sim_lse_cols(a, b, B, L, S, K, SCALE_COARSE, torch.empty(B * L, ts, device=DEV),
                         torch.empty(B * L, ts, device=DEV), lse_rows, torch.empty(B, groups, S, device=DEV),
                         torch.empty(B, groups, S, device=DEV), lse_cols, split, col_mask=cm)
        conf = torch.full((B, L, S), float("nan"), device=DEV)
        bv, bi = torch.empty(B, L, device=DEV), torch.empty(B, L, device=DEV, dtype=torch.int32)
        colmax = torch.full((B, S), -1, device=DEV, dtype=torch.int32)
        ops.sim_conf_colmax(a, b, lse_rows, lse_cols, conf, B, L, S, K, SCALE_COARSE, torch.empty(B * L, ts, device=DEV),
                            torch.empty(B * L, ts, device=DEV, dtype=torch.int32), bv, bi, colmax, split)
        torch.cuda.synchronize()
        sim = torch.einsum("blk,bsk->bls", _q(af, split).double(), _q(bf, split).double()) * SCALE_COARSE
        sim = sim - 1e9 * (cm == 0).double()[:, None, :]
        masked = (cm == 0)
        assert torch.isinf(lse_cols[masked]).all() and (lse_cols[masked] > 0).all(), "masked columns: lse_cols != +inf"
        _close(f"col_mask split={split} lse_rows", lse_rows, torch.logsumexp(sim, 2).float(), 1e-5, 1e-4)
        _close(f"col_mask split={split} lse_cols", lse_cols[~masked], torch.logsumexp(sim, 1).float()[~masked],
               1e-5, 1e-4)
        assert (conf.transpose(1, 2)[masked] == 0).all(), "masked columns: conf is not exactly 0"
        _close(f"col_mask split={split} conf", conf, (torch.softmax(sim, 1) * torch.softmax(sim, 2)).float(),
               5e-4, 1e-7)
        assert torch.equal(colmax, conf.max(1).values.view(torch.int32)), "column maxima under the mask"
        assert (bi[1].long() == 333).all(), "image 1: every row's best column is its one valid column"



def check_match_select_colmax():
    """opp_match_select_colmax (value-based mutual test against the column maxima) on planted conf maps
    against the reference's mask expression (coarse_matching.py:142-172): exact ties keep every tied
    row, the keypoints are one shared [1, N, 3] bank (bank_shared) or one per image."""
    B, L, hc, wc = 3, 2500, 20, 24
    S = hc * wc
    g = torch.Generator().manual_seed(0)
    conf = torch.rand(B, L, S, generator=g) * 0.3
    for b in range(B):
        cols = torch.randperm(S, generator=g)[:200]
        rows = torch.randperm(L, generator=g)[:200]
        conf[b, rows, cols] = 0.5 + 0.5 * torch.rand(200, generator=g)
        # ties: rows 0-29 of the planted ones copied into 30 other rows (same row maxima, tied columns)
        twins = torch.tensor([r for r in torch.randperm(L, generator=g).tolist() if r not in set(rows.tolist())][:30])
        conf[b, twins] = conf[b, rows[:30]]
    conf = conf.to(DEV)
    pt_val, pt_idx = conf.max(2)
    colmax = conf.max(1).values.contiguous().view(torch.int32)
    scale = torch.rand(B, 2, device=DEV) + 0.5
    for shared in (True, False):
        kpts = torch.rand(1 if shared else B, L, 3, device=DEV)
        cap = B * L
        outs = [torch.full((cap,), -1, device=DEV, dtype=torch.int64) for _ in range(3)]
        mconf, mk3, mkc = torch.empty(cap, device=DEV), torch.empty(cap, 3, device=DEV), torch.empty(cap, 2, device=DEV)
        cnt = torch.zeros(1, device=DEV, dtype=torch.int32)
        ops.match_select_colmax(pt_val.contiguous(), pt_idx.int().contiguous(), colmax, kpts, scale, B, L, hc, wc,
                                0.4, 2, 8.0, torch.empty((B * L + 1023) // 1024 + 2, device=DEV, dtype=torch.int32),
                                *outs, mconf, mk3, mkc, cnt, bank_shared=shared)
        torch.cuda.synchronize()
        M = int(cnt.item())
        mask = (conf > 0.4).view(B, L, hc, wc).clone()
        mask[:, :, :2] = False
        mask[:, :, :, :2] = False
        mask = mask.view(B, L, S) * (conf == conf.max(2, keepdim=True)[0]) * (conf == conf.max(1, keepdim=True)[0])
        mv, aj = mask.max(2)
        rb, ri = torch.where(mv)
        rj = aj[rb, ri]
        tied = int((torch.bincount(rb * S + rj) > 1).sum())
        print(f"  match_select_colmax bank_shared={shared}: M={M} ref={len(rb)}, {tied} columns matched by tied rows")
        assert M == len(rb) and M > 100 and tied >= 10, (M, len(rb), tied)
        assert torch.equal(outs[0][:M], rb) and torch.equal(outs[1][:M], ri) and torch.equal(outs[2][:M], rj)
        assert torch.equal(mconf[:M], conf[rb, ri, rj])
        assert torch.equal(mk3[:M], kpts[0, ri] if shared else kpts[rb, ri])
        _close("match_select_colmax mkpts_c", mkc[:M], torch.stack([rj % wc, rj // wc], 1) * (8.0 * scale[rb][:, [1, 0]]),
               1e-6, 1e-5)


CHECKS = {
    "linear_act": check_linear_act,
    "linear_ln": check_linear_ln,
    "linear_q": check_linear_q,
    "linear_act_shared": check_linear_act_shared,
    "conv": check_conv,
    "conv_up_odd_clusters": check_conv_up_odd_clusters,
    "conv_win": check_conv_win,
    "conv_layers": check_conv_layers,
    "conv_launch_invariance": check_conv_launch_invariance,
    "conv_win_production": check_conv_win_production,
    "conv1_gemm": check_conv1_gemm,
    "kpt_encode": check_kpt_encode,
    "kv_state": check_kv_state,
    "fine": check_fine,
    "full_attention": check_full_attention,
    "loftr_kernels": check_loftr_kernels,
    "sim_colmax": check_sim_colmax,
    "sim_lse_cols": check_sim_lse_cols,
    "kv_single_plane": check_kv_single_plane,
    "row_gemms": check_row_gemms,
    "row_launch_invariance": check_row_launch_invariance,
    "row_dyn": check_row_dyn,
    "row_masks": check_row_masks,
    "sim_col_mask": check_sim_col_mask,
    "match_select_colmax": check_match_select_colmax,
}


# run only in a child process whose environment selects the launch configuration
CHILD_CHECKS = {"conv_up": _conv_up_cases,
                "conv_layers_split1": functools.partial(_conv_layers, 1),
                "conv_layers_split0": functools.partial(_conv_layers, 0),
                "conv_batch_slices": _conv_batch_slices,
                "conv_win_production_tiles": _conv_win_production,
                **{f"conv_variant_{tag}": functools.partial(_conv_variant, tag) for tag in INVARIANCE_VARIANTS},
                "row_gemms_split1": functools.partial(_row_layers, 1),
                "row_gemms_split0": functools.partial(_row_layers, 0),
                "row_batch_slices": _row_batch_slices,
                **{f"row_variant_{tag}": functools.partial(_row_variant, tag) for tag in ROW_VARIANTS}}
assert not CHECKS.keys() & CHILD_CHECKS.keys(), "`--one name` must name one function"


def main(argv):
    if len(argv) == 2 and argv[0] == "--one":
        print(f"[{argv[1]}]")
        {**CHECKS, **CHILD_CHECKS}[argv[1]]()
        print(f"[{argv[1]}] OK (peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated by torch)")
        return 0
    names = argv or list(CHECKS)
    failed = []
    for n in names:
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", n], timeout=600)
            if r.returncode != 0:
                failed.append(n)
        except subprocess.TimeoutExpired:
            print(f"[{n}] TIMEOUT")
            failed.append(n)
    print("FAILED:" if failed else "ALL KERNEL CHECKS PASSED", failed)
    return 1 if failed else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
