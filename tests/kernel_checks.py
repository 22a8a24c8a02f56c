"""Per-kernel numerics checks of libopp_b200.so against plain fp32 torch math on the same
(fp16-rounded) inputs.  Used by tests/test_kernels_gpu.py (pytest -m gpu) and runnable as a script
(`python tests/kernel_checks.py [name ...]`), where every check runs in its own subprocess so that
a device-side trap in one kernel cannot poison the others.
"""
import math
import subprocess
import sys
import os

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from onepose_plus_plus_b200 import _lib, ops  # noqa: E402

DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def _close(name, got, ref, rtol, atol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    worst = (err / tol).max().item() if err.numel() else 0.0
    print(f"  {name}: max_abs_err={err.max().item() if err.numel() else 0:.3e} "
          f"worst/tol={worst:.3f} bad={bad}/{err.numel()}")
    assert bad == 0, f"{name}: {bad} elements out of tolerance (worst {worst:.2f}x)"


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


def _conv_case(split, B, H, W, cin, cin_pad, cout, cout_pad, k, stride, act, resid, tokens, up=False):
    xf = torch.zeros(B, H, W, cin_pad, device=DEV)
    xf[..., :cin] = _rand(B, H, W, cin, seed=1)
    wf = torch.zeros(cout_pad, k, k, cin_pad, device=DEV)
    wf[:cout, :, :, :cin] = _rand(cout, k, k, cin, scale=1.0 / math.sqrt(k * k * cin), seed=2)
    bias = torch.zeros(cout_pad, device=DEV)
    bias[:cout] = _rand(cout, seed=3) * 0.1
    pad = k // 2
    oh, ow = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    pl = 2 if split else 1
    x16 = _planes(xf, split)
    w16 = _planes(wf.reshape(cout_pad, -1), split)
    res = resf = None
    if resid:
        resf = torch.zeros(B, oh, ow, cout_pad, device=DEV)
        resf[..., :cout] = _rand(B, oh, ow, cout, seed=4)
        res = _planes(resf, split)
    out = torch.full((B, oh, ow, pl * cout_pad), float("nan"), device=DEV, dtype=torch.half)
    tok = pe = None
    if tokens:
        tok = torch.full((B, oh * ow, pl * cout_pad), float("nan"), device=DEV, dtype=torch.half)
        pe = _rand(oh * ow, cout_pad, seed=5)
    up16 = upf = None
    if up:   # FPN top-down merge: + bilinear x2 (align_corners=True) of a coarser map, fused in the epilogue
        upf = torch.zeros(B, oh // 2, ow // 2, cout_pad, device=DEV)
        upf[..., :cout] = _rand(B, oh // 2, ow // 2, cout, seed=6)
        up16 = _planes(upf, split)
    _lib.call("opp_conv2d_nhwc", _lib.ptr(x16), _lib.ptr(w16), _lib.ptr(bias), _lib.ptr(res),
              _lib.ptr(out), B, H, W, cin_pad, cout_pad, k, stride, act, 0.01, _lib.ptr(tok),
              _lib.ptr(pe), _lib.ptr(up16), split, _lib.stream())
    torch.cuda.synchronize()
    ref = F.conv2d(_q(xf, split).double().permute(0, 3, 1, 2), _q(wf, split).double().permute(0, 3, 1, 2),
                   bias.double(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    if up:
        ref = ref + F.interpolate(_q(upf, split).double().permute(0, 3, 1, 2), scale_factor=2.0, mode="bilinear",
                                  align_corners=True).permute(0, 2, 3, 1)
    if resid:
        ref = ref + _q(resf, split).double()
    if act == 1:
        ref = torch.relu(ref)
    elif act == 2:
        ref = F.leaky_relu(ref, 0.01)
    ref = ref.float()
    name = f"conv split={split} k={k} s={stride} {cin}->{cout} {H}x{W} act={act} resid={resid} up={up}"
    got = _unplanes(out, split)
    _close(name, got, ref, *_tol(split, (2e-3, 3e-3), (2e-5, 2e-5)))
    if cout_pad > cout:
        assert got[..., cout:].abs().max().item() == 0.0, "padding channels must stay zero"
    if tokens:
        _close(name + " tok", _unplanes(tok, split), ref.reshape(B, oh * ow, cout_pad) + pe,
               *_tol(split, (2e-3, 3e-3), (2e-5, 2e-5)))


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
    env = dict(os.environ, OPP_CLUSTER=str(cluster))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", "conv_up"], env=env, timeout=600)
    assert r.returncode == 0, f"fused-upsample conv checks failed with OPP_CLUSTER={cluster} ({sms} SMs)"


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
            cy, cx = (j_ids // wc).cpu(), (j_ids % wc).cpu()
            bad_t = bad_o = 0
            for m in range(M):
                for (win, org, got, dense) in ((7, -3, t_w, t_d), (5, -2, o_w, o_d)):
                    for ly in range(win):
                        for lx in range(win):
                            y, x = 4 * int(cy[m]) + org + ly, 4 * int(cx[m]) + org + lx
                            inside = 0 <= y < H and 0 <= x < W
                            if win == 5 and not inside:
                                continue      # the gather never reads these
                            want = dense[int(b_ids[m]), y, x] if inside else torch.zeros_like(got[m, ly, lx])
                            if not torch.equal(got[m, ly, lx], want):
                                if win == 7:
                                    bad_t += 1
                                else:
                                    bad_o += 1
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


def check_sim():
    for split in (0, 1):
        for (B, L, S, K) in [(2, 700, 520, 256), (1, 300, 100, 256), (1, 5000, 4096, 256)]:
            af = _rand(B, L, K, scale=0.9, seed=1)
            bf = _rand(B, S, K, scale=0.9, seed=2)
            a, b = _planes(af, split), _planes(bf, split)
            scale = 1.0 / (256 * 0.0801)
            sim = (torch.einsum("blk,bsk->bls", _q(af, split).double(), _q(bf, split).double()) * scale)
            lse_pt_ref = torch.logsumexp(sim, 2).float()   # over query cells, per 3D point
            lse_px_ref = torch.logsumexp(sim, 1).float()   # over 3D points, per query cell
            lib = _lib.load()
            ts, tl = lib.opp_sim_tiles(S), lib.opp_sim_tiles(L)

            def lse(x, y, rows, cols, tiles):
                pm = torch.empty(B * rows, tiles, device=DEV)
                ps = torch.empty(B * rows, tiles, device=DEV)
                out = torch.empty(B, rows, device=DEV)
                _lib.call("opp_sim_lse", _lib.ptr(x), _lib.ptr(y), _lib.ptr(pm), _lib.ptr(ps), B, rows,
                          cols, K, scale, split, _lib.stream())
                _lib.call("opp_lse_finalize", _lib.ptr(pm), _lib.ptr(ps), _lib.ptr(out), B * rows, tiles,
                          _lib.stream())
                return out

            lse_pt = lse(a, b, L, S, ts)
            lse_px = lse(b, a, S, L, tl)
            torch.cuda.synchronize()
            _close(f"sim split={split} lse_pt B={B} L={L} S={S}", lse_pt, lse_pt_ref, 1e-5, 1e-4)
            _close("sim lse_px", lse_px, lse_px_ref, 1e-5, 1e-4)

            conf = torch.full((B, L, S), float("nan"), device=DEV)

            def best(x, y, own, other, own_is_pt, rows, cols, tiles, conf_out):
                pv = torch.empty(B * rows, tiles, device=DEV)
                pi = torch.empty(B * rows, tiles, device=DEV, dtype=torch.int32)
                bv = torch.empty(B, rows, device=DEV)
                bi = torch.empty(B, rows, device=DEV, dtype=torch.int32)
                _lib.call("opp_sim_conf", _lib.ptr(x), _lib.ptr(y), _lib.ptr(own), _lib.ptr(other),
                          own_is_pt, _lib.ptr(conf_out), _lib.ptr(pv), _lib.ptr(pi), B, rows, cols, K,
                          scale, split, _lib.stream())
                _lib.call("opp_best_finalize", _lib.ptr(pv), _lib.ptr(pi), _lib.ptr(bv), _lib.ptr(bi),
                          B * rows, tiles, _lib.stream())
                return bv, bi

            pt_val, pt_idx = best(a, b, lse_pt, lse_px, 1, L, S, ts, conf)
            px_val, px_idx = best(b, a, lse_px, lse_pt, 0, S, L, tl, None)
            torch.cuda.synchronize()
            conf_ref = (torch.softmax(sim, 1) * torch.softmax(sim, 2)).float()
            _close("sim conf", conf, conf_ref, 5e-4, 1e-7)
            # maxima must agree with the conf matrix the kernel itself wrote (index-exact)
            v, i = conf.max(2)
            assert torch.equal(pt_idx.long(), i), "row argmax mismatch"
            assert torch.equal(pt_val, v), "row max mismatch"
            v, i = conf.max(1)
            _close("sim col max", px_val, v, 1e-5, 1e-9)
            agree = (px_idx.long() == i).float().mean().item()
            print(f"  col argmax agreement {agree:.6f}")
            assert agree > 0.999


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
    ref = torch.relu(F.conv2d(imgf.double(), _q(w64, split)[:, :49].reshape(C, 1, 7, 7).double(),
                              _q(w64, split)[:, 49].double(), stride=2, padding=3)).permute(0, 2, 3, 1).float()
    _close(f"conv1_gemm split={split} u8={u8} {H}x{W}", _unplanes(out, split), ref,
           *_tol(split, (2e-3, 2e-3), (2e-5, 2e-5)))


def check_conv1_gemm():
    for split in (0, 1):
        _conv1_gemm_case(split, 2, 96, 128, 128, False)
        _conv1_gemm_case(split, 1, 72, 200, 128, True)     # ragged 16x16 im2col tiles, uint8 image


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
    for split in (0, 1):
        B, S, d = 2, 1000, 256
        kvf = torch.cat([_rand(B, S, d, seed=1).abs() + 0.1, _rand(B, S, d, seed=2)], 2)
        kv = _planes(kvf, split)
        mw = _rand(d, d, scale=0.06, seed=3)
        chunks = _lib.load().opp_kv_chunks_b(S, B)
        pl = 2 if split else 1
        part = torch.empty(B, chunks, 8, 33, 32, device=DEV)
        mt = torch.empty(B, d, pl * d, device=DEV, dtype=torch.half)
        ksum = torch.empty(B, d, device=DEV)
        _lib.call("opp_kv_partial", _lib.ptr(kv), _lib.ptr(part), B, S, d, split, _lib.stream())
        _lib.call("opp_kv_finalize", _lib.ptr(part), _lib.ptr(mw), _lib.ptr(mt), _lib.ptr(ksum), B,
                  chunks, d, float(S), split, _lib.stream())
        torch.cuda.synchronize()
        kvq = _q(kvf, split).double()
        K = kvq[..., :d].view(B, S, 8, 32)
        V = kvq[..., d:].view(B, S, 8, 32)
        KV = torch.einsum("bshd,bshv->bhdv", K, V) / S
        ref_ksum = K.sum(1).reshape(B, d).float()
        # mt[b][c][h*32+dd] = sum_v mw[c][h*32+v] KV[b][h][dd][v]
        ref_mt = torch.einsum("chv,bhdv->bchd", mw.double().view(d, 8, 32), KV).reshape(B, d, d).float()
        _close(f"kv ksum split={split}", ksum, ref_ksum, 1e-5, 1e-3)
        _close("kv mt", _unplanes(mt, split), ref_mt, *_tol(split, (2e-3, 1e-4), (2e-5, 1e-6)))


def check_match_select():
    B, L, hc, wc = 3, 2500, 20, 24
    S = hc * wc
    g = torch.Generator().manual_seed(0)
    conf = torch.rand(B, L, S, generator=g).to(DEV) * 0.3
    # plant mutual maxima
    for b in range(B):
        perm = torch.randperm(S, generator=g)[:200]
        rows = torch.randperm(L, generator=g)[:200]
        conf[b, rows, perm] = 0.5 + 0.5 * torch.rand(200, generator=g).to(DEV)
    pt_val, pt_idx = conf.max(2)
    px_idx = conf.max(1).indices
    kpts = torch.rand(B, L, 3, device=DEV)
    scale = torch.rand(B, 2, device=DEV) + 0.5
    cap = B * min(L, S)
    scratch = torch.empty((B * L + 1023) // 1024 + 2, device=DEV, dtype=torch.int32)
    b_ids = torch.empty(cap, device=DEV, dtype=torch.int64)
    i_ids, j_ids = torch.empty_like(b_ids), torch.empty_like(b_ids)
    mconf = torch.empty(cap, device=DEV)
    mk3 = torch.empty(cap, 3, device=DEV)
    mkc = torch.empty(cap, 2, device=DEV)
    cnt = torch.zeros(1, device=DEV, dtype=torch.int32)
    pt_idx32, px_idx32 = pt_idx.int(), px_idx.int()
    _lib.call("opp_match_select", _lib.ptr(pt_val), _lib.ptr(pt_idx32), _lib.ptr(px_idx32),
              _lib.ptr(kpts), _lib.ptr(scale), B, L, hc, wc, 0.4, 2, 8.0, _lib.ptr(scratch),
              _lib.ptr(b_ids), _lib.ptr(i_ids), _lib.ptr(j_ids), _lib.ptr(mconf), _lib.ptr(mk3),
              _lib.ptr(mkc), _lib.ptr(cnt), 0, _lib.stream())
    torch.cuda.synchronize()
    M = int(cnt.item())
    # reference semantics (coarse_matching.py:142-172)
    mask = conf > 0.4
    mask = mask.view(B, L, hc, wc)
    mask[:, :, :2] = False
    mask[:, :, :, :2] = False
    mask = mask.view(B, L, S)
    mask = mask * (conf == conf.max(2, keepdim=True)[0]) * (conf == conf.max(1, keepdim=True)[0])
    mv, aj = mask.max(2)
    rb, ri = torch.where(mv)
    rj = aj[rb, ri]
    print(f"  match_select: M={M} ref={len(rb)}")
    assert M == len(rb) and M > 100
    assert torch.equal(b_ids[:M], rb) and torch.equal(i_ids[:M], ri) and torch.equal(j_ids[:M], rj)
    assert torch.equal(mconf[:M], conf[rb, ri, rj])
    assert torch.equal(mk3[:M], kpts[rb, ri])
    ref_c = torch.stack([rj % wc, rj // wc], 1) * (8.0 * scale[rb][:, [1, 0]])
    _close("match_select mkpts_c", mkc[:M], ref_c, 1e-6, 1e-5)


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
            lib = _lib.load()
            ts, tl = lib.opp_sim_tiles(S), lib.opp_sim_tiles(L)
            lse_pt, lse_px = torch.empty(B, L, device=DEV), torch.empty(B, S, device=DEV)
            ops.sim_lse(a, b, B, L, S, K, scale, torch.empty(B * L, ts, device=DEV),
                        torch.empty(B * L, ts, device=DEV), lse_pt, split)
            ops.sim_lse(b, a, B, S, L, K, scale, torch.empty(B * S, tl, device=DEV),
                        torch.empty(B * S, tl, device=DEV), lse_px, split)
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
    ops.kv_state(kv, part, mw, mt, ksum, B, S, d, float(S), True, kv_split=False)
    torch.cuda.synchronize()
    kvq = kv.double().view(B, S, 2 * d)
    K, V = kvq[..., :d].view(B, S, 8, 32), kvq[..., d:].view(B, S, 8, 32)
    KV = torch.einsum("bshd,bshv->bhdv", K, V) / S
    ref_mt = torch.einsum("chv,bhdv->bchd", mw.double().view(d, 8, 32), KV).reshape(B, d, d).float()
    _close("kv1 ksum", ksum, K.sum(1).reshape(B, d).float(), 1e-5, 1e-3)
    _close("kv1 mt", _unplanes(mt, 1), ref_mt, 2e-5, 1e-6)


CHECKS = {
    "linear_act": check_linear_act,
    "linear_ln": check_linear_ln,
    "linear_q": check_linear_q,
    "linear_act_shared": check_linear_act_shared,
    "conv": check_conv,
    "conv_up_odd_clusters": check_conv_up_odd_clusters,
    "conv_win": check_conv_win,
    "sim": check_sim,
    "conv1_gemm": check_conv1_gemm,
    "kpt_encode": check_kpt_encode,
    "kv_state": check_kv_state,
    "match_select": check_match_select,
    "fine": check_fine,
    "full_attention": check_full_attention,
    "loftr_kernels": check_loftr_kernels,
    "sim_colmax": check_sim_colmax,
    "sim_lse_cols": check_sim_lse_cols,
    "kv_single_plane": check_kv_single_plane,
}


# run only in a child process whose environment selects the launch configuration
CHILD_CHECKS = {"conv_up": _conv_up_cases}


def main(argv):
    if len(argv) == 2 and argv[0] == "--one":
        print(f"[{argv[1]}]")
        {**CHECKS, **CHILD_CHECKS}[argv[1]]()
        print(f"[{argv[1]}] OK")
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
