"""pytest -m gpu: the token-row GEMM epilogues on the accumulator registers — exact ties in the
dual-softmax passes, bit-identical repeat calls (no order-dependent merges), and a ragged last N tile."""
import pytest
import torch

from onepose_plus_plus_b200 import _lib, ops
from tests.kernel_checks import DEV, _close, _planes, _q, _rand, _unplanes

pytestmark = pytest.mark.gpu

SCALE = 1.0 / (256 * 0.0801)


def _sim_inputs(B, L, S, K, split, dup_rows=False, dup_cols=False):
    af = _rand(B, L, K, scale=0.9, seed=1)
    bf = _rand(B, S, K, scale=0.9, seed=2)
    if dup_rows:     # rows L/2.. repeat rows 0..: every column maximum is tied
        af[:, L // 2:] = af[:, : L - L // 2]
    if dup_cols:     # columns S/2.. repeat columns 0..: every row maximum is tied
        bf[:, S // 2:] = bf[:, : S - S // 2]
    return af, bf, _planes(af, split), _planes(bf, split)


def _lse_cols(a, b, B, L, S, K, split):
    ts, groups = ops.sim_tiles(S), (L + 31) // 32
    out = {"lse_rows": torch.full((B, L), float("nan"), device=DEV),
           "lse_cols": torch.full((B, S), float("nan"), device=DEV),
           "col_m": torch.full((B, groups, S), float("nan"), device=DEV),
           "col_s": torch.full((B, groups, S), float("nan"), device=DEV)}
    ops.sim_lse_cols(a, b, B, L, S, K, SCALE, torch.empty(B * L, ts, device=DEV), torch.empty(B * L, ts, device=DEV),
                     out["lse_rows"], out["col_m"], out["col_s"], out["lse_cols"], split)
    return out


def _conf_colmax(a, b, lse_rows, lse_cols, B, L, S, K, split):
    ts = ops.sim_tiles(S)
    out = {"conf": torch.full((B, L, S), float("nan"), device=DEV),
           "bv": torch.empty(B, L, device=DEV), "bi": torch.empty(B, L, device=DEV, dtype=torch.int32),
           "colmax": torch.full((B, S), -1, device=DEV, dtype=torch.int32)}
    ops.sim_conf_colmax(a, b, lse_rows, lse_cols, out["conf"], B, L, S, K, SCALE, torch.empty(B * L, ts, device=DEV),
                        torch.empty(B * L, ts, device=DEV, dtype=torch.int32), out["bv"], out["bi"],
                        out["colmax"], split)
    return out


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("dup", ["rows", "cols"])
def test_dual_softmax_exact_ties(split, dup):
    """Duplicated rows / columns give bit-equal conf values; the row argmax is the first tied column
    and the value-based mutual test (rowmax == colmax[argmax]) selects what torch selects."""
    B, L, S, K = 2, 700, 520, 256      # 520 columns: two full N tiles and an 8-column last tile
    af, bf, a, b = _sim_inputs(B, L, S, K, split, dup_rows=dup == "rows", dup_cols=dup == "cols")
    st = _lse_cols(a, b, B, L, S, K, split)
    r = _conf_colmax(a, b, st["lse_rows"], st["lse_cols"], B, L, S, K, split)
    torch.cuda.synchronize()
    conf = r["conf"]
    if dup == "rows":
        h = L - L // 2
        assert torch.equal(conf[:, L // 2:].view(torch.int32), conf[:, :h].view(torch.int32)), "tied rows differ"
    else:
        h = S - S // 2
        assert torch.equal(conf[:, :, S // 2:].view(torch.int32), conf[:, :, :h].view(torch.int32)), \
            "tied columns differ"
    sim = torch.einsum("blk,bsk->bls", _q(af, split).double(), _q(bf, split).double()) * SCALE
    _close(f"tied conf split={split} dup={dup}", conf, (torch.softmax(sim, 1) * torch.softmax(sim, 2)).float(),
           5e-4, 1e-7)
    rowmax = conf.max(2, keepdim=True).values
    first = (conf == rowmax).int().argmax(2)          # torch.argmax: the first maximal index
    assert torch.equal(r["bv"], rowmax[..., 0]), "row maxima differ"
    assert torch.equal(r["bi"].long(), first), "row argmax is not the first tied column"
    assert torch.equal(r["colmax"], conf.max(1).values.view(torch.int32)), "column maxima are not the bits of conf.max(1)"
    mutual = (conf == rowmax) & (conf == conf.max(1, keepdim=True).values)
    sel = torch.gather(r["colmax"], 1, r["bi"].long()) == r["bv"].view(torch.int32)
    assert torch.equal(sel, mutual.any(2)), "mutual-nearest selection differs from torch"


@pytest.mark.parametrize("split", [0, 1])
def test_dual_softmax_repeat_bit_identical(split):
    B, L, S, K = 2, 1300, 1000, 256
    _, _, a, b = _sim_inputs(B, L, S, K, split)
    runs = []
    for _ in range(2):
        st = _lse_cols(a, b, B, L, S, K, split)
        st.update(_conf_colmax(a, b, st["lse_rows"], st["lse_cols"], B, L, S, K, split))
        runs.append(st)
    torch.cuda.synchronize()
    for k, v in runs[0].items():
        assert torch.equal(v.view(torch.int32), runs[1][k].view(torch.int32)), f"{k} differs between two calls"


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("rows", [600, 12000])   # 600: N-split cluster (DSMEM statistics); 12000: whole rows
def test_linear_ln_repeat_bit_identical(split, rows):
    n, k0 = 256, 256
    a0 = _planes(_rand(rows, k0, seed=1), split)
    w = _planes(_rand(1, n, k0, scale=0.05, seed=3), split)
    gamma, beta = 1 + 0.1 * _rand(n, seed=4), 0.1 * _rand(n, seed=5)
    res = _planes(_rand(rows, n, seed=6), split)
    pl = 2 if split else 1
    outs = []
    for _ in range(2):
        o16 = torch.full((rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
        o32 = torch.full((rows, n), float("nan"), device=DEV)
        ops.linear_ln(a0, None, w, False, gamma, beta, 1, rows, split, resid=res, out16=o16, out32=o32)
        outs.append((o16, o32))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0].view(torch.int16), outs[1][0].view(torch.int16)), "out16 differs between calls"
    assert torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32)), "out32 differs between calls"
    assert not torch.isnan(outs[0][1]).any(), "unwritten LayerNorm output"


@pytest.mark.parametrize("split", [0, 1])
def test_linear_act_ragged_last_tile(split):
    """N = 272: a 256-column tile and a 16-column last tile (linear_act needs N % 16 == 0)."""
    rows, k0, n, act_cols = 1000, 256, 272, 256
    a0f, wf = _rand(rows, k0, seed=1), _rand(n, k0, scale=0.05, seed=3)
    pl = 2 if split else 1
    out = torch.full((rows, pl * n), float("nan"), device=DEV, dtype=torch.half)
    _lib.call("opp_linear_act_f16", _lib.ptr(_planes(a0f, split)), k0, None, 0, _lib.ptr(_planes(wf, split)),
              _lib.ptr(out), rows, n, 1, act_cols, split, _lib.stream())
    torch.cuda.synchronize()
    ref = (_q(a0f, split).double() @ _q(wf, split).double().t()).float()
    ref[:, :act_cols] = torch.relu(ref[:, :act_cols])
    tol = (2e-5, 2e-5) if split else (2e-3, 2e-3)
    _close(f"linear_act N=272 split={split}", _unplanes(out, split), ref, *tol)
