"""pytest -m gpu: the token-row GEMMs' ring slot width (GemmShape.bk).  Layers whose full-width tile is
above 128 columns (the coarse transformer's N = 256 / 512 projections, the dual-softmax passes) fill
and release each 64-column ring stage as two 32-column slots (64-byte swizzle), the others as one;
$OPP_ROWS_BK=32|64 forces one width for every token-row GEMM.  The width sets the fp32 accumulation
order, so it must depend on the layer only: these tests check every token-row entry point at both
widths against fp64 at the forward's launch configurations, that the rule gives a batch-1 launch
(N split, LayerNorm pair cluster) the width of the batch-64 one and the same bits per image, and
that the lazy conf_matrix stays bit-equal to the eager one.

The engine reads its knobs once per process, so every case runs in a child process: either an entry
of tests/kernel_checks.py (`--one name`), a pytest node, or a function of this module
(`python <this file> name ...`)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
KERNEL_CHECKS = os.path.join(ROOT, "tests", "kernel_checks.py")


def _run(argv, timeout=1500, **env):
    r = subprocess.run([sys.executable, *argv], env=dict(os.environ, **env), timeout=timeout)
    assert r.returncode == 0, f"{argv} failed in a child process with {env}"


# kernel_checks entries at a forced slot width: every ROW_GEMMS launch (bench batch 64 and batch 1:
# N split, LayerNorm pair cluster, a0_shared, concatenated A, w_batched, the fine stage with the row
# count on the host and on the device) against fp64 with its pinned tile, the device-count edges,
# row masks, N-tile-width invariance, and the dual-softmax passes (column masks, row counts)
ROW_CHECKS = ["row_gemms_split1", "row_gemms_split0", "row_dyn", "row_masks", "row_launch_invariance",
              "linear_act", "linear_ln", "linear_q", "linear_act_shared", "sim_colmax", "sim_lse_cols",
              "sim_col_mask"]
FORCED = [(c, "32") for c in ROW_CHECKS] + [("row_gemms_split1", "64"), ("sim_lse_cols", "64")]


@pytest.mark.gpu
@pytest.mark.parametrize("check,bk", FORCED, ids=[f"{c}-bk{b}" for c, b in FORCED])
def test_row_checks_at_slot_width(check, bk):
    _run([KERNEL_CHECKS, "--one", check], OPP_ROWS_BK=bk, OPP_LOG_TILES="2")


@pytest.mark.gpu
@pytest.mark.parametrize("bk", ["32", "64"])
def test_row_epilogues_at_slot_width(bk):
    """exact dual-softmax ties, bit-identical repeat calls (also the LayerNorm pair cluster) and a
    ragged last N tile (N = 272) at one slot width"""
    _run(["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
          os.path.join(ROOT, "tests", "test_rows_epilogue_gpu.py")], OPP_ROWS_BK=bk)


@pytest.mark.gpu
@pytest.mark.parametrize("bk", ["", "32", "64"])
def test_lazy_conf_bit_identical_at_slot_width(bk):
    """the lazy conf_matrix against the eager one (and the uint8 resident bank), bit for bit"""
    _run(["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
          os.path.join(ROOT, "tests", "test_model_gpu.py") + "::test_resident_bank_uint8_and_lazy_conf_are_bit_identical"],
         **({"OPP_ROWS_BK": bk} if bk else {}))


def _rule_bk(n):
    """the width rows_chunk_k gives a layer of N output columns: 32 above a 128-column full-width tile"""
    block_n = (n + 15) & ~15 if n <= 256 else (256 if n % 256 == 0 else 128 if n % 128 == 0 else 256)
    return 32 if block_n > 128 else 64


def rule(split):
    """every ROW_GEMMS launch at batch 64 and batch 1 under the default rule: its slot width is the
    layer's (the same at both batches, whatever the tile, cluster or N split)"""
    from tests import kernel_checks as kc
    split = int(split)
    failed = []
    for spec in kc.ROW_GEMMS:
        name, n = spec[0], spec[5]
        seen = {}
        for B in (64, 1):
            t, _ = kc._row_gemm(split, spec, B)
            seen[B] = t
            print(f"  {name} batch {B}: block_n {t['block_n']} pair {t['pair']} stages {t['stages']} bk {t['bk']}")
        if not seen[64]["bk"] == seen[1]["bk"] == _rule_bk(n):
            failed.append(f"{name}: bk {seen[64]['bk']} (batch 64), {seen[1]['bk']} (batch 1), rule {_rule_bk(n)}")
    assert not failed, f"split={split}: {failed}"


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["1", "0"])
def test_row_slot_width_rule(split):
    _run([os.path.abspath(__file__), "rule", split], OPP_LOG_TILES="2")


def batch_images():
    """image 0 of batch-64 launches against a batch-1 launch of the same image under the default
    knobs (batch 1 takes the latency N split): linear_q (EpiQ, batches = B), the K'/V rows and mlp0
    with its concatenated A operand (EpiStoreF16, one launch over B * S rows), bit for bit"""
    import torch
    from tests import kernel_checks as kc
    specs = {s[0]: s for s in kc.ROW_GEMMS}
    differ = []
    for split in (1, 0):
        for name in ("linear_q 2D", "wkv 2D", "mlp0 2D"):
            spec = specs[name]
            inp = kc._row_inputs(split, spec, 64)
            out, _ = kc._row_outputs(split, spec, 64, inp["rows"])
            with kc._tile_log() as new:
                kc._row_launch(split, spec, 64, inp, out)
                torch.cuda.synchronize()
            t64 = kc._launch_tile(new, 0, spec[5], spec[3] + spec[4], 0, kc._EPI_LOG[spec[1]])
            one = dict(inp, a0=inp["a0"][:kc.ROW_S].contiguous(),
                       a1=inp["a1"][:kc.ROW_S].contiguous() if inp["a1"] is not None else None)
            if "ksum" in inp:
                one["ksum"] = inp["ksum"][:1].contiguous()
            o1, _ = kc._row_outputs(split, spec, 1, kc.ROW_S)
            with kc._tile_log() as new:
                kc._row_launch(split, spec, 1, one, o1)
                torch.cuda.synchronize()
            t1 = kc._launch_tile(new, 0, spec[5], spec[3] + spec[4], 0, kc._EPI_LOG[spec[1]])
            print(f"  {name} split={split}: batch 64 block_n {t64['block_n']} bk {t64['bk']}, "
                  f"batch 1 block_n {t1['block_n']} bk {t1['bk']}")
            assert t64["bk"] == t1["bk"] == 32, (name, t64, t1)
            assert not torch.isnan(o1.float()).any(), f"{name}: unwritten outputs"
            if not kc._bits_equal(o1, out[:kc.ROW_S]):
                differ.append(f"{name} split={split}: {int((o1 != out[:kc.ROW_S]).sum())} elements")
            torch.cuda.empty_cache()
    assert not differ, f"batch-1 launches differ from image 0 of batch-64 launches: {differ}"


@pytest.mark.gpu
def test_batch1_rows_bit_equal_batch64():
    _run([os.path.abspath(__file__), "batch_images"], OPP_LOG_TILES="2")


if __name__ == "__main__":
    globals()[sys.argv[1]](*sys.argv[2:])
