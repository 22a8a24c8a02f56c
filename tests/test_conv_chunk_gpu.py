"""pytest -m gpu: the conv engine's ring slot width (GemmShape.bk).  3x3 conv layers whose padded
output width is above 128 fill and release each 64-channel ring stage as two 32-channel slots
(64-byte swizzle), the others as one; $OPP_CONV_BK=32|64 forces one width for every conv layer.  The
width sets the fp32 accumulation order, so it must depend on the layer only: these tests check the
32-wide kernels against fp64, the window convolutions against the dense ones bit for bit at both
widths, and that the outputs at 32 do not depend on the launch configuration.

The engine reads its knobs once per process, so every case runs in a child process: either an entry
of tests/kernel_checks.py (`--one name`) or a function of this module (`python <this file> name ...`)."""
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
KERNEL_CHECKS = os.path.join(ROOT, "tests", "kernel_checks.py")


def _run(argv, timeout=1200, **env):
    r = subprocess.run([sys.executable, *argv], env=dict(os.environ, **env), timeout=timeout)
    assert r.returncode == 0, f"{argv} failed in a child process with {env}"


# kernel_checks entries at a forced chunk width: fp64 checks of 128 / 208 (16-channel tail) / 256
# channels, stride 2, 1x1, tokens, the fused upsample-add (EpiConvUp, accumulator over the ring), and
# the window convolutions A and B (A_WIN, also with the row count on the device) bit-equal to the
# dense ones at the window positions
FORCED = [("conv", "32"), ("conv_up", "32"), ("conv_win", "32"), ("conv_win", "64"),
          ("conv_win_production_tiles", "32"), ("conv_win_production_tiles", "64")]


@pytest.mark.gpu
@pytest.mark.parametrize("check,bk", FORCED, ids=[f"{c}-bk{b}" for c, b in FORCED])
def test_conv_checks_at_chunk_width(check, bk):
    _run([KERNEL_CHECKS, "--one", check], OPP_CONV_BK=bk, OPP_LOG_TILES="1")


@pytest.mark.gpu
@pytest.mark.parametrize("bk", ["64", "32"])
def test_fine_windows_equal_dense_at_chunk_width(bk):
    """the model's window head (layer1_outconv2 on the match windows) against its dense map, bit for bit"""
    _run(["-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
          os.path.join(ROOT, "tests", "test_model_gpu.py") + "::test_fine_windows_path_equals_dense_map"],
         OPP_CONV_BK=bk)


# The backbone's convolutions (kernel_checks.BACKBONE_CONVS) under the default chunk-width rule: the
# tile configuration the fp16x3 mode runs with at bench.py's batch 64, (mma_n, N tiles, ring stages,
# cluster, bk), and in the fp16 mode (mma_n, N tiles, bk).
BACKBONE_TILES = {
    "layer1 conv1":      ((128, 1, 3, 2, 64), (128, 1, 64)),
    "layer1 conv2":      ((128, 1, 3, 2, 64), (128, 1, 64)),
    "layer2.0 conv1":    ((208, 1, 2, 2, 32), (208, 1, 32)),
    "layer2.0 down":     ((208, 1, 2, 2, 64), (208, 1, 64)),
    "layer2 conv2":      ((208, 1, 2, 2, 32), (208, 1, 32)),
    "layer3.0 conv1":    ((256, 1, 2, 2, 32), (256, 1, 32)),
    "layer3.0 down":     ((256, 1, 2, 2, 64), (256, 1, 64)),
    "layer3 conv2":      ((256, 1, 2, 2, 32), (256, 1, 32)),
    "layer3_outconv":    ((256, 1, 2, 2, 64), (256, 1, 64)),
    "layer2_outconv":    ((128, 2, 2, 2, 64), (256, 1, 64)),
    "layer2_outconv2.0": ((256, 1, 2, 2, 32), (256, 1, 32)),
    "layer2_outconv2.3": ((208, 1, 2, 2, 32), (208, 1, 32)),
    "layer1_outconv":    ((208, 1, 2, 2, 64), (208, 1, 64)),
    "layer1_outconv2.0": ((208, 1, 2, 2, 32), (208, 1, 32)),
    "layer1_outconv2.3": ((128, 1, 3, 2, 64), (128, 1, 64)),
}


def layers(split):
    """every BACKBONE_CONVS launch against fp64, and its tile configuration against BACKBONE_TILES"""
    from tests import kernel_checks as kc
    split = int(split)
    assert set(BACKBONE_TILES) == {c[0] for c in kc.BACKBONE_CONVS}
    failed = []
    for name, (want1, want0) in BACKBONE_TILES.items():
        try:
            _, _, t, (lo, hi) = kc._backbone_conv(split, name)
            got = (t["mma_n"], -(-t["n"] // t["block_n"]), t["stages"], t["cluster"], t["bk"])
            print(f"  {name}: mma_n {got[0]} N tiles {got[1]} stages {got[2]} alias {t['alias']} cluster {got[3]} "
                  f"bk {got[4]} tiles per cluster {lo}-{hi}")
            want = want1 if split else want0
            have = got if split else (got[0], got[1], got[4])
            assert have == want, f"{name}: tile {have}, expected {want}"
            assert hi >= 8, f"{name}: only {hi} tiles per cluster"
        except AssertionError as e:   # go on: which launches fail locates a defect
            print(f"  {name}: FAILED: {e}")
            failed.append(name)
    assert not failed, f"split={split}: {failed}"


@pytest.mark.gpu
@pytest.mark.parametrize("split", ["1", "0"])
def test_conv_layers_chunk_widths(split):
    _run([os.path.abspath(__file__), "layers", split], OPP_LOG_TILES="1")


# Launch configurations forced through the engine's knobs at bk = 32, and the tile fields each must
# show: outputs must be bit-identical to the default configuration's.
VARIANTS = {
    "default": ({}, {"layer1 conv2": {"cluster": 2, "stages": 3}, "layer2 conv2": {"cluster": 2, "stages": 2},
                     "layer3 conv2 batch 1": {"mma_n": 64, "block_n": 64}}),
    "cluster4": ({"OPP_CLUSTER": "4"}, {"layer1 conv2": {"cluster": 4}, "layer3_outconv": {"cluster": 4}}),
    "stages2": ({"OPP_STAGES": "2"}, {"layer1 conv2": {"stages": 2}}),
    "nsplit0": ({"OPP_NSPLIT": "0"}, {"layer3 conv2 batch 1": {"mma_n": 256, "block_n": 256}}),
}
VARIANT_LAUNCHES = ["layer1 conv2", "layer2 conv2", "layer3_outconv", "layer1_outconv", "layer3 conv2 batch 1"]


def variant(tag, out_dir):
    """VARIANT_LAUNCHES (fp16x3) under this process's knobs, saved to out_dir/<tag>.pt; the default
    configuration is also checked against fp64"""
    import torch
    from tests import kernel_checks as kc
    want = VARIANTS[tag][1]
    saved = {}
    for name in VARIANT_LAUNCHES:
        if name == "layer3 conv2 batch 1":
            with kc._tile_log() as new:
                out, tok = kc._conv_case(1, 1, 64, 64, 256, 256, 256, 256, 3, 1, 1, True, False,
                                         check=tag == "default", accum_tol=True)
            t = kc._conv_tile(new, 256, 256, 3)
        else:
            out, tok, t, _ = kc._backbone_conv(1, name, check=tag == "default")
        print(f"  [{tag}] {name}: mma_n {t['mma_n']} block_n {t['block_n']} stages {t['stages']} "
              f"cluster {t['cluster']} bk {t['bk']}")
        assert t["bk"] == 32, f"[{tag}] {name}: bk {t['bk']}"
        assert all(t[f] == v for f, v in want.get(name, {}).items()), f"[{tag}] {name}: tile {t}, expected {want[name]}"
        saved[name] = (out.cpu(), tok.cpu() if tok is not None else None)
    torch.save(saved, os.path.join(out_dir, f"{tag}.pt"))


@pytest.mark.gpu
def test_conv_launch_invariance_chunk32():
    import torch
    from tests import kernel_checks as kc
    with tempfile.TemporaryDirectory() as d:
        for tag, (env, _) in VARIANTS.items():
            _run([os.path.abspath(__file__), "variant", tag, d], OPP_CONV_BK="32", OPP_LOG_TILES="1", **env)
        base = torch.load(os.path.join(d, "default.pt"))
        differ = []
        for tag in VARIANTS:
            if tag == "default":
                continue
            for name, tensors in torch.load(os.path.join(d, f"{tag}.pt")).items():
                for what, a, b in zip(("out", "tok"), tensors, base[name]):
                    if a is not None and not kc._bits_equal(a, b):
                        differ.append(f"{tag}: {name} {what} ({int((a != b).sum())} fp16 elements)")
    assert not differ, f"outputs at bk = 32 depend on the launch configuration: {differ}"


if __name__ == "__main__":
    globals()[sys.argv[1]](*sys.argv[2:])
