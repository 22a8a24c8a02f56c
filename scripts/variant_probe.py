"""One library build on the GPU: kernel checks of every wgmma-engine epilogue and of the kernels behind
runtime options, golden end-to-end parity, and batch-64 forward timing with a per-op breakdown,
for each option set given on the command line.

    OPP_B200_LIB=variants/libopp_<name>.so python scripts/variant_probe.py <tag> [opt=val,opt=val ...]

Prints one JSON line."""
import io
import json
import os
import sys
import time
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_plus_plus_b200 import _lib  # noqa: E402
from oracle import workload  # noqa: E402
from tests import golden_io, kernel_checks, parity  # noqa: E402

tag = sys.argv[1] if len(sys.argv) > 1 else "probe"
configs = [dict((kv.split("=")[0], int(kv.split("=")[1])) for kv in a.split(",") if kv)
           for a in (sys.argv[2:] or [""])]
B = 64
res = {"tag": tag, "lib": _lib.LIB_PATH, "checks": {}, "timing": {}, "golden": {}}
t_start = time.time()


def guarded(name, fn):
    try:
        fn()
        torch.cuda.synchronize()
        res["checks"][name] = "ok"
    except BaseException as e:  # noqa: BLE001  (a device trap surfaces as RuntimeError)
        res["checks"][name] = f"FAIL: {type(e).__name__}: {str(e)[:300]}"
        traceback.print_exc()


def golden(label):
    for case in golden_io.cases():
        data, z = golden_io.load(case)
        got = parity.run_cuda(data)
        if not torch.is_tensor(got.get("conf_matrix")):
            got["conf_matrix"] = got["conf_matrix"].materialize()
        res["golden"][f"{case}[{label}]"] = parity.compare(got, {k: z[k] for k in z.files}, max_borderline=0)


def c5_shape():
    """BASELINE configs[4]: 640x480 image (60x80 coarse cells), 20000 points, window 5 — end-to-end
    parity against the oracle on a planted bank (not yet part of the pytest -m gpu suite)."""
    from oracle import oracle
    sd = workload.synthetic_state_dict(0)
    data, _ = workload.planted_workload(sd, 480, 640, 20000, 3000, batch=1)
    ref = {k: v.clone() for k, v in data.items()}
    oracle.forward(sd, ref)
    got = parity.run_cuda(data)
    res["golden"]["c5_shape"] = parity.compare(got, ref)
    err = (got["conf_matrix"].cpu() - ref["conf_matrix"]).abs().max().item()
    assert err <= 1e-3, f"conf_matrix max err {err:.2e}"


_STEP = {}


def make_step():
    """the bench's resident step (batch B, 512x512, shared 5000-point planted bank)"""
    if _STEP:
        return _STEP["fn"]
    sd = workload.synthetic_state_dict(0)
    model = parity.cuda_model()
    data, _ = workload.planted_workload(sd, 512, 512, 5000, 3000, batch=1)
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(100)
    imgs = (data["query_image"] + 0.02 * torch.randn(B, 1, 512, 512, generator=g)).clamp(0, 1).to(dev)
    scale = data["query_image_scale"].expand(B, -1).contiguous().to(dev)
    bank = {k: data[k].to(dev) for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db")}

    def step():
        d = {"query_image": imgs, "query_image_scale": scale,
             **{k: v.expand(B, -1, -1) for k, v in bank.items()}}
        model(d)
        return d

    _STEP["fn"] = step
    return step


def timing(label):
    step = make_step()
    for _ in range(3):
        d = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        d = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    rows = _lib.profile_ops(step, io.StringIO())
    res["timing"][label] = {
        "batch": B, "ms_per_forward": ms, "images_per_s": B / ms * 1e3, "M": int(d["b_ids"].numel()),
        "ops_ms": {k: round(v[1], 3) for k, v in sorted(rows.items(), key=lambda kv_: -kv_[1][1])}}


# options: (historic: C-ABI switches, since removed) except "colmax" / "lse_cols", host-flow switches of the
# model (column maxima of conf / column log-sum-exp from the first pass instead of a second GEMM).  Every config
# starts from the defaults; its label lists the options it turns on.
EXPERIMENTAL_CHECK = {}
DEFAULTS = {"colmax": 1, "lse_cols": 1, "kv1": 1, "lazy": 0}
MODEL_ATTR = {"colmax": "coarse_colmax", "lse_cols": "coarse_lse_cols", "kv1": "kv_single_plane",
              "lazy": "conf_matrix_mode"}
ATTR_VALUE = {"lazy": {0: "eager", 1: "lazy"}}


def apply(cfg):
    for k, v in {**DEFAULTS, **cfg}.items():
        if k in MODEL_ATTR:
            try:
                setattr(parity.cuda_model(), MODEL_ATTR[k], ATTR_VALUE[k][v] if k in ATTR_VALUE else bool(v))
            except RuntimeError:   # no CUDA device (dry run of the script logic)
                pass
        else:
            raise KeyError(k)


first = True
for cfg in configs:
    label = ",".join(f"{k}={v}" for k, v in cfg.items()) or "default"
    if first:   # the engine's epilogues do not depend on the runtime options
        apply({})
        for name in ("linear_ln", "conv", "linear_act", "linear_q", "sim"):
            guarded(name, kernel_checks.CHECKS[name])
        guarded("conv1_gemm", kernel_checks.CHECKS["conv1_gemm"])
        guarded("c5_shape", c5_shape)
        first = False
    for k, v in cfg.items():
        if v and k in EXPERIMENTAL_CHECK:   # these set and restore their own option
            guarded(f"{EXPERIMENTAL_CHECK[k]}[{label}]", kernel_checks.CHECKS[EXPERIMENTAL_CHECK[k]])
    apply(cfg)
    guarded(f"kv_state[{label}]", kernel_checks.check_kv_state)
    guarded(f"golden[{label}]", lambda label=label: golden(label))
    guarded(f"timing[{label}]", lambda label=label: timing(label))
apply({})

res["seconds"] = round(time.time() - t_start, 1)
print(json.dumps(res))
