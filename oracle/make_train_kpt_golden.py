"""Writes tests/golden/reference/train_kpt.npz: KeypointEncoding_linear of the UNMODIFIED reference
(utils/position_encoding.py:46-79 after utils/normalize.py:16-26), forward and backward in fp64 on the
CPU, on the seeded case of make_case (B = 2, N = 301), so that the tests need nothing from the
reference tree.  Stored: the output [B, 256, N] and the gradient of each of the eight encoder
parameters under objective() (sampled entries plus absmax, coarse_loss.put_sampled).  The weights are
workload.synthetic_state_dict(0).

    python -m oracle.make_train_kpt_golden
"""
import copy
import os
import sys

import numpy as np
import torch

from . import oracle, workload
from .coarse_loss import put_sampled

SAMPLES = 1024
PARAMS = tuple(f"encoder.{i}.{k}" for i in (0, 3, 6, 9) for k in ("weight", "bias"))


def make_case(seed=0, B=2, N=301):
    """keypoints3d fp64 [B, N, 3] (an object-sized box off the origin), descriptors [B, 256, N] and the
    objective's weights g [B, 256, N]."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    kpts = torch.rand(B, N, 3, generator=g, dtype=f64) * torch.tensor([0.12, 0.08, 0.1], dtype=f64) + \
        torch.tensor([0.3, -0.2, 0.9], dtype=f64)
    return {"kpts": kpts, "desc": torch.randn(B, 256, N, generator=g, dtype=f64),
            "g": torch.randn(B, 256, N, generator=g, dtype=f64)}


def objective(out, case):
    return (out * case["g"].to(out)).sum()


def reference_encoding(sd, case):
    """(output, [d param in PARAMS order]) of the reference module in fp64."""
    from . import ref_shims
    ref_shims.install()
    from src.models.OnePosePlus.utils.normalize import normalize_3d_keypoints  # type: ignore
    model = ref_shims.build_reference_model(sd, copy.deepcopy(oracle.DEFAULT_CONFIG))
    enc = model.kpt_3d_pos_encoding.double().train()
    out = enc(normalize_3d_keypoints(case["kpts"]), case["desc"])
    params = [dict(enc.named_parameters())[n] for n in PARAMS]
    return out.detach(), list(torch.autograd.grad(objective(out, case), params))


def main():
    sd = workload.synthetic_state_dict(0)
    case = make_case()
    out, grads = reference_encoding(sd, case)
    res = {}
    put_sampled(res, "out", out, k=SAMPLES)
    for n, g in zip(PARAMS, grads):
        put_sampled(res, f"d_{n}", g, k=SAMPLES)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "train_kpt.npz")
    np.savez_compressed(path, **res)
    print(f"train_kpt -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
