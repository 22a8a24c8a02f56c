"""Writes tests/golden/reference/train_coarse_tf.npz: the coarse LocalFeatureTransformer of the
UNMODIFIED reference (six linear-attention layers, 3 x (self, cross)), forward and backward in fp64 on
the CPU, on the seeded case of make_case (B = 2, S = 12 x 16, N = 301), without a mask and with a pad
mask that drops the last columns of batch element 1, so that the GPU tests need nothing from the
reference tree.  Stored per case: the two outputs and the gradients of both inputs and of the 60
parameters under objective(), each as sampled entries plus its absmax (coarse_loss.put_sampled).
The inputs are regenerated from their seeds (make_case, workload.synthetic_state_dict(0)).

    python -m oracle.make_train_coarse_tf_golden
"""
import copy
import os
import sys

import numpy as np
import torch

from . import oracle, workload
from .coarse_loss import put_sampled

# the parameters of one coarse layer, in train_fine.layer_params order
LAYER_PARAMS = ("q_proj.weight", "k_proj.weight", "v_proj.weight", "merge.weight", "mlp.0.weight", "mlp.2.weight",
                "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias")
COARSE_PARAMS = tuple(f"loftr_coarse.layers.{n}.{p}" for n in range(6) for p in LAYER_PARAMS)
SAMPLES = 128
CASES = ("plain", "masked")


def make_case(seed=0, B=2, hc=12, wc=16, N=301, masked=False):
    """desc3d fp64 [B, 256, N] (the keypoint-encoding output's layout), desc2d [B, hc*wc, 256], the
    pad mask bool [B, hc*wc] (batch element B - 1 loses its last wc // 4 columns) or None, and the
    objective's weights w3 [B, N, 256], w2 [B, hc*wc, 256]."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    S = hc * wc
    desc3d = torch.randn(B, 256, N, generator=g, dtype=f64)
    desc2d = torch.randn(B, S, 256, generator=g, dtype=f64)
    w3 = torch.randn(B, N, 256, generator=g, dtype=f64)
    w2 = torch.randn(B, S, 256, generator=g, dtype=f64)
    mask = None
    if masked:
        mask = torch.ones(B, hc, wc, dtype=torch.bool)
        mask[B - 1, :, wc - wc // 4:] = False
        mask = mask.reshape(B, S)
    return {"desc3d": desc3d, "desc2d": desc2d, "mask": mask, "w3": w3, "w2": w2}


def objective(d3, d2, case):
    return (d3 * case["w3"].to(d3)).sum() + (d2 * case["w2"].to(d2)).sum()


def coarse_module(sd, dtype=torch.float64, device="cpu"):
    """The drop-in model's loftr_coarse with the weights of sd."""
    from onepose_plus_plus_b200 import OnePosePlus_model
    model = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    model.load_state_dict(sd, strict=True)
    return model.loftr_coarse.to(device=device, dtype=dtype).train()


def _grads(tf, d3, d2, desc3d, desc2d, case):
    loss = objective(d3, d2, case)
    params = dict(tf.named_parameters())
    names = [n[len("loftr_coarse."):] for n in COARSE_PARAMS]
    grads = torch.autograd.grad(loss, [desc3d, desc2d] + [params[n] for n in names])
    return d3.detach(), d2.detach(), grads[0], grads[1], list(grads[2:])


def reference_coarse(sd, case):
    """The reference LocalFeatureTransformer in fp64: (d3, d2, d desc3d, d desc2d, [d param])."""
    from . import ref_shims
    ref_shims.install()
    tf = ref_shims.build_reference_model(sd, copy.deepcopy(oracle.DEFAULT_CONFIG)).loftr_coarse.double().train()
    desc3d = case["desc3d"].clone().requires_grad_(True)
    desc2d = case["desc2d"].clone().requires_grad_(True)
    d3, d2 = tf(desc3d, desc2d, case["mask"])
    return _grads(tf, d3, d2, desc3d, desc2d, case)


def train_path_coarse(tf, case, dtype=torch.float64, device="cpu"):
    """train_path.transformer with autograd on `tf` (a coarse LocalFeatureTransformer in `dtype`):
    (d3, d2, d desc3d, d desc2d, [d param in COARSE_PARAMS order])."""
    from onepose_plus_plus_b200 import train_path
    desc3d = case["desc3d"].to(device=device, dtype=dtype).requires_grad_(True)
    desc2d = case["desc2d"].to(device=device, dtype=dtype).requires_grad_(True)
    mask = None if case["mask"] is None else case["mask"].to(device)
    d3, d2 = train_path.transformer(tf, desc3d, desc2d, mask)
    return _grads(tf, d3, d2, desc3d, desc2d, case)


def tensor_names():
    return ["d3", "d2", "d_desc3d", "d_desc2d"] + ["d_" + n for n in COARSE_PARAMS]


def flat_results(r):
    """(d3, d2, d desc3d, d desc2d, [d param]) -> list in tensor_names() order."""
    return [r[0], r[1], r[2], r[3]] + list(r[4])


def main():
    sd = workload.synthetic_state_dict(0)
    out = {}
    for name in CASES:
        case = make_case(masked=name == "masked")
        for key, t in zip(tensor_names(), flat_results(reference_coarse(sd, case))):
            put_sampled(out, f"{name}_{key}", t, k=SAMPLES)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "train_coarse_tf.npz")
    np.savez_compressed(path, **out)
    print(f"train_coarse_tf -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
