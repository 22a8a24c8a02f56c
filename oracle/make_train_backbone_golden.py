"""Writes tests/golden/reference/train_backbone.npz: the ResNetFPN_8_2 backbone of the UNMODIFIED
reference, forward and backward in fp64 on the CPU, on the seeded case of make_case (B = 2, 96 x 128
image, upstream gradients for both outputs), with the backbone in train mode (batch-statistics
BatchNorm) and in eval mode (running statistics, as pretrained_fix leaves it), so that the GPU tests
need nothing from the reference tree.  Stored per case: both outputs, the gradient of every backbone
parameter under objective() (sampled entries plus absmax, coarse_loss.put_sampled) and every
BatchNorm's running_mean / running_var / num_batches_tracked after the step (in full).  The weights are
workload.synthetic_state_dict(0) (perturbed BatchNorm).

    python -m oracle.make_train_backbone_golden
"""
import copy
import os
import sys

import numpy as np
import torch

from . import oracle, workload
from .coarse_loss import put_sampled

SAMPLES = 128
CASES = ("train", "eval")


def make_case(seed=0, B=2, H=96, W=128):
    """image fp64 [B, 1, H, W] in [0, 1) and the objective's weights g_c [B, 256, H/8, W/8],
    g_f [B, 128, H/2, W/2]."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    return {"img": torch.rand(B, 1, H, W, generator=g, dtype=f64),
            "g_c": torch.randn(B, 256, H // 8, W // 8, generator=g, dtype=f64),
            "g_f": torch.randn(B, 128, H // 2, W // 2, generator=g, dtype=f64)}


def objective(feat_c, feat_f, case):
    return (feat_c * case["g_c"].to(feat_c)).sum() + (feat_f * case["g_f"].to(feat_f)).sum()


def backbone_module(sd, dtype=torch.float64, device="cpu", train=True):
    """The drop-in model's backbone with the weights of sd."""
    from onepose_plus_plus_b200 import OnePosePlus_model
    model = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    model.load_state_dict(sd, strict=True)
    return model.backbone.to(device=device, dtype=dtype).train(train)


def param_names(bb):
    return [n for n, _ in bb.named_parameters()]


def buffer_names(bb):
    return [n for n, _ in bb.named_buffers()]


def run(bb, fwd, case, dtype=torch.float64, device="cpu"):
    """(feat_c, feat_f, [d param in named_parameters order], {buffer name: buffer after the step})."""
    img = case["img"].to(device=device, dtype=dtype)
    feat_c, feat_f = fwd(bb, img)
    params = [p for _, p in bb.named_parameters()]
    grads = torch.autograd.grad(objective(feat_c, feat_f, case), params)
    return feat_c.detach(), feat_f.detach(), list(grads), {n: b.detach().clone() for n, b in bb.named_buffers()}


def reference_backbone(sd, case, train=True):
    from . import ref_shims
    ref_shims.install()
    bb = ref_shims.build_reference_model(sd, copy.deepcopy(oracle.DEFAULT_CONFIG)).backbone.double().train(train)
    return run(bb, lambda m, x: tuple(m(x)), case)


def main():
    sd = workload.synthetic_state_dict(0)
    out = {}
    case = make_case()
    names = param_names(backbone_module(sd))
    for name in CASES:
        feat_c, feat_f, grads, bufs = reference_backbone(sd, case, train=name == "train")
        put_sampled(out, f"{name}_feat_c", feat_c, k=SAMPLES)
        put_sampled(out, f"{name}_feat_f", feat_f, k=SAMPLES)
        for n, g in zip(names, grads):
            put_sampled(out, f"{name}_d_{n}", g, k=SAMPLES)
        for n, b in bufs.items():
            out[f"{name}_buf_{n}"] = b.numpy()
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "train_backbone.npz")
    np.savez_compressed(path, **out)
    print(f"train_backbone -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
