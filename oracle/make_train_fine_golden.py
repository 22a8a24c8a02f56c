"""Writes tests/golden/reference/train_fine.npz: the fine level of a training step — FinePreprocess,
the fine LocalFeatureTransformer, FineMatching and Loss.compute_fine_loss of the UNMODIFIED reference,
in fp64 on the CPU — on the seeded case of make_case (B = 2, border cells, repeated (b, j) cells), so
that the GPU tests need nothing from the reference tree.  Stored: expec_f, the fine loss, and the
gradients of feat_f and of every fine parameter (1024 sampled entries and the absmax of each, as
coarse_loss.npz does).  The inputs are regenerated from their seeds (make_case,
workload.synthetic_state_dict(0)).

    python -m oracle.make_train_fine_golden
"""
import contextlib
import copy
import os
import sys

import numpy as np
import torch

from . import oracle, workload
from .coarse_loss import LOSS_CONFIG, put_sampled

# the parameters of one fine layer, in train_fine.layer_params order
LAYER_PARAMS = ("q_proj.weight", "k_proj.weight", "v_proj.weight", "merge.weight", "mlp.0.weight", "mlp.2.weight",
                "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias")
FINE_PARAMS = tuple(f"loftr_fine.layers.{n}.{p}" for n in range(2) for p in LAYER_PARAMS)


def make_case(seed=0, B=2, hc=4, wc=5, stride=4, n3d=24, M=40):
    """feat_f fp64 [B, 128, hc*stride, wc*stride], descriptors3d_db [B, 128, n3d], M matches whose
    cells include the four corners of both images and three repeated (b, j) cells, expec_f_gt [M, 2]
    (some beyond the correct threshold 1)."""
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    feat = torch.randn(B, 128, hc * stride, wc * stride, generator=g, dtype=f64)
    desc = torch.randn(B, 128, n3d, generator=g, dtype=f64)
    b = torch.randint(0, B, (M,), generator=g)
    i = torch.randint(0, n3d, (M,), generator=g)
    j = torch.randint(0, hc * wc, (M,), generator=g)
    corners = torch.tensor([0, wc - 1, (hc - 1) * wc, hc * wc - 1])
    b[:8], j[:8] = torch.arange(8) // 4, corners.repeat(2)
    b[-3:], j[-3:] = b[8:11], j[8:11]                     # the GT padding draws with replacement
    gt = (torch.rand(M, 2, generator=g, dtype=f64) * 2.6 - 1.3)
    return {"feat_f": feat, "desc3d": desc, "b_ids": b, "i_ids": i, "j_ids": j, "expec_f_gt": gt,
            "q_hw_c": (hc, wc), "q_hw_f": (hc * stride, wc * stride), "q_hw_i": (hc * 8, wc * 8)}


def fine_data(case):
    return {"b_ids": case["b_ids"], "i_ids": case["i_ids"], "j_ids": case["j_ids"], "q_hw_c": case["q_hw_c"],
            "q_hw_f": case["q_hw_f"], "q_hw_i": case["q_hw_i"],
            "mkpts_query_c": torch.zeros(len(case["b_ids"]), 2, dtype=case["feat_f"].dtype),
            "mkpts_3d_db": torch.zeros(len(case["b_ids"]), 3, dtype=case["feat_f"].dtype)}


def reference_fine(sd, case):
    """The reference modules and loss in fp64: (expec_f, loss, d feat_f, {name: d param})."""
    from . import ref_shims
    ref_shims.install()
    from src.lightning_model.losses import Loss as RefLoss   # type: ignore
    model = ref_shims.build_reference_model(sd, copy.deepcopy(oracle.DEFAULT_CONFIG)).double().train()
    feat = case["feat_f"].clone().requires_grad_(True)
    data = fine_data(case)
    f3d, f2d = model.fine_preprocess(data, case["desc3d"], feat)
    f3d, f2d = model.loftr_fine(f3d, f2d)
    model.fine_matching(f3d, f2d, data)
    loss = RefLoss(LOSS_CONFIG).compute_fine_loss(data["expec_f"], case["expec_f_gt"])
    loss.backward()
    params = dict(model.named_parameters())
    return data["expec_f"].detach(), loss.detach(), feat.grad, {n: params[n].grad for n in FINE_PARAMS}


def fine_module(sd, dtype=torch.float64, device="cpu"):
    """The drop-in model's loftr_fine with the weights of sd."""
    from onepose_plus_plus_b200 import OnePosePlus_model
    model = OnePosePlus_model(copy.deepcopy(oracle.DEFAULT_CONFIG))
    model.load_state_dict(sd, strict=True)
    return model.loftr_fine.to(device=device, dtype=dtype).train()


def objective(expec_f, case, weights=None):
    """The fine loss (losses.Loss, the reference formula) or, with weights [M, 3], sum(expec_f * weights)
    (the fine loss passes no gradient to the std column)."""
    if weights is not None:
        return (expec_f * weights).sum()
    from onepose_plus_plus_b200 import losses
    return losses.Loss(LOSS_CONFIG).compute_fine_loss(expec_f, case["expec_f_gt"].to(expec_f))


@contextlib.contextmanager
def default_dtype(dtype):
    """train_path.fine_matching builds its grid with torch.linspace in the default dtype."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        yield
    finally:
        torch.set_default_dtype(prev)


def train_path_fine(fine, case, dtype=torch.float64, device="cpu", weights=None):
    """train_path.fine_preprocess -> transformer -> fine_matching with autograd on `fine` (a fine
    LocalFeatureTransformer in `dtype`): (expec_f, loss, d feat_f, [d param in FINE_PARAMS order])."""
    from onepose_plus_plus_b200 import train_path
    feat = case["feat_f"].to(device=device, dtype=dtype).requires_grad_(True)
    data = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in fine_data(case).items()}
    f3d, f2d = train_path.fine_preprocess(5, 128, data, case["desc3d"].to(device=device, dtype=dtype), feat)
    f3d, f2d = train_path.transformer(fine, f3d, f2d)
    with default_dtype(dtype):
        train_path.fine_matching(f3d, f2d, data, True)
    loss = objective(data["expec_f"], case, weights)
    params = dict(fine.named_parameters())
    names = [n[len("loftr_fine."):] for n in FINE_PARAMS]
    grads = torch.autograd.grad(loss, [feat] + [params[n] for n in names])
    return data["expec_f"].detach(), loss.detach(), grads[0], list(grads[1:])


def main():
    sd = workload.synthetic_state_dict(0)
    case = make_case()
    expec, loss, dfeat, dparams = reference_fine(sd, case)
    out = {"expec_f": expec.numpy(), "loss": np.float64(loss.item())}
    put_sampled(out, "d_feat_f", dfeat)
    for n, t in dparams.items():
        put_sampled(out, "d_" + n, t)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "train_fine.npz")
    np.savez_compressed(path, **out)
    print(f"train_fine -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
