"""fp64 restatement of the coarse focal loss of training (Loss.compute_coarse_loss,
src/lightning_model/losses.py:18-58, focal branch) on the dual-softmax confidence, and of its
closed-form gradient with respect to the two feature sets (DESIGN §7 f4):

    sim = s A B^T, p = softmax over L, q = softmax over S, c = p q
    g = d loss / d c (0 where the clamp is active), R_i = sum_j g c, C_j = sum_i g c
    d sim = 2 g c - p C - q R,  dA = s dsim B,  dB = s dsim^T A

Masked query columns (query_image_mask) have q = c = 0.  Also the seeded input cases of the
tests and the generator of tests/golden/reference/coarse_loss.npz (what the unmodified reference
computes on them, through autograd):

    python -m oracle.coarse_loss
"""
import os
import sys

import numpy as np
import torch

# configs/experiment/train.yaml:130-144 (loss section)
LOSS_CONFIG = {"coarse_type": "focal", "coarse_weight": 1.0, "fine_type": "l2_with_std", "fine_weight": 0.81,
               "focal_alpha": 0.5, "focal_gamma": 2.0, "pos_weight": 1.0, "neg_weight": 1.0,
               "fine_correct_thr": 1.0}
TEMPERATURE = 0.1
LO, HI = 1e-6, 1 - 1e-6


def scale_of(c=256, temperature=TEMPERATURE):
    return 1.0 / (c * (temperature + 1e-4))


def dual_softmax(a, b, scale, mask=None):
    """(p, q, c) in the dtype of a / b; mask bool [B, S] (False = padding)."""
    sim = scale * torch.einsum("blk,bsk->bls", a, b)
    keep = torch.ones_like(sim, dtype=torch.bool) if mask is None else mask.bool()[:, None, :].expand_as(sim)
    p = torch.softmax(sim, 1)
    q = torch.softmax(sim.masked_fill(~keep, float("-inf")), 2)
    return p, q, p * q


def softmax_stats(a, b, scale, mask=None):
    """fp64 softmax statistics of sim = scale A B^T: (row max, row log-sum-exp) over the kept columns
    of each row and (column max, column log-sum-exp) over every row of each column."""
    sim = scale * torch.einsum("blk,bsk->bls", a.double(), b.double())
    col_max, col_lse = sim.amax(1), torch.logsumexp(sim, 1)
    if mask is not None:
        sim = sim.masked_fill(~mask.bool()[:, None, :], float("-inf"))
    return sim.amax(2), torch.logsumexp(sim, 2), col_max, col_lse


def focal_loss_and_grads(a, b, gt, scale, mask=None, alpha=0.5, gamma=2.0, pos_w=1.0, neg_w=1.0, with_rc=False):
    """fp64 loss, dA, dB (torch tensors on the device of a); with_rc also R [B, L] and C [B, S]."""
    a, b = a.double(), b.double()
    p, q, c = dual_softmax(a, b, scale, mask)
    ct = c.clamp(LO, HI)
    passes = (c >= LO) & (c <= HI)
    pos, neg = gt == 1, gt == 0
    npos, nneg = int(pos.sum()), int(neg.sum())
    l_pos = -alpha * (1 - ct) ** gamma * torch.log(ct)
    l_neg = -(1 - alpha) * ct ** gamma * torch.log1p(-ct)
    if npos == 0 and nneg == 0:
        loss = torch.tensor(float("nan"), dtype=torch.float64)
    else:
        loss = ((pos_w * l_pos[pos].sum() / npos) if npos else 0.0) + ((neg_w * l_neg[neg].sum() / nneg) if nneg else 0.0)
    d_pos = alpha * gamma * (1 - ct) ** (gamma - 1) * torch.log(ct) - alpha * (1 - ct) ** gamma / ct
    d_neg = -(1 - alpha) * gamma * ct ** (gamma - 1) * torch.log1p(-ct) + (1 - alpha) * ct ** gamma / (1 - ct)
    g = torch.zeros_like(c)
    if npos:
        g = torch.where(pos, d_pos * (pos_w / npos), g)
    if nneg:
        g = torch.where(neg, d_neg * (neg_w / nneg), g)
    gc = g * passes * c
    dsim = 2 * gc - p * gc.sum(1, keepdim=True) - q * gc.sum(2, keepdim=True)
    da = scale * torch.einsum("bls,bsk->blk", dsim, b)
    db = scale * torch.einsum("bls,blk->bsk", dsim, a)
    loss = torch.as_tensor(loss, dtype=torch.float64)
    if with_rc:
        return loss, da, db, gc.sum(2), gc.sum(1)
    return loss, da, db


def make_case(name, batch=2, rows=40, cols=48, k=256, seed=0):
    """Seeded (a, b, gt, mask) of one test case (CPU, fp32 features):
      random     — unrelated features, ~5% positives, a few gt values that are neither class
      planted    — rows planted on columns (strong matches), gt on the plants
      no_pos     — planted, gt all 0
      no_neg     — planted, gt 1 or 2 (2 = neither) only
      clamp      — planted with large gain: c hits both clamp bounds
      masked     — planted, query_image_mask pads the last columns of every image"""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(batch, rows, k, generator=g)
    b = torch.randn(batch, cols, k, generator=g)
    gt = torch.zeros(batch, rows, cols, dtype=torch.int16)
    mask = None
    if name == "random":
        gt[torch.rand(batch, rows, cols, generator=g) < 0.05] = 1
        gt[torch.rand(batch, rows, cols, generator=g) < 0.01] = 2
        return a * 1.5, b * 1.5, gt, mask
    gain = 3.0 if name == "clamp" else 0.6
    n = min(rows, cols) // 2
    for bi in range(batch):
        ri = torch.randperm(rows, generator=g)[:n]
        cj = torch.randperm(cols, generator=g)[:n]
        b[bi, cj] = a[bi, ri] + 0.3 * torch.randn(n, k, generator=g)
        gt[bi, ri, cj] = 1
    a, b = a * gain, b * gain
    if name == "no_pos":
        gt.zero_()
    elif name == "no_neg":
        gt[gt == 0] = 2
    elif name == "masked":
        mask = torch.ones(batch, cols, dtype=torch.bool)
        mask[:, cols - cols // 4:] = False
        mask[1:, cols - cols // 3:] = False
    return a, b, gt, mask


CASES = ("random", "planted", "no_pos", "no_neg", "clamp", "masked")
# golden cases: the planted train-sized batch (B = 2, L = 300, S = 192) with and without the mask, and
# a width that is not a multiple of the kernels' 64-row tiles
GOLDEN_CASES = {"planted_300x192": ("planted", 2, 300, 192), "masked_300x192": ("masked", 2, 300, 192),
                "planted_130x150": ("planted", 2, 130, 150), "clamp_300x192": ("clamp", 2, 300, 192)}


def reference_loss_and_grads(a, b, gt, scale, mask=None, config=None):
    """Autograd through the UNMODIFIED reference Loss.compute_coarse_loss (imported from the
    reference tree through oracle/ref_shims.py) on the fp64 dual softmax of a, b; config: the loss
    section (LOSS_CONFIG by default)."""
    from . import ref_shims
    ref_shims.install()
    from src.lightning_model.losses import Loss as RefLoss   # type: ignore
    a = a.double().clone().requires_grad_(True)
    b = b.double().clone().requires_grad_(True)
    sim = scale * torch.einsum("blk,bsk->bls", a, b)
    if mask is not None:
        neg = torch.zeros_like(sim)
        neg[~mask.bool()[:, None].expand_as(sim)] = -1e9
        sim = sim + neg
    conf = torch.softmax(sim, 1) * torch.softmax(sim, 2)
    loss = RefLoss(LOSS_CONFIG if config is None else config).compute_coarse_loss(conf, gt)
    loss.backward()
    return loss.detach(), a.grad, b.grad


def put_sampled(out, name, t, k=1024, seed=7):
    gen = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, t.numel(), (min(k, t.numel()),), generator=gen)
    out[name + "_idx"] = idx.numpy()
    out[name] = t.detach().flatten()[idx].numpy()
    out[name + "_absmax"] = np.float64(t.abs().max().item())


def main():
    out = {}
    for key, (name, batch, rows, cols) in GOLDEN_CASES.items():
        a, b, gt, mask = make_case(name, batch, rows, cols)
        loss, da, db = reference_loss_and_grads(a, b, gt, scale_of(), mask)
        out[key + "_loss"] = np.float64(loss.item())
        put_sampled(out, key + "_da", da)
        put_sampled(out, key + "_db", db)
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                        "coarse_loss.npz")
    np.savez_compressed(path, **out)
    print(f"coarse_loss -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
