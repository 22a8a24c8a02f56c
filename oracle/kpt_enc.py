"""fp64 restatement of the keypoint-encoder backward that csrc/opp_train_kpt.cu implements
(KeypointEncoding_linear, utils/position_encoding.py:46-79, norm_method "instancenorm"), written out
by hand so that the CPU suite can check the manual formulas against autograd.

Per point:  a_l = W_l z_{l-1} + b_l,  y_l = (a_l - mean a_l) r_l,  r_l = (var a_l + eps)^-1/2 (biased),
z_l = relu(y_l) for the hidden layers (z_0 = the normalised keypoint), out = W_4 z_3 + b_4 + desc.
Backward from g = d out:  dz_3 = W_4ᵀ g;  dy = [y > 0] dz;  da = r (dy - mean dy - y mean(dy y));
dz_{l-1} = W_lᵀ da;  dW_l = sum_p da ⊗ z_{l-1};  db_l = sum_p da.
"""
import torch

EPS = 1e-5


def forward(params, x0, desc, eps=EPS):
    """params = [W1, b1, ..., W4, b4] (nn.Linear layouts); x0 [B, N, 3] normalised keypoints;
    desc [B, 256, N].  Returns (out [B, 256, N], the per-layer (z_in, y, r) of the hidden layers)."""
    z, cache = x0, []
    for i in range(3):
        a = z @ params[2 * i].T + params[2 * i + 1]
        mu = a.mean(-1, keepdim=True)
        r = 1.0 / torch.sqrt(((a - mu) ** 2).mean(-1, keepdim=True) + eps)
        y = (a - mu) * r
        cache.append((z, y, r))
        z = torch.clamp(y, min=0)
    out = z @ params[6].T + params[7]
    return desc + out.transpose(1, 2), (cache, z)


def backward(params, x0, g, eps=EPS):
    """The eight parameter gradients for the upstream gradient g [B, 256, N] of forward's output."""
    _, (cache, z3) = forward(params, x0, torch.zeros_like(g), eps)
    g = g.transpose(1, 2)                                # [B, N, 256]
    grads = [None] * 8
    grads[6] = torch.einsum("bnc,bnk->ck", g, z3)
    grads[7] = g.sum((0, 1))
    dz = g @ params[6]
    for i in (2, 1, 0):
        z_in, y, r = cache[i]
        dy = torch.where(y > 0, dz, torch.zeros_like(dz))
        da = r * (dy - dy.mean(-1, keepdim=True) - y * (dy * y).mean(-1, keepdim=True))
        grads[2 * i] = torch.einsum("bnc,bnk->ck", da, z_in)
        grads[2 * i + 1] = da.sum((0, 1))
        dz = da @ params[2 * i]
    return grads
