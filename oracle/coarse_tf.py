"""fp64 restatement of the linear attention of the coarse transformer (linear_attention.py:29-61, as
train_path._linear_attention) and of the manual backward the opp_coarse_tf_* kernels implement
(DESIGN §7 f4).  Shapes as in _linear_attention: q [B, L, H, D], k / v [B, S, H, D], masks [B, L] /
[B, S] with 0/1 entries or None.  Per head, with m the masks and n = S (masked rows included):

    K = elu(k) + 1, KV = sum_s (K_s m_s) (v_s m_s / n)^T, ksum = sum_s K_s m_s
    Q = (elu(q) + 1) m, A = Q KV, Z = 1 / (Q . ksum + eps), out = A Z n

    dU = g Z n, dden = -n Z^2 (g . A), dQ = KV dU + ksum dden, dq = dQ m elu'(q)
    dKV = sum_l Q_l dU_l^T, dksum = sum_l Q_l dden_l
    dk_s = m_s (dKV v_s / n + dksum) elu'(k_s), dv_s = (m_s / n) dKV^T K_s

elu'(x) = 1 for x > 0, else exp(x).  The forward's state and the backward's two passes are written
out separately, as the kernels split them.
"""
import torch


def _elu1(x):
    return torch.where(x > 0, x + 1, torch.exp(torch.clamp(x, max=0)))


def _elu1_grad(x):
    return torch.where(x > 0, torch.ones_like(x), torch.exp(torch.clamp(x, max=0)))


def _ones(t, n):
    return torch.ones(t.shape[0], n, dtype=t.dtype, device=t.device)


def state(k, v, kv_mask=None):
    """(KV [B, H, D, D], ksum [B, H, D]) of the source rows."""
    n = k.shape[1]
    m = (_ones(k, n) if kv_mask is None else kv_mask.to(k.dtype))[:, :, None, None]
    K = _elu1(k) * m
    return torch.einsum("nshd,nshv->nhdv", K, v * m / n), K.sum(1)


def forward(q, k, v, q_mask=None, kv_mask=None, eps=1e-6):
    n = k.shape[1]
    KV, ksum = state(k, v, kv_mask)
    m = (_ones(q, q.shape[1]) if q_mask is None else q_mask.to(q.dtype))[:, :, None, None]
    Q = _elu1(q) * m
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, ksum) + eps)
    return torch.einsum("nlhd,nhdv->nlhv", Q, KV) * Z[..., None] * n


def backward_q(q, KV, ksum, n, dout, q_mask=None, eps=1e-6):
    """Query pass: (dq, dKV, dksum)."""
    m = (_ones(q, q.shape[1]) if q_mask is None else q_mask.to(q.dtype))[:, :, None, None]
    Q = _elu1(q) * m
    A = torch.einsum("nlhd,nhdv->nlhv", Q, KV)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, ksum) + eps)
    dU = dout * Z[..., None] * n
    dden = -n * Z ** 2 * (dout * A).sum(-1)
    dQ = torch.einsum("nhdv,nlhv->nlhd", KV, dU) + ksum[:, None] * dden[..., None]
    dq = dQ * m * _elu1_grad(q)
    dKV = torch.einsum("nlhd,nlhv->nhdv", Q, dU)
    dksum = torch.einsum("nlhd,nlh->nhd", Q, dden)
    return dq, dKV, dksum


def backward_kv(k, v, dKV, dksum, kv_mask=None):
    """Source pass: (dk, dv), v_len = the source's length."""
    n = k.shape[1]
    m = (_ones(k, n) if kv_mask is None else kv_mask.to(k.dtype))[:, :, None, None]
    dk = m * (torch.einsum("nhdv,nshv->nshd", dKV, v) / n + dksum[:, None]) * _elu1_grad(k)
    dv = (m / n) * torch.einsum("nhdv,nshd->nshv", dKV, _elu1(k))
    return dk, dv


def backward(q, k, v, dout, q_mask=None, kv_mask=None, eps=1e-6):
    """(dq, dk, dv) of forward(q, k, v, q_mask, kv_mask, eps) for the output gradient dout."""
    KV, ksum = state(k, v, kv_mask)
    dq, dKV, dksum = backward_q(q, KV, ksum, k.shape[1], dout, q_mask, eps)
    dk, dv = backward_kv(k, v, dKV, dksum, kv_mask)
    return dq, dk, dv
