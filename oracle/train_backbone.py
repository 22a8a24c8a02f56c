"""fp64 restatements of the index arithmetic of the backbone's training kernels
(csrc/opp_train_backbone.cu) that autograd does not expose, checked against autograd on the CPU
(tests/test_train_backbone_cpu.py), and of the BatchNorm running-statistics update:

  * conv_dgrad: the data gradient of a k x k convolution (pad k // 2) as a gather: input pixel i
    receives from tap k_y of output row (i + pad - k_y) / stride where that is an integer in range;
  * up2x_taps / up2x_bwd: the output positions of the align_corners bilinear x2 upsample that read
    each input position, with ATen's fp32 source index, and the gather backward built on them;
  * bn_running_update: F.batch_norm's update of running_mean / running_var.
"""
import numpy as np
import torch


def conv_dgrad(dy, w, stride, in_hw):
    """dx [B, Ci, H, W] of conv2d(x, w, stride, padding=k // 2) for dy [B, Co, Ho, Wo], fp64."""
    B, Co, Ho, Wo = dy.shape
    _, Ci, k, _ = w.shape
    H, W = in_hw
    pad = k // 2
    dx = torch.zeros(B, Ci, H, W, dtype=torch.float64)
    dy, w = dy.double(), w.double()
    for ky in range(k):
        for kx in range(k):
            for i in range(H):
                ty = i + pad - ky
                if ty < 0 or ty % stride or ty // stride >= Ho:
                    continue
                for j in range(W):
                    tx = j + pad - kx
                    if tx < 0 or tx % stride or tx // stride >= Wo:
                        continue
                    dx[:, :, i, j] += torch.einsum("bo,oc->bc", dy[:, :, ty // stride, tx // stride], w[:, :, ky, kx])
    return dx


def _src(d, n_in):
    """ATen's fp32 source index of output position d (align_corners, out = 2 n_in): (i0, i1, lambda1)."""
    scale = np.float32(n_in - 1) / np.float32(2 * n_in - 1) if n_in > 1 else np.float32(0)
    src = np.float32(scale * np.float32(d))
    i0 = int(src)
    i1 = i0 + (1 if i0 < n_in - 1 else 0)
    return i0, i1, float(np.float32(src - np.float32(i0)))


def up2x_taps(i, n_in):
    """{output position: weight} of the output positions in [2i - 3, 2i + 4] that read input position i."""
    taps = {}
    for d in range(max(0, 2 * i - 3), min(2 * n_in - 1, 2 * i + 4) + 1):
        i0, i1, l1 = _src(d, n_in)
        wv = (1.0 - l1 if i0 == i else 0.0) + (l1 if i1 == i else 0.0)
        if i0 == i or i1 == i:
            taps[d] = wv
    return taps


def up2x_bwd(dout, in_hw):
    """din [B, C, h, w] of interpolate(x, scale_factor=2, bilinear, align_corners=True), fp64 gather."""
    h, w = in_hw
    dout = dout.double()
    ry = torch.zeros(h, 2 * h, dtype=torch.float64)
    rx = torch.zeros(w, 2 * w, dtype=torch.float64)
    for i in range(h):
        for d, wv in up2x_taps(i, h).items():
            ry[i, d] = wv
    for j in range(w):
        for d, wv in up2x_taps(j, w).items():
            rx[j, d] = wv
    return torch.einsum("iy,bcyx,jx->bcij", ry, dout, rx)


def bn_running_update(x, running_mean, running_var, momentum):
    """(running_mean, running_var) after one train-mode F.batch_norm of x [B, C, H, W], fp64."""
    x = x.double().transpose(0, 1).flatten(1)
    n = x.shape[1]
    mean, var = x.mean(1), x.var(1, unbiased=False)
    return ((1 - momentum) * running_mean.double() + momentum * mean,
            (1 - momentum) * running_var.double() + momentum * var * n / (n - 1))
