"""Keypoint encoder of the training forward on the device (model.kpt_encoder_train_mode "kernels", CUDA,
train mode).

One autograd Function replaces train_path.keypoint_encoding(enc, normalize_3d_keypoints(kpts), desc):
the normalisation statistics (opp_kpt_stats, the inference kernel), then the 3-32-64-128-256 MLP with a
per-point InstanceNorm + ReLU after each hidden layer and the descriptor add, forward and backward in
fp32 on the CUDA cores (csrc/opp_train_kpt.cu).

The Function returns contiguous rows [B, N, 256] = descriptorsᵀ + encoding; keypoint_encoding hands
out their [B, 256, N] transpose, the tensor train_path.keypoint_encoding returns.  Memory: the forward
keeps the keypoints and the per-batch statistics [B, 4] and no activation; the backward recomputes each
point's forward in shared memory.  Weight gradients are summed per group of opp_kpt_train_group() rows
into partials, WGRAD_SLICE_GROUPS partials per call, added in group order without floating-point
atomics: two calls give the same bits.
"""
import torch

from . import ops

MODES = ("autograd", "kernels")
CHANNELS = (3, 32, 64, 128, 256)
LINEARS = (0, 3, 6, 9)             # indices of the nn.Linear modules in enc.encoder
WGRAD_SLICE_GROUPS = 128           # partials of one opp_kpt_train_bwd call (128 x 170 KiB = 21.3 MiB)


def check(model, data):
    """Raise for what the kernels do not cover (model.kpt_encoder_train_mode "kernels")."""
    if model.precision == "fp16":
        raise ValueError('kpt_encoder_train_mode "kernels" needs precision "fp16x3", as the other device stages '
                         'of the training step: with single fp16 operands the coarse matches differ from the eager '
                         'fp32 ones')
    enc = model.kpt_3d_pos_encoding.encoder
    lin = [m for m in enc if isinstance(m, torch.nn.Linear)]
    chans = tuple([lin[0].in_features] + [m.out_features for m in lin]) if lin else ()
    norms = [m for m in enc if isinstance(m, torch.nn.InstanceNorm1d)]
    if chans != CHANNELS or len(enc) != 10 or any(m.eps != 1e-5 or m.affine for m in norms):
        raise NotImplementedError(f'kpt_encoder_train_mode "kernels" is built for the channels {list(CHANNELS)} '
                                  f'(InstanceNorm eps 1e-5, no affine), not {list(chans)}')
    if data["keypoints3d"].requires_grad:
        raise NotImplementedError('kpt_encoder_train_mode "kernels" does not differentiate keypoints3d (the '
                                  'normalisation reads the extents of batch element 0)')
    if _descriptors(data).requires_grad:
        raise NotImplementedError('kpt_encoder_train_mode "kernels" does not differentiate the 3D descriptors')
    if any(p.dtype != torch.float32 for p in enc.parameters()):
        raise NotImplementedError('kpt_encoder_train_mode "kernels" runs fp32 parameters')


def use_kernels(model, data):
    """True when the keypoint encoder of this training forward runs on the kernels (validated)."""
    mode = model.kpt_encoder_train_mode
    if mode not in MODES:
        raise ValueError(f"kpt_encoder_train_mode must be one of {MODES}, not {mode!r}")
    if mode != "kernels" or not model.training or not data["keypoints3d"].is_cuda:
        return False
    check(model, data)
    return True


def _descriptors(data):
    return data["descriptors3d_coarse_db"] if "descriptors3d_coarse_db" in data else data["descriptors3d_db"]


def params(enc):
    """The Function's parameter inputs: (weight, bias) of encoder.0, .3, .6, .9."""
    return [p for i in LINEARS for p in (enc.encoder[i].weight, enc.encoder[i].bias)]


def pack(tensors):
    """The weight pack of opp_kpt_train_fwd / _bwd: W1ᵀ b1 W2ᵀ b2 W3ᵀ b3 W4ᵀ b4, then W2 W3 W4."""
    w, b = tensors[0::2], tensors[1::2]
    parts = [t for i in range(4) for t in (w[i].detach().t(), b[i].detach())] + [t.detach() for t in w[1:]]
    return torch.cat([t.reshape(-1) for t in parts]).float().contiguous()


class KeypointEncoderStage(torch.autograd.Function):
    """rows [B, N, 256] = (descriptors + encoder(normalize_3d_keypoints(kpts)))ᵀ on the kernels.
    Inputs: keypoints3d [B, N, 3], descriptors [B, 256, N], then params(enc)."""

    @staticmethod
    def forward(ctx, kpts, desc, *tensors):
        kpts = kpts.detach().float().contiguous()
        B, N, _ = kpts.shape
        dev = kpts.device
        stats = torch.empty(B, 4, dtype=torch.float32, device=dev)
        ops.kpt_stats(kpts, stats)
        out = torch.empty(B, N, CHANNELS[-1], dtype=torch.float32, device=dev)
        ops.kpt_train_fwd(kpts, stats, desc.detach().float().contiguous(), pack(tensors), out)
        ctx.save_for_backward(kpts, stats, *tensors)
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, dout):
        need = ctx.needs_input_grad[2:]
        nothing = (None,) * (2 + len(need))
        if dout is None or not any(need):
            return nothing
        kpts, stats, *tensors = ctx.saved_tensors
        B, N, _ = kpts.shape
        rows, group, nparams = B * N, ops.kpt_train_group(), ops.kpt_train_params()
        step = WGRAD_SLICE_GROUPS * group
        part = torch.empty(-(-min(rows, step) // group) * nparams, dtype=torch.float32, device=kpts.device)
        flat = torch.empty(nparams, dtype=torch.float32, device=kpts.device)
        dout = dout.float().contiguous()
        w = pack(tensors)
        for r0 in range(0, rows, step):
            ops.kpt_train_bwd(kpts, stats, dout, w, r0, min(step, rows - r0), part, flat, r0 > 0)
        grads, off = [], 0
        for t, want in zip(tensors, need):
            grads.append(flat[off:off + t.numel()].view(t.shape) if want else None)
            off += t.numel()
        return (None, None, *grads)


def keypoint_encoding(enc, kpts, descriptors):
    """train_path.keypoint_encoding(enc, train_path.normalize_3d_keypoints(kpts), descriptors) on the
    kernels: [B, 256, N], the transpose of the contiguous rows the Function returns."""
    return KeypointEncoderStage.apply(kpts, descriptors, *params(enc)).transpose(1, 2)
