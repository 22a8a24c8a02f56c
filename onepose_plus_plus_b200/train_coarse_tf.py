"""Coarse transformer of the training forward on the device (model.coarse_transformer_train_mode
"kernels", CUDA, train mode).

One autograd Function replaces train_path.transformer(model.loftr_coarse, ...): the self / cross
LoFTR layers (d_model 256, 8 heads, linear attention) forward and backward in fp32 on the CUDA cores.
The projections, the merge and the MLP run on the fine level's token-row GEMMs
(opp_fine_train_linear / _wgrad), the attention and the 256-channel LayerNorm on the opp_coarse_tf_*
kernels (csrc/opp_train_coarse_tf.cu).

Rows: one [B*(S+N), 256] buffer holds both sequences, the 2D rows [0, B*S) and then the 3D rows
[B*S, B*S + B*N).  Both sequences go through one weight set, so each projection, LayerNorm and MLP is
one GEMM over all rows and each weight gradient sums both sequences; only the attention kernels tell
the sequences apart.

Memory: the forward keeps the input of every layer and nothing else.  The backward runs the layers in
reverse; each layer's forward is recomputed from its saved input, then differentiated.  The weight
gradients are summed in row slices of at most WGRAD_SLICE_GROUPS partials.  Every sum runs in a fixed
order without floating-point atomics: two calls give the same bits.
"""
import torch

from . import ops
from .train_fine import layer_params

MODES = ("autograd", "kernels")
D = 256
WGRAD_SLICE_GROUPS = 64      # partials of one opp_fine_train_wgrad call (64 MiB at 512 x 512)
GROUP_ROWS = 256             # rows per partial (opp_fine_train_groups)


def check(model, data):
    """Raise for what the kernels do not cover (model.coarse_transformer_train_mode "kernels")."""
    tf = model.loftr_coarse
    if any(layer.attention_type != "linear" for layer in tf.layers):
        raise NotImplementedError('coarse_transformer_train_mode "kernels" is built for linear attention, '
                                  'not "full"')
    if tf.d_model != 256 or tf.nhead != 8 or any(layer.nhead != 8 or layer.dim != 32 for layer in tf.layers):
        raise NotImplementedError('coarse_transformer_train_mode "kernels" is built for d_model 256 and 8 heads')
    bad = [n for n in tf.layer_names if n not in ("self", "cross")]
    if bad or len(tf.layer_names) != len(tf.layers):
        raise NotImplementedError(f'coarse_transformer_train_mode "kernels" is built for "self" / "cross" layers, '
                                  f'not {bad}')
    mask = data.get("query_image_mask")
    if mask is not None and not bool(((mask == 0) | (mask == 1)).all()):
        raise ValueError("query_image_mask must be 0/1-valued (a pad mask) for coarse_transformer_train_mode "
                         '"kernels"')


def use_kernels(model, data):
    """True when the coarse transformer of this training forward runs on the kernels (validated)."""
    mode = model.coarse_transformer_train_mode
    if mode not in MODES:
        raise ValueError(f"coarse_transformer_train_mode must be one of {MODES}, not {mode!r}")
    if mode != "kernels" or not model.training or not data["query_image"].is_cuda:
        return False
    check(model, data)
    return True


def _pack(params):
    """Per layer: (w_qkv [768, 256], w_merge, w_mlp0, w_mlp2, ln1 gamma, beta, ln2 gamma, beta)."""
    out = []
    for i in range(0, len(params), 10):
        p = [t.detach().float().contiguous() for t in params[i:i + 10]]
        out.append((torch.cat(p[0:3], 0).contiguous(), *p[3:]))
    return out


class _Geo:
    """The two sequences of the row buffer and the 2D mask (uint8 [B*S] or None)."""

    def __init__(self, B, S, N, mask):
        self.B, self.S, self.N, self.mask = B, S, N, mask
        self.rows = B * (S + N)

    def split(self, t):
        """(2D rows, 3D rows) of a row buffer."""
        return t[:self.B * self.S], t[self.B * self.S:]


class _Work:
    """Buffers of one layer: the forward state (xm = [layer input | LN1 output], q | k | v, message,
    merge output, ReLU output, mlp output, LayerNorm statistics), the attention states of the 2D and
    the 3D rows and the partials; for the backward also the gradient temporaries."""

    def __init__(self, g, dev, backward):
        def e(*s):
            return torch.empty(*s, dtype=torch.float32, device=dev)
        R, B = g.rows, g.B
        self.f = dict(xm=e(R, 2 * D), qkv=e(R, 3 * D), a=e(R, D), m0=e(R, D), st1=e(R, 2), r=e(R, 2 * D),
                      h2=e(R, D), st2=e(R, 2))
        self.state = (e(B, 8, 32, 32), e(B, 8, 32), e(B, 8, 32, 32), e(B, 8, 32))     # 2D rows, 3D rows
        self.part = e(B * max(ops.coarse_tf_chunks(g.S), ops.coarse_tf_chunks(g.N)) * ops.COARSE_TF_STATE)
        groups = ops.fine_train_groups(R)
        self.lnpart = e(groups * 2 * D)
        if backward:
            self.t = dict(t256a=e(R, D), t256b=e(R, D), t512a=e(R, 2 * D), t512b=e(R, 2 * D), t768=e(R, 3 * D))
            self.dstate = (e(B, 8, 32, 32), e(B, 8, 32), e(B, 8, 32, 32), e(B, 8, 32))
            self.wpart = e(min(groups, WGRAD_SLICE_GROUPS) * (2 * D) * (2 * D))


def _sources(g, cross, state):
    """(kv, ksum, v_len) read by the 2D queries and by the 3D queries: self layers attend within a
    sequence, cross layers to the other one."""
    kv2, ks2, kv3, ks3 = state
    own2, own3 = (kv2, ks2, g.S), (kv3, ks3, g.N)
    return (own3, own2) if cross else (own2, own3)


def _attn_fwd(g, cross, W, qkv, out):
    q2, q3 = g.split(qkv)
    kv2, ks2, kv3, ks3 = W.state
    ops.coarse_tf_kv(q2, g.mask, g.B, W.part, kv2, ks2)
    ops.coarse_tf_kv(q3, None, g.B, W.part, kv3, ks3)
    src2, src3 = _sources(g, cross, W.state)
    o2, o3 = g.split(out)
    ops.coarse_tf_attn(q2, g.mask, g.B, *src2, o2)
    ops.coarse_tf_attn(q3, None, g.B, *src3, o3)


def _attn_bwd(g, cross, W, qkv, dout, dqkv):
    """dqkv (overwritten): the q columns from the query pass, the k / v columns from the source pass of
    the state each sequence's rows form; each state is read by one query sequence."""
    q2, q3 = g.split(qkv)
    d2, d3 = g.split(dout)
    dq2, dq3 = g.split(dqkv)
    src2, src3 = _sources(g, cross, W.state)
    dkv2, dks2, dkv3, dks3 = W.dstate
    dsrc2, dsrc3 = ((dkv3, dks3), (dkv2, dks2)) if cross else ((dkv2, dks2), (dkv3, dks3))
    ops.coarse_tf_attn_bwd_q(q2, g.mask, g.B, *src2, d2, dq2, W.part, *dsrc2)
    ops.coarse_tf_attn_bwd_q(q3, None, g.B, *src3, d3, dq3, W.part, *dsrc3)
    ops.coarse_tf_attn_bwd_kv(q2, g.mask, g.B, dkv2, dks2, dq2)
    ops.coarse_tf_attn_bwd_kv(q3, None, g.B, dkv3, dks3, dq3)


def _layer_fwd(p, cross, g, W, x, y):
    """LoFTREncoderLayer.forward on both sequences: y = x + LN2(mlp([x, LN1(merge(attn))]))."""
    wqkv, wm, w0, w2, g1, b1, g2, b2 = p
    F = W.f
    F["xm"][:, :D].copy_(x)
    ops.fine_train_linear(x, wqkv, True, F["qkv"])
    _attn_fwd(g, cross, W, F["qkv"], F["a"])
    ops.fine_train_linear(F["a"], wm, True, F["m0"])
    ops.coarse_tf_ln(F["m0"], g1, b1, None, F["xm"][:, D:], F["st1"])
    ops.fine_train_linear(F["xm"], w0, True, F["r"], ops.EPI_RELU)
    ops.fine_train_linear(F["r"], w2, True, F["h2"])
    ops.coarse_tf_ln(F["h2"], g2, b2, x, y, F["st2"])


def _wgrad(g, a, part, dw):
    """dw += g.T @ a in row slices of at most WGRAD_SLICE_GROUPS partials (dw starts at zero)."""
    step = WGRAD_SLICE_GROUPS * GROUP_ROWS
    for r0 in range(0, g.shape[0], step):
        ops.fine_train_wgrad(g[r0:r0 + step], a[r0:r0 + step], part, dw, True)


def _layer_bwd(p, G, cross, g, W, x, dy, dx, want_w):
    """Backward of _layer_fwd (its state in W): dx = dy + d(mlp input)[:, :256] + dqkv W_qkv (dx None:
    not formed); the weight gradients G (w_qkv, merge, mlp0, mlp2, ln1 [2, 256], ln2 [2, 256])."""
    wqkv, wm, w0, w2, g1, _, g2, _ = p
    gqkv, gm, g0, g2w, gln1, gln2 = G
    F, T = W.f, W.t
    dh2 = T["t256a"]
    ops.coarse_tf_ln_bwd(F["h2"], g2, F["st2"], dy, dh2, W.lnpart, gln2, False)
    if want_w:
        _wgrad(dh2, F["r"], W.wpart, g2w)
    dh1 = T["t512a"]
    ops.fine_train_linear(dh2, w2, False, dh1, ops.EPI_MASK, aux=F["r"])        # ReLU: r > 0 <=> h1 > 0
    if want_w:
        _wgrad(dh1, F["xm"], W.wpart, g0)
    dxm = T["t512b"]
    ops.fine_train_linear(dh1, w0, False, dxm)
    dm0 = T["t256a"]
    ops.coarse_tf_ln_bwd(F["m0"], g1, F["st1"], dxm[:, D:], dm0, W.lnpart, gln1, False)
    if want_w:
        _wgrad(dm0, F["a"], W.wpart, gm)
    da = T["t256b"]
    ops.fine_train_linear(dm0, wm, False, da)
    dqkv = T["t768"]
    _attn_bwd(g, cross, W, F["qkv"], da, dqkv)
    if want_w:
        _wgrad(dqkv, x, W.wpart, gqkv)
    if dx is not None:
        ops.fine_train_linear(dqkv, wqkv, False, dx, ops.EPI_ADD, aux=dxm[:, :D], aux2=dy)


class CoarseTransformerStage(torch.autograd.Function):
    """(d3 [B, N, 256], d2 [B, S, 256]) = train_path.transformer(loftr_coarse, ...) on the kernels.
    Inputs: the 3D tokens [B, N, 256], the 2D tokens [B, S, 256], the 2D mask (uint8 [B, S] or None),
    the layer names, then the 10 parameters of each layer (train_fine.layer_params order)."""

    @staticmethod
    def forward(ctx, d3, d2, mask, names, *params):
        B, N, _ = d3.shape
        S = d2.shape[1]
        dev = d2.device
        g = _Geo(B, S, N, None if mask is None else mask.reshape(-1))
        P = _pack(params)
        x = torch.empty(g.rows, D, dtype=torch.float32, device=dev)
        x2, x3 = g.split(x)
        x2.view(B, S, D).copy_(d2)
        x3.view(B, N, D).copy_(d3)
        W = _Work(g, dev, backward=False)
        xs = [x]
        for i, name in enumerate(names):
            y = torch.empty_like(x)
            _layer_fwd(P[i], name == "cross", g, W, xs[-1], y)
            xs.append(y)
        out = xs.pop()
        ctx.save_for_backward(mask, *xs, *params)
        ctx.geo, ctx.names, ctx.dtypes = (B, S, N), tuple(names), (d3.dtype, d2.dtype)
        y2, y3 = g.split(out)
        return y3.view(B, N, D).to(d3.dtype), y2.view(B, S, D).to(d2.dtype)

    @staticmethod
    def backward(ctx, dd3, dd2):
        mask, *rest = ctx.saved_tensors
        names = ctx.names
        xs, params = rest[:len(names)], rest[len(names):]
        need = ctx.needs_input_grad
        want_x, want_w = need[0] or need[1], any(need[4:])
        grads = [None] * len(params)
        if not (want_x or want_w):
            return (None, None, None, None, *grads)
        (B, S, N), dev = ctx.geo, xs[0].device
        g = _Geo(B, S, N, None if mask is None else mask.reshape(-1))
        P = _pack(params)
        W = _Work(g, dev, backward=True)
        f32 = dict(dtype=torch.float32, device=dev)
        G = [(torch.zeros(3 * D, D, **f32), torch.zeros(D, D, **f32), torch.zeros(2 * D, 2 * D, **f32),
              torch.zeros(D, 2 * D, **f32), torch.zeros(2, D, **f32), torch.zeros(2, D, **f32)) for _ in names]
        dy = torch.empty(g.rows, D, **f32)
        dy2, dy3 = g.split(dy)
        dy2.view(B, S, D).copy_(dd2)
        dy3.view(B, N, D).copy_(dd3)
        dx = torch.empty_like(dy) if (want_x or len(names) > 1) else None
        for i in reversed(range(len(names))):
            cross = names[i] == "cross"
            _layer_fwd(P[i], cross, g, W, xs[i], W.t["t256b"])          # recompute; the output is not kept
            out = dx if (i > 0 or want_x) else None
            _layer_bwd(P[i], G[i], cross, g, W, xs[i], dy, out, want_w)
            if out is not None:
                dy, dx = dx, dy
        del W, dx
        d3 = d2 = None
        if want_x:
            dx2, dx3 = g.split(dy)
            d3 = dx3.view(B, N, D).to(ctx.dtypes[0]) if need[0] else None
            d2 = dx2.view(B, S, D).to(ctx.dtypes[1]) if need[1] else None
        if want_w:
            grads = []
            for gqkv, gm, g0, g2w, gln1, gln2 in G:
                grads += [gqkv[:D], gqkv[D:2 * D], gqkv[2 * D:], gm, g0, g2w, gln1[0], gln1[1], gln2[0], gln2[1]]
            grads = [t if n else None for t, n in zip(grads, need[4:])]
        return (d3, d2, None, None, *grads)


def coarse_transformer(tf, desc3d, desc2d, query_mask=None):
    """train_path.transformer(tf, desc3d, desc2d, query_mask) on the kernels: desc3d [B, 256, N],
    desc2d [B, S, 256], query_mask 0/1 [B, S] or None; returns (d3 [B, N, 256], d2 [B, S, 256])."""
    B, S, _ = desc2d.shape
    mask = None
    if query_mask is not None:
        mask = (query_mask.reshape(B, S) != 0).to(torch.uint8).contiguous()
    params = [p for layer in tf.layers for p in layer_params(layer)]
    return CoarseTransformerStage.apply(desc3d.transpose(1, 2), desc2d, mask, tuple(tf.layer_names), *params)
