"""Fine level of the training forward on the device (model.fine_train_mode "kernels", CUDA, train mode).

One autograd Function replaces train_path.fine_preprocess -> transformer(model.loftr_fine, ...) ->
train_path.fine_matching.  Its input is the backbone's fine map feat_f [B, 128, Hf, Wf] (fp32), the
bank's descriptors3d_db, the match ids and the parameters of the two fine layers; its output is
data["expec_f"] [M, 3] with a grad_fn, so losses.Loss is unchanged.  The opp_fine_train_* kernels
(csrc/opp_train_fine.cu) gather the 5 x 5 windows straight from feat_f and run both layers and the
heatmap expectation in fp32, forward and backward; no [B, 25*128, L] unfold tensor exists.

Memory: the matches are processed in chunks of CHUNK, each through a workspace of about 430 KB per
match.  The forward keeps nothing but expec_f; the backward recomputes a chunk's forward, then runs
its backward, and accumulates the weight gradients chunk after chunk (a fixed order).  d feat_f is
formed once at the end from the window gradients of every match, as a gather per fine pixel.
Every sum runs in a fixed order without floating-point atomics: two calls give the same bits.
"""
import torch

from . import ops

MODES = ("autograd", "kernels")
CHUNK = 192      # matches per pass through the workspace
D = 128
TOK = 26         # 25 window tokens + the 3D token per match


def check(model, data):
    """Raise for what the kernels do not cover (model.fine_train_mode "kernels")."""
    cfg = model.config
    if model.precision == "fp16":
        raise ValueError('fine_train_mode "kernels" needs precision "fp16x3": with single fp16 operands the '
                         'coarse matches the fine level refines differ from the eager fp32 ones')
    if not cfg["loftr_fine"]["enable"] or not cfg["fine_matching"]["enable"]:
        raise NotImplementedError('fine_train_mode "kernels" needs loftr_fine.enable and fine_matching.enable')
    if model.fine_preprocess.W != 5:
        raise NotImplementedError(f'fine_train_mode "kernels" is built for window size 5, not {model.fine_preprocess.W}')
    if list(model.loftr_fine.layer_names) != ["self", "cross"]:
        raise NotImplementedError('fine_train_mode "kernels" is built for the fine layers ["self", "cross"]')
    if data["descriptors3d_db"].requires_grad:
        raise NotImplementedError('fine_train_mode "kernels" does not differentiate descriptors3d_db')


def use_kernels(model, data):
    """True when the fine level of this training forward runs on the kernels (validated)."""
    mode = model.fine_train_mode
    if mode not in MODES:
        raise ValueError(f"fine_train_mode must be one of {MODES}, not {mode!r}")
    if mode != "kernels" or not model.training or not data["query_image"].is_cuda:
        return False
    check(model, data)
    return True


def layer_params(layer):
    """The 10 parameters of a fine LoFTREncoderLayer, in the Function's order."""
    return (layer.q_proj.weight, layer.k_proj.weight, layer.v_proj.weight, layer.merge.weight,
            layer.mlp[0].weight, layer.mlp[2].weight, layer.norm1.weight, layer.norm1.bias,
            layer.norm2.weight, layer.norm2.bias)


def _pack(params):
    """Per layer: (w_qkv [384, 128], w_merge, w_mlp0, w_mlp2, ln1 gamma, beta, ln2 gamma, beta)."""
    out = []
    for p in (params[:10], params[10:]):
        p = [t.detach().float().contiguous() for t in p]
        out.append((torch.cat(p[0:3], 0).contiguous(), *p[3:]))
    return out


class _Work:
    """Per-chunk buffers: the saved state of both layers (layer input | LayerNorm-1 output in xm,
    q | k | v, attention message, merge output, ReLU output, mlp output, LayerNorm statistics), the
    stage output and, for the backward, the gradient temporaries."""

    def __init__(self, rows, dev, backward):
        def e(*s):
            return torch.empty(*s, dtype=torch.float32, device=dev)
        self.layers = [dict(xm=e(rows, 2 * D), qkv=e(rows, 3 * D), a=e(rows, D), m0=e(rows, D), st1=e(rows, 2),
                            r=e(rows, 2 * D), h2=e(rows, D), st2=e(rows, 2)) for _ in range(2)]
        self.out = e(rows, D)
        if backward:
            self.t = dict(t128a=e(rows, D), t128b=e(rows, D), t256a=e(rows, 2 * D), t256b=e(rows, 2 * D),
                          t384=e(rows, 3 * D), dy2=e(rows, D), dy1=e(rows, D))
            self.part = e(ops.fine_train_groups(rows) * 4 * D * 2 * D)

    def view(self, rows):
        layers = [{k: v[:rows] for k, v in s.items()} for s in self.layers]
        t = {k: v[:rows] for k, v in self.t.items()} if hasattr(self, "t") else None
        return layers, self.out[:rows], t


def _layer_fwd(p, cross, S, y, m):
    """LoFTREncoderLayer.forward on both sequences: y = x + LN2(mlp([x, LN1(merge(attn))]))."""
    wqkv, wm, w0, w2, g1, b1, g2, b2 = p
    x = S["xm"][:, :D]
    ops.fine_train_linear(x, wqkv, True, S["qkv"])
    ops.fine_train_attention(S["qkv"], S["a"], m, cross)
    ops.fine_train_linear(S["a"], wm, True, S["m0"])
    ops.fine_train_ln(S["m0"], g1, b1, None, S["xm"][:, D:], S["st1"])
    ops.fine_train_linear(S["xm"], w0, True, S["r"], ops.EPI_RELU)
    ops.fine_train_linear(S["r"], w2, True, S["h2"])
    ops.fine_train_ln(S["h2"], g2, b2, x, y, S["st2"])


def _layer_bwd(p, g, cross, S, T, dy, dx, m, part, acc, want_w):
    """Backward of _layer_fwd: dx = dy + d(mlp input)[:, :128] + dqkv W_qkv (dx None: not formed);
    the weight gradients g (w_qkv, merge, mlp0, mlp2, ln1 [2, 128], ln2 [2, 128]) accumulate."""
    wqkv, wm, w0, w2, g1, _, g2, _ = p
    gqkv, gm, g0, g2w, gln1, gln2 = g
    x = S["xm"][:, :D]
    dh2 = T["t128a"]
    ops.fine_train_ln_bwd(S["h2"], g2, S["st2"], dy, dh2, part, gln2, acc)
    if want_w:
        ops.fine_train_wgrad(dh2, S["r"], part, g2w, acc)
    dh1 = T["t256a"]
    ops.fine_train_linear(dh2, w2, False, dh1, ops.EPI_MASK, aux=S["r"])        # ReLU: r > 0 <=> h1 > 0
    if want_w:
        ops.fine_train_wgrad(dh1, S["xm"], part, g0, acc)
    dxm = T["t256b"]
    ops.fine_train_linear(dh1, w0, False, dxm)
    dm0 = T["t128a"]
    ops.fine_train_ln_bwd(S["m0"], g1, S["st1"], dxm[:, D:], dm0, part, gln1, acc)
    if want_w:
        ops.fine_train_wgrad(dm0, S["a"], part, gm, acc)
    da = T["t128b"]
    ops.fine_train_linear(dm0, wm, False, da)
    dqkv = T["t384"]
    ops.fine_train_attention_bwd(S["qkv"], da, dqkv, m, cross)
    if want_w:
        ops.fine_train_wgrad(dqkv, x, part, gqkv, acc)
    if dx is not None:
        ops.fine_train_linear(dqkv, wqkv, False, dx, ops.EPI_ADD, aux=dxm[:, :D], aux2=dy)


def _chunks(M):
    for m0 in range(0, M, CHUNK):
        yield m0, min(M, m0 + CHUNK)


def _forward_chunk(P, work, feat, desc3d, ids, geo, m0, m1):
    m = m1 - m0
    (L1, L2), out, T = work.view(m * TOK)
    b, i, j = (t[m0:m1] for t in ids)
    ops.fine_train_gather(feat, desc3d, b, i, j, *geo, L1["xm"])
    _layer_fwd(P[0], False, L1, L2["xm"][:, :D], m)
    _layer_fwd(P[1], True, L2, out, m)
    return L1, L2, out, T


class FineStage(torch.autograd.Function):
    """expec_f = fine_matching(transformer(loftr_fine, fine_preprocess(feat_f, ...))) on the kernels.
    Inputs: feat_f, descriptors3d_db (no gradient), b_ids, i_ids, j_ids, geo = (hc, wc, stride), then
    the 20 parameters of the two layers (layer_params order)."""

    @staticmethod
    def forward(ctx, feat, desc3d, b_ids, i_ids, j_ids, geo, *params):
        M = b_ids.numel()
        P = _pack(params)
        expec = torch.empty(M, 3, dtype=torch.float32, device=feat.device)
        if M:
            work = _Work(min(M, CHUNK) * TOK, feat.device, backward=False)
            for m0, m1 in _chunks(M):
                _, _, out, _ = _forward_chunk(P, work, feat, desc3d, (b_ids, i_ids, j_ids), geo, m0, m1)
                ops.fine_train_match(out, m1 - m0, expec[m0:m1])
        ctx.save_for_backward(feat, desc3d, b_ids, i_ids, j_ids, *params)
        ctx.geo = geo
        return expec

    @staticmethod
    def backward(ctx, dexpec):
        feat, desc3d, b_ids, i_ids, j_ids, *params = ctx.saved_tensors
        geo, need = ctx.geo, ctx.needs_input_grad
        need_feat, want_w = need[0], any(need[6:])
        M, dev = b_ids.numel(), feat.device
        f32 = dict(dtype=torch.float32, device=dev)
        G = [(torch.zeros(3 * D, D, **f32), torch.zeros(D, D, **f32), torch.zeros(2 * D, 2 * D, **f32),
              torch.zeros(D, 2 * D, **f32), torch.zeros(2, D, **f32), torch.zeros(2, D, **f32)) for _ in range(2)]
        dx0 = torch.empty(M * TOK, D, **f32) if need_feat and M else None
        if M and (need_feat or want_w):
            P = _pack(params)
            dexpec = dexpec.float().contiguous()
            work = _Work(min(M, CHUNK) * TOK, dev, backward=True)
            for c, (m0, m1) in enumerate(_chunks(M)):
                m = m1 - m0
                L1, L2, out, T = _forward_chunk(P, work, feat, desc3d, (b_ids, i_ids, j_ids), geo, m0, m1)
                ops.fine_train_match_bwd(out, dexpec[m0:m1], m, T["dy2"])
                _layer_bwd(P[1], G[1], True, L2, T, T["dy2"], T["dy1"], m, work.part, c > 0, want_w)
                _layer_bwd(P[0], G[0], False, L1, T, T["dy1"], dx0[m0 * TOK:m1 * TOK] if need_feat else None, m,
                           work.part, c > 0, want_w)
            del work, T, L1, L2, out
        dfeat = None
        if need_feat:
            dfeat = torch.empty_like(feat)
            if M:
                hc, wc, stride = geo
                B = feat.shape[0]
                cells = (b_ids * (hc * wc) + j_ids).contiguous()
                _, col_ptr, col_rows = ops.gt_index(torch.zeros_like(b_ids), torch.arange(M, device=dev), cells,
                                                    (1, M, B * hc * wc))
                ops.fine_train_gather_bwd(dx0, col_ptr, col_rows, hc, wc, stride, dfeat)
            else:
                dfeat.zero_()
        grads = []
        for gqkv, gm, g0, g2w, gln1, gln2 in G:
            grads += [gqkv[:D], gqkv[D:2 * D], gqkv[2 * D:], gm, g0, g2w, gln1[0], gln1[1], gln2[0], gln2[1]]
        grads = [g if n else None for g, n in zip(grads, need[6:])]
        return (dfeat, None, None, None, None, None, *grads)


def fine_stage(model, data, feat_f):
    """Writes data["W"], data["expec_f"] (with grad_fn) and data["mkpts_query_f"] as train_path's
    fine_preprocess -> transformer -> fine_matching do (fine_matching.py:28-110)."""
    W = model.fine_preprocess.W
    data["W"] = W
    b_ids, i_ids, j_ids = data["b_ids"], data["i_ids"], data["j_ids"]
    assert b_ids.numel() != 0, "M is always >0, when training, see coarse_matching.py"
    hc, wc = (int(n) for n in data["q_hw_c"])
    hf, wf = (int(n) for n in data["q_hw_f"])
    stride = hf // hc
    if (hf - 1) // stride + 1 != hc or (wf - 1) // stride + 1 != wc:
        raise ValueError(f"fine map {hf}x{wf} and coarse grid {hc}x{wc} do not give unfold's L = hc*wc")
    params = [p for layer in model.loftr_fine.layers for p in layer_params(layer)]
    desc3d = data["descriptors3d_db"].detach().float().contiguous()
    ids = [t.contiguous() for t in (b_ids, i_ids, j_ids)]
    expec = FineStage.apply(feat_f.float().contiguous(), desc3d, *ids, (hc, wc, stride), *params)
    data["expec_f"] = expec
    with torch.no_grad():
        scale = data["q_hw_i"][0] / data["q_hw_f"][0]
        qs = scale * data["query_image_scale"][b_ids][:, [1, 0]] if "query_image_scale" in data else scale
        data["mkpts_query_f"] = data["mkpts_query_c"] + (expec[:, :2] * (W // 2) * qs)[: len(data["mkpts_query_c"])]
