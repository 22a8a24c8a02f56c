"""ResNet-FPN backbone of the training forward on the device (model.backbone_train_mode "kernels",
CUDA, train mode).

One autograd Function replaces train_path.backbone(model.backbone, img): the 22 convolutions, the 17
BatchNorms with their ReLU / LeakyReLU and residual adds, and the two bilinear x2 upsample-adds of the
FPN, forward and backward (csrc/opp_train_backbone.cu).  The convolutions' forward, data gradient and
weight gradient run on the tensor cores in 3xTF32 (each operand split into tf32 hi + lo, three MMAs
per k8 step); the rest runs in fp32.

BatchNorm follows each module's own .training: batch statistics over N·H·W (biased variance, the
module's eps), with running_mean / running_var / num_batches_tracked updated in place once per forward
as F.batch_norm does; or, for a module in eval mode (pretrained_fix calls backbone.eval()), its running
statistics; that form runs the forward only (frozen parameters, as pretrained_fix leaves them).

Memory: the forward keeps the segment inputs (x0, the layer1.0 output, x1, the layer2.0 output, x2, the
layer3.0 output, x3, x2_out), the output x3_out and the per-BN mean / inverse std, and nothing else.
The backward walks the segments in reverse (FPN 1/2, FPN 1/4, layer3_outconv, the six blocks, conv1);
each segment's forward is recomputed from its saved input with the saved statistics, then
differentiated, and each recomputed tensor is dropped after its last reader.  Weight gradients are
summed in slices of WGRAD_SLICE_GROUPS partials.  Every sum runs in a fixed order without
floating-point atomics: two calls give the same bits, running statistics included.
"""
import torch

from . import ops

MODES = ("autograd", "kernels")
WGRAD_SLICE_GROUPS = 32      # partials of one opp_backbone_train_conv_wgrad call (44 MiB at 196 x 196 x 3 x 3)

BLOCKS = ("layer1.0", "layer1.1", "layer2.0", "layer2.1", "layer3.0", "layer3.1")


def _block_convs(name, down):
    return (f"{name}.conv1", f"{name}.conv2") + ((f"{name}.downsample.0",) if down else ())


def _block_bns(name, down):
    return (f"{name}.bn1", f"{name}.bn2") + ((f"{name}.downsample.1",) if down else ())


CONVS = (("conv1",) + sum((_block_convs(b, b.endswith(".0") and b != "layer1.0") for b in BLOCKS), ()) +
         ("layer3_outconv", "layer2_outconv", "layer2_outconv2.0", "layer2_outconv2.3", "layer1_outconv",
          "layer1_outconv2.0", "layer1_outconv2.3"))
BNS = (("bn1",) + sum((_block_bns(b, b.endswith(".0") and b != "layer1.0") for b in BLOCKS), ()) +
       ("layer2_outconv2.1", "layer1_outconv2.1"))


def check(model, data):
    """Raise for what the kernels do not cover (model.backbone_train_mode "kernels")."""
    img = data["query_image"]
    if img.requires_grad:
        raise NotImplementedError('backbone_train_mode "kernels" does not differentiate query_image')
    if img.dim() != 4 or img.size(1) != 1:
        raise ValueError(f"query_image must be [B, 1, H, W], not {tuple(img.shape)}")
    if img.size(2) % 8 or img.size(3) % 8:
        raise ValueError(f"query_image is {img.size(2)} x {img.size(3)}: the FPN adds need H and W to be "
                         f"multiples of 8")
    bb = model.backbone
    mods = dict(bb.named_modules())
    if any(p.dtype != torch.float32 for p in bb.parameters()) or img.dtype != torch.float32:
        raise NotImplementedError('backbone_train_mode "kernels" runs fp32 parameters and images')
    if any(not mods[n].training for n in BNS) and any(p.requires_grad for p in bb.parameters()):
        raise NotImplementedError('backbone_train_mode "kernels" differentiates batch-statistics BatchNorm only: '
                                  'a backbone in eval mode (pretrained_fix) must have frozen parameters')
    if img.size(0) * (img.size(2) // 8) * (img.size(3) // 8) == 1 and any(
            mods[n].training for n in BNS):
        raise ValueError("Expected more than 1 value per channel when training (a 1 x 1 coarse map at batch 1)")


def use_kernels(model, data):
    """True when the backbone of this training forward runs on the kernels (validated)."""
    mode = model.backbone_train_mode
    if mode not in MODES:
        raise ValueError(f"backbone_train_mode must be one of {MODES}, not {mode!r}")
    if mode != "kernels" or not model.training or not data["query_image"].is_cuda:
        return False
    check(model, data)
    return True


def params(bb):
    """The Function's parameter inputs: the 22 convolution weights (CONVS order), then (gamma, beta) of
    the 17 BatchNorms (BNS order)."""
    mods = dict(bb.named_modules())
    return [mods[n].weight for n in CONVS] + [p for n in BNS for p in (mods[n].weight, mods[n].bias)]


def _empty(shape, dev):
    return torch.empty(shape, dtype=torch.float32, device=dev)


class _Net:
    """The parameters by name, the BN statistics and the kernel calls of one forward / backward."""

    def __init__(self, bb, tensors, dev):
        self.dev = dev
        self.w = {n: t.detach().contiguous() for n, t in zip(CONVS, tensors[:len(CONVS)])}
        gb = tensors[len(CONVS):]
        self.gamma = {n: gb[2 * i].detach().contiguous() for i, n in enumerate(BNS)}
        self.beta = {n: gb[2 * i + 1].detach().contiguous() for i, n in enumerate(BNS)}
        mods = dict(bb.named_modules())
        self.mods = {n: mods[n] for n in BNS}
        self.stride = {n: mods[n].stride[0] for n in CONVS}
        self.stats = {}              # BN name -> (mean, invstd), from the forward
        self.record = False          # forward: compute the statistics (and update the running ones)

    # forward pieces -----------------------------------------------------------------------------
    def conv(self, name, x):
        B, _, H, W = x.shape
        w = self.w[name]
        ho, wo = ops.conv_out_hw(H, W, w.shape[2], self.stride[name])
        y = _empty((B, w.shape[0], ho, wo), self.dev)
        ops.backbone_conv(x, w, self.stride[name], y)
        return y

    def _stats(self, name, h):
        if not self.record:
            return self.stats[name]
        m = self.mods[name]
        B, C, H, W = h.shape
        batch = m.training or m.running_mean is None
        if not batch:
            st = (m.running_mean.detach().float().contiguous(),
                  torch.rsqrt(m.running_var.detach().float() + m.eps).contiguous())
        else:
            st = (_empty(C, self.dev), _empty(C, self.dev))
            rm = rv = None
            factor = 0.0
            if m.training and m.track_running_stats:
                m.num_batches_tracked.add_(1)
                factor = (1.0 / float(m.num_batches_tracked) if m.momentum is None else m.momentum)
                rm, rv = m.running_mean, m.running_var
                if rm.dtype != torch.float32 or not rm.is_contiguous() or not rv.is_contiguous():
                    raise NotImplementedError("running statistics must be contiguous fp32")
            ops.backbone_bn_stats(h, m.eps, ops.backbone_bn_part(B, C, H * W, self.dev), *st, rm, rv, factor)
        self.stats[name] = (st[0], st[1], batch)
        return self.stats[name]

    def bn(self, name, h, act, res=None, out=None):
        mean, invstd, _ = self._stats(name, h)
        y = h if out is None else out
        ops.backbone_bn_act(h, mean, invstd, self.gamma[name], self.beta[name], res, act, y)
        return y

    def block(self, name, x, keep=False):
        """BasicBlock.forward; keep: also return the intermediates the backward reads."""
        down = name in ("layer2.0", "layer3.0")
        h1 = self.conv(f"{name}.conv1", x)
        a1 = self.bn(f"{name}.bn1", h1, "relu", out=_empty(h1.shape, self.dev) if keep else None)
        h2 = self.conv(f"{name}.conv2", a1)
        hd = r = None
        if down:
            hd = self.conv(f"{name}.downsample.0", x)
            r = self.bn(f"{name}.downsample.1", hd, "none", out=_empty(hd.shape, self.dev) if keep else None)
        y = self.bn(f"{name}.bn2", h2, "relu", res=x if r is None else r, out=_empty(h2.shape, self.dev) if keep else None)
        if not keep:
            return y
        return y, (h1, a1, h2, hd)

    def fpn(self, pre, lat_name, x, coarse, keep=False):
        """layer{k}_outconv2(layer{k}_outconv(x) + up(coarse)); keep: also the intermediates."""
        lat = self.conv(lat_name, x)
        ops.backbone_up2x_add(coarse, lat, lat)
        h = self.conv(f"{pre}.0", lat)
        t = self.bn(f"{pre}.1", h, "leaky", out=_empty(h.shape, self.dev) if keep else None)
        out = self.conv(f"{pre}.3", t)
        if not keep:
            return out
        return out, (lat, h, t)

    # backward pieces ----------------------------------------------------------------------------
    def wgrad(self, name, x, dy, want):
        if not want(name):
            return
        w = self.w[name]
        dw = torch.zeros_like(w)
        B, _, ho, wo = dy.shape
        pixels = B * ho * wo
        group = ops.backbone_wgrad_group()
        step = WGRAD_SLICE_GROUPS * group
        part = _empty(min(pixels, step) // group * w.numel() + w.numel(), self.dev)
        for p0 in range(0, pixels, step):
            ops.backbone_conv_wgrad(x, dy, self.stride[name], dw, part, p0, min(step, pixels - p0), True)
        self.grads[name] = dw

    def dgrad(self, name, dy, x_shape, out=None, accumulate=False):
        dx = _empty(x_shape, self.dev) if out is None else out
        ops.backbone_conv_dgrad(dy, self.w[name], self.stride[name], dx, accumulate)
        return dx

    def bn_bwd(self, name, h, y, dy, act, dres=None):
        """dh (written over dy) and the BN's (dgamma, dbeta); dres = d residual when given."""
        mean, invstd, batch = self.stats[name]
        B, C, H, W = h.shape
        dgb = _empty((2, C), self.dev)
        ops.backbone_bn_act_bwd(h, y, dy, mean, invstd, self.gamma[name], act, batch,
                                ops.backbone_bn_part(B, C, H * W, self.dev), dy, dres, dgb)
        self.grads[name] = dgb
        return dy

    def block_bwd(self, name, x, dy, want, dx_out, accumulate):
        """Backward of block(name) from its input x; dy is consumed.  dx_out: the input gradient
        buffer (+= when accumulate) or None when not needed."""
        down = name in ("layer2.0", "layer3.0")
        y, (h1, a1, h2, hd) = self.block(name, x, keep=True)
        dr = dx_out if (not down and dx_out is not None and not accumulate) else _empty(dy.shape, self.dev)
        dh2 = self.bn_bwd(f"{name}.bn2", h2, y, dy, "relu", dres=dr)
        del y
        self.wgrad(f"{name}.conv2", a1, dh2, want)
        da1 = self.dgrad(f"{name}.conv2", dh2, a1.shape)
        del dh2, h2
        dh1 = self.bn_bwd(f"{name}.bn1", h1, a1, da1, "relu")
        del a1, h1
        self.wgrad(f"{name}.conv1", x, dh1, want)
        if down:
            dhd = self.bn_bwd(f"{name}.downsample.1", hd, None, dr, "none")
            del hd
            self.wgrad(f"{name}.downsample.0", x, dhd, want)
            if dx_out is not None:
                self.dgrad(f"{name}.downsample.0", dhd, x.shape, dx_out, accumulate)
            del dhd, dr
        if dx_out is not None:
            self.dgrad(f"{name}.conv1", dh1, x.shape, dx_out, True)

    def fpn_bwd(self, pre, lat_name, x, coarse, dout, want, dcoarse, dx_out, accumulate_coarse):
        """Backward of fpn(...): dcoarse (+)= the upsample path's gradient, dx_out = the lateral
        input's gradient (overwritten) or None; dout is consumed."""
        _, (lat, h, t) = self.fpn(pre, lat_name, x, coarse, keep=True)
        self.wgrad(f"{pre}.3", t, dout, want)
        dt = self.dgrad(f"{pre}.3", dout, t.shape)
        del dout
        dh = self.bn_bwd(f"{pre}.1", h, t, dt, "leaky")
        del t, h
        self.wgrad(f"{pre}.0", lat, dh, want)
        dlat = self.dgrad(f"{pre}.0", dh, lat.shape)
        del dh, lat
        ops.backbone_up2x_bwd(dlat, dcoarse, accumulate_coarse)
        self.wgrad(lat_name, x, dlat, want)
        if dx_out is not None:
            self.dgrad(lat_name, dlat, x.shape, dx_out)


# the backward's segments, last first: (conv names, BN names) whose gradients each one produces
_SEGMENTS = (
    (("layer1_outconv2.0", "layer1_outconv2.3", "layer1_outconv"), ("layer1_outconv2.1",)),
    (("layer2_outconv2.0", "layer2_outconv2.3", "layer2_outconv"), ("layer2_outconv2.1",)),
    (("layer3_outconv",), ()),
) + tuple((_block_convs(b, b in ("layer2.0", "layer3.0")), _block_bns(b, b in ("layer2.0", "layer3.0")))
          for b in reversed(BLOCKS)) + ((("conv1",), ("bn1",)),)


class BackboneStage(torch.autograd.Function):
    """(x3_out [B, 256, H/8, W/8], x1_out [B, 128, H/2, W/2]) = train_path.backbone(bb, img) on the
    kernels.  Inputs: the backbone module (structure, BN modes and running statistics), the image
    [B, 1, H, W], then params(bb)."""

    @staticmethod
    def forward(ctx, bb, img, *tensors):
        dev = img.device
        net = _Net(bb, tensors, dev)
        net.record = True
        img = img.detach().contiguous()
        x0 = net.bn("bn1", net.conv("conv1", img), "relu")
        segs = [x0]
        for name in BLOCKS:
            segs.append(net.block(name, segs[-1]))
        x3 = segs[-1]
        x3_out = net.conv("layer3_outconv", x3)
        x2_out = net.fpn("layer2_outconv2", "layer2_outconv", segs[4], x3_out)
        x1_out = net.fpn("layer1_outconv2", "layer1_outconv", segs[2], x2_out)
        stats = [t for n in BNS for t in net.stats[n][:2]]
        ctx.batch = tuple(net.stats[n][2] for n in BNS)
        ctx.save_for_backward(img, *segs, x3_out, x2_out, *stats, *tensors)
        ctx.bb = bb
        ctx.set_materialize_grads(False)
        return x3_out, x1_out

    @staticmethod
    def backward(ctx, d_x3_out, d_x1_out):
        need = ctx.needs_input_grad[2:]
        nothing = (None, None) + (None,) * len(need)
        if not any(need) or (d_x3_out is None and d_x1_out is None):
            return nothing
        saved = ctx.saved_tensors
        img, segs, (x3_out, x2_out) = saved[0], list(saved[1:8]), saved[8:10]
        stats = saved[10:10 + 2 * len(BNS)]
        tensors = saved[10 + 2 * len(BNS):]
        dev = img.device
        net = _Net(ctx.bb, tensors, dev)
        net.stats = {n: (stats[2 * i], stats[2 * i + 1], ctx.batch[i]) for i, n in enumerate(BNS)}
        net.grads = {}
        need_conv = dict(zip(CONVS, need[:len(CONVS)]))
        need_bn = {n: need[len(CONVS) + 2 * i] or need[len(CONVS) + 2 * i + 1] for i, n in enumerate(BNS)}

        def want(name):
            return need_conv[name]

        # how many segments (last first) the walk has to reach
        seg_need = [any(need_conv[c] for c in cs) or any(need_bn[b] for b in bs) for cs, bs in _SEGMENTS]
        last = max(i for i, v in enumerate(seg_need) if v)

        x1, x2, x3 = segs[2], segs[4], segs[6]
        d3 = (torch.zeros_like(x3_out) if d_x3_out is None else d_x3_out.float().contiguous().clone())
        dx1 = dx2 = None
        fpn = d_x1_out is not None
        if fpn:
            d2o = _empty(x2_out.shape, dev)
            dx1 = _empty(x1.shape, dev) if last >= 3 else None
            net.fpn_bwd("layer1_outconv2", "layer1_outconv", x1, x2_out, d_x1_out.float().contiguous().clone(),
                        want, d2o, dx1, False)
            if last >= 1:
                dx2 = _empty(x2.shape, dev) if last >= 3 else None
                net.fpn_bwd("layer2_outconv2", "layer2_outconv", x2, x3_out, d2o, want, d3, dx2, True)
            del d2o
        if last >= 2:
            net.wgrad("layer3_outconv", x3, d3, want)
            dy = net.dgrad("layer3_outconv", d3, x3.shape) if last >= 3 else None
            del d3
            # blocks, last first; segs[i] is the input of BLOCKS[i]
            for k, name in enumerate(reversed(BLOCKS)):
                i = len(BLOCKS) - 1 - k
                if last < 3 + k:
                    break
                x = segs[i]
                if last < 4 + k:
                    dx, acc = None, False
                elif name == "layer2.0":
                    dx, acc = (dx1, True) if dx1 is not None else (_empty(x.shape, dev), False)
                elif name == "layer3.0":
                    dx, acc = (dx2, True) if dx2 is not None else (_empty(x.shape, dev), False)
                else:
                    dx, acc = _empty(x.shape, dev), False
                net.block_bwd(name, x, dy, want, dx, acc)
                dy = dx
            if last >= 3 + len(BLOCKS):
                h0 = net.conv("conv1", img)
                dh0 = net.bn_bwd("bn1", h0, segs[0], dy, "relu")
                del h0
                net.wgrad("conv1", img, dh0, want)
        grads = [net.grads.get(n) if need_conv[n] else None for n in CONVS]
        for i, n in enumerate(BNS):
            dgb = net.grads.get(n)
            grads += [dgb[0] if dgb is not None and need[len(CONVS) + 2 * i] else None,
                      dgb[1] if dgb is not None and need[len(CONVS) + 2 * i + 1] else None]
        return (None, None, *grads)


def backbone(bb, img):
    """train_path.backbone(bb, img) on the kernels: (feat_c [B, 256, H/8, W/8], feat_f [B, 128, H/2, W/2])."""
    return BackboneStage.apply(bb, img, *params(bb))
