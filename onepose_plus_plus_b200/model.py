"""Drop-in for the reference ``OnePosePlus_model`` (src/models/OnePosePlus/OnePosePlusModel.py:25-201).

Same constructor (``config, profiler=None, debug=False``), same config keys, same 195 state-dict
keys (so ``load_state_dict(strict=True)`` of a reference checkpoint works), same in-place
``forward(data)`` contract — but ``forward`` runs the whole coarse-to-fine matcher through the
sm_90a kernels of ``libopp_b200.so``.  The ``nn.Module`` tree below only *holds* parameters with
the reference's names and initialisers; there is no PyTorch math on the hot path and no fallback:
CPU tensors, training mode, or a missing extension raise.

Scope (DESIGN.md): inference (``eval()``, no autograd), linear attention; extensions of the input
path (resident bank, uint8 frames, lazy ``conf_matrix``, CUDA-graph replay) are documented at
``forward`` / ``set_bank`` / ``enable_cuda_graphs``.
"""
import contextlib
import math
import operator
import os

import torch
import torch.nn as nn

from . import ops

__all__ = ["OnePosePlus_model", "build_backbone"]


# ---------------------------------------------------------------------------------------------
# parameter containers — names / shapes / initialisers follow the reference
# ---------------------------------------------------------------------------------------------
def _conv(cin, cout, k, stride=1):
    return nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2, bias=False)


class BasicBlock(nn.Module):
    """backbone/resnet.py:20-45"""

    def __init__(self, in_planes, planes, stride=1):
        super().__init__()
        self.conv1 = _conv(in_planes, planes, 3, stride)
        self.conv2 = _conv(planes, planes, 3)
        self.bn1 = nn.BatchNorm2d(planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = None if stride == 1 else nn.Sequential(
            nn.Conv2d(in_planes, planes, kernel_size=1, stride=stride, padding=0, bias=False),
            nn.BatchNorm2d(planes))


class ResNetFPN_8_2(nn.Module):
    """backbone/resnet.py:85-164 (parameters only; compute is in OnePosePlus_model._backbone)"""

    def __init__(self, config):
        super().__init__()
        if config["block_type"] != "BasicBlock":
            raise NotImplementedError("only BasicBlock backbones are built (resnet.py:80-83)")
        d0 = config["initial_dim"]
        b = config["block_dims"]
        self.block_dims = b
        self.output_layers = config["output_layers"]
        self.conv1 = nn.Conv2d(1, d0, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(d0)
        self.layer1 = nn.Sequential(BasicBlock(d0, b[0], 1), BasicBlock(b[0], b[0], 1))
        self.layer2 = nn.Sequential(BasicBlock(b[0], b[1], 2), BasicBlock(b[1], b[1], 1))
        self.layer3 = nn.Sequential(BasicBlock(b[1], b[2], 2), BasicBlock(b[2], b[2], 1))
        self.layer3_outconv = _conv(b[2], b[2], 1)
        self.layer2_outconv = _conv(b[1], b[2], 1)
        self.layer2_outconv2 = nn.Sequential(_conv(b[2], b[2], 3), nn.BatchNorm2d(b[2]),
                                             nn.LeakyReLU(), _conv(b[2], b[1], 3))
        self.layer1_outconv = _conv(b[0], b[1], 1)
        self.layer1_outconv2 = nn.Sequential(_conv(b[1], b[1], 3), nn.BatchNorm2d(b[1]),
                                             nn.LeakyReLU(), _conv(b[1], b[0], 3))
        for m in self.modules():  # resnet.py:126-131
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)


def build_backbone(config):
    """backbone/__init__.py:7-15"""
    if config["type"] == "ResNetFPN":
        if list(config["resolution"]) == [8, 2]:
            return ResNetFPN_8_2(config["resnetfpn"])
        raise NotImplementedError
    raise ValueError("reaching this line! LOFTR_BACKBONE.TYEP and RESOLUTION are not correct")


class PositionEncodingSine(nn.Module):
    """utils/position_encoding.py:8-42 — keeps the reference's floor-division quirk."""

    def __init__(self, d_model, max_shape=(256, 256)):
        super().__init__()
        max_shape = tuple(max_shape)
        pe = torch.zeros((d_model, *max_shape))
        y_position = torch.ones(max_shape).cumsum(0).float().unsqueeze(0)
        x_position = torch.ones(max_shape).cumsum(1).float().unsqueeze(0)
        div_term = torch.exp(torch.arange(0, d_model // 2, 2).float()
                             * (-math.log(10000.0) / d_model // 2))[:, None, None]
        pe[0::4] = torch.sin(x_position * div_term)
        pe[1::4] = torch.cos(x_position * div_term)
        pe[2::4] = torch.sin(y_position * div_term)
        pe[3::4] = torch.cos(y_position * div_term)
        self.register_buffer("pe", pe.unsqueeze(0), persistent=False)


class KeypointEncoding_linear(nn.Module):
    """utils/position_encoding.py:46-79 (parameters only)"""

    def __init__(self, inp_dim, feature_dim, layers, norm_method="batchnorm"):
        super().__init__()
        if norm_method != "instancenorm":
            raise NotImplementedError("kernel implements norm_method 'instancenorm' (shipped configs)")
        channels = [inp_dim] + list(layers) + [feature_dim]
        mods = []
        for i in range(1, len(channels)):
            mods.append(nn.Linear(channels[i - 1], channels[i], bias=True))
            if i < len(channels) - 1:
                mods.append(nn.InstanceNorm1d(channels[i]))
                mods.append(nn.ReLU())
        self.encoder = nn.Sequential(*mods)
        nn.init.constant_(self.encoder[-1].bias, 0.0)


class LoFTREncoderLayer(nn.Module):
    """loftr_module/transformer.py:7-63 (parameters only)"""

    def __init__(self, d_model, nhead, attention="linear", norm_method="layernorm", rezero=None):
        super().__init__()
        if attention not in ("linear", "full"):
            raise NotImplementedError(f"attention {attention!r}: 'linear' and 'full' are built")
        self.attention_type = attention
        if norm_method != "layernorm":
            raise NotImplementedError("only norm_method='layernorm' is built")
        if rezero is not None:
            raise NotImplementedError("rezero is not built (null in the shipped configs)")
        self.dim = d_model // nhead
        self.nhead = nhead
        self.q_proj = nn.Linear(d_model, d_model, bias=False)
        self.k_proj = nn.Linear(d_model, d_model, bias=False)
        self.v_proj = nn.Linear(d_model, d_model, bias=False)
        self.merge = nn.Linear(d_model, d_model, bias=False)
        self.mlp = nn.Sequential(nn.Linear(d_model * 2, d_model * 2, bias=False), nn.ReLU(True),
                                 nn.Linear(d_model * 2, d_model, bias=False))
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)


class LocalFeatureTransformer(nn.Module):
    """loftr_module/transformer.py:97-131 (parameters only)"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.d_model = config["d_model"]
        self.nhead = config["nhead"]
        self.layer_names = list(config["layer_names"]) * config["layer_iter_n"]
        if config["redraw_interval"] is not None:
            assert config["redraw_interval"] % 2 == 0
        if config["type"] != "LoFTR":
            raise ValueError()
        if config["final_proj"]:
            raise NotImplementedError("final_proj is False in every shipped config")
        layers = []
        for name in self.layer_names:
            if name not in ("self", "cross"):
                raise NotImplementedError
            layers.append(LoFTREncoderLayer(config["d_model"], config["nhead"], config["attention"],
                                            config["norm_method"], config["rezero"]))
        self.layers = nn.ModuleList(layers)
        for p in self.parameters():  # transformer.py:128-131
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)


class CoarseMatching(nn.Module):
    """utils/coarse_matching.py:45-75 (configuration only)"""

    def __init__(self, config, profiler=None):
        super().__init__()
        self.config = config
        if config["feat_norm_method"] != "sqrt_feat_dim":
            raise ValueError("only feat_norm_method 'sqrt_feat_dim' is built")
        if config["type"] != "dual-softmax":
            raise NotImplementedError()
        self.temperature = config["dual_softmax"]["temperature"]
        self.thr = config["thr"]
        self.border_rm = config["border_rm"]


class FinePreprocess(nn.Module):
    """loftr_module/fine_preprocess.py:8-30 (configuration only)"""

    def __init__(self, config, cf_res=None, feat_ids=None, feat_dims=None):
        super().__init__()
        self.config = config
        self.W = config["window_size"]


class FineMatching(nn.Module):
    """utils/fine_matching.py:10-27 (configuration only)"""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self._type = config["s2d"]["type"]
        if self._type != "heatmap":
            raise NotImplementedError()


def _pad16(c):
    return (c + 15) // 16 * 16


# ---------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------
_VERSION_OF = operator.attrgetter("_version")


class _OutPack:
    """The per-match outputs of a forward carved out of ONE byte buffer.  In CUDA-graph mode the
    graph owns the buffers it writes, so the caller gets copies: one clone of the pack (one
    kernel) instead of one per output tensor."""

    def __init__(self, nbytes, dev):
        self.buf = torch.empty((nbytes + 15) & ~15, dtype=torch.uint8, device=dev)
        self.fields = []
        self._off = 0

    @staticmethod
    def nbytes(cap, fcap):
        # b_ids, i_ids, j_ids (int64), mconf, mkpts_3d_db [.,3], mkpts_query_c [.,2]; expec_f [.,3],
        # mkpts_query_f [.,2]; 16 B alignment slack per field
        # + gt_mask (bool, all False at inference: coarse_matching.py:233 with no GT)
        return cap * (3 * 8 + 4 + 12 + 8 + 1) + fcap * (12 + 8) + 16 * 9

    def new(self, key, shape, dtype):
        n = dtype.itemsize
        for d in shape:
            n *= d
        off = (self._off + 15) & ~15
        self.fields.append((key, off, n, dtype, tuple(shape)))
        self._off = off + n
        return self.buf[off:off + n].view(dtype).view(shape)

    def views(self, buf, M):
        """The first M rows of every field of `buf` (a clone of self.buf): one typed alias of the
        buffer per dtype + one as_strided per field (this runs on the host after the forward's only
        sync, so every tensor op here is latency)."""
        bases, out = {}, {}
        for k, off, n, dt, shape in self.fields:
            base = bases.get(dt)
            if base is None:
                base = bases[dt] = buf.view(dt)
            tail = shape[1:]
            stride = (tail[0], 1) if tail else (1,)
            out[k] = torch.as_strided(base, (M,) + tail, stride, off // dt.itemsize)
        return out


class _Engine(nn.Module):
    """What the 2D-3D matcher (OnePosePlus_model) and the 2D-2D matcher (loftr.LoFTR_for_OnePose_Plus)
    share: weight preparation for the kernels, the name-keyed workspace, the ResNet-FPN backbone
    and the d_model-256 encoder layer, all as sequences of C-ABI calls."""

    def _init_engine(self, precision, coarse_attention="linear"):
        precision = precision or os.environ.get("OPP_B200_PRECISION", "fp16x3")
        if precision not in ("fp16x3", "fp16"):
            raise ValueError(f"unknown precision {precision!r}")
        self.precision = precision
        self._coarse_attention = coarse_attention
        self._plan = None
        self._plan_sig = None
        self._sig_tensors = None
        self._apply_epoch = 0
        self._ws = {}
        self._ws_epoch = 0
        self._graphs = {}

    @property
    def kv_single_plane(self):
        return True   # read-only, reported by bench.py: the K'/V rows have no other layout

    def _pe_module(self):
        return getattr(self, "dense_pos_encoding", None)

    def _ensure_plan(self, dev):
        sig = self._signature()
        if self._plan is None or self._plan_sig != sig or self._plan["device"] != dev:
            self._plan = self._prepare(dev)
            self._plan["device"] = dev
            self._plan_sig = sig
            self._graphs = {}

    @property
    def split(self):
        return self.precision == "fp16x3"

    # ------------------------------------------------------------------ weight preparation
    def _apply(self, fn, *args, **kwargs):
        # .cuda() / .to() / .half(): parameters are replaced -> re-read the tensor list
        self._sig_tensors = None
        self._apply_epoch += 1
        return super()._apply(fn, *args, **kwargs)

    def _signature(self):
        """Cheap identity of the weights: the parameter / buffer tensors are listed once (the list
        is rebuilt after _apply or load_state_dict(assign=True)); per forward only their in-place
        version counters are read (load_state_dict, optimizer steps and .copy_() bump them)."""
        ts = self._sig_tensors
        if ts is None:
            ts = self._sig_tensors = list(self.state_dict(keep_vars=True).values())
        return (self.precision, self._apply_epoch, sum(map(_VERSION_OF, ts)))

    def load_state_dict(self, *args, **kwargs):
        self._sig_tensors = None
        self._apply_epoch += 1
        return super().load_state_dict(*args, **kwargs)

    @torch.no_grad()
    def _prepare(self, device):
        """Fold eval-mode BatchNorm into the convolutions (w' = w*g/sqrt(var+eps),
        b' = beta - mean*g/sqrt(var+eps)), pad 196-channel tensors to 208, reorder weights to the
        kernels' layouts and convert GEMM operands to fp16 planes (hi | lo)."""
        sd = {k: v.detach().to(device=device, dtype=torch.float32) if v.is_floating_point() else v
              for k, v in self.state_dict().items()}
        split = self.split
        P = {}

        def fold(wkey, bnkey):
            w = sd[wkey + ".weight"]
            if bnkey is None:
                return w, torch.zeros(w.shape[0], device=device)
            g = sd[bnkey + ".weight"] / torch.sqrt(sd[bnkey + ".running_var"] + 1e-5)
            return w * g[:, None, None, None], sd[bnkey + ".bias"] - sd[bnkey + ".running_mean"] * g

        def conv(name, wkey, bnkey):
            w, b = fold("backbone." + wkey, None if bnkey is None else "backbone." + bnkey)
            co, ci, k, _ = w.shape
            wp = torch.zeros(_pad16(co), k, k, _pad16(ci), device=device)
            wp[:co, :, :, :ci] = w.permute(0, 2, 3, 1)
            bp = torch.zeros(_pad16(co), device=device)
            bp[:co] = b
            P[name] = (ops.to_planes(wp.reshape(_pad16(co), -1), split), bp.contiguous())

        # conv1 runs as ONE 64-wide K chunk of the wgmma engine: W[c] = (49 folded taps, folded
        # bias, 14 zeros) against im2col rows (49 taps, 1.0, 14 zeros) — ops.conv1_gemm
        w, b = fold("backbone.conv1", "backbone.bn1")
        w64 = torch.zeros(w.shape[0], 64, device=device)
        w64[:, :49] = w.view(w.shape[0], 49)
        w64[:, 49] = b
        P["conv1"] = ops.to_planes(w64, split)
        for li in (1, 2, 3):
            for bi in (0, 1):
                p = f"layer{li}.{bi}"
                conv(p + ".conv1", p + ".conv1", p + ".bn1")
                conv(p + ".conv2", p + ".conv2", p + ".bn2")
                if li > 1 and bi == 0:
                    conv(p + ".down", p + ".downsample.0", p + ".downsample.1")
        conv("layer3_outconv", "layer3_outconv", None)
        conv("layer2_outconv", "layer2_outconv", None)
        conv("layer2_outconv2.0", "layer2_outconv2.0", "layer2_outconv2.1")
        conv("layer2_outconv2.3", "layer2_outconv2.3", None)
        conv("layer1_outconv", "layer1_outconv", None)
        conv("layer1_outconv2.0", "layer1_outconv2.0", "layer1_outconv2.1")
        conv("layer1_outconv2.3", "layer1_outconv2.3", None)

        if "kpt_3d_pos_encoding.encoder.0.weight" in sd:
            P["kpt_mlp"] = [(sd[f"kpt_3d_pos_encoding.encoder.{i}.weight"].t().contiguous(),
                             sd[f"kpt_3d_pos_encoding.encoder.{i}.bias"].contiguous()) for i in (0, 3, 6, 9)]

        def layer(prefix):
            g = lambda k: sd[prefix + k]  # noqa: E731
            tp = lambda t: ops.to_planes(t, split)  # noqa: E731
            return {
                "wq": tp(g("q_proj.weight")),
                "wkv": tp(torch.cat([g("k_proj.weight"), g("v_proj.weight")], 0)),
                "wqkv": tp(torch.cat([g("q_proj.weight"), g("k_proj.weight"), g("v_proj.weight")], 0)),
                "merge32": g("merge.weight").contiguous(),
                "merge16": tp(g("merge.weight")),
                "mlp0": tp(g("mlp.0.weight")),
                "mlp2": tp(g("mlp.2.weight")),
                "n1": (g("norm1.weight").contiguous(), g("norm1.bias").contiguous()),
                "n2": (g("norm2.weight").contiguous(), g("norm2.bias").contiguous()),
            }

        P["coarse"] = [layer(f"loftr_coarse.layers.{i}.") for i in range(len(self.loftr_coarse.layers))]
        P["fine"] = [layer(f"loftr_fine.layers.{i}.") for i in range(len(self.loftr_fine.layers))]
        P["pe"] = {}
        return P

    def _pe_tokens(self, hc, wc, device):
        key = (hc, wc)
        if key not in self._plan["pe"]:
            pem = self._pe_module()
            if pem is None:
                pe = torch.zeros(hc * wc, 256, device=device)
            else:
                pe = pem.pe[0, :, :hc, :wc].to(device)
                pe = pe.permute(1, 2, 0).reshape(hc * wc, -1).contiguous()
            self._plan["pe"][key] = pe
        return self._plan["pe"][key]

    def _buf(self, name, shape, dtype, device):
        """Workspace tensor `name`: ONE backing allocation per name, grown to the largest size ever
        requested (high-water mark) and viewed at the requested shape — memory stays bounded when
        point counts / image sizes change from object to object (a long-running service), and the
        steady state allocates nothing.  `_ws_epoch` counts (re)allocations: captured CUDA graphs
        hold raw pointers and are dropped when it moves."""
        nbytes = dtype.itemsize * math.prod(shape)
        ent = self._ws.get(name)
        if ent is None or ent[0].device != device or ent[0].numel() < nbytes:
            ent = (torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device), {})
            self._ws[name] = ent
            self._ws_epoch += 1
        key = (tuple(shape), dtype)
        v = ent[1].get(key)
        if v is None:
            if len(ent[1]) >= 16:
                ent[1].clear()
            v = ent[0][:nbytes].view(dtype).view(tuple(shape))
            ent[1][key] = v
        return v

    def clear_workspace(self):
        """Drop the cached workspace (re-created by the next forward) and captured graphs."""
        self._ws = {}
        self._graphs = {}
        self._ws_epoch += 1

    def workspace_bytes(self):
        return sum(e[0].numel() for e in self._ws.values())

    # ------------------------------------------------------------------ stages
    def _backbone(self, img, defer_fine=False, fpn_stream=None, coarse_only=False):
        """ResNetFPN_8_2.forward (backbone/resnet.py:141-164) -> coarse tokens (+pe), fine map.
        defer_fine: stop before layer1_outconv2 and return its input (the merged 1/2-resolution
        map) instead of the fine map; the caller finishes with _fine_head_dense or, when the
        matches are few, _fine_head_windows.  fpn_stream (latency mode): the top-down path below
        the coarse output — which nothing needs before the fine stage — is enqueued on that stream
        so that it runs beside the coarse transformer; the caller joins it before the fine head.
        coarse_only: stop after the coarse tokens (the fine map is None)."""
        P = self._plan
        dev = img.device
        B, _, H, W = img.shape
        f16 = torch.float16
        split = self.split
        pl = 2 if split else 1

        def cv(name, x, out_name, ksize, stride, act=0, resid=None, **kw):
            w, b = P[name]
            Bn, h, wd, _ = x.shape
            oh, ow = (h - 1) // stride + 1, (wd - 1) // stride + 1
            out = self._buf(out_name, (Bn, oh, ow, pl * w.shape[0]), f16, dev)
            return ops.conv2d_nhwc(x, w, b, out, ksize, stride, split, act, resid, **kw)

        x0 = ops.conv1_gemm(img, P["conv1"], self._buf("conv1_cols", (B * (H // 2) * (W // 2), pl * 64), f16, dev),
                            self._buf("x0", (B, H // 2, W // 2, pl * 128), f16, dev), split)

        def block(prefix, x, tag, stride):
            t = cv(prefix + ".conv1", x, tag + "_t", 3, stride, act=1)
            sc = x if stride == 1 else cv(prefix + ".down", x, tag + "_ds", 1, stride)
            return cv(prefix + ".conv2", t, tag + "_o", 3, 1, act=1, resid=sc)

        x1 = block("layer1.1", block("layer1.0", x0, "l1a", 1), "l1b", 1)
        x2 = block("layer2.1", block("layer2.0", x1, "l2a", 2), "l2b", 1)
        x3 = block("layer3.1", block("layer3.0", x2, "l3a", 2), "l3b", 1)
        hc, wc = x3.shape[1:3]
        S = hc * wc
        tok = self._buf("q2_0", (B, S, pl * 256), f16, dev)
        x3_out = cv("layer3_outconv", x3, "x3_out", 1, 1, tok=tok, pe=self._pe_tokens(hc, wc, dev))
        if coarse_only:
            return tok, None, (hc, wc)

        def top_down():
            # FPN top-down merge fused into the lateral 1x1 conv epilogue (resnet.py:149-157)
            x2_lat = cv("layer2_outconv", x2, "x2_lat", 1, 1, up=x3_out)
            t = cv("layer2_outconv2.0", x2_lat, "x2_h", 3, 1, act=2)
            x2_out = cv("layer2_outconv2.3", t, "x2_out", 3, 1)
            return cv("layer1_outconv", x1, "x1_lat", 1, 1, up=x2_out)

        if fpn_stream is not None:
            fpn_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(fpn_stream):
                x1_lat = top_down()
        else:
            x1_lat = top_down()
        if defer_fine:
            return tok, x1_lat, (hc, wc)
        return tok, self._fine_head_dense(x1_lat), (hc, wc)

    def _fine_head_dense(self, x1_lat):
        """layer1_outconv2 (resnet.py:155-157) on the whole 1/2-resolution map."""
        P, split = self._plan, self.split
        pl = 2 if split else 1
        B, h, w, _ = x1_lat.shape
        (w0, b0), (w1, b1) = P["layer1_outconv2.0"], P["layer1_outconv2.3"]
        t = self._buf("x1_h", (B, h, w, pl * w0.shape[0]), torch.float16, x1_lat.device)
        ops.conv2d_nhwc(x1_lat, w0, b0, t, 3, 1, split, 2)
        out = self._buf("x1_out", (B, h, w, pl * w1.shape[0]), torch.float16, x1_lat.device)
        return ops.conv2d_nhwc(t, w1, b1, out, 3, 1, split, 0)

    def _fine_head_windows(self, x1_lat, b_ids, j_ids, M, wc, stride, count=None):
        """The same two convolutions evaluated only where fine_preprocess.py:40-47 reads them: the
        5x5 window of each coarse match (conv A on its 7x7 neighbourhood, conv B on the window).
        Returns the compact window tensor [M, 5, 8, pl*128] (values identical to the dense map's at
        those positions).  M is the capacity when `count` (device-side match count) is given."""
        P, split = self._plan, self.split
        pl = 2 if split else 1
        dev = x1_lat.device
        (w0, b0), (w1, b1) = P["layer1_outconv2.0"], P["layer1_outconv2.3"]
        t = self._buf("x1_h_win", (M, 7, 8, pl * w0.shape[0]), torch.float16, dev)
        ops.conv_win(x1_lat, w0, b0, t, 7, split, M, act=2, b_ids=b_ids, j_ids=j_ids, wc=wc, stride=stride,
                     org=-3, count=count)
        out = self._buf("x1_out_win", (M, 5, ops.conv_win_pitch(5), pl * w1.shape[0]), torch.float16, dev)
        return ops.conv_win(t, w1, b1, out, 5, split, M, count=count)

    def _windows_pay(self, M, B, hf, wf):
        """Sparse vs dense layer1_outconv2: M-tile counts weighted by the output widths (208 / 128):
        2 (3) windows per 128-row tile against hf*wf/128 tiles per image."""
        return M * (208 / 2 + 128 / 3) < 0.85 * B * (hf * wf / 128) * (208 + 128)

    def _src_state(self, L, tag, src, B, ls, src_mask=None, v_len=None):
        """Source side of linear attention for one layer (linear_attention.py:46,55-57 +
        transformer.py:78-79,85): K' = elu(Wk src)+1, V = Wv src, per-head KV / Ksum, with `merge`
        folded in -> (Mt [B, 256, pl*256] fp16, Ksum [B, 256] fp32).  v_len (default ls): the
        length the query side multiplies back by (linear_attention.py:55,61).  The K'/V rows are ONE
        fp16 plane in both operand modes: their only consumer sums them over thousands of tokens, so
        the 2^-12 rounding averages out (oracle experiment: conf changes by 1e-4)."""
        dev = src.device
        f16 = torch.float16
        split = self.split
        pl = 2 if split else 1
        kv16 = self._buf(tag + "kv16", (B * ls, 512), f16, dev)
        ops.linear_act(src, None, L["wkv"], kv16, B * ls, 2, 256, split, out_split=False,
                       row_mask=src_mask)
        part = self._buf(tag + "part", (B, ops.kv_chunks(ls, B), 8, 33, 32), torch.float32, dev)
        mt = self._buf(tag + "mt", (B, 256, pl * 256), f16, dev)
        ksum = self._buf(tag + "ksum", (B, 256), torch.float32, dev)
        ops.kv_state(kv16, part, L["merge32"], mt, ksum, B, ls, 256, ls if v_len is None else v_len, split)
        return mt, ksum

    def _encoder_layer(self, L, tag, x, src, B, lx, ls, out, x_shared=False, state=None, x_mask=None,
                       src_mask=None, state_batched=False):
        """LoFTREncoderLayer.forward (transformer.py:65-94) with linear attention
        (linear_attention.py:29-61) for d_model 256.  x, src, out: fp16 planes [B, len, pl*256].
        x_shared: x is [1, lx, ..] — one object's tokens, the same for every image of the batch.
        state = (Mt [1, ...], Ksum [B, 256]): precomputed source state shared by the batch
        (state_batched: Mt is [B, ...], one per image).
        x_mask / src_mask (uint8 [B * len]): padded positions of query_image_mask — Q rows resp.
        K', V rows are zeroed (linear_attention.py:49-53)."""
        dev = x.device
        f16 = torch.float16
        split = self.split
        pl = 2 if split else 1
        msg = self._buf(tag + "msg", (B * lx, pl * 256), f16, dev)
        if self._coarse_attention == "full":
            # FullAttention (linear_attention.py:64-95): q/k/v projections, softmax(QK^T/sqrt(D))V per
            # head, merge + LayerNorm (transformer.py:77-86).  Cold path (no shipped config).
            if x_mask is not None or src_mask is not None:
                raise NotImplementedError("query_image_mask with attention='full' is not built")
            q16 = self._buf(tag + "qz", (B * lx, pl * 256), f16, dev)
            ops.linear_act(x, None, L["wq"], q16, lx if x_shared else B * lx, 0, 0, split,
                           batches=B if x_shared else 1, a0_shared=x_shared)
            kv16 = self._buf(tag + "kv16", (B * ls, pl * 512), f16, dev)
            ops.linear_act(src, None, L["wkv"], kv16, B * ls, 0, 0, split)
            att = self._buf(tag + "att", (B * lx, pl * 256), f16, dev)
            ops.full_attention(q16, kv16, att, B, lx, ls, 8, 32, split)
            ops.linear_ln(att, None, L["merge16"], False, *L["n1"], 1, B * lx, split, out16=msg)
        else:
            if state is None:
                mt, ksum = self._src_state(L, tag, src, B, ls, src_mask)
                mt_batched = True
            else:
                mt, ksum = state
                mt_batched = state_batched
            qz = self._buf(tag + "qz", (B * lx, pl * 256), f16, dev)
            ops.linear_q(x, L["wq"], ksum, qz, B, lx, ls, split, x_shared=x_shared, row_mask=x_mask)
            ops.linear_ln(qz, None, mt, mt_batched, *L["n1"], B, lx, split, out16=msg)
        h = self._buf(tag + "h", (B * lx, pl * 512), f16, dev)
        if x_shared:
            ops.linear_act(x, msg, L["mlp0"], h, lx, 1, 512, split, batches=B, a0_shared=True)
            ops.linear_ln(h, None, L["mlp2"], False, *L["n2"], B, lx, split, resid=x, out16=out,
                          resid_shared=True)
        else:
            ops.linear_act(x, msg, L["mlp0"], h, B * lx, 1, 512, split)
            ops.linear_ln(h, None, L["mlp2"], False, *L["n2"], 1, B * lx, split, resid=x, out16=out)


class OnePosePlus_model(_Engine):
    def __init__(self, config, profiler=None, debug=False, precision=None):
        """`precision` (extension; default from $OPP_B200_PRECISION or "fp16x3"):
        "fp16x3" = 2-term fp16 split operands, three wgmma MMAs per K-step (fp32-grade, the
        parity mode); "fp16" = single fp16 operands (fast, ~1e-2 deviations on high-gain inputs)."""
        super().__init__()
        self.config = config
        self.profiler = profiler
        self.debug = debug
        self._init_engine(precision, config["loftr_coarse"]["attention"])
        self.backbone = build_backbone(config["loftr_backbone"])
        if config["positional_encoding"]["enable"]:
            self.dense_pos_encoding = PositionEncodingSine(
                config["loftr_coarse"]["d_model"],
                max_shape=config["positional_encoding"]["pos_emb_shape"])
        else:
            self.dense_pos_encoding = None
        if config["keypoints_encoding"]["enable"]:
            if config["keypoints_encoding"]["type"] != "mlp_linear":
                raise NotImplementedError
            self.kpt_3d_pos_encoding = KeypointEncoding_linear(
                inp_dim=3, feature_dim=config["keypoints_encoding"]["descriptor_dim"],
                layers=config["keypoints_encoding"]["keypoints_encoder"],
                norm_method=config["keypoints_encoding"]["norm_method"])
        else:
            raise NotImplementedError("keypoints_encoding.enable=False is not built")
        self.loftr_coarse = LocalFeatureTransformer(config["loftr_coarse"])
        self.coarse_matching = CoarseMatching(config["coarse_matching"], profiler=profiler)
        self.fine_preprocess = FinePreprocess(config["loftr_fine"],
                                              cf_res=config["loftr_backbone"]["resolution"])
        self.loftr_fine = LocalFeatureTransformer(config["loftr_fine"])
        self.fine_matching = FineMatching(config["fine_matching"])
        if config["loftr_coarse"]["d_model"] != 256 or config["loftr_coarse"]["nhead"] != 8:
            raise NotImplementedError("coarse kernels are built for d_model 256, 8 heads")
        if config["loftr_fine"]["d_model"] != 128 or config["loftr_fine"]["nhead"] != 8:
            raise NotImplementedError("fine kernels are built for d_model 128, 8 heads")
        if config["loftr_fine"]["attention"] != "linear":
            raise NotImplementedError("the fine-level kernels implement attention='linear' (every shipped "
                                      "config); 'full' is built for the coarse transformer only")
        if config["loftr_fine"]["window_size"] != 5:
            raise NotImplementedError("fine kernels are built for window_size 5")
        b = config["loftr_backbone"]["resnetfpn"]
        if list(b["block_dims"]) != [128, 196, 256] or b["initial_dim"] != 128 \
                or list(b["output_layers"]) != [3, 1]:
            raise NotImplementedError("backbone kernels are built for dims 128/[128,196,256], outputs [3,1]")

        self.loftr_backbone_pretrained = config["loftr_backbone"]["pretrained"]
        if self.loftr_backbone_pretrained is not None:
            # OnePosePlusModel.py:79-94: initialise the backbone from a LoFTR checkpoint
            ckpt = torch.load(self.loftr_backbone_pretrained, "cpu")["state_dict"]
            for k in list(ckpt.keys()):
                if "backbone" in k:
                    ckpt[k[k.find("backbone") + len("backbone") + 1:]] = ckpt[k]
                ckpt.pop(k)
            self.backbone.load_state_dict(ckpt)
            if config["loftr_backbone"]["pretrained_fix"]:
                for p in self.backbone.parameters():
                    p.requires_grad = False
        self._bank = None
        self._bank_set = None
        self._side_stream = None
        self._fwd_count = 0
        self.use_cuda_graphs = os.environ.get("OPP_B200_GRAPHS", "0") == "1"
        # data["conf_matrix"]: "eager" = fp32 [B, N, S] written every forward (reference contract,
        # coarse_matching.py:119; what the training loss reads); "lazy" = a LazyConfMatrix handle
        # that materialises on demand (no inference consumer reads the matrix:
        # inference_OnePosePlus_worker.py:20-31); "skip" = key not written.
        self.conf_matrix_mode = os.environ.get("OPP_B200_CONF", "eager")
        # fine level of .train() on CUDA: "autograd" = train_path's PyTorch functions, "kernels" = the
        # opp_fine_train_* kernels forward and backward (train_fine.py; no unfold tensor)
        self.fine_train_mode = os.environ.get("OPP_B200_FINE_TRAIN", "autograd")
        # coarse transformer of .train() on CUDA: "autograd" = train_path.transformer, "kernels" = the
        # opp_coarse_tf_* kernels forward and backward, recomputing one layer at a time (train_coarse_tf.py)
        self.coarse_transformer_train_mode = os.environ.get("OPP_B200_COARSE_TF_TRAIN", "autograd")
        # backbone of .train() on CUDA: "autograd" = train_path.backbone (cuDNN), "kernels" = the
        # opp_backbone_train_* kernels forward and backward (convolutions on the tensor cores in 3xTF32),
        # recomputing one segment at a time (train_backbone.py)
        self.backbone_train_mode = os.environ.get("OPP_B200_BACKBONE_TRAIN", "autograd")
        # keypoint encoder of .train() on CUDA: "autograd" = train_path.keypoint_encoding, "kernels" = the
        # opp_kpt_train_* kernels forward and backward, recomputing each point's MLP (train_kpt.py)
        self.kpt_encoder_train_mode = os.environ.get("OPP_B200_KPT_TRAIN", "autograd")
        # layer1_outconv2 (the last two 3x3 convolutions of the FPN, 1/2 resolution) evaluated only on
        # the 5x5 windows the fine stage reads: "auto" = when cheaper than the dense map (by the
        # match count), "sparse" / "dense" = always / never
        self.fine_windows = os.environ.get("OPP_B200_FINE_WINDOWS", "auto")

    # read-only, reported by bench.py: coarse matching is always the one-pass dual softmax
    @property
    def coarse_colmax(self):
        return True

    @property
    def coarse_lse_cols(self):
        return True

    # pickling (Ray ships the module object): drop device-side caches
    def __getstate__(self):
        st = self.__dict__.copy()
        st["_plan"], st["_plan_sig"], st["_ws"], st["_sig_tensors"] = None, None, {}, None
        st["_bank"], st["_graphs"], st["_side_stream"] = None, {}, None
        st["_bank_set"] = None
        st.pop("_aux", None)
        st.pop("_aux_fpn", None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        for k, v in (("_sig_tensors", None), ("_apply_epoch", 0), ("_ws_epoch", 0), ("_bank", None),
                     ("_bank_set", None),
                     ("_graphs", {}), ("_fwd_count", 0), ("use_cuda_graphs", False), ("_side_stream", None),
                     ("fine_windows", "auto")):
            self.__dict__.setdefault(k, v)

    # ------------------------------------------------------------------ descriptor bank
    def _encode_bank(self, kpts, dcoarse, dfine, persistent, l1_v_len=None):
        """Image-independent part of the forward for one descriptor bank (SURVEY §8e/f2): keypoint
        normalisation + encoding (normalize.py:16-26, position_encoding.py:54-60) and — when the
        bank is ONE object ([1, N, .]) and the coarse transformer starts with (self, cross) — the
        3D side of the first self layer plus the 3D-as-source attention state of the first cross
        layer (transformer.py:148-159: both read only 3D tokens).  l1_v_len: the v_len that layer-1
        state is divided by (default N; a bank set pads to N_max and its forward queries with N_max)."""
        dev = kpts.device
        f16 = torch.float16
        pl = 2 if self.split else 1
        Bb, N = kpts.shape[:2]
        alloc = (lambda name, shape, dt: torch.empty(shape, dtype=dt, device=dev)) if persistent else \
            (lambda name, shape, dt: self._buf("bank_" + name, shape, dt, dev))
        st = {"Bb": Bb, "N": N, "kpts": kpts, "fine": dfine, "sig": self._plan_sig}
        d3 = alloc("d3_in", (Bb, N, pl * 256), f16)
        ops.kpt_encode(kpts, dcoarse, self._plan["kpt_mlp"], alloc("stats", (Bb, 4), torch.float32), d3,
                       self.split)
        st["d3_in"] = d3
        names = self.loftr_coarse.layer_names
        linear = self.config["loftr_coarse"]["attention"] == "linear"
        if Bb == 1 and linear and len(names) >= 2 and names[0] == "self" and names[1] == "cross":
            d3_l0 = alloc("d3_l0", (1, N, pl * 256), f16)
            self._encoder_layer(self._plan["coarse"][0], "c3s_", d3, d3, 1, N, N, d3_l0)
            mt, ksum = self._src_state(self._plan["coarse"][1], "c3s_", d3_l0, 1, N, v_len=l1_v_len)
            st["d3_l0"] = d3_l0
            st["l1_mt"] = alloc("l1_mt", mt.shape, f16).copy_(mt)
            st["l1_ksum"] = alloc("l1_ksum", ksum.shape, torch.float32).copy_(ksum)
        return st

    def set_bank(self, keypoints3d, descriptors3d_db, descriptors3d_coarse_db=None):
        """Make one object's descriptor bank resident on the model's device (extension; the
        reference re-uploads the bank with every frame: inference_OnePosePlus_worker.py:54-56, and
        only `preload`s it in demo mode: OnePosePlus_inference_dataset.py:58-59).  Shapes as in the
        reference data dict with a leading 1 (or none): keypoints3d [1, N, 3], descriptors3d_db
        [1, 128, N], descriptors3d_coarse_db [1, 256, N].  Afterwards `forward(data)` uses this bank
        whenever `data` carries no "keypoints3d"; the keypoint encoding, the 3D side of the first
        self layer and the 3D source state of the first cross layer are computed once per object."""
        self._bank = {"raw": self._prep_bank(keypoints3d, descriptors3d_db, descriptors3d_coarse_db),
                      "state": None}
        self._bank_set = None
        return self

    def _prep_bank(self, keypoints3d, descriptors3d_db, descriptors3d_coarse_db=None):
        """One object's bank on the model's device: (kpts [1,N,3], coarse [1,256,N], fine [1,128,N]) fp32."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("set_bank: move the model to a CUDA device first (there is no CPU path)")

        def prep(t):
            t = torch.as_tensor(t)
            if t.dim() == 2:
                t = t[None]
            if t.dim() != 3 or t.shape[0] != 1:
                raise ValueError(f"set_bank expects ONE object ([1, ...] tensors), got {tuple(t.shape)}")
            return t.to(device=dev, dtype=torch.float32).contiguous()

        kp = prep(keypoints3d)
        fine = prep(descriptors3d_db)
        coarse = prep(descriptors3d_coarse_db) if descriptors3d_coarse_db is not None else fine
        N = kp.shape[1]
        if kp.shape[2] != 3 or fine.shape[2] != N or coarse.shape[2] != N or coarse.shape[1] != 256:
            raise ValueError("set_bank: expected keypoints3d [1,N,3], descriptors3d_db [1,128,N], "
                             f"descriptors3d_coarse_db [1,256,N]; got {tuple(kp.shape)}, {tuple(fine.shape)}, "
                             f"{tuple(coarse.shape)}")
        return kp, coarse, fine

    def set_banks(self, banks):
        """Make a SET of K objects' descriptor banks resident (extension with no counterpart in the
        reference, which matches every frame of a batch against one object).  `banks`: a list of K
        (keypoints3d, descriptors3d_db, descriptors3d_coarse_db=None) tuples shaped as for
        set_bank; the point counts N_k may differ.  Afterwards `forward(data)` reads
        data["object_ids"] (int [B], entries in [0, K); CPU avoids a read-back: a CUDA tensor is
        copied to the host to be validated before any launch) and matches frame b against
        object object_ids[b]: every output equals that of set_bank(*banks[object_ids[b]]) and a
        forward of frame b alone (each object's keypoints normalised by its own extents), with the
        frames' matches in the usual ascending (b, i) order; i_ids index the frame's own object and
        mkpts_3d_db come from it.  conf_matrix is [B, N_max, S] with rows >= N_k of a frame exactly 0.
        Replaces a bank of set_bank; clear_bank() drops both.  Not built: query_image_mask with a
        set (NotImplementedError) and training (train() raises while a set is resident)."""
        names = self.loftr_coarse.layer_names
        if self.config["loftr_coarse"]["attention"] != "linear" or names[:2] != ["self", "cross"]:
            raise NotImplementedError("bank sets are built for linear coarse attention starting with (self, cross)")
        if self.training:
            raise NotImplementedError("bank sets are built for inference: call eval() first")
        banks = list(banks)
        if not banks:
            raise ValueError("set_banks: empty list of banks")
        raw = []
        for bk in banks:
            if not isinstance(bk, (tuple, list)) or len(bk) not in (2, 3):
                raise ValueError("set_banks: every bank is (keypoints3d, descriptors3d_db[, descriptors3d_coarse_db])")
            raw.append(self._prep_bank(*bk))
            if raw[-1][0].shape[1] < 1:
                raise ValueError("set_banks: an object without keypoints")
        if len({r[2].shape[1] for r in raw}) != 1:
            raise ValueError("set_banks: descriptors3d_db channel counts differ between objects")
        self._bank = None
        self._bank_set = {"raw": raw, "state": None}
        return self

    def clear_bank(self):
        self._bank = None
        self._bank_set = None

    def train(self, mode=True):
        if mode and getattr(self, "_bank_set", None) is not None:
            raise NotImplementedError("training with a resident bank set is not built: clear_bank() first")
        return super().train(mode)

    def _resident_bank_state(self):
        b = self._bank
        if b["state"] is None or b["state"]["sig"] != self._plan_sig:
            b["state"] = self._encode_bank(*b["raw"], persistent=True)
        return b["state"]

    def _encode_bank_set(self, raw):
        """Image-independent state of a bank set: every object encoded once, unpadded, by the
        one-object code (_encode_bank: its own keypoint extents, the first (self, cross) cache), then
        stored padded to N_max = max N_k.  Rows >= n_rows[k] of kpts / d3_l0 and columns >= n_rows[k]
        of fine are padding: the forward masks them (row_mask, row_count) and no output reads them,
        whatever they hold."""
        dev = raw[0][0].device
        n = [r[0].shape[1] for r in raw]
        K, Nm = len(raw), max(n)
        pl = 2 if self.split else 1
        st = {"K": K, "N": Nm, "sig": self._plan_sig,
              "kpts": torch.zeros(K, Nm, 3, device=dev),
              "fine": torch.zeros(K, raw[0][2].shape[1], Nm, device=dev),
              "d3_l0": torch.zeros(K, Nm, pl * 256, dtype=torch.float16, device=dev),
              "l1_mt": torch.empty(K, 256, pl * 256, dtype=torch.float16, device=dev),
              "l1_ksum": torch.empty(K, 256, dtype=torch.float32, device=dev),
              "n_rows": torch.tensor(n, dtype=torch.int32, device=dev),
              "rows": torch.arange(Nm, dtype=torch.int32, device=dev)}
        for k, (kp, coarse, fine) in enumerate(raw):
            # the forward's layer-1 query multiplies by v_len = N_max (_coarse_transformer), so the
            # cached state divides by N_max: KV/N_max * N_max is the one-object KV/N_k * N_k
            one = self._encode_bank(kp, coarse, fine, persistent=False, l1_v_len=Nm)
            st["kpts"][k, :n[k]] = kp[0]
            st["fine"][k, :, :n[k]] = fine[0]
            st["d3_l0"][k, :n[k]] = one["d3_l0"][0]
            st["l1_mt"][k] = one["l1_mt"][0]
            st["l1_ksum"][k] = one["l1_ksum"][0]
        return st

    def _resident_set_state(self):
        s = self._bank_set
        if s["state"] is None or s["state"]["sig"] != self._plan_sig:
            s["state"] = self._encode_bank_set(s["raw"])
        return s["state"]

    def _set_frame_state(self, oid, B):
        """The bank state of a forward with a bank set: per-frame copies of the cached first-layer
        state (index_select on the device-side object ids, so a CUDA graph captures the gather and
        serves every assignment of objects to frames), the frames' row counts and the uint8 row
        mask [B * N_max] (0 on padding).  kpts / fine stay [K, ...] and are read through
        bank_of_batch."""
        st = self._resident_set_state()
        dev, Nm = oid.device, st["N"]

        def gather(name, src):
            return torch.index_select(src, 0, oid, out=self._buf(name, (B,) + tuple(src.shape[1:]), src.dtype, dev))

        n_b = gather("set_n_rows", st["n_rows"])
        mask = self._buf("set_row_mask", (B, Nm), torch.bool, dev)
        torch.lt(st["rows"][None], n_b[:, None], out=mask)
        return {"Bb": B, "N": Nm, "kpts": st["kpts"], "fine": st["fine"],
                "d3_l0": gather("set_d3_l0", st["d3_l0"]), "l1_mt": gather("set_l1_mt", st["l1_mt"]),
                "l1_ksum": gather("set_l1_ksum", st["l1_ksum"]), "row_count": n_b,
                "row_mask": mask.view(torch.uint8).view(-1), "bank_of_batch": oid}

    def _coarse_transformer(self, q2, bank, B, S, N, qmask=None):
        """LocalFeatureTransformer.forward (transformer.py:133-171): self layers update each
        sequence from itself; cross layers update BOTH from the pre-update tensors.  `bank` is the
        state of _encode_bank; with one shared object the 3D work of the first (self, cross) pair
        that does not depend on the image comes from it.  qmask (uint8 [B*S]) = query_image_mask:
        it masks the 2D side only (transformer.py:150-159)."""
        dev = q2.device
        f16 = torch.float16
        pl = 2 if self.split else 1
        names = self.loftr_coarse.layer_names
        shared = bank["Bb"] == 1 and B > 1
        cur2, cur3 = q2, bank.get("d3_in")
        # bank set (_set_frame_state): uint8 [B*N], 0 on the padding of each frame's object.  As a
        # source its K'/V rows are zero, as a query its rows stay finite; v_len = N (padded) cancels
        # between the KV state (/v_len) and the query (*v_len), the cached layer-1 state included
        # (_encode_bank_set builds it with v_len = N)
        rmask = bank.get("row_mask")
        first = 0
        both = self._both
        if "d3_l0" in bank:
            # layer 0 (self): 2D side only; layer 1 (cross): the 2D side reads the cached 3D source
            # state, the 3D side reads the shared 3D tokens in place (no per-image copies)
            L0, L1 = self._plan["coarse"][0], self._plan["coarse"][1]
            o2 = self._buf("q2_1", (B, S, pl * 256), f16, dev)
            self._encoder_layer(L0, "c2_", cur2, cur2, B, S, S, o2, x_mask=qmask, src_mask=qmask)
            d3 = bank["d3_l0"]
            if rmask is None:
                ksum_b = self._buf("l1_ksum_b", (B, 256), torch.float32, dev)
                ksum_b.copy_(bank["l1_ksum"].expand(B, -1))
                state = (bank["l1_mt"], ksum_b)
            else:   # bank set: per-frame states and tokens, gathered already
                state = (bank["l1_mt"], bank["l1_ksum"])
            o2b = self._buf("q2_0", (B, S, pl * 256), f16, dev)
            o3 = self._buf("d3_0", (B, N, pl * 256), f16, dev)
            both(lambda: self._encoder_layer(L1, "c2_", o2, None, B, S, N, o2b, state=state, x_mask=qmask,
                                             state_batched=rmask is not None),
                 lambda: self._encoder_layer(L1, "c3_", d3, o2, B, N, S, o3, x_shared=rmask is None, src_mask=qmask,
                                             x_mask=rmask))
            cur2, cur3 = o2b, o3
            first = 2
        elif shared:
            cur3 = self._buf("d3_0", (B, N, pl * 256), f16, dev)
            cur3.copy_(bank["d3_in"].expand(B, -1, -1))
        for i in range(first, len(names)):
            L = self._plan["coarse"][i]
            nxt = (i + 1) % 2
            o2 = self._buf(f"q2_{nxt}", (B, S, pl * 256), f16, dev)
            o3 = self._buf(f"d3_{nxt}", (B, N, pl * 256), f16, dev)
            self_layer = names[i] == "self"
            both(lambda: self._encoder_layer(L, "c2_", cur2, cur2 if self_layer else cur3, B, S,
                                             S if self_layer else N, o2, x_mask=qmask,
                                             src_mask=qmask if self_layer else rmask),
                 lambda: self._encoder_layer(L, "c3_", cur3, cur3 if self_layer else cur2, B, N,
                                             N if self_layer else S, o3, x_mask=rmask,
                                             src_mask=rmask if self_layer else qmask))
            cur2, cur3 = o2, o3
        return cur2, cur3

    def _both(self, f2, f3):
        """The 2D-side and the 3D-side update of a layer are independent (cross layers read the
        pre-update tensors, transformer.py:154-159).  At small batches each persistent GEMM fills a
        fraction of the 132 SMs, so in latency (CUDA-graph) mode the two sides are enqueued on two
        streams and run side by side; otherwise one after the other."""
        side = self._side_stream
        if side is None:
            f2()
            f3()
            return
        cur = torch.cuda.current_stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            f3()
        f2()
        cur.wait_stream(side)

    def _coarse_matching(self, q2, d3, bank, img_scale, B, N, hc, wc, cell, out, qmask=None, pack=None, side=None):
        """CoarseMatching.forward + get_coarse_match (coarse_matching.py:76-242), inference branch.
        Enqueues everything up to the ordered match lists (capacity B*N) and the device-side
        match count; nothing here synchronises.  Fills `out` with the full-capacity tensors."""
        dev = q2.device
        S = hc * wc
        f32, i32 = torch.float32, torch.int32
        split = self.split
        cm = self.coarse_matching
        scale = 1.0 / (256.0 * (cm.temperature + 1e-4))  # (a/16).(b/16)/(T+1e-4)
        ts = ops.sim_tiles(S)
        pm_pt = self._buf("pm_pt", (B * N, ts), f32, dev)
        ps_pt = self._buf("ps_pt", (B * N, ts), f32, dev)
        lse_pt = self._buf("lse_pt", (B, N), f32, dev)
        lse_px = self._buf("lse_px", (B, S), f32, dev)
        # bank set: rows >= row_count[b] are the padding of frame b's object
        rows_b, bank_of_batch = bank.get("row_count"), bank.get("bank_of_batch")
        groups = (N + 31) // 32
        col_m = self._buf("lse_col_m", (B, groups, S), f32, dev)
        col_s = self._buf("lse_col_s", (B, groups, S), f32, dev)
        ops.sim_lse_cols(d3, q2, B, N, S, 256, scale, pm_pt, ps_pt, lse_pt, col_m, col_s, lse_px, split,
                         col_mask=qmask, side_stream=side, row_count=rows_b)
        mode = self.conf_matrix_mode
        conf = torch.empty((B, N, S), dtype=f32, device=dev) if mode == "eager" else None  # caller's
        pi_pt = self._buf("pi_pt", (B * N, ts), i32, dev)
        pt_val = self._buf("pt_val", (B, N), f32, dev)
        pt_idx = self._buf("pt_idx", (B, N), i32, dev)
        # capacity: one match per 3D point; the value-based mutual test keeps every row of an exact
        # tie (as the reference's mask does), so a query cell can match more than one point
        cap = B * N
        scratch = self._buf("match_scratch", ((B * N + 1023) // 1024 + 2,), i32, dev)
        count = self._buf("match_count", (1,), i32, dev)
        new = pack.new if pack is not None else (
            lambda key, shape, dtype: torch.empty(shape, dtype=dtype, device=dev))
        b_ids = new("b_ids", (cap,), torch.int64)
        i_ids = new("i_ids", (cap,), torch.int64)
        j_ids = new("j_ids", (cap,), torch.int64)
        mconf = new("mconf", (cap,), f32)
        mk3 = new("mkpts_3d_db", (cap, 3), f32)
        mkc = new("mkpts_query_c", (cap, 2), f32)
        colmax = self._buf("colmax", (B, S), i32, dev)
        ops.sim_conf_colmax(d3, q2, lse_pt, lse_px, conf, B, N, S, 256, scale, pm_pt, pi_pt,
                            pt_val, pt_idx, colmax, split, row_count=rows_b)
        ops.match_select_colmax(pt_val, pt_idx, colmax, bank["kpts"], img_scale, B, N, hc, wc,
                                cm.thr, cm.border_rm, cell, scratch, b_ids, i_ids, j_ids, mconf,
                                mk3, mkc, count, bank_shared=bank["Bb"] == 1, bank_of_batch=bank_of_batch,
                                row_count=rows_b)
        if mode == "lazy":
            conf = LazyConfMatrix(self, d3, q2, lse_pt, lse_px, B, N, S, scale, rows_b)
        out.update({"conf_matrix": conf, "b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids, "mconf": mconf,
                    "mkpts_3d_db": mk3, "mkpts_query_c": mkc})
        return count, cap

    def _materialize_conf(self, d3, q2, lse_pt, lse_px, B, N, S, scale, rows_b=None):
        """conf_matrix on demand (LazyConfMatrix): re-runs the conf pass of the forward with the fp32
        store (for a bank set it stores 0 on the padded rows); its row and column maxima go to scratch."""
        dev = q2.device
        ts = ops.sim_tiles(S)
        conf = torch.empty((B, N, S), dtype=torch.float32, device=dev)
        part = (self._buf("lz_pv", (B * N, ts), torch.float32, dev), self._buf("lz_pi", (B * N, ts), torch.int32, dev),
                self._buf("lz_bv", (B, N), torch.float32, dev), self._buf("lz_bi", (B, N), torch.int32, dev))
        ops.sim_conf_colmax(d3, q2, lse_pt, lse_px, conf, B, N, S, 256, scale, *part,
                            self._buf("lz_colmax", (B, S), torch.int32, dev), self.split, row_count=rows_b)
        return conf

    def _fine(self, fine_map, bank, ids, M, img_scale, hc, wc, q_hw_i, out, count=None, pack=None, windows_hw=None):
        """FinePreprocess (fine_preprocess.py:32-55) -> loftr_fine -> FineMatching
        (fine_matching.py:28-110) on the first M entries of the match lists.  With `count` (the
        device-side match counter) M is only the CAPACITY: every kernel reads the real number of
        matches on the device, so nothing here needs the host to know it."""
        dev = fine_map.device
        f16, f32 = torch.float16, torch.float32
        split = self.split
        pl = 2 if split else 1
        if windows_hw is None:
            B, hf, wf, _ = fine_map.shape
        else:
            hf, wf = windows_hw     # fine_map = compact windows of _fine_head_windows
        stride = hf // hc
        rows = 26 * M
        x = [self._buf(f"fx{k}", (rows, pl * 128), f16, dev) for k in range(2)]
        x32 = self._buf("fx32", (rows, 128), f32, dev)
        fine_layers = self.loftr_fine.layer_names if self.config["loftr_fine"]["enable"] else []
        b_ids, i_ids, j_ids, mkc = ids
        dyn = {} if count is None else {"count": count}
        dyn26 = {} if count is None else {"count": count, "rows_per_count": 26}
        ops.fine_gather(fine_map, bank["fine"], b_ids, i_ids, j_ids, None if fine_layers else x32, x[0], M,
                        hf, wf, wc, stride, bank["N"], split, bank_shared=bank["Bb"] == 1,
                        windows=windows_hw is not None, bank_of_batch=bank.get("bank_of_batch"), **dyn)
        cur = 0
        if fine_layers:
            qkv = self._buf("f_qkv", (rows, pl * 384), f16, dev)
            att = self._buf("f_att", (rows, pl * 128), f16, dev)
            msg = self._buf("f_msg", (rows, pl * 128), f16, dev)
            h = self._buf("f_h", (rows, pl * 256), f16, dev)
            for i, name in enumerate(fine_layers):
                L = self._plan["fine"][i]
                last = i == len(fine_layers) - 1
                ops.linear_act(x[cur], None, L["wqkv"], qkv, rows, 2, 256, split, **dyn26)
                ops.fine_attention(qkv, att, M, name == "cross", split, **dyn)
                ops.linear_ln(att, None, L["merge16"], False, *L["n1"], 1, rows, split, out16=msg, **dyn26)
                ops.linear_act(x[cur], msg, L["mlp0"], h, rows, 1, 256, split, **dyn26)
                ops.linear_ln(h, None, L["mlp2"], False, *L["n2"], 1, rows, split, resid=x[cur],
                              out16=None if last else x[1 - cur], out32=x32 if last else None, **dyn26)
                cur = 1 - cur
        if pack is not None:
            expec_f, mkpts_f = pack.new("expec_f", (M, 3), f32), pack.new("mkpts_query_f", (M, 2), f32)
        else:
            expec_f = torch.empty((M, 3), dtype=f32, device=dev)
            mkpts_f = torch.empty((M, 2), dtype=f32, device=dev)
        fine_scale = float(q_hw_i[0] / hf)
        ops.fine_match(x32, mkc, b_ids, img_scale, expec_f, mkpts_f, M, fine_scale, **dyn)
        out.update({"expec_f": expec_f, "mkpts_query_f": mkpts_f})

    # ------------------------------------------------------------------ input checks
    def _check_inputs(self, data):
        """Shape / dtype validation of the reference data dict (the kernels index raw pointers:
        a wrong batch or point count would read out of bounds instead of raising like PyTorch)."""
        img = data["query_image"]
        if not torch.is_tensor(img) or not img.is_cuda:
            raise RuntimeError("OnePosePlus_model has no CPU path: move the model and data to "
                               "a CUDA device")
        if img.dim() != 4 or img.shape[1] != 1:
            raise ValueError(f"query_image must be [B, 1, H, W], got {tuple(img.shape)}")
        if img.dtype != torch.uint8 and not img.is_floating_point():
            raise TypeError(f"query_image must be floating point in [0, 1] or uint8, got {img.dtype}")
        B, _, H, W = img.shape
        if H % 8 or W % 8 or H < 16 or W < 16:
            raise ValueError("query_image height/width must be multiples of 8 (>= 16)")
        if self.dense_pos_encoding is not None:
            mh, mw = self.dense_pos_encoding.pe.shape[2:]
            if H // 8 > mh or W // 8 > mw:
                raise ValueError(f"image {H}x{W} exceeds positional_encoding.pos_emb_shape {mh}x{mw} (x8)")
        scale = data.get("query_image_scale")
        if scale is not None and tuple(scale.shape) != (B, 2):
            raise ValueError(f"query_image_scale must be [B, 2] = [{B}, 2], got {tuple(scale.shape)}")
        if self._bank_set is not None:
            given = [k for k in ("keypoints3d", "descriptors3d_db", "descriptors3d_coarse_db") if k in data]
            if given:
                raise ValueError(f"a bank set is resident (set_banks): data must not carry {given}")
        if "keypoints3d" not in data:
            if self._bank is None and self._bank_set is None:
                raise KeyError("data has no 'keypoints3d' and no bank is resident (set_bank)")
            return img, scale, None
        kp, dfine = data["keypoints3d"], data["descriptors3d_db"]
        dco = data["descriptors3d_coarse_db"] if "descriptors3d_coarse_db" in data else dfine
        if kp.dim() != 3 or kp.shape[2] != 3:
            raise ValueError(f"keypoints3d must be [B, N, 3], got {tuple(kp.shape)}")
        N = kp.shape[1]
        if N < 1:
            raise ValueError("keypoints3d is empty")
        for name, t, c in (("descriptors3d_db", dfine, 128 if self.config["fine_matching"]["enable"] else None),
                           ("descriptors3d_coarse_db", dco, 256)):
            if t.dim() != 3 or t.shape[2] != N or (c is not None and t.shape[1] != c):
                raise ValueError(f"{name} must be [B, {c}, N={N}], got {tuple(t.shape)}")
        for name, t in (("keypoints3d", kp), ("descriptors3d_db", dfine), ("descriptors3d_coarse_db", dco)):
            if t.shape[0] not in (1, B):
                raise ValueError(f"{name} has batch {t.shape[0]}, query_image has batch {B}")
            if not t.is_cuda or t.device != img.device:
                raise RuntimeError(f"{name} must be on the same CUDA device as query_image")
        if len({kp.shape[0], dfine.shape[0], dco.shape[0]}) != 1:
            raise ValueError("keypoints3d / descriptors3d_db / descriptors3d_coarse_db disagree on the batch size")
        return img, scale, (kp, dco, dfine)

    def _check_object_ids(self, data, B):
        """data["object_ids"] of a forward with a bank set, validated on the host (a CUDA tensor is
        read back once): int [B], entries in [0, K).  Returns it as int32 on the host, or None
        without a bank set."""
        oid = data.get("object_ids")
        if self._bank_set is None:
            if oid is not None:
                raise ValueError("data has 'object_ids' but no bank set is resident (set_banks)")
            return None
        if oid is None:
            raise ValueError("a bank set is resident (set_banks): data needs 'object_ids' (int [B])")
        oid = torch.as_tensor(oid)
        if oid.dtype not in (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64):
            raise ValueError(f"object_ids must be an integer tensor, got {oid.dtype}")
        if tuple(oid.shape) != (B,):
            raise ValueError(f"object_ids must be [B] = [{B}], got {tuple(oid.shape)}")
        oid = oid.cpu()
        K = len(self._bank_set["raw"])
        if int(oid.min()) < 0 or int(oid.max()) >= K:
            raise ValueError(f"object_ids entries must be in [0, {K}), got {oid.tolist()}")
        return oid.to(torch.int32)

    # ------------------------------------------------------------------ forward
    def forward(self, data):
        """Same contract as the reference (OnePosePlusModel.py:96-201): reads query_image,
        keypoints3d, descriptors3d_db, descriptors3d_coarse_db (optional), query_image_scale
        (optional); writes bs, q_hw_i, q_hw_c, q_hw_f, conf_matrix, b_ids, i_ids, j_ids, gt_mask,
        m_bids, mkpts_3d_db, mkpts_query_c, mconf, W, expec_f, mkpts_query_f; returns None.
        Extensions: query_image may be uint8 (x/255 folded into conv1); the bank keys may be
        absent after set_bank(); a bank given as [1, N, .] tensors or stride-0 expanded views is
        encoded once for the whole batch."""
        if self.training:
            # train_onepose_plus.py: differentiable PyTorch path on the same parameters (the CUDA
            # kernels implement the inference forward only) — see train_path.py
            from . import train_path
            return train_path.forward_train(self, data)
        return self._forward(data)

    def _forward(self, data, prologue=None):
        """forward(data); `prologue` (tracking.py) produces query_image on the device first: its
        `inputs` (tensors, host or device) are copied to the device and `run(inputs, query_image)`
        enqueues the kernels that write the image — in CUDA-graph mode inside the same graph, with
        `key` added to the graph's signature."""
        img, img_scale, bank_raw = self._check_inputs(data)
        oid = self._check_object_ids(data, img.shape[0])
        if prologue is not None and (img.dtype != torch.uint8 or not img.is_contiguous()):
            raise ValueError("a prologue writes query_image in place: it must be a contiguous uint8 tensor")
        qmask = data.get("query_image_mask")
        if qmask is not None and oid is not None:
            raise NotImplementedError("query_image_mask together with a bank set is not built")
        if qmask is not None:
            # OnePosePlusModel.py:158: mask at coarse resolution, flattened to [B, S]; nonzero = valid
            B_, H_, W_ = img.shape[0], img.shape[2], img.shape[3]
            if qmask.numel() != B_ * (H_ // 8) * (W_ // 8) or qmask.shape[0] != B_:
                raise ValueError(f"query_image_mask must be [B, H/8, W/8] = [{B_}, {H_ // 8}, {W_ // 8}], "
                                 f"got {tuple(qmask.shape)}")
            qmask = (qmask.to(img.device) != 0).to(torch.uint8).reshape(-1).contiguous()
        self._fwd_count += 1
        # kernels are enqueued on the current stream of the tensors' device
        # (switching the current device costs two driver calls per forward: only when it is not current)
        on_dev = contextlib.nullcontext() if torch.cuda.current_device() == img.device.index else torch.cuda.device(img.device)
        with torch.no_grad(), on_dev:
            dev = img.device
            self._ensure_plan(dev)
            if img.dtype != torch.uint8 and img.dtype != torch.float32:
                img = img.float()
            img = img.contiguous()
            if img_scale is not None:
                img_scale = img_scale.to(device=dev, dtype=torch.float32).contiguous()
            if oid is not None:   # pinned: the upload does not wait for the stream
                oid = oid.pin_memory().to(dev, non_blocking=True)
            B, _, H, W = img.shape
            fine_on = self.config["fine_matching"]["enable"]
            data.update({"bs": B, "q_hw_i": img.shape[2:], "q_hw_c": torch.Size((H // 8, W // 8)),
                         "q_hw_f": torch.Size((H // 2, W // 2))})
            if fine_on:
                data["W"] = self.fine_preprocess.W   # fine_preprocess.py:33 (not reached when disabled)
            if self.use_cuda_graphs:
                if qmask is not None:
                    raise NotImplementedError("query_image_mask is not supported in CUDA-graph mode")
                out, M = self._replay(img, img_scale, bank_raw, fine_on, prologue, oid=oid)
                if out is None:
                    # more matches than the captured fine stage holds (exact ties keep every tied row,
                    # so the count can exceed B * min(N, S)): this call runs eagerly, the graph stays
                    out, count, cap = self._enqueue(img, img_scale, bank_raw, fine_on, dynamic=False, oid=oid)
                    M = out.pop("M")
            else:
                if prologue is not None:
                    prologue.run([t.to(dev) for t in prologue.inputs], img)
                out, count, cap = self._enqueue(img, img_scale, bank_raw, fine_on, dynamic=False, qmask=qmask,
                                                oid=oid)
                M = out.pop("M")
            self._publish(data, out, M, dev, fine_on)

    def _enqueue(self, img, img_scale, bank_raw, fine_on, dynamic, qmask=None, oid=None):
        """The whole forward as kernel launches on the current stream.  dynamic=False: one host
        sync reads the match count M between the coarse and the fine stage (the reference syncs in
        torch.where, coarse_matching.py:170) and the fine stage runs on exactly M matches.
        dynamic=True: no sync at all — the fine stage is launched at its capacity
        (B * min(N, S) matches) and reads M on the device; this is the capturable form."""
        B, _, H, W = img.shape
        # layer1_outconv2 is deferred: after the coarse stage it runs on the match windows only
        # (fine_windows "auto": when that is cheaper; "sparse" / "dense" force one path), and not
        # at all when fine matching is disabled
        win_ok = fine_on and self.fine_windows != "dense" and self.fine_preprocess.W == 5
        # latency mode (CUDA-graph capture at small batch): FPN top-down path on its own stream
        fpn_stream = None
        if dynamic and B <= 2 and os.environ.get("OPP_B200_TWO_STREAMS") != "0":
            fpn_stream = self._aux_stream(img.device, "_aux_fpn")
        q2, fine_in, (hc, wc) = self._backbone(img, defer_fine=True, fpn_stream=fpn_stream)
        fstride = fine_in.shape[1] // hc
        win_ok = win_ok and fstride == 4
        if oid is not None:
            bank = self._set_frame_state(oid, B)
        elif bank_raw is None:
            bank = self._resident_bank_state()
        else:
            kp, dco, dfine = bank_raw
            # one object for the whole batch ([1, N, .] tensors or stride-0 expanded views)
            one = kp.shape[0] == 1 or (B > 1 and kp.stride(0) == 0 and dco.stride(0) == 0
                                       and dfine.stride(0) == 0)
            if one:
                kp, dco, dfine = kp[:1], dco[:1], dfine[:1]
            bank = self._encode_bank(kp.float().contiguous(), dco.float().contiguous(),
                                     dfine.float().contiguous(), persistent=False)
        N = bank["N"]
        # latency mode at small batch: both sides of every layer run concurrently (see _both)
        small = B * (max(hc * wc, N) // 256 + 1) <= 37
        if os.environ.get("OPP_B200_TWO_STREAMS") == "0":   # A/B switch for the latency probe
            small = False
        side = self._aux_stream(img.device) if (dynamic and small) else None
        self._side_stream = side
        try:
            q2, d3 = self._coarse_transformer(q2, bank, B, hc * wc, N, qmask)
        finally:
            self._side_stream = None
        out = {}
        pack = None
        if dynamic:
            S = hc * wc
            cap = B * N
            fcap = min(cap, B * min(N, S))
            pack = _OutPack(_OutPack.nbytes(cap, fcap), img.device)
            out["gt_mask"] = pack.new("gt_mask", (cap,), torch.bool)   # zeroed once by _replay, never written
        count, cap = self._coarse_matching(q2, d3, bank, img_scale, B, N, hc, wc, float(H / hc), out, qmask,
                                           pack=pack, side=side)
        ids = (out["b_ids"], out["i_ids"], out["j_ids"], out["mkpts_query_c"])
        hf, wf = fine_in.shape[1:3]
        if fpn_stream is not None:
            torch.cuda.current_stream().wait_stream(fpn_stream)
        if dynamic:
            if fine_on:
                # the host does not know M: windows at capacity (the kernels read M on the device)
                # for the small batches this mode is meant for, else the dense map
                if win_ok and (self.fine_windows == "sparse" or B <= 8):
                    fw = self._fine_head_windows(fine_in, out["b_ids"], out["j_ids"], fcap, wc, fstride, count=count)
                    self._fine(fw, bank, ids, fcap, img_scale, hc, wc, (H, W), out, count=count, pack=pack,
                               windows_hw=(hf, wf))
                else:
                    self._fine(self._fine_head_dense(fine_in), bank, ids, fcap, img_scale, hc, wc, (H, W), out,
                               count=count, pack=pack)
            out["fcap"] = fcap
            out["pack"] = pack
        else:
            M = int(count.item())  # the one host sync of the forward
            if fine_on and M > 0:
                if win_ok and (self.fine_windows == "sparse" or self._windows_pay(M, B, hf, wf)):
                    fw = self._fine_head_windows(fine_in, out["b_ids"], out["j_ids"], M, wc, fstride)
                    self._fine(fw, bank, ids, M, img_scale, hc, wc, (H, W), out, windows_hw=(hf, wf))
                else:
                    self._fine(self._fine_head_dense(fine_in), bank, ids, M, img_scale, hc, wc, (H, W), out)
            out["M"] = M
        return out, count, cap

    def _aux_stream(self, dev, name="_aux"):
        st = getattr(self, name, None)
        if st is None or st.device != dev:
            st = torch.cuda.Stream(device=dev)
            setattr(self, name, st)
        return st

    # ------------------------------------------------------------------ CUDA graphs
    def enable_cuda_graphs(self, on=True):
        """Latency mode (extension): capture the forward once per input signature
        (B, H, W, N, dtypes) and replay it — one graph launch instead of ~115 kernel launches from
        Python, one host sync at the END (to size the outputs) instead of one in the middle.  The
        results are the same bits as the eager path.  Returned tensors are copies (the graph owns
        its buffers); conf_matrix_mode "eager" therefore costs an extra copy of the matrix —
        prefer "lazy"/"skip" here.  With a bank set, pass object_ids as a CPU tensor: a CUDA one
        is read back to validate it before any launch, which waits for the work queued before the
        forward (a second host sync)."""
        self.use_cuda_graphs = bool(on)
        if not on:
            self._graphs = {}
        return self

    def _replay(self, img, img_scale, bank_raw, fine_on, prologue=None, oid=None):
        resident = bank_raw is None
        if oid is not None:
            # object_ids is a graph input: one graph per bank set serves every assignment
            bkey = ("set", id(self._bank_set))
        elif resident:
            bkey = ("resident", id(self._bank))
        else:
            one = bank_raw[0].shape[0] == 1 or (img.shape[0] > 1 and all(t.stride(0) == 0 for t in bank_raw))
            if one:
                bank_raw = tuple(t[:1] for t in bank_raw)
            bkey = tuple((tuple(t.shape), t.dtype) for t in bank_raw)
        key = (tuple(img.shape), img.dtype, img_scale is not None, bkey, fine_on, self.conf_matrix_mode,
               self.fine_windows)
        if prologue is not None:
            key = key + (prologue.key,)
        ent = self._graphs.get(key)
        if ent is not None and ent["ws_epoch"] != self._ws_epoch:
            ent = None            # a workspace buffer was re-allocated: the captured pointers are stale
        if ent is None:
            if len(self._graphs) >= 8:
                self._graphs.clear()
            s_img = torch.empty_like(img)
            s_scale = torch.empty_like(img_scale) if img_scale is not None else None
            s_bank = None if resident else tuple(torch.empty_like(t.contiguous()) for t in bank_raw)
            s_pro = None if prologue is None else [torch.empty(t.shape, dtype=t.dtype, device=img.device)
                                                   for t in prologue.inputs]

            def load():
                if s_pro is None:
                    s_img.copy_(img)
                else:
                    for d, t in zip(s_pro, prologue.inputs):
                        d.copy_(t)
                if s_scale is not None:
                    s_scale.copy_(img_scale)
                if s_bank is not None:
                    for d, t in zip(s_bank, bank_raw):
                        d.copy_(t)
            load()
            s_oid = None if oid is None else oid.clone()
            # warm-up outside the capture: sizes the workspace, sets kernel attributes
            if s_pro is not None:
                prologue.run(s_pro, s_img)
            self._enqueue(s_img, s_scale, s_bank, fine_on, dynamic=True, oid=s_oid)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            count_host = torch.empty(1, dtype=torch.int32, pin_memory=True)
            with torch.cuda.graph(g):
                if s_pro is not None:
                    prologue.run(s_pro, s_img)   # first node: query_image from the prologue's inputs
                out, count, cap = self._enqueue(s_img, s_scale, s_bank, fine_on, dynamic=True, oid=s_oid)
                count_host.copy_(count, non_blocking=True)   # last node of the graph: M lands in pinned memory
            out["gt_mask"].zero_()
            ent = {"graph": g, "out": out, "count": count_host, "ws_epoch": self._ws_epoch,
                   "inputs": (s_img, s_scale, s_bank, s_pro), "oid": s_oid,
                   # the key holds id() of the resident bank / set: holding the object keeps that id
                   # from being reused by a later set_bank / set_banks while this graph exists
                   "bank_ref": self._bank_set if oid is not None else (self._bank if resident else None)}
            self._graphs[key] = ent
        s_img, s_scale, s_bank, s_pro = ent["inputs"]
        if s_pro is None:
            s_img.copy_(img)
        else:
            for d, t in zip(s_pro, prologue.inputs):
                d.copy_(t)
        if s_scale is not None:
            s_scale.copy_(img_scale)
        if s_bank is not None:
            for d, t in zip(s_bank, bank_raw):
                d.copy_(t)
        if oid is not None:
            ent["oid"].copy_(oid)
        ent["graph"].replay()
        if s_pro is not None:
            img.copy_(s_img)   # the caller's query_image receives what the prologue wrote
        src = ent["out"]
        torch.cuda.current_stream().synchronize()        # the only host sync, after everything is queued
        M = int(ent["count"][0])
        if M > src["fcap"]:
            return None, M    # the fine stage ran on the first fcap matches only: the caller re-runs eagerly
        pack = src["pack"]
        out = pack.views(pack.buf.clone(), M)    # one copy kernel
        out["sized"] = True
        out["conf_matrix"] = None
        if torch.is_tensor(src["conf_matrix"]):
            out["conf_matrix"] = src["conf_matrix"].clone()
        elif src["conf_matrix"] is not None:     # lazy handle: re-issue it for this forward
            out["conf_matrix"] = LazyConfMatrix(self, *src["conf_matrix"]._args)
        return out, M

    def _publish(self, data, out, M, dev, fine_on):
        """Write the reference's output keys (coarse_matching.py:231-241, fine_matching.py:46-55,107-110)."""
        if out["conf_matrix"] is not None:
            data["conf_matrix"] = out["conf_matrix"]
        # graph mode hands in tensors that are already M rows long (sized=True)
        cut = (lambda t: t) if out.get("sized") else (lambda t: t[:M])
        b_ids = cut(out["b_ids"])
        data.update({
            "b_ids": b_ids, "i_ids": cut(out["i_ids"]), "j_ids": cut(out["j_ids"]),
            "gt_mask": cut(out["gt_mask"]) if "gt_mask" in out else torch.zeros(M, dtype=torch.bool, device=dev),
            "m_bids": b_ids, "mkpts_3d_db": cut(out["mkpts_3d_db"]), "mkpts_query_c": cut(out["mkpts_query_c"]),
            "mconf": cut(out["mconf"]),
        })
        if not fine_on:
            data["mkpts_query_f"] = data["mkpts_query_c"]
        elif M == 0:
            data.update({"expec_f": torch.empty(0, 3, device=dev), "mkpts_query_f": data["mkpts_query_c"]})
        else:
            data.update({"expec_f": cut(out["expec_f"]), "mkpts_query_f": cut(out["mkpts_query_f"])})


class LazyConfMatrix:
    """Handle stored in data["conf_matrix"] when `model.conf_matrix_mode == "lazy"`: the dual-softmax
    statistics of the forward are kept, the 4 B x N x S bytes of the matrix are only written when
    somebody asks (`.materialize()` / `torch.as_tensor(handle.materialize())`).  Valid until the
    model's next forward (it reads the model's workspace)."""

    def __init__(self, model, d3, q2, lse_pt, lse_px, B, N, S, scale, rows_b=None):
        self._model, self._args = model, (d3, q2, lse_pt, lse_px, B, N, S, scale, rows_b)
        self._epoch = model._fwd_count
        self.shape = torch.Size((B, N, S))
        self._value = None

    def materialize(self):
        if self._value is None:
            if self._model._fwd_count != self._epoch:
                raise RuntimeError("LazyConfMatrix is stale: the model ran another forward since")
            with torch.no_grad(), torch.cuda.device(self._args[1].device):
                self._value = self._model._materialize_conf(*self._args)
        return self._value
