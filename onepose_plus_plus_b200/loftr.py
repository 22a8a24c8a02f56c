"""Drop-in for ``LoFTR_for_OnePose_Plus`` (src/KeypointFreeSfM/loftr_for_sfm/loftr.py:16-167) — the
2D-2D detector-free matcher OnePose++ uses for its keypoint-free SfM mapping and as the detector
of demo.py — on the same sm_90a kernels as the 2D-3D matcher (SURVEY §8 f3).

Same constructor (``config, enable_fine_matching=True``; config = the lower-cased dict of
``loftr_for_onepose_plus_cfg.py``), same state-dict keys (``backbone.*``, ``loftr_coarse.layers.N.*``,
``loftr_fine.layers.N.*``; ``pos_encoding.pe`` non-persistent), same in-place ``forward(data)``
contract: reads ``image0, image1`` (+ ``scale0, scale1``), writes ``bs, hw*_i/c/f, conf_matrix,
b_ids, i_ids, j_ids, gt_mask, m_bids, mkpts0_c, mkpts1_c, mconf, W, expec_f, mkpts0_f, mkpts1_f``.
What differs from the 2D-3D path (submodules/LoFTR/src/loftr): both sequences are image tokens,
8 coarse layers with SEQUENTIAL cross updates (transformer.py:96-97), temperature 0.1 / threshold
0.2 / border removal on all sides of both grids (coarse_matching.py), W x W windows (W = 9) from
both fine maps and the centre token of image 0's window correlated with image 1's
(fine_matching.py).

Built: inference with predicted coarse matches, images of equal size per call, linear attention,
``fine_concat_coarse_feat`` False (the shipped configuration); the fine-only branch with given
coarse matches (``mkpts0_c`` / ``mkpts1_c`` in data, B = 1) and the ``extract_coarse_feature`` /
``extract_fine_feature`` sampling at the fine matches (B = 1), which the keypoint-free SfM
refinement calls (loftr.py:81-165).  Not built (raise): padding masks (``mask0/mask1``), training
mode, B > 1 on the fine-only branch or with extraction.
"""
import math

import torch
import torch.nn as nn

from . import ops
from .model import (LocalFeatureTransformer, ResNetFPN_8_2, _Engine)

__all__ = ["LoFTR_for_OnePose_Plus"]


class _PositionEncodingSine(nn.Module):
    """submodules/LoFTR/src/loftr/utils/position_encoding.py:11-36 (both frequency tables)"""

    def __init__(self, d_model, max_shape=(256, 256), temp_bug_fix=True):
        super().__init__()
        pe = torch.zeros((d_model, *max_shape))
        y_position = torch.ones(max_shape).cumsum(0).float().unsqueeze(0)
        x_position = torch.ones(max_shape).cumsum(1).float().unsqueeze(0)
        k = torch.arange(0, d_model // 2, 2).float()
        if temp_bug_fix:
            div_term = torch.exp(k * (-math.log(10000.0) / (d_model // 2)))
        else:   # the historical table (backward compatibility of released checkpoints)
            div_term = torch.exp(k * (-math.log(10000.0) / d_model // 2))
        div_term = div_term[:, None, None]
        pe[0::4], pe[1::4] = torch.sin(x_position * div_term), torch.cos(x_position * div_term)
        pe[2::4], pe[3::4] = torch.sin(y_position * div_term), torch.cos(y_position * div_term)
        self.register_buffer("pe", pe.unsqueeze(0), persistent=False)


def _transformer(cfg):
    # LoFTR's LocalFeatureTransformer takes (d_model, nhead, layer_names, attention) only
    return LocalFeatureTransformer({"d_model": cfg["d_model"], "nhead": cfg["nhead"], "type": "LoFTR",
                                    "layer_names": list(cfg["layer_names"]), "layer_iter_n": 1,
                                    "attention": cfg["attention"], "norm_method": "layernorm", "rezero": None,
                                    "redraw_interval": None, "final_proj": False})


class LoFTR_for_OnePose_Plus(_Engine):
    def __init__(self, config, enable_fine_matching=True, precision=None):
        super().__init__()
        self.config = config
        self.enable_fine_matching = enable_fine_matching
        if config["backbone_type"] != "ResNetFPN" or tuple(config["resolution"]) != (8, 2):
            raise ValueError(f"LOFTR.BACKBONE_TYPE {config['backbone_type']} / resolution not supported.")
        rf = config["resnetfpn"]
        if rf["initial_dim"] != 128 or list(rf["block_dims"]) != [128, 196, 256]:
            raise NotImplementedError("backbone kernels are built for dims 128/[128,196,256]")
        if config["coarse"]["d_model"] != 256 or config["coarse"]["nhead"] != 8 or \
                config["fine"]["d_model"] != 128 or config["fine"]["nhead"] != 8:
            raise NotImplementedError("kernels are built for d_model 256/128, 8 heads")
        if config["coarse"]["attention"] != "linear" or config["fine"]["attention"] != "linear":
            raise NotImplementedError("the 2D-2D matcher is built for attention='linear'")
        if config["match_coarse"]["match_type"] != "dual_softmax":
            raise NotImplementedError("match_type 'sinkhorn' is not built")
        if config["fine_concat_coarse_feat"]:
            raise NotImplementedError("fine_concat_coarse_feat=True is not built (False in loftr_for_onepose_plus_cfg.py)")
        self.W = config["fine_window_size"]
        if self.W % 2 != 1 or not 3 <= self.W <= 9:
            raise NotImplementedError("fine window sizes 3, 5, 7, 9 are built")
        self._init_engine(precision, "linear")
        self.backbone = ResNetFPN_8_2({"block_type": "BasicBlock", "initial_dim": rf["initial_dim"],
                                       "block_dims": list(rf["block_dims"]), "output_layers": [3, 1]})
        self.pos_encoding = _PositionEncodingSine(config["coarse"]["d_model"],
                                                  temp_bug_fix=config["coarse"]["temp_bug_fix"])
        self.loftr_coarse = _transformer(config["coarse"])
        self.loftr_fine = _transformer(config["fine"])

    def _pe_module(self):
        return self.pos_encoding

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_plan"], st["_plan_sig"], st["_ws"], st["_sig_tensors"], st["_graphs"] = None, None, {}, None, {}
        return st

    # ------------------------------------------------------------------ stages
    def _coarse(self, t0, t1, B, S0, S1):
        """LoFTR LocalFeatureTransformer.forward (loftr_module/transformer.py:81-101): self layers on
        both images, then cross layers one after the other — feat1 reads the UPDATED feat0."""
        dev = t0.device
        f16 = torch.float16
        pl = 2 if self.split else 1
        cur0, cur1 = t0, t1
        for i, name in enumerate(self.loftr_coarse.layer_names):
            L = self._plan["coarse"][i]
            n0 = self._buf(f"lt0_{i % 2}", (B, S0, pl * 256), f16, dev)
            n1 = self._buf(f"lt1_{i % 2}", (B, S1, pl * 256), f16, dev)
            if name == "self":
                self._encoder_layer(L, "c2_", cur0, cur0, B, S0, S0, n0)
                self._encoder_layer(L, "c3_", cur1, cur1, B, S1, S1, n1)
            else:
                self._encoder_layer(L, "c2_", cur0, cur1, B, S0, S1, n0)
                self._encoder_layer(L, "c3_", cur1, n0, B, S1, S0, n1)
            cur0, cur1 = n0, n1
        return cur0, cur1

    def _coarse_select(self, t0, t1, B, hc, wc, H, s0, s1, conf=None):
        """LoFTR utils/coarse_matching.py:74-107, 133-259 on B pairs of final coarse tokens: the
        one-pass dual softmax and the mutual-nearest selection (threshold, border on all sides,
        coordinates times the scales).  conf fp32 [B, S, S] receives the matrix; None skips it.
        Returns (M, b_ids, i_ids, j_ids, mconf, mkpts0_c, mkpts1_c) trimmed to the M matches (one host
        sync, for the count)."""
        dev = t0.device
        f32, i32 = torch.float32, torch.int32
        split = self.split
        S = hc * wc
        mc = self.config["match_coarse"]
        scale = 1.0 / (256.0 * mc["dsmax_temperature"])
        ts = ops.sim_tiles(S)
        pm, ps = self._buf("pm_pt", (B * S, ts), f32, dev), self._buf("ps_pt", (B * S, ts), f32, dev)
        lse0, lse1 = self._buf("lse_pt", (B, S), f32, dev), self._buf("lse_px", (B, S), f32, dev)
        groups = (S + 31) // 32
        ops.sim_lse_cols(t0, t1, B, S, S, 256, scale, pm, ps, lse0, self._buf("lse_col_m", (B, groups, S), f32, dev),
                         self._buf("lse_col_s", (B, groups, S), f32, dev), lse1, split)
        pt_val, pt_idx = self._buf("pt_val", (B, S), f32, dev), self._buf("pt_idx", (B, S), i32, dev)
        colmax = self._buf("colmax", (B, S), i32, dev)
        ops.sim_conf_colmax(t0, t1, lse0, lse1, conf, B, S, S, 256, scale, pm, self._buf("pi_pt", (B * S, ts), i32, dev),
                            pt_val, pt_idx, colmax, split)
        cap = B * S
        count = self._buf("match_count", (1,), i32, dev)
        b_ids, i_ids, j_ids = (torch.empty(cap, dtype=torch.int64, device=dev) for _ in range(3))
        mconf = torch.empty(cap, dtype=f32, device=dev)
        mk0, mk1 = torch.empty((cap, 2), dtype=f32, device=dev), torch.empty((cap, 2), dtype=f32, device=dev)
        ops.match_select_2d(pt_val, pt_idx, colmax, s0, s1, B, hc, wc, hc, wc, mc["thr"], mc["border_rm"],
                            float(H / hc), self._buf("match_scratch", ((cap + 1023) // 1024 + 2,), i32, dev),
                            b_ids, i_ids, j_ids, mconf, mk0, mk1, count)
        M = int(count.item())   # the one host sync (the reference syncs in torch.where)
        return M, b_ids[:M], i_ids[:M], j_ids[:M], mconf[:M], mk0[:M], mk1[:M]

    def _fine_layer(self, L, x, src, G, T, out16, out32=None):
        """LoFTREncoderLayer.forward (d_model 128) on G groups of T tokens: x, src [G*T, pl*128]."""
        dev = x.device
        f16 = torch.float16
        split = self.split
        pl = 2 if split else 1
        rows = G * T
        q = self._buf("lf_q", (rows, pl * 128), f16, dev)
        kv = self._buf("lf_kv", (rows, pl * 256), f16, dev)
        att = self._buf("lf_att", (rows, pl * 128), f16, dev)
        msg = self._buf("lf_msg", (rows, pl * 128), f16, dev)
        h = self._buf("lf_h", (rows, pl * 256), f16, dev)
        ops.linear_act(x, None, L["wq"], q, rows, 2, 128, split)           # Q = elu(q_proj x) + 1
        ops.linear_act(src, None, L["wkv"], kv, rows, 2, 128, split)       # K' = elu(k_proj s) + 1 | V
        ops.seq_attention(q, kv, att, G, T, T, split)
        ops.linear_ln(att, None, L["merge16"], False, *L["n1"], 1, rows, split, out16=msg)
        ops.linear_act(x, msg, L["mlp0"], h, rows, 1, 256, split)
        ops.linear_ln(h, None, L["mlp2"], False, *L["n2"], 1, rows, split, resid=x, out16=out16, out32=out32)

    def _fine_layers(self, xa, xb, x32, M):
        """LocalFeatureTransformer.forward of the fine level (transformer.py:81-101) on the 2M gathered
        windows in xa (sequence-major); xb is the second ping-pong buffer, x32 receives the fp32 output."""
        WW = self.W * self.W
        half = M * WW
        cur, nxt = xa, xb
        names = self.loftr_fine.layer_names
        for li, name in enumerate(names):
            L = self._plan["fine"][li]
            last = li == len(names) - 1
            if name == "self":      # both windows at once: 2M groups attending to themselves
                self._fine_layer(L, cur, cur, 2 * M, WW, nxt, x32 if last else None)
            else:                   # sequential: window 0 from window 1, then window 1 from the NEW window 0
                self._fine_layer(L, cur[:half], cur[half:], M, WW, nxt[:half], x32[:half] if last else None)
                self._fine_layer(L, cur[half:], nxt[:half], M, WW, nxt[half:], x32[half:] if last else None)
            cur, nxt = nxt, cur
        if not names:
            raise NotImplementedError("a fine transformer without layers is not built")

    @staticmethod
    def _given_cells(mk0, mk1, hw_i, hc, wc, scale0, scale1):
        """The fine-only branch's conversion of given coarse matches (loftr.py:87-109): clip x to
        [0, w - 2] and y to [0, h - 2] IN PLACE, then cell = round(mkpts / (8 * scale[[1, 0]])) (half to
        even) as y * wc + x in the keypoints' dtype.  scale0 / scale1: per-match fp32 [M, 2] or None.
        Returns (i_ids, j_ids) int64; ValueError when a cell lies outside [0, hc * wc) (an x that rounds
        to wc wraps into the next row, as in the reference)."""
        h, w = int(hw_i[0]), int(hw_i[1])
        for mk in (mk0, mk1):
            mk[:, 0] = torch.clip(mk[:, 0], min=0, max=w - 2)
            mk[:, 1] = torch.clip(mk[:, 1], min=0, max=h - 2)
        scale = h / hc
        ids = []
        for mk, sc in ((mk0, scale0), (mk1, scale1)):
            r = torch.round(mk / (scale * sc[:, [1, 0]] if sc is not None else scale))
            ids.append((r[:, 1] * wc + r[:, 0]).long())
        S = hc * wc
        if ids[0].numel() and not bool(torch.stack([ids[0].min() >= 0, ids[1].min() >= 0, ids[0].max() < S,
                                                    ids[1].max() < S]).all()):
            raise ValueError(f"a given coarse match lies outside the {hc}x{wc} coarse grid (cell id not in [0, {S}))")
        return ids[0], ids[1]

    def _fine_given(self, fine_store, img0, img1, i_ids, j_ids, M, hc, wc, hf, wf, H, scales):
        """Fine level on M given cells (fine_preprocess.py:30-59, transformer, fine_matching.py:17-74) of
        image pairs (img0[m], img1[m]) of one map store.  Returns (expec_f fp32 [M, 3], delta fp32 [M, 2])
        with delta = coords * (W // 2) * 2 * scales[img1] rounded as fine_matching rounds it; the
        caller adds mkpts1_c in its own dtype."""
        dev = fine_store.device
        split = self.split
        pl = 2 if split else 1
        WW = self.W * self.W
        rows = 2 * M * WW
        f16, f32 = torch.float16, torch.float32
        xa = self._buf("lf_xa", (rows, pl * 128), f16, dev)
        xb = self._buf("lf_xb", (rows, pl * 128), f16, dev)
        x32 = self._buf("lf_x32", (rows, 128), f32, dev)
        ops.fine_gather_2d_images(fine_store, img0, img1, i_ids, j_ids, xa, M, hf, wf, wc, hf // hc, self.W, split)
        self._fine_layers(xa, xb, x32, M)
        expec_f = torch.empty((M, 3), dtype=f32, device=dev)
        delta = torch.empty((M, 2), dtype=f32, device=dev)
        zeros = torch.zeros((M, 2), dtype=f32, device=dev)     # mkpts1_f = 0 + offset: the offset alone
        ops.fine_match_2d(x32, zeros, img1, scales, expec_f, delta, M, self.W, float(H / hf))
        return expec_f, delta

    def _extract(self, coarse_store, fine_store, img0, img1, mk0f, mk1f, imghw, coarse, fine):
        """loftr.py:131-165: sample_feature_from_featuremap at mkpts0_f / mkpts1_f, nearest from the raw
        coarse map (before the position encoding), bilinear from the fine map.  imghw fp32 [N, 2] =
        scale * (h, w) per image of the stores."""
        out = {}
        pl = 2 if self.split else 1
        if coarse:
            c = coarse_store.shape[-1] // pl
            out["feat_coarse_b_0"] = ops.sample_feature(coarse_store, c, self.split, mk0f, imghw, True, img0)
            out["feat_coarse_b_1"] = ops.sample_feature(coarse_store, c, self.split, mk1f, imghw, True, img1)
        if fine:
            c = fine_store.shape[-1] // pl
            out["feat_ext0"] = ops.sample_feature(fine_store, c, self.split, mk0f, imghw, False, img0)
            out["feat_ext1"] = ops.sample_feature(fine_store, c, self.split, mk1f, imghw, False, img1)
        return out

    # ------------------------------------------------------------------ forward
    def forward(self, data, **kwargs):
        if self.training:
            raise NotImplementedError("LoFTR_for_OnePose_Plus is the inference matcher: call .eval()")
        if "mask0" in data or "mask1" in data:
            raise NotImplementedError("padding masks (mask0 / mask1) are not built")
        ext_c, ext_f = bool(kwargs.get("extract_coarse_feature")), bool(kwargs.get("extract_fine_feature"))
        if "mkpts0_c" in data or ext_c or ext_f:
            return self._forward_given(data, ext_c, ext_f)
        im0, im1 = data["image0"], data["image1"]
        if not (torch.is_tensor(im0) and im0.is_cuda and im1.is_cuda):
            raise RuntimeError("LoFTR_for_OnePose_Plus has no CPU path: move the model and data to a CUDA device")
        if im0.dim() != 4 or im0.shape[1] != 1 or im1.shape != im0.shape:
            raise ValueError(f"image0 / image1 must both be [B, 1, H, W] of one size, got {tuple(im0.shape)}, "
                             f"{tuple(im1.shape)} (differently sized pairs: one call per size)")
        B, _, H, W = im0.shape
        if H % 8 or W % 8 or H < 48 or W < 48:
            raise ValueError("image height/width must be multiples of 8 (>= 48)")
        for k in ("scale0", "scale1"):
            if k in data and tuple(data[k].shape) != (B, 2):
                raise ValueError(f"{k} must be [B, 2]")
        if ("scale0" in data) != ("scale1" in data):
            raise ValueError("scale0 and scale1 come together")
        with torch.no_grad(), torch.cuda.device(im0.device):
            dev = im0.device
            self._ensure_plan(dev)
            split = self.split
            pl = 2 if split else 1
            f16, f32 = torch.float16, torch.float32
            img = torch.cat([im0, im1], 0)
            if img.dtype not in (torch.uint8, torch.float32):
                img = img.float()
            tok, fine_map, (hc, wc) = self._backbone(img.contiguous())     # loftr.py:46-49 (one batched pass)
            S = hc * wc
            hf, wf = fine_map.shape[1:3]
            data.update({"bs": B, "hw0_i": im0.shape[2:], "hw1_i": im1.shape[2:],
                         "hw0_c": torch.Size((hc, wc)), "hw1_c": torch.Size((hc, wc)),
                         "hw0_f": torch.Size((hf, wf)), "hw1_f": torch.Size((hf, wf))})
            t0, t1 = self._coarse(tok[:B], tok[B:], B, S, S)
            conf = torch.empty((B, S, S), dtype=f32, device=dev)
            s0 = data["scale0"].to(device=dev, dtype=f32).contiguous() if "scale0" in data else None
            s1 = data["scale1"].to(device=dev, dtype=f32).contiguous() if "scale1" in data else None
            M, b_ids, i_ids, j_ids, mconf, mk0, mk1 = self._coarse_select(t0, t1, B, hc, wc, H, s0, s1, conf)
            data.update({"conf_matrix": conf, "b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids,
                         "gt_mask": torch.zeros(M, dtype=torch.bool, device=dev), "m_bids": b_ids,
                         "mkpts0_c": mk0, "mkpts1_c": mk1, "mconf": mconf})
            if not self.enable_fine_matching:
                data.update({"mkpts0_f": data["mkpts0_c"], "mkpts1_f": data["mkpts1_c"]})
                return
            # ---- fine level (fine_preprocess.py:30-59, transformer.py:81-101, fine_matching.py:17-74)
            data["W"] = self.W
            if M == 0:
                data.update({"expec_f": torch.empty(0, 3, device=dev), "mkpts0_f": data["mkpts0_c"],
                             "mkpts1_f": data["mkpts1_c"]})
                return
            WW = self.W * self.W
            rows = 2 * M * WW
            xa = self._buf("lf_xa", (rows, pl * 128), f16, dev)
            xb = self._buf("lf_xb", (rows, pl * 128), f16, dev)
            x32 = self._buf("lf_x32", (rows, 128), f32, dev)
            ops.fine_gather_2d(fine_map[:B], fine_map[B:], b_ids, i_ids, j_ids, xa, M, hf, wf, wc, hf, wf, wc,
                               hf // hc, self.W, split)
            self._fine_layers(xa, xb, x32, M)
            expec_f = torch.empty((M, 3), dtype=f32, device=dev)
            mk1f = torch.empty((M, 2), dtype=f32, device=dev)
            ops.fine_match_2d(x32, data["mkpts1_c"], b_ids, s1, expec_f, mk1f, M, self.W, float(H / hf))
            data.update({"expec_f": expec_f, "mkpts0_f": data["mkpts0_c"], "mkpts1_f": mk1f})

    def _forward_given(self, data, ext_c, ext_f):
        """forward() with given coarse matches (loftr.py:81-121) and/or the feature extraction at the
        fine matches (loftr.py:131-165); B = 1 as the reference requires."""
        im0, im1 = data["image0"], data["image1"]
        if not (torch.is_tensor(im0) and im0.is_cuda and im1.is_cuda):
            raise RuntimeError("LoFTR_for_OnePose_Plus has no CPU path: move the model and data to a CUDA device")
        if im0.dim() != 4 or im0.shape[1] != 1 or im1.shape != im0.shape:
            raise ValueError(f"image0 / image1 must both be [B, 1, H, W] of one size, got {tuple(im0.shape)}, "
                             f"{tuple(im1.shape)}")
        B, _, H, W = im0.shape
        if B != 1:
            raise NotImplementedError("the fine-only branch and the feature extraction are built for B = 1 "
                                      "(loftr.py:82 and sample_feature_from_featuremap assert it)")
        if H % 8 or W % 8 or H < 48 or W < 48:
            raise ValueError("image height/width must be multiples of 8 (>= 48)")
        for k in ("scale0", "scale1"):
            if k in data and tuple(data[k].shape) != (B, 2):
                raise ValueError(f"{k} must be [B, 2]")
        if ("scale0" in data) != ("scale1" in data):
            raise ValueError("scale0 and scale1 come together")
        given = "mkpts0_c" in data
        hc, wc = H // 8, W // 8
        hf, wf = H // 2, W // 2
        dev = im0.device
        with torch.no_grad(), torch.cuda.device(dev):
            s0 = data["scale0"].to(device=dev, dtype=torch.float32) if "scale0" in data else None
            s1 = data["scale1"].to(device=dev, dtype=torch.float32) if "scale1" in data else None
            if given:
                mk0, mk1 = data["mkpts0_c"], data["mkpts1_c"]
                if not (mk0.is_cuda and mk1.is_cuda and mk0.dim() == 2 and mk0.shape[1] == 2 and mk1.shape == mk0.shape):
                    raise ValueError("mkpts0_c / mkpts1_c must be CUDA tensors [M, 2] of one length")
                M = mk0.shape[0]
                b_ids = torch.zeros((M,), dtype=torch.int64, device=dev)
                i_ids, j_ids = self._given_cells(mk0, mk1, im0.shape[2:], hc, wc,
                                                 s0[b_ids] if s0 is not None else None,
                                                 s1[b_ids] if s1 is not None else None)
            self._ensure_plan(dev)
            img = torch.cat([im0, im1], 0)
            if img.dtype not in (torch.uint8, torch.float32):
                img = img.float()
            tok, fine_map, _ = self._backbone(img.contiguous())
            pl = 2 if self.split else 1
            coarse_map = self._buf("x3_out", (2, hc, wc, pl * 256), torch.float16, dev)   # before the encoding
            data.update({"bs": B, "hw0_i": im0.shape[2:], "hw1_i": im1.shape[2:],
                         "hw0_c": torch.Size((hc, wc)), "hw1_c": torch.Size((hc, wc)),
                         "hw0_f": torch.Size((hf, wf)), "hw1_f": torch.Size((hf, wf))})
            if given:
                data.update({"m_bids": b_ids, "b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids,
                             "mconf": torch.ones_like(b_ids)})
            else:
                S = hc * wc
                t0, t1 = self._coarse(tok[:B], tok[B:], B, S, S)
                conf = torch.empty((B, S, S), dtype=torch.float32, device=dev)
                M, b_ids, i_ids, j_ids, mconf, mk0, mk1 = self._coarse_select(
                    t0, t1, B, hc, wc, H, s0.contiguous() if s0 is not None else None,
                    s1.contiguous() if s1 is not None else None, conf)
                data.update({"conf_matrix": conf, "b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids,
                             "gt_mask": torch.zeros(M, dtype=torch.bool, device=dev), "m_bids": b_ids,
                             "mkpts0_c": mk0, "mkpts1_c": mk1, "mconf": mconf})
            img0 = torch.zeros((M,), dtype=torch.int64, device=dev)
            img1 = torch.ones((M,), dtype=torch.int64, device=dev)
            if not self.enable_fine_matching:
                data.update({"mkpts0_f": data["mkpts0_c"], "mkpts1_f": data["mkpts1_c"]})
            else:
                data["W"] = self.W
                if M == 0:
                    data.update({"expec_f": torch.empty(0, 3, device=dev), "mkpts0_f": data["mkpts0_c"],
                                 "mkpts1_f": data["mkpts1_c"]})
                else:
                    sc = torch.cat([s0, s1], 0).contiguous() if s1 is not None else None
                    expec_f, delta = self._fine_given(fine_map, img0, img1, i_ids, j_ids, M, hc, wc, hf, wf, H, sc)
                    data.update({"expec_f": expec_f, "mkpts0_f": data["mkpts0_c"],
                                 "mkpts1_f": data["mkpts1_c"] + delta})
            if ext_c or ext_f:
                imghw = torch.cat([data["scale0"].to(dev).float() * torch.tensor([H, W], dtype=torch.float32, device=dev),
                                   data["scale1"].to(dev).float() * torch.tensor([H, W], dtype=torch.float32, device=dev)], 0)
                data.update(self._extract(coarse_map, fine_map, img0, img1, data["mkpts0_f"].contiguous(),
                                          data["mkpts1_f"].contiguous(), imghw.contiguous(), ext_c, ext_f))

    # ------------------------------------------------------------------ SfM coarse matching
    def image_tokens(self, images_u8, image_chunk=16):
        """The coarse tokens of N images, each image once: conv1 .. layer3 and layer3_outconv with the
        position-encoding epilogue, bit-equal to the tokens forward() computes for the same image.
        The FPN branches that only the fine level reads are skipped.  images_u8 uint8 [N, 1, H, W] on
        the device; the backbone runs on `image_chunk` images at a time, so its workspace stays that
        of one chunk.  Returns (fp16 planes [N, S, pl*256], (hc, wc))."""
        N, _, H, W = images_u8.shape
        dev = images_u8.device
        self._ensure_plan(dev)
        hc, wc = H // 8, W // 8
        store = torch.empty((N, hc * wc, (2 if self.split else 1) * 256), dtype=torch.float16, device=dev)
        for c0 in range(0, N, image_chunk):
            tok, _, _ = self._backbone(images_u8[c0:c0 + image_chunk].contiguous(), coarse_only=True)
            store[c0:c0 + image_chunk].copy_(tok)
        return store, (hc, wc)

    @torch.no_grad()
    def coarse_matches_for_pairs(self, images_u8, scales, pair_idx, pair_batch=32, image_chunk=16):
        """Coarse-only matching of many pairs over one image set (the keypoint-free SfM coarse match,
        coarse_match_worker.py:44-76): the backbone once per image (image_tokens), then the coarse
        transformer, the dual softmax and the selection on `pair_batch` pairs at a time, without the
        confidence matrix.  One host sync per pair batch, for its match count.
        images_u8 uint8 [N, 1, H, W] (CUDA), scales fp32 [N, 2] (the per-image scale0 / scale1),
        pair_idx int64 [P, 2] (image indices).  Returns a dict of device tensors over all pairs, in
        pair order and within a pair in (i) order as forward() gives them: b_ids (the pair index),
        i_ids, j_ids, mkpts0_c, mkpts1_c, mconf, and offsets int64 [P + 1] (host) delimiting the
        pairs."""
        if self.training:
            raise NotImplementedError("LoFTR_for_OnePose_Plus is the inference matcher: call .eval()")
        if not (torch.is_tensor(images_u8) and images_u8.is_cuda and images_u8.dtype == torch.uint8):
            raise TypeError("images_u8 must be a uint8 CUDA tensor [N, 1, H, W]")
        N, C, H, W = images_u8.shape
        if C != 1 or H % 8 or W % 8 or H < 48 or W < 48:
            raise ValueError(f"images must be [N, 1, H, W] with H, W multiples of 8 (>= 48), got {tuple(images_u8.shape)}")
        pair_idx = torch.as_tensor(pair_idx, dtype=torch.int64).reshape(-1, 2)
        if tuple(scales.shape) != (N, 2):
            raise ValueError(f"scales must be [N, 2] = [{N}, 2], got {tuple(scales.shape)}")
        if pair_idx.numel() and (int(pair_idx.min()) < 0 or int(pair_idx.max()) >= N):
            raise ValueError("pair_idx names an image outside [0, N)")
        if pair_batch < 1:
            raise ValueError("pair_batch must be >= 1")
        with torch.cuda.device(images_u8.device):
            dev = images_u8.device
            store, (hc, wc) = self.image_tokens(images_u8, image_chunk)
            S = hc * wc
            scales = scales.to(device=dev, dtype=torch.float32)
            pidx = pair_idx.to(dev)
            P = pair_idx.shape[0]
            out = {k: [] for k in ("b_ids", "i_ids", "j_ids", "mkpts0_c", "mkpts1_c", "mconf")}
            counts = []
            for p0 in range(0, P, pair_batch):
                idx = pidx[p0:p0 + pair_batch]
                B = idx.shape[0]
                t0, t1 = self._coarse(store[idx[:, 0]], store[idx[:, 1]], B, S, S)
                s0, s1 = scales[idx[:, 0]].contiguous(), scales[idx[:, 1]].contiguous()
                M, b_ids, i_ids, j_ids, mconf, mk0, mk1 = self._coarse_select(t0, t1, B, hc, wc, H, s0, s1)
                for k, v in zip(out, (b_ids + p0, i_ids, j_ids, mk0, mk1, mconf)):
                    out[k].append(v)
                counts.append(torch.bincount(b_ids, minlength=B).cpu() if M else torch.zeros(B, dtype=torch.int64))
            res = {k: torch.cat(v) if v else torch.empty((0, 2) if k.startswith("mkpts") else (0,),
                                                          dtype=torch.float32 if k[0] == "m" else torch.int64,
                                                          device=dev)
                   for k, v in out.items()}
            offsets = torch.zeros(P + 1, dtype=torch.int64)
            if P:
                torch.cumsum(torch.cat(counts), 0, out=offsets[1:])
            res["offsets"] = offsets
            return res

    # ------------------------------------------------------------------ SfM refinement (fine matching)
    def image_maps(self, images_u8, image_chunk=16):
        """The full backbone of N images, each image once, kept in two stores: the fine map (1/2
        resolution, 128 channels) and the raw coarse map (layer3_outconv's output before the position
        encoding, 1/8 resolution, 256 channels), both NHWC fp16 with a lo plane when split.  A store
        holds planes * 2 * (H/2 * W/2 * 128 + H/8 * W/8 * 256) bytes per image: 37.7 MB at 512 x 512
        with the split fp16 planes.  The backbone runs `image_chunk` images at a time.  Returns
        (fine fp16 [N, H/2, W/2, pl*128], coarse fp16 [N, H/8, W/8, pl*256])."""
        N, _, H, W = images_u8.shape
        dev = images_u8.device
        self._ensure_plan(dev)
        pl = 2 if self.split else 1
        hc, wc = H // 8, W // 8
        fine = torch.empty((N, H // 2, W // 2, pl * 128), dtype=torch.float16, device=dev)
        coarse = torch.empty((N, hc, wc, pl * 256), dtype=torch.float16, device=dev)
        for c0 in range(0, N, image_chunk):
            chunk = images_u8[c0:c0 + image_chunk].contiguous()
            _, fmap, _ = self._backbone(chunk)
            fine[c0:c0 + image_chunk].copy_(fmap)
            coarse[c0:c0 + image_chunk].copy_(self._buf("x3_out", (chunk.shape[0], hc, wc, pl * 256), torch.float16, dev))
        return fine, coarse

    @torch.no_grad()
    def fine_matches_for_pairs(self, images_u8, scales, pair_idx, mkpts0_c, mkpts1_c, offsets, pair_batch=32,
                               image_chunk=16, match_batch=8192):
        """The fine-only forward with both extractions (forward(data, extract_coarse_feature=True,
        extract_fine_feature=True) with mkpts0_c / mkpts1_c given, fine_match_worker.py:28-31) for many
        pairs over one image set: the full backbone once per image (image_maps), then for batches of
        up to `pair_batch` pairs (and about `match_batch` matches) the window gather from the stores,
        the fine layers, the expectation and the four samplings.  No host sync inside the loop: the
        match counts are known from offsets.
        images_u8 uint8 [N, 1, H, W] (CUDA); scales fp32 [N, 2] (each image's scale); pair_idx int64
        [P, 2] (image indices); mkpts0_c / mkpts1_c [M, 2] fp32 or fp64 CUDA tensors of all pairs
        concatenated, pair p owning rows offsets[p]:offsets[p + 1] (offsets int64 [P + 1], host).  Like
        forward, mkpts*_c are clipped IN PLACE.  ValueError, before any launch, for a cell id outside
        the coarse grid.  Returns a dict of device tensors over all matches: i_ids, j_ids, expec_f,
        mkpts1_f (mkpts1_c's dtype), feat_coarse_b_0/1 fp32 [M, 256], feat_ext0/1 fp32 [M, 128]."""
        if self.training:
            raise NotImplementedError("LoFTR_for_OnePose_Plus is the inference matcher: call .eval()")
        if not (torch.is_tensor(images_u8) and images_u8.is_cuda and images_u8.dtype == torch.uint8):
            raise TypeError("images_u8 must be a uint8 CUDA tensor [N, 1, H, W]")
        N, C, H, W = images_u8.shape
        if C != 1 or H % 8 or W % 8 or H < 48 or W < 48:
            raise ValueError(f"images must be [N, 1, H, W] with H, W multiples of 8 (>= 48), got {tuple(images_u8.shape)}")
        if not self.enable_fine_matching:
            raise NotImplementedError("fine_matches_for_pairs needs enable_fine_matching=True")
        pair_idx = torch.as_tensor(pair_idx, dtype=torch.int64).reshape(-1, 2)
        P = pair_idx.shape[0]
        offsets = torch.as_tensor(offsets, dtype=torch.int64).cpu()
        M = int(offsets[-1]) if P else 0
        if tuple(scales.shape) != (N, 2):
            raise ValueError(f"scales must be [N, 2] = [{N}, 2], got {tuple(scales.shape)}")
        if tuple(offsets.shape) != (P + 1,) or int(offsets[0]) != 0 or bool((offsets[1:] < offsets[:-1]).any()):
            raise ValueError("offsets must be int64 [P + 1], ascending from 0")
        if not (mkpts0_c.is_cuda and mkpts1_c.is_cuda and tuple(mkpts0_c.shape) == (M, 2) and mkpts1_c.shape == mkpts0_c.shape):
            raise ValueError(f"mkpts0_c / mkpts1_c must be CUDA tensors [{M}, 2]")
        if pair_idx.numel() and (int(pair_idx.min()) < 0 or int(pair_idx.max()) >= N):
            raise ValueError("pair_idx names an image outside [0, N)")
        if pair_batch < 1 or match_batch < 1:
            raise ValueError("pair_batch and match_batch must be >= 1")
        dev = images_u8.device
        with torch.cuda.device(dev):
            hc, wc, hf, wf = H // 8, W // 8, H // 2, W // 2
            scales = scales.to(device=dev, dtype=torch.float32).contiguous()
            pair_of = torch.repeat_interleave(torch.arange(P), offsets[1:] - offsets[:-1]).to(dev)
            pidx = pair_idx.to(dev)
            img0, img1 = pidx[pair_of, 0].contiguous(), pidx[pair_of, 1].contiguous()
            i_ids, j_ids = self._given_cells(mkpts0_c, mkpts1_c, (H, W), hc, wc, scales[img0], scales[img1])
            fine, coarse = self.image_maps(images_u8, image_chunk)
            imghw = (scales * torch.tensor([H, W], dtype=torch.float32, device=dev)).contiguous()
            res = {"i_ids": i_ids, "j_ids": j_ids, "expec_f": torch.empty((M, 3), device=dev),
                   "mkpts1_f": torch.empty_like(mkpts1_c),
                   "feat_coarse_b_0": torch.empty((M, 256), device=dev), "feat_coarse_b_1": torch.empty((M, 256), device=dev),
                   "feat_ext0": torch.empty((M, 128), device=dev), "feat_ext1": torch.empty((M, 128), device=dev)}
            off = offsets.tolist()
            p0 = 0
            while p0 < P:
                p1 = p0 + 1               # at least one pair, then up to pair_batch within match_batch
                while p1 < P and p1 - p0 < pair_batch and off[p1 + 1] - off[p0] <= match_batch:
                    p1 += 1
                a, b = off[p0], off[p1]
                p0 = p1
                if a == b:
                    continue
                m = b - a
                expec_f, delta = self._fine_given(fine, img0[a:b], img1[a:b], i_ids[a:b], j_ids[a:b], m, hc, wc, hf,
                                                  wf, H, scales)
                res["expec_f"][a:b] = expec_f
                res["mkpts1_f"][a:b] = mkpts1_c[a:b] + delta
                ext = self._extract(coarse, fine, img0[a:b], img1[a:b], mkpts0_c[a:b].contiguous(),
                                    res["mkpts1_f"][a:b].contiguous(), imghw, True, True)
                for k, v in ext.items():
                    res[k][a:b] = v
            return res
