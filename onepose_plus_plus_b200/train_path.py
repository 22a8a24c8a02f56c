"""Training-mode forward of ``OnePosePlus_model`` — differentiable PyTorch (autograd) path.

The sm_90a kernels of this package implement the *inference* forward; their backward passes are
not built.  ``train_onepose_plus.py`` (PL_OnePosePlus.training_step:
src/lightning_model/OnePosePlus_lightning_model.py:54-60) however calls ``self.matcher(batch)`` in
``.train()`` mode, back-propagates through ``conf_matrix`` / ``expec_f`` (losses.py:125-133) and
relies on the ground-truth padding of the coarse matches (coarse_matching.py:177-217).  So that the
drop-in keeps that script running, ``forward`` dispatches here whenever ``self.training`` is set:
the same parameters (the module tree of model.py holds ordinary nn.Conv2d / BatchNorm2d / Linear /
LayerNorm modules with the reference's names), evaluated with library PyTorch ops in the
reference's order, BatchNorm in batch-statistics mode exactly as ``nn.Module.train()`` leaves it.
This is the slow path by construction (SURVEY §8 f4 "keep the PyTorch path for self.training");
``.eval()`` always runs the CUDA kernels and never falls back to this module.  The one exception is
the coarse supervision: with ``model.conf_matrix_mode == "lazy"`` on CUDA tensors the L x S
confidence matrix is not built — the statistics and the match selection run on the inference
kernels and ``data["conf_matrix"]`` is a TrainConfHandle that ``losses.Loss`` differentiates with
the opp_coarse_focal kernels (DESIGN §7 f4).  With ``model.fine_train_mode == "kernels"`` on CUDA
tensors the fine level (fine_preprocess -> loftr_fine -> fine_matching) runs on the
opp_fine_train_* kernels instead (train_fine.py), and with model.coarse_transformer_train_mode ==
"kernels" the coarse transformer runs on the opp_coarse_tf_* kernels (train_coarse_tf.py).  With
model.backbone_train_mode == "kernels" the ResNet-FPN backbone runs on the opp_backbone_train_*
kernels, its convolutions on the tensor cores in 3xTF32, BatchNorm following each module's .training
(train_backbone.py).  With model.kpt_encoder_train_mode == "kernels" the keypoint-encoder MLP runs on
the opp_kpt_train_* kernels (train_kpt.py).  The ground truth the padding draws from is data["conf_matrix_gt"] or, in its place, the
correspondence list data["gt_sparse"] (train_gt.py).

Every function cites the reference lines it follows.
"""
import torch
import torch.nn.functional as F

from . import train_backbone, train_coarse_tf, train_fine, train_gt, train_kpt


def _block(blk, x):
    """BasicBlock.forward (backbone/resnet.py:36-45)"""
    y = F.relu(blk.bn1(blk.conv1(x)))
    y = blk.bn2(blk.conv2(y))
    if blk.downsample is not None:
        x = blk.downsample(x)
    return F.relu(x + y)


def backbone(bb, x):
    """ResNetFPN_8_2.forward (backbone/resnet.py:141-164), output_layers [3, 1]"""
    x0 = F.relu(bb.bn1(bb.conv1(x)))
    x1 = _block(bb.layer1[1], _block(bb.layer1[0], x0))
    x2 = _block(bb.layer2[1], _block(bb.layer2[0], x1))
    x3 = _block(bb.layer3[1], _block(bb.layer3[0], x2))
    x3_out = bb.layer3_outconv(x3)
    x3_up = F.interpolate(x3_out, scale_factor=2.0, mode="bilinear", align_corners=True)
    x2_out = bb.layer2_outconv2(bb.layer2_outconv(x2) + x3_up)
    x2_up = F.interpolate(x2_out, scale_factor=2.0, mode="bilinear", align_corners=True)
    x1_out = bb.layer1_outconv2(bb.layer1_outconv(x1) + x2_up)
    return x3_out, x1_out


def normalize_3d_keypoints(kpts):
    """utils/normalize.py:16-26 (extents of batch element 0, per-batch mean)"""
    ext = kpts[0].max(0).values - kpts[0].min(0).values
    return (kpts - kpts.mean(-2)[:, None]) / (ext.max() * 0.6)


def keypoint_encoding(enc, kpts, descriptors):
    """KeypointEncoding_linear.forward (utils/position_encoding.py:54-79): nn.InstanceNorm1d applied
    to [B, N, C] normalises each point over its C features (biased variance, eps 1e-5)."""
    x = kpts
    for m in enc.encoder:
        if isinstance(m, torch.nn.InstanceNorm1d):
            mu = x.mean(-1, keepdim=True)
            x = (x - mu) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + m.eps)
        else:
            x = m(x)
    return descriptors + x.transpose(2, 1)


def _linear_attention(q, k, v, q_mask=None, kv_mask=None, eps=1e-6):
    """LinearAttention.forward (loftr_module/linear_attention.py:29-61)"""
    Q, K = F.elu(q) + 1, F.elu(k) + 1
    if q_mask is not None:
        Q = Q * q_mask[:, :, None, None]
    if kv_mask is not None:
        K = K * kv_mask[:, :, None, None]
        v = v * kv_mask[:, :, None, None]
    v_len = v.size(1)
    v = v / v_len
    KV = torch.einsum("nshd,nshv->nhdv", K, v)
    Z = 1 / (torch.einsum("nlhd,nhd->nlh", Q, K.sum(1)) + eps)
    return (torch.einsum("nlhd,nhdv,nlh->nlhv", Q, KV, Z) * v_len).contiguous()


def _encoder_layer(layer, x, source, x_mask=None, source_mask=None):
    """LoFTREncoderLayer.forward (loftr_module/transformer.py:65-94)"""
    bs = x.size(0)
    q = layer.q_proj(x).view(bs, -1, layer.nhead, layer.dim)
    k = layer.k_proj(source).view(bs, -1, layer.nhead, layer.dim)
    v = layer.v_proj(source).view(bs, -1, layer.nhead, layer.dim)
    msg = _linear_attention(q, k, v, x_mask, source_mask)
    msg = layer.norm1(layer.merge(msg.view(bs, -1, layer.nhead * layer.dim)))
    msg = layer.norm2(layer.mlp(torch.cat([x, msg], 2)))
    return x + msg


def transformer(tf, desc3d, desc2d, query_mask=None):
    """LocalFeatureTransformer.forward (loftr_module/transformer.py:133-171): cross layers update
    both sequences from the pre-update tensors; the mask applies to the 2D side only."""
    d3 = desc3d.transpose(1, 2)
    d2 = desc2d
    for layer, name in zip(tf.layers, tf.layer_names):
        if name == "self":
            d2, d3 = _encoder_layer(layer, d2, d2, query_mask, query_mask), _encoder_layer(layer, d3, d3)
        else:
            d2, d3 = (_encoder_layer(layer, d2, d3, x_mask=query_mask),
                      _encoder_layer(layer, d3, d2, source_mask=query_mask))
    return d3, d2


@torch.no_grad()
def _coarse_matches(cm, conf, data, training):
    """CoarseMatching.get_coarse_match (utils/coarse_matching.py:125-242) including the training
    branch: a random subset of the predictions padded with ground-truth matches (:177-217)."""
    hc, wc = data["q_hw_c"]
    B, L, S = conf.shape
    mask = (conf > cm.thr).view(B, L, hc, wc).clone()
    if cm.border_rm > 0:     # mask_border (:10-20): the `-b:0` slices are empty, only top/left are cleared
        mask[:, :, :cm.border_rm] = False
        mask[:, :, :, :cm.border_rm] = False
    mask = mask.view(B, L, S)
    mask = mask * (conf == conf.max(2, keepdim=True)[0]) * (conf == conf.max(1, keepdim=True)[0])
    mask_v, all_j = mask.max(2)
    b_ids, i_ids = torch.where(mask_v)
    j_ids = all_j[b_ids, i_ids]
    mconf = conf[b_ids, i_ids, j_ids]
    return _pad_matches(cm, b_ids, i_ids, j_ids, mconf, (B, L, S), data, training)


@torch.no_grad()
def _pad_matches(cm, b_ids, i_ids, j_ids, mconf, shape, data, training):
    """get_coarse_match from the predicted matches on: training padding (:177-217), coordinates."""
    hc, wc = data["q_hw_c"]
    dev = b_ids.device
    B, L, S = shape
    tcfg = cm.config["train"]
    if training and tcfg["train_padding"]:
        n_max = int(B * min(L, S) * tcfg["train_coarse_percent"])
        n_pred = len(b_ids)
        pad_min = tcfg["train_pad_num_gt_min"]
        assert pad_min < n_max, "min-num-gt-pad should be less than num-train-matches"
        if n_pred <= n_max - pad_min:
            pred_idx = torch.arange(n_pred, device=dev)
        else:
            pred_idx = torch.randint(n_pred, (n_max - pad_min,), device=dev)
        gt = train_gt.gt_of(data)
        if gt is not None:      # the list is in the order of torch.where: the same draws pick the same paddings
            if tuple(gt.shape) != (B, L, S):
                raise ValueError(f"gt_sparse has shape {tuple(gt.shape)}, the confidence {(B, L, S)}")
            if gt.device != dev:
                raise ValueError(f"gt_sparse is on {gt.device}, the matches on {dev}")
            sb, si, sj = gt.b_ids, gt.i_ids, gt.j_ids
        else:
            sb, si, sj = torch.where(data["conf_matrix_gt"])
        assert len(sb) != 0
        pad_idx = torch.randint(len(sb), (max(n_max - n_pred, pad_min),), device=dev)
        zeros = torch.zeros(len(sb), device=dev)   # confidence of the gt paddings is 0
        b_ids, i_ids, j_ids, mconf = (torch.cat([x[pred_idx], y[pad_idx]], 0) for x, y in
                                      ((b_ids, sb), (i_ids, si), (j_ids, sj), (mconf, zeros)))
    scale = data["q_hw_i"][0] / hc
    scale_total = scale * data["query_image_scale"][b_ids][:, [1, 0]] if "query_image_scale" in data else scale
    mkpts_query = torch.stack([j_ids % wc, j_ids // wc], 1) * scale_total
    keep = mconf != 0
    return {"b_ids": b_ids, "i_ids": i_ids, "j_ids": j_ids, "gt_mask": mconf == 0, "m_bids": b_ids[keep],
            "mkpts_3d_db": data["keypoints3d"][b_ids, i_ids][keep], "mkpts_query_c": mkpts_query[keep],
            "mconf": mconf[keep]}


def dual_softmax(cm, feat3d, feat2d, mask_query):
    """conf_matrix of CoarseMatching.forward (utils/coarse_matching.py:96-119), with autograd"""
    c = feat3d.shape[-1]
    sim = torch.einsum("nlc,nsc->nls", feat3d / c ** 0.5, feat2d / c ** 0.5) / (cm.temperature + 1e-4)
    if mask_query is not None:
        neg = torch.zeros_like(sim)
        neg[~mask_query.bool()[:, None].expand_as(sim)] = -1e9
        sim = sim + neg
    return F.softmax(sim, 1) * F.softmax(sim, 2)


def coarse_matching(cm, feat3d, feat2d, data, mask_query, training, lazy_split=None):
    """CoarseMatching.forward (utils/coarse_matching.py:76-123).  lazy_split (CUDA, the model's
    conf_matrix_mode "lazy"): the matrix is not built; data["conf_matrix"] is a TrainConfHandle and
    the matches come from the inference kernels (split = the model's fp16x3 operand mode)."""
    if lazy_split is None:
        conf = dual_softmax(cm, feat3d, feat2d, mask_query)
        data["conf_matrix"] = conf
        data.update(_coarse_matches(cm, conf, data, training))
        return
    handle, b_ids, i_ids, j_ids, mconf = _lazy_coarse(cm, feat3d, feat2d, data, mask_query, lazy_split)
    data["conf_matrix"] = handle
    data.update(_pad_matches(cm, b_ids, i_ids, j_ids, mconf, tuple(handle.shape), data, training))


class TrainConfHandle:
    """data["conf_matrix"] in training with conf_matrix_mode "lazy": the autograd-connected features
    and the softmax statistics of their fp32 sim (opp_coarse_focal_stats — the same sim the loss
    kernels recompute), instead of the [B, L, S] matrix.  onepose_plus_plus_b200.losses.Loss
    evaluates the coarse loss and its backward from it.
      .shape        torch.Size([B, L, S])
      .max()        max of the matrix (detached 0-d tensor, from the selection pass's row maxima)
      .materialize() the matrix the eager mode writes, with autograd (same formula)."""

    def __init__(self, cm, feat3d, feat2d, mask_query, rowmax=None):
        from . import ops
        B, L, C = feat3d.shape
        S = feat2d.shape[1]
        self.cm, self.feat3d, self.feat2d, self.mask_query = cm, feat3d, feat2d, mask_query
        self.scale = 1.0 / (C * (cm.temperature + 1e-4))    # (a / sqrt(C)) . (b / sqrt(C)) / (T + 1e-4)
        self.shape = torch.Size((B, L, S))
        with torch.no_grad():
            self.a32 = feat3d.detach().float().contiguous()
            self.b32 = feat2d.detach().float().contiguous()
            self.col_mask = (mask_query != 0).to(torch.uint8).reshape(B, S).contiguous() \
                if mask_query is not None else None
            self.st_rows, self.st_cols = ops.coarse_focal_stats(self.a32, self.b32, self.col_mask, self.scale)
        self._rowmax = rowmax

    def max(self):
        if self._rowmax is None:
            raise RuntimeError("this handle was built without the selection pass's row maxima")
        return self._rowmax.max()

    def materialize(self):
        return dual_softmax(self.cm, self.feat3d, self.feat2d, self.mask_query)


@torch.no_grad()
def _lazy_coarse(cm, feat3d, feat2d, data, mask_query, split):
    """Match selection with the inference kernels (opp_sim_lse_cols + finalisers on fp16 hi/lo planes,
    opp_sim_conf_colmax, opp_match_select_colmax): threshold, top/left border, mutual nearest
    neighbour by value, matches in (b, l) order, mconf = the row maxima.  The loss statistics of the
    handle are computed separately, from the fp32 features (TrainConfHandle)."""
    from . import ops
    B, L, C = feat3d.shape
    S = feat2d.shape[1]
    hc, wc = data["q_hw_c"]
    dev, f32, i32, i64 = feat3d.device, torch.float32, torch.int32, torch.int64
    scale = 1.0 / (C * (cm.temperature + 1e-4))
    a16, b16 = ops.to_planes(feat3d.detach().float(), split), ops.to_planes(feat2d.detach().float(), split)
    col_mask = (mask_query != 0).to(torch.uint8).reshape(B, S).contiguous() if mask_query is not None else None
    ts, groups = ops.sim_tiles(S), (L + 31) // 32
    pm, ps = torch.empty(B * L, ts, dtype=f32, device=dev), torch.empty(B * L, ts, dtype=f32, device=dev)
    lse_rows, lse_cols = torch.empty(B, L, dtype=f32, device=dev), torch.empty(B, S, dtype=f32, device=dev)
    col_m, col_s = (torch.empty(B, groups, S, dtype=f32, device=dev) for _ in range(2))
    ops.sim_lse_cols(a16, b16, B, L, S, C, scale, pm, ps, lse_rows, col_m, col_s, lse_cols, split,
                     col_mask=col_mask)
    del col_m, col_s, ps
    pi = torch.empty(B * L, ts, dtype=i32, device=dev)
    rowmax, rowarg = torch.empty(B, L, dtype=f32, device=dev), torch.empty(B, L, dtype=i32, device=dev)
    colmax = torch.empty(B, S, dtype=i32, device=dev)
    ops.sim_conf_colmax(a16, b16, lse_rows, lse_cols, None, B, L, S, C, scale, pm, pi, rowmax, rowarg, colmax,
                        split)
    del a16, b16, pm, pi
    cap = B * L
    ids = [torch.empty(cap, dtype=i64, device=dev) for _ in range(3)]
    mconf = torch.empty(cap, dtype=f32, device=dev)
    count = torch.empty(1, dtype=i32, device=dev)
    ops.match_select_colmax(rowmax, rowarg, colmax, data["keypoints3d"].detach().float().contiguous(), None, B, L,
                            hc, wc, cm.thr, cm.border_rm, 1.0,
                            torch.empty((cap + 1023) // 1024 + 2, dtype=i32, device=dev), *ids, mconf,
                            torch.empty(cap, 3, dtype=f32, device=dev), torch.empty(cap, 2, dtype=f32, device=dev),
                            count)
    n = int(count.item())
    handle = TrainConfHandle(cm, feat3d, feat2d, mask_query, rowmax)
    return (handle, *(t[:n] for t in ids), mconf[:n])


def fine_preprocess(W, d_model, data, desc3d_db, feat_f):
    """FinePreprocess.forward (loftr_module/fine_preprocess.py:32-55)"""
    data["W"] = W
    if data["b_ids"].shape[0] == 0:
        return (torch.empty(0, d_model, 1, device=feat_f.device),
                torch.empty(0, W * W, d_model, device=feat_f.device))
    stride = data["q_hw_f"][0] // data["q_hw_c"][0]
    unf = F.unfold(feat_f, kernel_size=(W, W), stride=stride, padding=W // 2)
    n, cww, l = unf.shape
    unf = unf.view(n, cww // (W * W), W * W, l).permute(0, 3, 2, 1)   # 'n (c ww) l -> n l ww c'
    f3d = desc3d_db.permute(0, 2, 1)[data["b_ids"], data["i_ids"], :].unsqueeze(-1)
    return f3d, unf[data["b_ids"], data["j_ids"]]


def fine_matching(feat3d, feat2d, data, training):
    """FineMatching.forward (utils/fine_matching.py:28-110), s2d heatmap"""
    M, WW, C = feat2d.shape
    W = int(WW ** 0.5)
    scale = data["q_hw_i"][0] / data["q_hw_f"][0]
    if M == 0:
        assert not training, "M is always >0, when training, see coarse_matching.py"
        data.update({"expec_f": torch.empty(0, 3, device=feat3d.device), "mkpts_query_f": data["mkpts_query_c"]})
        return
    f0 = feat3d[:, feat3d.shape[1] // 2, :]
    heat = torch.softmax(torch.einsum("mc,mrc->mr", f0, feat2d) / C ** 0.5, 1)
    lin = torch.linspace(-1, 1, W, device=heat.device)
    grid = torch.stack([lin.repeat(W), lin.repeat_interleave(W)], 1)     # (x, y), x fastest
    coords = heat @ grid
    var = heat @ grid ** 2 - coords ** 2
    std = torch.sqrt(torch.clamp(var, min=1e-10)).sum(-1)
    data["expec_f"] = torch.cat([coords, std[:, None]], -1)
    with torch.no_grad():
        qs = scale * data["query_image_scale"][data["b_ids"]][:, [1, 0]] if "query_image_scale" in data else scale
        data["mkpts_query_f"] = data["mkpts_query_c"] + (coords * (W // 2) * qs)[: len(data["mkpts_query_c"])]


def forward_train(model, data):
    """OnePosePlus_model.forward (OnePosePlusModel.py:96-201) with autograd, module in train mode."""
    cfg = model.config
    mode = model.conf_matrix_mode
    if mode == "skip":
        raise ValueError('conf_matrix_mode "skip" cannot train: the coarse loss reads data["conf_matrix"] '
                         '(use "lazy" for the matrix-free handle)')
    if model.loftr_backbone_pretrained and cfg["loftr_backbone"]["pretrained_fix"]:
        model.backbone.eval()                                      # OnePosePlusModel.py:109-113
    img = data["query_image"]
    lazy_split = model.split if mode == "lazy" and img.is_cuda else None
    if lazy_split is False:
        # single fp16 operands would select matches from a sim that differs from the eager fp32 one
        raise ValueError('conf_matrix_mode "lazy" in train mode needs precision "fp16x3" (the match '
                         'selection runs on the fp32-grade split operands)')
    fine_kernels = train_fine.use_kernels(model, data)
    coarse_tf_kernels = train_coarse_tf.use_kernels(model, data)
    backbone_kernels = train_backbone.use_kernels(model, data)
    kpt_kernels = train_kpt.use_kernels(model, data)
    data.update({"bs": img.size(0), "q_hw_i": img.shape[2:]})
    if backbone_kernels:
        feat_c, feat_f = train_backbone.backbone(model.backbone, img)
    else:
        feat_c, feat_f = backbone(model.backbone, img)
    data.update({"q_hw_c": feat_c.shape[2:], "q_hw_f": feat_f.shape[2:]})
    if model.dense_pos_encoding is not None:
        feat_c = feat_c + model.dense_pos_encoding.pe[:, :, :feat_c.size(2), :feat_c.size(3)]
    q_c = feat_c.flatten(2).transpose(1, 2)                        # 'n c h w -> n (h w) c'
    dsel = data["descriptors3d_coarse_db"] if "descriptors3d_coarse_db" in data else data["descriptors3d_db"]
    if kpt_kernels:
        d3 = train_kpt.keypoint_encoding(model.kpt_3d_pos_encoding, data["keypoints3d"], dsel)
    else:
        d3 = keypoint_encoding(model.kpt_3d_pos_encoding, normalize_3d_keypoints(data["keypoints3d"]), dsel)
    qmask = data["query_image_mask"].flatten(-2) if "query_image_mask" in data else None
    if coarse_tf_kernels:
        d3, q_c = train_coarse_tf.coarse_transformer(model.loftr_coarse, d3, q_c, qmask)
    else:
        d3, q_c = transformer(model.loftr_coarse, d3, q_c, qmask)
    coarse_matching(model.coarse_matching, d3, q_c, data, qmask, model.training, lazy_split)
    if not cfg["fine_matching"]["enable"]:
        data.update({"mkpts_query_f": data["mkpts_query_c"]})
        return
    if fine_kernels:
        train_fine.fine_stage(model, data, feat_f)
        return
    f3d, f2d = fine_preprocess(model.fine_preprocess.W, cfg["loftr_fine"]["d_model"], data,
                               data["descriptors3d_db"], feat_f)
    if f2d.size(0) != 0 and cfg["loftr_fine"]["enable"]:
        f3d, f2d = transformer(model.loftr_fine, f3d, f2d)
    else:
        f3d = f3d.transpose(1, 2)
    fine_matching(f3d, f2d, data, model.training)
