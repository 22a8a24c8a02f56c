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
``.eval()`` always runs the CUDA kernels and never falls back to this module.

Every function cites the reference lines it follows.
"""
import torch
import torch.nn.functional as F


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
    dev = conf.device
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


def coarse_matching(cm, feat3d, feat2d, data, mask_query, training):
    """CoarseMatching.forward (utils/coarse_matching.py:76-123)"""
    c = feat3d.shape[-1]
    sim = torch.einsum("nlc,nsc->nls", feat3d / c ** 0.5, feat2d / c ** 0.5) / (cm.temperature + 1e-4)
    if mask_query is not None:
        neg = torch.zeros_like(sim)
        neg[~mask_query.bool()[:, None].expand_as(sim)] = -1e9
        sim = sim + neg
    conf = F.softmax(sim, 1) * F.softmax(sim, 2)
    data["conf_matrix"] = conf
    data.update(_coarse_matches(cm, conf, data, training))


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
    if model.loftr_backbone_pretrained and cfg["loftr_backbone"]["pretrained_fix"]:
        model.backbone.eval()                                      # OnePosePlusModel.py:109-113
    img = data["query_image"]
    data.update({"bs": img.size(0), "q_hw_i": img.shape[2:]})
    feat_c, feat_f = backbone(model.backbone, img)
    data.update({"q_hw_c": feat_c.shape[2:], "q_hw_f": feat_f.shape[2:]})
    if model.dense_pos_encoding is not None:
        feat_c = feat_c + model.dense_pos_encoding.pe[:, :, :feat_c.size(2), :feat_c.size(3)]
    q_c = feat_c.flatten(2).transpose(1, 2)                        # 'n c h w -> n (h w) c'
    dsel = data["descriptors3d_coarse_db"] if "descriptors3d_coarse_db" in data else data["descriptors3d_db"]
    d3 = keypoint_encoding(model.kpt_3d_pos_encoding, normalize_3d_keypoints(data["keypoints3d"]), dsel)
    qmask = data["query_image_mask"].flatten(-2) if "query_image_mask" in data else None
    d3, q_c = transformer(model.loftr_coarse, d3, q_c, qmask)
    coarse_matching(model.coarse_matching, d3, q_c, data, qmask, model.training)
    if not cfg["fine_matching"]["enable"]:
        data.update({"mkpts_query_f": data["mkpts_query_c"]})
        return
    f3d, f2d = fine_preprocess(model.fine_preprocess.W, cfg["loftr_fine"]["d_model"], data,
                               data["descriptors3d_db"], feat_f)
    if f2d.size(0) != 0 and cfg["loftr_fine"]["enable"]:
        f3d, f2d = transformer(model.loftr_fine, f3d, f2d)
    else:
        f3d = f3d.transpose(1, 2)
    fine_matching(f3d, f2d, data, model.training)
