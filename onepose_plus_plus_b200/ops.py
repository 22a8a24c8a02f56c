"""Thin tensor-level wrappers over the C ABI (include/opp_b200.h).  Each wrapper checks dtype /
contiguity, passes raw device pointers and the current CUDA stream, and raises on error.  There
is deliberately no alternative code path: without libopp_b200.so these functions raise."""
import torch

from . import _lib

ptr, call, stream = _lib.ptr, _lib.call, _lib.stream


def to_planes(x, split):
    """fp32 tensor [..., C] -> fp16 storage [..., planes*C]: (hi | lo) planes when split."""
    hi = x.half()
    if not split:
        return hi.contiguous()
    lo = (x - hi.float()).half()
    return torch.cat([hi, lo], -1).contiguous()


def from_planes(t, split):
    """Inverse of to_planes (returns fp32)."""
    if not split:
        return t.float()
    c = t.shape[-1] // 2
    return t[..., :c].float() + t[..., c:].float()


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def conv1_gemm(image, w64, a_buf, out, split):
    """conv1 7x7/2 + folded BN + ReLU as im2col + ONE 64-wide wgmma K chunk (bias rides in K column
    49).  image fp32 or uint8 [B,1,H,W]; w64 fp16 [C, planes*64]; a_buf fp16 [B*H/2*W/2, planes*64]."""
    B, _, H, W = image.shape
    if image.dtype not in (torch.float32, torch.uint8):
        raise TypeError(f"image: expected float32 or uint8, got {image.dtype}")
    call("opp_conv1_im2col", ptr(image), int(image.dtype == torch.uint8), ptr(a_buf), B, H, W, int(split),
         stream())
    rows = B * (H // 2) * (W // 2)
    call("opp_linear_act_f16", ptr(a_buf), 64, None, 0, ptr(w64), ptr(out), rows, w64.shape[0], 1,
         (w64.shape[0] + 31) // 32 * 32, int(split), stream())
    return out


def conv2d_nhwc(x, w, bias, out, ksize, stride, split, act=0, resid=None, slope=0.01, tok=None,
                pe=None, up=None):
    """x NHWC fp16 [B,H,W,planes*Cin_pad]; w fp16 [Cout_pad, planes*k*k*Cin_pad];
    act 0 none / 1 relu / 2 leaky; up: coarser NHWC map added as bilinear x2 (align_corners)."""
    _chk(x, torch.float16, "x")
    _chk(w, torch.float16, "w")
    _chk(resid, torch.float16, "resid")
    B, H, W, C = x.shape
    planes = 2 if split else 1
    call("opp_conv2d_nhwc", ptr(x), ptr(w), ptr(bias), ptr(resid), ptr(out), B, H, W, C // planes,
         w.shape[0], ksize, stride, act, float(slope), ptr(tok), ptr(pe), ptr(up), int(split), stream())
    return out


def kpt_encode(kpts, desc, mlp, stats, tok, split):
    B, N, _ = kpts.shape
    _chk(kpts, torch.float32, "keypoints3d")
    _chk(desc, torch.float32, "descriptors3d")
    call("opp_kpt_stats", ptr(kpts), ptr(stats), B, N, stream())
    (w1, b1), (w2, b2), (w3, b3), (w4, b4) = mlp
    call("opp_kpt_encode", ptr(kpts), ptr(stats), ptr(desc), ptr(w1), ptr(b1), ptr(w2), ptr(b2),
         ptr(w3), ptr(b3), ptr(w4), ptr(b4), ptr(tok), B, N, int(split), stream())


def linear_act(a0, a1, w, out, rows, act, act_cols, split, out_split=None, batches=1, a0_shared=False,
               count=None, rows_per_count=1, row_mask=None):
    """a_i fp16 [rows, planes*k_i]; w fp16 [n, planes*(k0+k1)]; out fp16 [rows, planes*n]
    (out_split=False with split=True: split operands, single-plane output [rows, n]).
    batches > 1: rows is per batch; a0_shared: a0 is [1, rows, ..] shared by every batch.
    count (int32 device tensor): `rows` is the capacity, the kernel uses count * rows_per_count rows.
    row_mask (uint8 [batches*rows]): rows with mask 0 are written as zeros."""
    _chk(row_mask, torch.uint8, "row_mask")
    _chk(a0, torch.float16, "a0")
    _chk(a1, torch.float16, "a1")
    _chk(w, torch.float16, "w")
    planes = 2 if split else 1
    k0 = a0.shape[-1] // planes
    k1 = a1.shape[-1] // planes if a1 is not None else 0
    if split and out_split is False:
        call("opp_linear_act_f16_out1", ptr(a0), k0, ptr(a1), k1, ptr(w), ptr(out), rows, w.shape[0], act,
             act_cols, ptr(row_mask), stream())
        return out
    if count is not None:
        call("opp_linear_act_f16_dyn", ptr(a0), k0, ptr(a1), k1, ptr(w), ptr(out), rows, ptr(count),
             rows_per_count, w.shape[0], act, act_cols, int(split), stream())
        return out
    if batches > 1 or a0_shared or row_mask is not None:
        call("opp_linear_act_f16_b", ptr(a0), k0, int(a0_shared), ptr(a1), k1, ptr(w), ptr(out), batches, rows,
             w.shape[0], act, act_cols, int(split), ptr(row_mask), stream())
        return out
    call("opp_linear_act_f16", ptr(a0), k0, ptr(a1), k1, ptr(w), ptr(out), rows, w.shape[0], act,
         act_cols, int(split), stream())
    return out


def linear_q(x16, wq, ksum, out, batches, rows, v_len, split, eps=1e-6, x_shared=False, row_mask=None):
    _chk(row_mask, torch.uint8, "row_mask")
    call("opp_linear_q_f16", ptr(x16), ptr(wq), ptr(ksum), ptr(out), batches, rows, wq.shape[0],
         float(v_len), float(eps), int(split), int(x_shared), ptr(row_mask), stream())
    return out


def linear_ln(a0, a1, w, w_batched, gamma, beta, batches, rows, split, resid=None, out16=None,
              out32=None, eps=1e-5, resid_shared=False, count=None, rows_per_count=1):
    _chk(a0, torch.float16, "a0")
    _chk(w, torch.float16, "w")
    _chk(resid, torch.float16, "resid")
    planes = 2 if split else 1
    k0 = a0.shape[-1] // planes
    k1 = a1.shape[-1] // planes if a1 is not None else 0
    n = w.shape[-2]
    if count is not None:
        call("opp_linear_ln_dyn", ptr(a0), k0, ptr(a1), k1, ptr(w), ptr(gamma), ptr(beta), float(eps),
             ptr(resid), ptr(out16), ptr(out32), rows, ptr(count), rows_per_count, n, int(split), stream())
        return
    call("opp_linear_ln", ptr(a0), k0, ptr(a1), k1, ptr(w), int(w_batched), ptr(gamma), ptr(beta),
         float(eps), ptr(resid), int(resid_shared), ptr(out16), ptr(out32), batches, rows, n, int(split),
         stream())


def full_attention(q16, kv16, out, batch, l, s, heads, head_dim, split):
    """softmax(Q K^T / sqrt(D)) V per head (attention: "full"); q16 [B*l, planes*H*D], kv16 [B*s, planes*2*H*D]."""
    _chk(q16, torch.float16, "q")
    _chk(kv16, torch.float16, "kv")
    call("opp_full_attention", ptr(q16), ptr(kv16), ptr(out), batch, l, s, heads, head_dim, int(split), stream())
    return out


def kv_chunks(s, batches=None):
    """Chunks per batch element of the K'V partial states (size of the `part` buffer)."""
    if batches is None:
        return _lib.load().opp_kv_chunks(s)
    return _lib.load().opp_kv_chunks_b(s, batches)


def kv_state(kv16, part, merge_w, mt, ksum, batches, s, d, v_len, split):
    """kv16: single-plane fp16 K'/V rows [batches * s, 2d]; split: plane mode of the mt output."""
    call("opp_kv_partial", ptr(kv16), ptr(part), batches, s, d, stream())
    call("opp_kv_finalize", ptr(part), ptr(merge_w), ptr(mt), ptr(ksum), batches, kv_chunks(s, batches), d,
         float(v_len), int(split), stream())


def sim_tiles(cols):
    return _lib.load().opp_sim_tiles(cols)


def sim_lse_cols(a, b, batches, rows, cols, k, scale, part_m, part_s, lse_rows, col_m, col_s, lse_cols,
                 split, col_mask=None, side_stream=None, row_count=None):
    """lse over columns for every row AND lse over rows for every column, one GEMM pass.
    col_mask uint8 [batches, cols]: masked columns (0) get sim - 1e9 and lse_cols = +inf (conf = 0).
    row_count int32 [batches] (bank sets): rows past the count drop out of lse_cols; their lse_rows
    are not meaningful.
    side_stream (latency mode): the two independent finalisers run side by side."""
    _chk(col_mask, torch.uint8, "col_mask")
    _chk(row_count, torch.int32, "row_count")
    tiles = sim_tiles(cols)
    groups = (rows + 31) // 32
    if row_count is not None:
        call("opp_sim_lse_cols_rows", ptr(a), ptr(b), ptr(part_m), ptr(part_s), ptr(col_m), ptr(col_s), batches,
             rows, cols, k, float(scale), int(split), ptr(col_mask), ptr(row_count), stream())
    else:
        call("opp_sim_lse_cols", ptr(a), ptr(b), ptr(part_m), ptr(part_s), ptr(col_m), ptr(col_s), batches,
             rows, cols, k, float(scale), int(split), ptr(col_mask), stream())
    if side_stream is not None:
        cur = torch.cuda.current_stream()
        side_stream.wait_stream(cur)
        with torch.cuda.stream(side_stream):
            call("opp_lse_finalize", ptr(part_m), ptr(part_s), ptr(lse_rows), batches * rows, tiles, stream())
    else:
        call("opp_lse_finalize", ptr(part_m), ptr(part_s), ptr(lse_rows), batches * rows, tiles, stream())
    call("opp_lse_col_finalize", ptr(col_m), ptr(col_s), ptr(lse_cols), batches, groups, cols, ptr(col_mask),
         stream())
    if side_stream is not None:
        cur.wait_stream(side_stream)


def sim_conf_colmax(a, b, lse_own, lse_other, conf, batches, rows, cols, k, scale, part_val, part_idx,
                    best_val, best_idx, colmax, split, row_count=None):
    """conf pass over rows = 3D points that also leaves max_l conf[b, l, s] (float bits) in colmax.
    row_count int32 [batches] (bank sets): rows past the count stay out of colmax and store conf 0."""
    _chk(row_count, torch.int32, "row_count")
    tiles = sim_tiles(cols)
    if row_count is not None:
        call("opp_sim_conf_colmax_rows", ptr(a), ptr(b), ptr(lse_own), ptr(lse_other), ptr(conf), ptr(part_val),
             ptr(part_idx), ptr(colmax), batches, rows, cols, k, float(scale), int(split), ptr(row_count), stream())
    else:
        call("opp_sim_conf_colmax", ptr(a), ptr(b), ptr(lse_own), ptr(lse_other), ptr(conf), ptr(part_val),
             ptr(part_idx), ptr(colmax), batches, rows, cols, k, float(scale), int(split), stream())
    call("opp_best_finalize", ptr(part_val), ptr(part_idx), ptr(best_val), ptr(best_idx),
         batches * rows, tiles, stream())


def match_select_colmax(pt_val, pt_idx, colmax, kpts, img_scale, batch, l, hc, wc, thr, border, cell,
                        scratch, b_ids, i_ids, j_ids, mconf, mkpts3d, mkpts_c, count, bank_shared=False,
                        bank_of_batch=None, row_count=None):
    """bank_of_batch / row_count int32 [batch] (bank sets, both or neither): kpts is [K, l, 3], read at
    the frame's object, and rows past the frame's count never match."""
    if bank_of_batch is not None or row_count is not None:
        _chk(bank_of_batch, torch.int32, "bank_of_batch")
        _chk(row_count, torch.int32, "row_count")
        call("opp_match_select_colmax_set", ptr(pt_val), ptr(pt_idx), ptr(colmax), ptr(kpts), ptr(img_scale),
             batch, l, hc, wc, float(thr), int(border), float(cell), ptr(scratch), ptr(b_ids),
             ptr(i_ids), ptr(j_ids), ptr(mconf), ptr(mkpts3d), ptr(mkpts_c), ptr(count), int(bank_shared),
             ptr(bank_of_batch), ptr(row_count), stream())
        return
    call("opp_match_select_colmax", ptr(pt_val), ptr(pt_idx), ptr(colmax), ptr(kpts), ptr(img_scale),
         batch, l, hc, wc, float(thr), int(border), float(cell), ptr(scratch), ptr(b_ids),
         ptr(i_ids), ptr(j_ids), ptr(mconf), ptr(mkpts3d), ptr(mkpts_c), ptr(count), int(bank_shared), stream())


GT_BYTES = {torch.bool: 1, torch.uint8: 1, torch.int16: 2}


def _gt_bytes(gt):
    if gt.dtype not in GT_BYTES:
        raise TypeError(f"conf_matrix_gt: expected bool, uint8 or int16, got {gt.dtype}")
    _chk(gt, gt.dtype, "conf_matrix_gt")
    return GT_BYTES[gt.dtype]


def coarse_focal_stats(a, b, col_mask, scale):
    """Softmax statistics of sim = scale * a b^T over each row / column, from the same fp32 sim the
    focal kernels recompute: (st_rows [B,L,2], st_cols [B,S,2]) = (max, log sum exp(sim - max))."""
    _chk(a, torch.float32, "feat3d")
    _chk(b, torch.float32, "feat2d")
    _chk(col_mask, torch.uint8, "col_mask")
    B, L, K = a.shape
    S = b.shape[1]
    nb = _lib.load().opp_coarse_focal_blocks(L)
    dev, f32 = a.device, torch.float32
    part_c = torch.empty(B, nb, S, 2, dtype=f32, device=dev)
    st_rows = torch.empty(B, L, 2, dtype=f32, device=dev)
    st_cols = torch.empty(B, S, 2, dtype=f32, device=dev)
    call("opp_coarse_focal_stats", ptr(a), ptr(b), ptr(col_mask), B, L, S, K, float(scale), ptr(part_c),
         ptr(st_rows), ptr(st_cols), stream())
    return st_rows, st_cols


def coarse_focal_fwd(a, b, st_rows, st_cols, gt, col_mask, scale, alpha, gamma, pos_w, neg_w):
    """Focal loss of the dual-softmax confidence (losses.py:18-58) from fp32 features a [B,L,256],
    b [B,S,256] and their coarse_focal_stats (st_rows, st_cols); returns (loss [1], counts int64
    [2] = (npos, nneg), wts [2], r [B,L], c [B,S]) — the last three are what coarse_focal_bwd reads."""
    _chk(a, torch.float32, "feat3d")
    _chk(b, torch.float32, "feat2d")
    _chk(col_mask, torch.uint8, "col_mask")
    gb = _gt_bytes(gt)
    B, L, K = a.shape
    S = b.shape[1]
    nb = _lib.load().opp_coarse_focal_blocks(L)
    dev, f32 = a.device, torch.float32
    part_loss = torch.empty(B * nb, 2, dtype=torch.float64, device=dev)
    part_cnt = torch.empty(B * nb, 2, dtype=torch.int64, device=dev)
    part_r = torch.empty(B, L, 2, dtype=torch.float64, device=dev)
    part_c = torch.empty(B, nb, S, 2, dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=f32, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    wts = torch.empty(2, dtype=f32, device=dev)
    r = torch.empty(B, L, dtype=torch.float64, device=dev)
    c = torch.empty(B, S, dtype=torch.float64, device=dev)
    call("opp_coarse_focal_fwd", ptr(a), ptr(b), ptr(st_rows), ptr(st_cols), ptr(gt), gb, ptr(col_mask), B, L,
         S, K, float(scale), float(alpha), float(gamma), float(pos_w), float(neg_w), ptr(part_loss),
         ptr(part_cnt), ptr(part_r), ptr(part_c), ptr(loss), ptr(counts), ptr(wts), ptr(r), ptr(c), stream())
    return loss, counts, wts, r, c


def coarse_focal_bwd(a, b, st_rows, st_cols, r, c, wts, grad, gt, col_mask, scale, alpha, gamma):
    """(d loss / d a, d loss / d b) * grad, grad a device scalar."""
    _chk(a, torch.float32, "feat3d")
    _chk(b, torch.float32, "feat2d")
    _chk(grad, torch.float32, "grad")
    _chk(col_mask, torch.uint8, "col_mask")
    gb = _gt_bytes(gt)
    B, L, K = a.shape
    S = b.shape[1]
    da, db = torch.empty_like(a), torch.empty_like(b)
    call("opp_coarse_focal_bwd", ptr(a), ptr(b), ptr(st_rows), ptr(st_cols), ptr(r), ptr(c), ptr(wts), ptr(grad),
         ptr(gt), gb, ptr(col_mask), B, L, S, K, float(scale), float(alpha), float(gamma), ptr(da), ptr(db),
         stream())
    return da, db


def _chk_gt_list(b_ids, i_ids, j_ids):
    for name, t in (("b_ids", b_ids), ("i_ids", i_ids), ("j_ids", j_ids)):
        _chk(t, torch.int64, "gt_sparse." + name)
    if not (b_ids.shape == i_ids.shape == j_ids.shape and b_ids.dim() == 1):
        raise ValueError("gt_sparse: b_ids, i_ids and j_ids must be 1-d tensors of one length")
    if b_ids.numel() >= 2 ** 31:
        raise ValueError("gt_sparse: more than 2^31 - 1 correspondences")


def gt_index(b_ids, i_ids, j_ids, shape):
    """Row and column index of a ground-truth list sorted by (b, i, j): (row_ptr int32 [B*L+1],
    col_ptr int32 [B*S+1], col_rows int32 [G] = the i of each column's entries, ascending)."""
    _chk_gt_list(b_ids, i_ids, j_ids)
    B, L, S = shape
    G, dev, i32 = b_ids.numel(), b_ids.device, torch.int32
    row_ptr = torch.empty(B * L + 1, dtype=i32, device=dev)
    col_ptr = torch.empty(B * S + 1, dtype=i32, device=dev)
    col_rows = torch.empty(G, dtype=i32, device=dev)
    fill = torch.empty(B * S, dtype=i32, device=dev)
    call("opp_gt_index", ptr(b_ids), ptr(i_ids), ptr(j_ids), G, B, L, S, ptr(row_ptr), ptr(col_ptr), ptr(col_rows),
         ptr(fill), stream())
    return row_ptr, col_ptr, col_rows


def coarse_focal_fwd_sparse(a, b, st_rows, st_cols, row_ptr, j_ids, col_mask, scale, alpha, gamma, pos_w, neg_w):
    """coarse_focal_fwd with the positives given as a list (row_ptr from gt_index, the list's j_ids):
    the same outputs, bit for bit, as the dense call on the dense form of the list."""
    _chk(a, torch.float32, "feat3d")
    _chk(b, torch.float32, "feat2d")
    _chk(col_mask, torch.uint8, "col_mask")
    _chk(row_ptr, torch.int32, "row_ptr")
    _chk(j_ids, torch.int64, "gt_sparse.j_ids")
    B, L, K = a.shape
    S = b.shape[1]
    if row_ptr.numel() != B * L + 1:
        raise ValueError(f"row_ptr has {row_ptr.numel()} entries, the features need {B * L + 1}")
    nb = _lib.load().opp_coarse_focal_blocks(L)
    dev, f32 = a.device, torch.float32
    part_loss = torch.empty(B * nb, 2, dtype=torch.float64, device=dev)
    part_cnt = torch.empty(B * nb, 2, dtype=torch.int64, device=dev)
    part_r = torch.empty(B, L, 2, dtype=torch.float64, device=dev)
    part_c = torch.empty(B, nb, S, 2, dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=f32, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    wts = torch.empty(2, dtype=f32, device=dev)
    r = torch.empty(B, L, dtype=torch.float64, device=dev)
    c = torch.empty(B, S, dtype=torch.float64, device=dev)
    call("opp_coarse_focal_fwd_sparse", ptr(a), ptr(b), ptr(st_rows), ptr(st_cols), ptr(row_ptr), ptr(j_ids),
         ptr(col_mask), B, L, S, K, float(scale), float(alpha), float(gamma), float(pos_w), float(neg_w),
         ptr(part_loss), ptr(part_cnt), ptr(part_r), ptr(part_c), ptr(loss), ptr(counts), ptr(wts), ptr(r), ptr(c),
         stream())
    return loss, counts, wts, r, c


def coarse_focal_bwd_sparse(a, b, st_rows, st_cols, r, c, wts, grad, row_ptr, j_ids, col_ptr, col_rows, col_mask,
                            scale, alpha, gamma):
    """coarse_focal_bwd with the positives given as a list and its gt_index."""
    _chk(a, torch.float32, "feat3d")
    _chk(b, torch.float32, "feat2d")
    _chk(grad, torch.float32, "grad")
    _chk(col_mask, torch.uint8, "col_mask")
    for name, t in (("row_ptr", row_ptr), ("col_ptr", col_ptr), ("col_rows", col_rows)):
        _chk(t, torch.int32, name)
    _chk(j_ids, torch.int64, "gt_sparse.j_ids")
    B, L, K = a.shape
    S = b.shape[1]
    if row_ptr.numel() != B * L + 1 or col_ptr.numel() != B * S + 1:
        raise ValueError("row_ptr / col_ptr do not belong to features of this shape")
    da, db = torch.empty_like(a), torch.empty_like(b)
    call("opp_coarse_focal_bwd_sparse", ptr(a), ptr(b), ptr(st_rows), ptr(st_cols), ptr(r), ptr(c), ptr(wts),
         ptr(grad), ptr(row_ptr), ptr(j_ids), ptr(col_ptr), ptr(col_rows), ptr(col_mask), B, L, S, K, float(scale),
         float(alpha), float(gamma), ptr(da), ptr(db), stream())
    return da, db


def fine_supervision(b_ids, i_ids, j_ids, fine_xy, shape, m_b, m_i, m_j, w_c, resolution, radius, img_scale):
    """expec_f_gt fp32 [M, 2] of the matches (m_b, m_i, m_j) from a ground-truth list sorted by
    (b, i, j) with fine locations fine_xy [G, 2]; img_scale fp32 [B, 2] (query_image_scale) or None."""
    _chk_gt_list(b_ids, i_ids, j_ids)
    _chk(fine_xy, torch.float32, "gt_sparse.fine_xy")
    for name, t in (("b_ids", m_b), ("i_ids", m_i), ("j_ids", m_j)):
        _chk(t, torch.int64, name)
    _chk(img_scale, torch.float32, "query_image_scale")
    B, L, S = shape
    if img_scale is not None and tuple(img_scale.shape) != (B, 2):
        raise ValueError(f"query_image_scale has shape {tuple(img_scale.shape)}, expected {(B, 2)}")
    M = m_b.numel()
    out = torch.empty(M, 2, dtype=torch.float32, device=m_b.device)
    call("opp_fine_supervision", ptr(b_ids), ptr(i_ids), ptr(j_ids), ptr(fine_xy), b_ids.numel(), B, L, S,
         ptr(m_b), ptr(m_i), ptr(m_j), M, int(w_c), int(resolution[0]), int(resolution[1]), int(radius),
         ptr(img_scale), ptr(out), stream())
    return out


def fine_gather(fine, desc3d, b_ids, i_ids, j_ids, x32, x16, m, hf, wf, wc, stride, n, split,
                bank_shared=False, count=None, windows=False, bank_of_batch=None):
    """windows: `fine` is the compact [m, 5, 8, planes*128] window tensor of conv_win.
    bank_of_batch int32 [B] (bank sets): desc3d is [K, 128, n], read at the frame's object."""
    _chk(desc3d, torch.float32, "descriptors3d_db")
    win = conv_win_pitch(5) if windows is True else int(windows)
    if bank_of_batch is not None:
        _chk(bank_of_batch, torch.int32, "bank_of_batch")
        call("opp_fine_gather_set", ptr(fine), ptr(desc3d), ptr(b_ids), ptr(i_ids), ptr(j_ids), ptr(x32),
             ptr(x16), m, hf, wf, wc, stride, n, int(split), int(bank_shared), win, ptr(count),
             ptr(bank_of_batch), stream())
        return
    call("opp_fine_gather", ptr(fine), ptr(desc3d), ptr(b_ids), ptr(i_ids), ptr(j_ids), ptr(x32),
         ptr(x16), m, hf, wf, wc, stride, n, int(split), int(bank_shared), win, ptr(count), stream())


def conv_win_pitch(win):
    """Row pitch of conv_win's compact output windows ([m, win, pitch, planes*Cout_pad])."""
    return _lib.load().opp_conv_win_pitch(win)


def conv_win(x, w, bias, out, win, split, m, act=0, slope=0.01, b_ids=None, j_ids=None, wc=0, stride=4,
             org=0, count=None):
    """3x3 convolution on per-match windows (opp_conv_win).  With j_ids: x is the dense NHWC map
    [B, H, W, planes*Cin_pad]; without: the compact output [m, win+2, 8, planes*Cin_pad] of the
    previous call.  out: [m, win, 8, planes*Cout_pad]."""
    _chk(x, torch.float16, "x")
    _chk(w, torch.float16, "w")
    planes = 2 if split else 1
    if j_ids is not None:
        B, H, W, C = x.shape
    else:
        B, H, W, C = 1, 0, 0, x.shape[-1]
    call("opp_conv_win", ptr(x), ptr(w), ptr(bias), ptr(out), ptr(b_ids), ptr(j_ids), m, ptr(count), B, H, W,
         C // planes, w.shape[0], win, wc, stride, org, act, float(slope), int(split), stream())
    return out


def fine_attention(qkv, msg, m, cross, split, eps=1e-6, count=None):
    call("opp_fine_attention", ptr(qkv), ptr(msg), m, int(cross), float(eps), int(split), ptr(count), stream())


def fine_match(x32, mkpts_c, b_ids, img_scale, expec_f, mkpts_f, m, fine_scale, count=None):
    call("opp_fine_match", ptr(x32), ptr(mkpts_c), ptr(b_ids), ptr(img_scale), ptr(expec_f),
         ptr(mkpts_f), m, float(fine_scale), ptr(count), stream())


# ---------------------------------------------------------------------------------------------
# LoFTR 2D-2D matcher (SURVEY §8 f3)
# ---------------------------------------------------------------------------------------------
def match_select_2d(pt_val, pt_idx, colmax, scale0, scale1, batch, h0, w0, h1, w1, thr, border, cell, scratch,
                    b_ids, i_ids, j_ids, mconf, mkpts0_c, mkpts1_c, count):
    call("opp_match_select_2d", ptr(pt_val), ptr(pt_idx), ptr(colmax), ptr(scale0), ptr(scale1), batch, h0, w0, h1,
         w1, float(thr), int(border), float(cell), ptr(scratch), ptr(b_ids), ptr(i_ids), ptr(j_ids), ptr(mconf),
         ptr(mkpts0_c), ptr(mkpts1_c), ptr(count), stream())


def fine_gather_2d(fine0, fine1, b_ids, i_ids, j_ids, x16, m, hf0, wf0, wc0, hf1, wf1, wc1, stride, window, split):
    _chk(fine0, torch.float16, "fine0")
    _chk(fine1, torch.float16, "fine1")
    call("opp_fine_gather_2d", ptr(fine0), ptr(fine1), ptr(b_ids), ptr(i_ids), ptr(j_ids), ptr(x16), m, hf0, wf0,
         wc0, hf1, wf1, wc1, stride, window, int(split), stream())


def seq_attention(q, kv, out, groups, l, s, split, eps=1e-6):
    _chk(q, torch.float16, "q")
    _chk(kv, torch.float16, "kv")
    call("opp_seq_attention", ptr(q), ptr(kv), ptr(out), groups, l, s, float(eps), int(split), stream())


def fine_match_2d(x32, mkpts1_c, b_ids, scale1, expec_f, mkpts1_f, m, window, fine_scale):
    call("opp_fine_match_2d", ptr(x32), ptr(mkpts1_c), ptr(b_ids), ptr(scale1), ptr(expec_f), ptr(mkpts1_f), m,
         window, float(fine_scale), stream())


# ---- training, fine level (opp_train_fine.cu; used by train_fine.py) ------------------------------
# Row operands are fp32 CUDA tensors addressed by (tensor, row stride); a column slice of a wider
# buffer (x[:, 128:]) passes its own data pointer with the buffer's stride.

def _ld(t):
    if t is None:
        return 0
    if t.dtype != torch.float32 or not t.is_cuda or t.stride(-1) != 1:
        raise ValueError("fine training operands are fp32 CUDA rows with unit column stride")
    return t.stride(0)


def fine_train_gather(feat, desc3d, b_ids, i_ids, j_ids, hc, wc, stride, x):
    _chk(feat, torch.float32, "feat_f")
    _chk(desc3d, torch.float32, "descriptors3d_db")
    _, _, hf, wf = feat.shape
    call("opp_fine_train_gather", ptr(feat), ptr(desc3d), ptr(b_ids), ptr(i_ids), ptr(j_ids), b_ids.numel(), hf, wf,
         hc, wc, desc3d.shape[2], stride, ptr(x), _ld(x), stream())


def fine_train_gather_bwd(dx, col_ptr, col_rows, hc, wc, stride, dfeat):
    B, _, hf, wf = dfeat.shape
    call("opp_fine_train_gather_bwd", ptr(dx), _ld(dx), ptr(col_ptr), ptr(col_rows), B, hf, wf, hc, wc, stride,
         ptr(dfeat), stream())


EPI_STORE, EPI_RELU, EPI_MASK, EPI_ADD = 0, 1, 2, 3


def fine_train_linear(a, w, trans_w, out, epi=EPI_STORE, aux=None, aux2=None):
    """out = epi(a @ w.T) (trans_w) or epi(a @ w); w contiguous fp32."""
    _chk(w, torch.float32, "weight")
    n, k = (w.shape[0], w.shape[1]) if trans_w else (w.shape[1], w.shape[0])
    call("opp_fine_train_linear", ptr(a), _ld(a), ptr(w), int(trans_w), a.shape[0], n, k, ptr(out), _ld(out), epi,
         ptr(aux), _ld(aux), ptr(aux2), _ld(aux2), stream())


def fine_train_wgrad(g, a, part, dw, accumulate):
    """dw (+)= g.T @ a, summed over row groups in a fixed order."""
    call("opp_fine_train_wgrad", ptr(g), _ld(g), ptr(a), _ld(a), g.shape[0], dw.shape[0], dw.shape[1], ptr(part),
         ptr(dw), int(accumulate), stream())


def fine_train_ln(x, gamma, beta, resid, y, stats):
    call("opp_fine_train_ln", ptr(x), _ld(x), ptr(gamma), ptr(beta), ptr(resid), _ld(resid), ptr(y), _ld(y),
         ptr(stats), x.shape[0], stream())


def fine_train_ln_bwd(x, gamma, stats, dy, dx, part, dgb, accumulate):
    call("opp_fine_train_ln_bwd", ptr(x), _ld(x), ptr(gamma), ptr(stats), ptr(dy), _ld(dy), ptr(dx), _ld(dx),
         x.shape[0], ptr(part), ptr(dgb), int(accumulate), stream())


def fine_train_attention(qkv, out, m, cross, eps=1e-6):
    call("opp_fine_train_attention", ptr(qkv), ptr(out), m, int(cross), eps, stream())


def fine_train_attention_bwd(qkv, dout, dqkv, m, cross, eps=1e-6):
    call("opp_fine_train_attention_bwd", ptr(qkv), ptr(dout), ptr(dqkv), m, int(cross), eps, stream())


def fine_train_match(x, m, expec_f):
    call("opp_fine_train_match", ptr(x), m, ptr(expec_f), stream())


def fine_train_match_bwd(x, dexpec, m, dx):
    _chk(dexpec, torch.float32, "grad of expec_f")
    call("opp_fine_train_match_bwd", ptr(x), ptr(dexpec), m, ptr(dx), stream())


def fine_train_groups(rows):
    return _lib.load().opp_fine_train_groups(rows)


# ---- training, coarse transformer (opp_train_coarse_tf.cu; used by train_coarse_tf.py) -----------
# A sequence is a row view [batches * len, ...] of the shared row buffer; masks are uint8 [batches * len].

COARSE_TF_STATE = 8 * 32 * 32 + 8 * 32      # floats per partial: KV [8][32][32], ksum [8][32]


def coarse_tf_chunks(length):
    return _lib.load().opp_coarse_tf_chunks(length)


def coarse_tf_part(batches, length, device):
    """The partial buffer of coarse_tf_kv / coarse_tf_attn_bwd_q for a sequence of `length` rows."""
    return torch.empty(batches, coarse_tf_chunks(length), COARSE_TF_STATE, dtype=torch.float32, device=device)


def _coarse_seq(qkv, mask, batches):
    rows = qkv.shape[0]
    if rows % batches:
        raise ValueError(f"{rows} rows do not split into {batches} batch elements")
    _chk(mask, torch.uint8, "mask")
    if mask is not None and mask.numel() != rows:
        raise ValueError(f"mask has {mask.numel()} entries for {rows} rows")
    return rows // batches


def coarse_tf_kv(qkv, mask, batches, part, kv, ksum):
    """kv [B, 8, 32, 32], ksum [B, 8, 32] (contiguous fp32, overwritten) of the source rows qkv."""
    length = _coarse_seq(qkv, mask, batches)
    _chk(kv, torch.float32, "kv")
    _chk(ksum, torch.float32, "ksum")
    call("opp_coarse_tf_kv", ptr(qkv), _ld(qkv), ptr(mask), batches, length, ptr(part), ptr(kv), ptr(ksum), stream())


def coarse_tf_attn(qkv, q_mask, batches, kv, ksum, v_len, out, eps=1e-6):
    length = _coarse_seq(qkv, q_mask, batches)
    call("opp_coarse_tf_attn", ptr(qkv), _ld(qkv), ptr(q_mask), batches, length, ptr(kv), ptr(ksum), float(v_len),
         float(eps), ptr(out), _ld(out), stream())


def coarse_tf_attn_bwd_q(qkv, q_mask, batches, kv, ksum, v_len, dout, dqkv, part, dkv, dksum, eps=1e-6):
    length = _coarse_seq(qkv, q_mask, batches)
    _chk(dkv, torch.float32, "dkv")
    _chk(dksum, torch.float32, "dksum")
    call("opp_coarse_tf_attn_bwd_q", ptr(qkv), _ld(qkv), ptr(q_mask), batches, length, ptr(kv), ptr(ksum),
         float(v_len), float(eps), ptr(dout), _ld(dout), ptr(dqkv), _ld(dqkv), ptr(part), ptr(dkv), ptr(dksum),
         stream())


def coarse_tf_attn_bwd_kv(qkv, mask, batches, dkv, dksum, dqkv):
    length = _coarse_seq(qkv, mask, batches)
    call("opp_coarse_tf_attn_bwd_kv", ptr(qkv), _ld(qkv), ptr(mask), batches, length, ptr(dkv), ptr(dksum),
         ptr(dqkv), _ld(dqkv), stream())


def coarse_tf_ln(x, gamma, beta, resid, y, stats):
    call("opp_coarse_tf_ln", ptr(x), _ld(x), ptr(gamma), ptr(beta), ptr(resid), _ld(resid), ptr(y), _ld(y),
         ptr(stats), x.shape[0], stream())


def coarse_tf_ln_bwd(x, gamma, stats, dy, dx, part, dgb, accumulate):
    call("opp_coarse_tf_ln_bwd", ptr(x), _ld(x), ptr(gamma), ptr(stats), ptr(dy), _ld(dy), ptr(dx), _ld(dx),
         x.shape[0], ptr(part), ptr(dgb), int(accumulate), stream())


# ---- training, backbone (opp_train_backbone.cu; used by train_backbone.py) ------------------------
# Maps are contiguous NCHW fp32 CUDA tensors; weights [c_out, c_in, k, k] with pad k // 2.

BB_ACT = {"none": 0, "relu": 1, "leaky": 2}


def backbone_wgrad_group():
    """Output pixels per weight-gradient partial (a slice of backbone_conv_wgrad starts at a multiple)."""
    return _lib.load().opp_backbone_train_wgrad_group()


def backbone_bn_part(batches, c, hw, device):
    """The fp64 partial buffer of backbone_bn_stats / backbone_bn_act_bwd for a [batches, c, hw] map."""
    parts = _lib.load().opp_backbone_train_bn_parts(batches, hw)
    return torch.empty(c * (2 * parts + 1), dtype=torch.float64, device=device)


def _conv_args(x, w, stride):
    _chk(x, torch.float32, "x")
    _chk(w, torch.float32, "w")
    B, C, H, W = x.shape
    co, ci, k, k2 = w.shape
    if ci != C or k != k2:
        raise ValueError(f"weight {tuple(w.shape)} does not fit input {tuple(x.shape)}")
    return B, C, H, W, co, k, int(stride)


def conv_out_hw(h, w, k, stride):
    pad = k // 2
    return (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1


def backbone_conv(x, w, stride, y):
    """y [B, c_out, ho, wo] = conv2d(x, w, stride, padding=k // 2)."""
    B, C, H, W, co, k, s = _conv_args(x, w, stride)
    _chk(y, torch.float32, "y")
    if tuple(y.shape) != (B, co, *conv_out_hw(H, W, k, s)):
        raise ValueError(f"y has shape {tuple(y.shape)}")
    call("opp_backbone_train_conv", ptr(x), ptr(w), B, C, H, W, co, k, s, ptr(y), stream())


def backbone_conv_dgrad(dy, w, stride, dx, accumulate):
    """dx [B, c_in, h, w] (+)= the input gradient of conv2d(., w, stride) for the output gradient dy."""
    B, C, H, W, co, k, s = _conv_args(dx, w, stride)
    _chk(dy, torch.float32, "dy")
    if tuple(dy.shape) != (B, co, *conv_out_hw(H, W, k, s)):
        raise ValueError(f"dy has shape {tuple(dy.shape)}")
    call("opp_backbone_train_conv_dgrad", ptr(dy), ptr(w), B, C, H, W, co, k, s, ptr(dx),
         int(accumulate), stream())


def backbone_conv_wgrad(x, dy, stride, dw, part, pix0, npix, accumulate):
    """dw (+)= the weight gradient over output pixels [pix0, pix0 + npix) of the flat (b, oy, ox) index;
    part fp32 with at least ceil(npix / group) * dw.numel() entries."""
    B, C, H, W, co, k, s = _conv_args(x, dw, stride)
    _chk(dy, torch.float32, "dy")
    _chk(part, torch.float32, "part")
    if tuple(dy.shape) != (B, co, *conv_out_hw(H, W, k, s)):
        raise ValueError(f"dy has shape {tuple(dy.shape)}")
    group = backbone_wgrad_group()
    if part.numel() < -(-npix // group) * dw.numel():
        raise ValueError("wgrad partial buffer too small")
    call("opp_backbone_train_conv_wgrad", ptr(x), ptr(dy), B, C, H, W, co, k, s, int(pix0), int(npix),
         ptr(part), ptr(dw), int(accumulate), stream())


def _bn_map(x):
    _chk(x, torch.float32, "x")
    B, C, H, W = x.shape
    return B, C, H * W


def backbone_bn_stats(x, eps, part, mean, invstd, running_mean=None, running_var=None, momentum=0.0):
    """mean / invstd [C] of x over (B, H, W); running_mean / running_var updated in place when given."""
    B, C, hw = _bn_map(x)
    for t, n in ((mean, "mean"), (invstd, "invstd"), (running_mean, "running_mean"), (running_var, "running_var")):
        _chk(t, torch.float32, n)
    call("opp_backbone_train_bn_stats", ptr(x), B, C, hw, float(eps), ptr(part), ptr(mean), ptr(invstd),
         ptr(running_mean), ptr(running_var), float(momentum), stream())


def backbone_bn_act(x, mean, invstd, gamma, beta, res, act, y):
    """y = act(gamma (x - mean) invstd + beta [+ res]), act "none" / "relu" / "leaky"."""
    B, C, hw = _bn_map(x)
    _chk(res, torch.float32, "res")
    _chk(y, torch.float32, "y")
    call("opp_backbone_train_bn_act", ptr(x), B, C, hw, ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(res),
         BB_ACT[act], ptr(y), stream())


def backbone_bn_act_bwd(x, y, dy, mean, invstd, gamma, act, batch_stats, part, dx, dres, dgb):
    """Backward of backbone_bn_act from its output y (None for act "none"): dx, dres (= d res, or None)
    and dgb [2, C] = (dgamma, dbeta), all overwritten; dx may be dy."""
    B, C, hw = _bn_map(x)
    for t, n in ((y, "y"), (dy, "dy"), (dx, "dx"), (dres, "dres"), (dgb, "dgb")):
        _chk(t, torch.float32, n)
    call("opp_backbone_train_bn_act_bwd", ptr(x), ptr(y), ptr(dy), B, C, hw, ptr(mean), ptr(invstd), ptr(gamma),
         BB_ACT[act], int(batch_stats), ptr(part), ptr(dx), ptr(dres), ptr(dgb), stream())


def backbone_up2x_add(x, lat, out):
    """out = lat + interpolate(x, scale_factor=2, bilinear, align_corners=True); out may be lat."""
    _chk(x, torch.float32, "x")
    _chk(lat, torch.float32, "lat")
    _chk(out, torch.float32, "out")
    B, C, h, w = x.shape
    if tuple(lat.shape) != (B, C, 2 * h, 2 * w) or lat.shape != out.shape:
        raise ValueError(f"lateral {tuple(lat.shape)} does not match 2x {tuple(x.shape)}")
    call("opp_backbone_train_up2x_add", ptr(x), ptr(lat), B, C, h, w, ptr(out), stream())


def backbone_up2x_bwd(dout, din, accumulate):
    """din [B, C, h, w] (+)= the backward of the x2 upsample for dout [B, C, 2h, 2w]."""
    _chk(dout, torch.float32, "dout")
    _chk(din, torch.float32, "din")
    B, C, h, w = din.shape
    if tuple(dout.shape) != (B, C, 2 * h, 2 * w):
        raise ValueError(f"dout {tuple(dout.shape)} does not match 2x {tuple(din.shape)}")
    call("opp_backbone_train_up2x_bwd", ptr(dout), B, C, h, w, ptr(din), int(accumulate), stream())


# ---- training, keypoint encoder (opp_train_kpt.cu; used by train_kpt.py) --------------------------
# Rows are the flat (b, n) index of keypoints3d [B, N, 3]; stats [B, 4] from kpt_stats.


def kpt_train_group():
    """Rows per weight-gradient partial of kpt_train_bwd (a slice starts at a multiple)."""
    return _lib.load().opp_kpt_train_group()


def kpt_train_params():
    """Floats of the flat parameter gradient: dW1 db1 dW2 db2 dW3 db3 dW4 db4."""
    return _lib.load().opp_kpt_train_params()


def kpt_train_pack_size():
    """Floats of the weight pack kpt_train_fwd / kpt_train_bwd read."""
    return _lib.load().opp_kpt_train_pack_size()


def kpt_stats(kpts, stats):
    """stats [B, 4] = (mean xyz of each batch element, 0.6 x the largest extent of element 0)."""
    _chk(kpts, torch.float32, "keypoints3d")
    _chk(stats, torch.float32, "stats")
    B, N, _ = kpts.shape
    if tuple(stats.shape) != (B, 4):
        raise ValueError(f"stats has shape {tuple(stats.shape)}, expected {(B, 4)}")
    call("opp_kpt_stats", ptr(kpts), ptr(stats), B, N, stream())


def _kpt_args(kpts, stats, pack):
    _chk(kpts, torch.float32, "keypoints3d")
    _chk(stats, torch.float32, "stats")
    _chk(pack, torch.float32, "pack")
    B, N, three = kpts.shape
    if three != 3 or tuple(stats.shape) != (B, 4):
        raise ValueError(f"keypoints3d {tuple(kpts.shape)} / stats {tuple(stats.shape)}")
    if pack.numel() != kpt_train_pack_size():
        raise ValueError(f"pack has {pack.numel()} floats, expected {kpt_train_pack_size()}")
    return B, N


def kpt_train_fwd(kpts, stats, desc, pack, out):
    """out [B * N, 256] = desc^T + the encoder MLP of the normalised keypoints; desc [B, 256, N]."""
    B, N = _kpt_args(kpts, stats, pack)
    _chk(desc, torch.float32, "descriptors")
    _chk(out, torch.float32, "out")
    if tuple(desc.shape) != (B, 256, N) or out.numel() != B * N * 256:
        raise ValueError(f"descriptors {tuple(desc.shape)} / out {tuple(out.shape)} for {B} x {N} keypoints")
    call("opp_kpt_train_fwd", ptr(kpts), ptr(stats), ptr(desc), ptr(pack), ptr(out), B, N, stream())


def kpt_train_bwd(kpts, stats, dout, pack, row0, nrows, part, dparams, accumulate):
    """dparams [kpt_train_params()] (+)= the parameter gradient for dout [B * N, 256] over the rows
    [row0, row0 + nrows); part fp32 with at least ceil(nrows / group) * kpt_train_params() entries."""
    B, N = _kpt_args(kpts, stats, pack)
    _chk(dout, torch.float32, "dout")
    _chk(part, torch.float32, "part")
    _chk(dparams, torch.float32, "dparams")
    if dout.numel() != B * N * 256 or dparams.numel() != kpt_train_params():
        raise ValueError(f"dout {tuple(dout.shape)} / dparams {tuple(dparams.shape)}")
    if part.numel() < -(-nrows // kpt_train_group()) * kpt_train_params():
        raise ValueError("wgrad partial buffer too small")
    call("opp_kpt_train_bwd", ptr(kpts), ptr(stats), ptr(dout), ptr(pack), B, N, int(row0), int(nrows), ptr(part),
         ptr(dparams), int(accumulate), stream())


def homography_warp(image, pack):
    """query_image fp32 [B, 1, h, w] -> a new tensor: kornia homography_warp (bilinear, zeros,
    align_corners=False) of the items whose pack warp flag is set, a copy of the others.
    pack fp32 [B, opp_train_batch_pack_size()] (train_batch._pack)."""
    _chk(image, torch.float32, "query_image")
    _chk(pack, torch.float32, "pack")
    B, C, h, w = image.shape
    if C != 1 or tuple(pack.shape) != (B, _lib.load().opp_train_batch_pack_size()):
        raise ValueError(f"homography_warp: image {tuple(image.shape)} / pack {tuple(pack.shape)}")
    out = torch.empty_like(image)
    call("opp_homography_warp_f32", ptr(image), ptr(pack), B, h, w, ptr(out), stream())
    return out


def train_gt(kp3d, assign, offsets, kp_offsets, n_kp, pack, img_scale, hw, w_c, S):
    """The ground-truth list of a training batch from the pose: (b_ids, i_ids, j_ids int64 [n],
    fine_xy fp32 [n, 2], status int32 [2]) — the first status[1] entries are the list, status[0]
    holds the error bits of opp_train_gt_build.  Nothing is synchronised here.
    kp3d fp32 [B, L, 3]; assign int64 [2, n]; offsets / kp_offsets int64 [B + 1] (device);
    n_kp = kp_offsets[-1] as a host int; img_scale fp32 [B, 2]; hw = (h, w) of the query image."""
    _chk(kp3d, torch.float32, "keypoints3d")
    _chk(assign, torch.int64, "assign")
    _chk(offsets, torch.int64, "offsets")
    _chk(kp_offsets, torch.int64, "kp_offsets")
    _chk(pack, torch.float32, "pack")
    _chk(img_scale, torch.float32, "query_image_scale")
    B, L, _ = kp3d.shape
    h, w = hw
    n = assign.shape[1]
    if assign.dim() != 2 or assign.shape[0] != 2 or offsets.numel() != B + 1 or kp_offsets.numel() != B + 1:
        raise ValueError("train_gt: assign must be [2, n] and offsets [B + 1]")
    if tuple(img_scale.shape) != (B, 2):
        raise ValueError(f"query_image_scale has shape {tuple(img_scale.shape)}, expected {(B, 2)}")
    if tuple(pack.shape) != (B, _lib.load().opp_train_batch_pack_size()):
        raise ValueError(f"train_gt: pack has shape {tuple(pack.shape)}")
    dev, i32 = kp3d.device, torch.int32
    ranks = ((w - 1) // 8 + 1) * ((h - 1) // 8 + 1)
    cell_owner = torch.empty(B * ranks, dtype=i32, device=dev)
    kp_owner = torch.empty(max(int(n_kp), 1), dtype=i32, device=dev)
    rank_of = torch.empty(n, dtype=i32, device=dev)
    fine = torch.empty(n, 2, dtype=torch.float32, device=dev)
    key = torch.empty(n, dtype=torch.int64, device=dev)
    key_xy = torch.empty(n, 2, dtype=torch.float32, device=dev)
    status = torch.empty(2, dtype=i32, device=dev)
    call("opp_train_gt_build", ptr(kp3d), ptr(assign), n, ptr(offsets), ptr(kp_offsets), int(n_kp), ptr(pack),
         ptr(img_scale), B, L, h, w, int(w_c), int(S), ptr(cell_owner), ptr(kp_owner), ptr(rank_of), ptr(fine),
         ptr(key), ptr(key_xy), ptr(status), stream())
    sorted_key, perm = torch.sort(key)          # the one library step: order by (b, i, j, rank)
    b_ids, i_ids, j_ids = (torch.empty(n, dtype=torch.int64, device=dev) for _ in range(3))
    fine_xy = torch.empty(n, 2, dtype=torch.float32, device=dev)
    call("opp_train_gt_compact", ptr(sorted_key), ptr(perm), n, ptr(key_xy), L, int(S), ranks, ptr(b_ids),
         ptr(i_ids), ptr(j_ids), ptr(fine_xy), ptr(status), stream())
    return b_ids, i_ids, j_ids, fine_xy, status


SFM_XY_LIMIT = 1 << 21      # the key packs x and y in 21 bits each and the image id in 20
SFM_MAX_IMAGES = 1 << 20


def sfm_points(matches, offsets, pair_img, images):
    """The 2D keypoint merge of the SfM coarse matching (opp_sfm_points.cu) over all pairs at once.
    matches fp32 [M, 5] (x0, y0, x1, y1, mconf) of P pairs in order; offsets int64 [P + 1] and
    pair_img int32 [P, 2] (image ids < images) on the device.  Returns (kpts fp32 [G, 2], scores
    fp32 [G], img_off int64 [images + 1], idx int64 [M, 2], status int32 [1]): image i's keypoints
    are kpts[img_off[i]:img_off[i + 1]] in id order, idx holds each match's two ids and status is
    non-zero when an endpoint was not found (it cannot be, for valid input).  Raises ValueError, before
    any launch, for coordinates the key cannot pack (outside [0, 2^21) or not finite), a negative or
    non-finite mconf, an image id outside [0, images) or offsets that do not partition the matches."""
    _chk(matches, torch.float32, "matches")
    _chk(offsets, torch.int64, "offsets")
    _chk(pair_img, torch.int32, "pair_img")
    P = pair_img.shape[0]
    M = matches.shape[0]
    if matches.dim() != 2 or matches.shape[1] != 5 or pair_img.dim() != 2 or pair_img.shape[1] != 2 \
            or tuple(offsets.shape) != (P + 1,):
        raise ValueError(f"sfm_points: matches {tuple(matches.shape)}, offsets {tuple(offsets.shape)}, "
                         f"pair_img {tuple(pair_img.shape)}")
    if P == 0 or M == 0 or not 0 < images <= SFM_MAX_IMAGES or 2 * M >= 2 ** 31:
        raise ValueError(f"sfm_points: P={P}, M={M}, images={images} outside the built range")
    xy, conf = matches[:, :4], matches[:, 4]
    ok = torch.stack([(xy >= 0).all(), (xy < SFM_XY_LIMIT).all(), (conf >= 0).all(), torch.isfinite(conf).all(),
                      (pair_img >= 0).all(), (pair_img < images).all(), offsets[0] == 0, offsets[-1] == M,
                      (offsets[1:] >= offsets[:-1]).all()])
    if not bool(ok.all()):
        names = ("x, y >= 0", f"x, y < {SFM_XY_LIMIT}", "mconf >= 0", "mconf finite", "image ids >= 0",
                 f"image ids < {images}", "offsets[0] == 0", f"offsets[-1] == {M}", "offsets ascending")
        bad = [n for n, v in zip(names, ok.tolist()) if not v]
        raise ValueError(f"sfm_points: input violates {', '.join(bad)}")
    dev, i32, i64 = matches.device, torch.int32, torch.int64
    n = 2 * M
    key = torch.empty(n, dtype=i64, device=dev)
    conf2 = torch.empty(n, dtype=torch.float32, device=dev)
    call("opp_sfm_points_emit", ptr(matches), M, ptr(offsets), ptr(pair_img), P, ptr(key), ptr(conf2), stream())
    sorted_key, perm = torch.sort(key, stable=True)     # library step: groups keep their appearance order
    scratch = torch.empty(_lib.load().opp_sfm_points_segments_scratch(n), dtype=i32, device=dev)
    start = torch.empty(n + 1, dtype=i32, device=dev)
    groups = torch.empty(1, dtype=i32, device=dev)
    call("opp_sfm_points_segments", ptr(sorted_key), n, ptr(scratch), ptr(start), ptr(groups), stream())
    G = int(groups.item())
    ukey, rank_key = torch.empty(G, dtype=i64, device=dev), torch.empty(G, dtype=i64, device=dev)
    sums = torch.empty(G, dtype=torch.float64, device=dev)
    img_off = torch.empty(images + 1, dtype=i64, device=dev)
    call("opp_sfm_points_sums", ptr(sorted_key), ptr(perm), ptr(conf2), ptr(start), G, int(images), ptr(ukey),
         ptr(sums), ptr(rank_key), ptr(img_off), stream())
    del key, sorted_key, perm, conf2, start, scratch
    _, perm1 = torch.sort(rank_key, stable=True)        # descending sum; ties keep ascending (x, y)
    img_key = torch.empty(G, dtype=i64, device=dev)
    call("opp_sfm_points_image_key", ptr(ukey), ptr(perm1), G, ptr(img_key), stream())
    _, perm2 = torch.sort(img_key, stable=True)         # then by image, keeping that order
    kpts = torch.empty(G, 2, dtype=torch.float32, device=dev)
    scores = torch.empty(G, dtype=torch.float32, device=dev)
    id_of = torch.empty(G, dtype=i64, device=dev)
    call("opp_sfm_points_rank", ptr(ukey), ptr(sums), ptr(img_off), ptr(perm1), ptr(perm2), G, ptr(kpts),
         ptr(scores), ptr(id_of), stream())
    idx = torch.empty(M, 2, dtype=i64, device=dev)
    status = torch.empty(1, dtype=i32, device=dev)
    call("opp_sfm_points_remap", ptr(matches), M, ptr(offsets), ptr(pair_img), P, ptr(ukey), ptr(img_off), ptr(id_of),
         ptr(idx), ptr(status), stream())
    return kpts, scores, img_off, idx, status


# ---- keypoint-free SfM refinement (opp_sfm_refine.cu; used by loftr.py and sfm_refine.py) ---------

def fine_gather_2d_images(fine, img0, img1, i_ids, j_ids, x16, m, hf, wf, wc, stride, window, split):
    """fine_gather_2d over a store of many images' fine maps: match m reads image img0[m] / img1[m]."""
    _chk(fine, torch.float16, "fine")
    for name, t in (("img0", img0), ("img1", img1), ("i_ids", i_ids), ("j_ids", j_ids)):
        _chk(t, torch.int64, name)
    call("opp_fine_gather_2d_images", ptr(fine), ptr(img0), ptr(img1), ptr(i_ids), ptr(j_ids), ptr(x16), m, hf, wf,
         wc, stride, window, int(split), stream())


def sample_feature(fmap, channels, split, kpts, imghw, nearest, img=None, out=None):
    """sample_feature_from_featuremap at kpts [n, 2] (fp32 or fp64, on the device) from the engine's
    NHWC fp16 map store [N, h, w, planes*channels]; img int64 [n] names each point's image (None:
    image 0), imghw fp32 [N, 2] = (h, w) * scale per image.  Returns fp32 [n, channels]."""
    _chk(fmap, torch.float16, "map")
    if kpts.dtype not in (torch.float32, torch.float64) or not kpts.is_cuda or not kpts.is_contiguous():
        raise TypeError("kpts must be a contiguous fp32 or fp64 CUDA tensor")
    _chk(imghw, torch.float32, "imghw")
    _chk(img, torch.int64, "img")
    N, hm, wm, C = fmap.shape
    if C != (2 if split else 1) * channels or kpts.dim() != 2 or kpts.shape[1] != 2 or tuple(imghw.shape) != (N, 2):
        raise ValueError(f"sample_feature: map {tuple(fmap.shape)}, kpts {tuple(kpts.shape)}, imghw {tuple(imghw.shape)}")
    n = kpts.shape[0]
    if out is None:
        out = torch.empty((n, channels), dtype=torch.float32, device=kpts.device)
    call("opp_sample_feature", ptr(fmap), ptr(img), ptr(kpts), int(kpts.dtype == torch.float64), n, hm, wm, channels,
         int(split), ptr(imghw), int(bool(nearest)), ptr(out), stream())
    return out


def sfm_refine_lookup(row_key, query):
    """row int64 [q]: the position in row_key (int64 [n]) of each query key, -1 when absent, -2 when the
    key occurs more than once."""
    _chk(row_key, torch.int64, "row_key")
    _chk(query, torch.int64, "query")
    row = torch.empty(query.shape[0], dtype=torch.int64, device=query.device)
    if query.shape[0] == 0:
        return row
    if row_key.shape[0] == 0:
        return row.fill_(-1)
    sorted_key, perm = torch.sort(row_key)     # library step, as in sfm_points
    call("opp_sfm_refine_lookup", ptr(sorted_key), ptr(perm), row_key.shape[0], ptr(query), query.shape[0], ptr(row),
         stream())
    return row


def sfm_refine_aggregate(c0, c1, f0, f1, row, track_off):
    """Track means and reference-side gathers of feature_aggregation_and_update: c0, c1 fp32 [R, dc],
    f0, f1 fp32 [R, df]; row int64 [K] (member -> row), track_off int64 [T + 1].  Returns (mean_c
    [T, dc], mean_f [T, df], ref_c [K, dc], ref_f [K, df])."""
    for name, t in (("c0", c0), ("c1", c1), ("f0", f0), ("f1", f1)):
        _chk(t, torch.float32, name)
    _chk(row, torch.int64, "row")
    _chk(track_off, torch.int64, "track_off")
    T, K, dc, df = track_off.shape[0] - 1, row.shape[0], c0.shape[1], f0.shape[1]
    dev = row.device
    mean_c, mean_f = torch.empty((T, dc), device=dev), torch.empty((T, df), device=dev)
    ref_c, ref_f = torch.empty((K, dc), device=dev), torch.empty((K, df), device=dev)
    call("opp_sfm_refine_aggregate", ptr(c0), ptr(c1), ptr(f0), ptr(f1), dc, df, ptr(row), ptr(track_off), T,
         ptr(mean_c), ptr(mean_f), ptr(ref_c), ptr(ref_f), stream())
    return mean_c, mean_f, ref_c, ref_f
