"""ctypes binding of ``libopp_b200.so`` (C ABI declared in ``include/opp_b200.h``).

There is no fallback: if the shared library is missing or a call fails, a ``RuntimeError`` is
raised.  Tensors are passed as raw device pointers; the current torch CUDA stream is used.
"""
import ctypes
import os
from ctypes import c_float, c_int, c_longlong, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OPP_B200_LIB") or os.path.join(_HERE, "libopp_b200.so")

_lib = None


def _sig(fn, argtypes):
    fn.argtypes = argtypes
    fn.restype = c_int


P, I, L, F = c_void_p, c_int, c_longlong, c_float

# name -> argtypes; must mirror include/opp_b200.h exactly (tests check every symbol resolves)
SIGNATURES = {
    "opp_conv2d_nhwc": [P, P, P, P, P, I, I, I, I, I, I, I, I, F, P, P, P, I, P],
    "opp_conv1_im2col": [P, I, P, I, I, I, I, P],
    "opp_kpt_stats": [P, P, I, I, P],
    "opp_kpt_encode": [P] * 12 + [I, I, I, P],
    "opp_linear_act_f16": [P, I, P, I, P, P, L, I, I, I, I, P],
    "opp_linear_act_f16_out1": [P, I, P, I, P, P, L, I, I, I, P, P],
    "opp_linear_act_f16_b": [P, I, I, P, I, P, P, I, L, I, I, I, I, P, P],
    "opp_linear_q_f16": [P, P, P, P, I, I, I, F, F, I, I, P, P],
    "opp_linear_ln": [P, I, P, I, P, I, P, P, F, P, I, P, P, I, L, I, I, P],
    "opp_full_attention": [P, P, P, I, I, I, I, I, I, P],
    "opp_kv_partial": [P, P, I, I, I, P],
    "opp_kv_finalize": [P, P, P, P, I, I, I, F, I, P],
    "opp_lse_finalize": [P, P, P, L, I, P],
    "opp_sim_lse_cols": [P, P, P, P, P, P, I, I, I, I, F, I, P, P],
    "opp_lse_col_finalize": [P, P, P, I, I, I, P, P],
    "opp_sim_conf_colmax": [P, P, P, P, P, P, P, P, I, I, I, I, F, I, P],
    "opp_best_finalize": [P, P, P, P, L, I, P],
    "opp_match_select_colmax": [P, P, P, P, P, I, I, I, I, F, I, F, P, P, P, P, P, P, P, P, I, P],
    "opp_fine_gather": [P, P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, P, P],
    "opp_sim_lse_cols_rows": [P, P, P, P, P, P, I, I, I, I, F, I, P, P, P],
    "opp_sim_conf_colmax_rows": [P, P, P, P, P, P, P, P, I, I, I, I, F, I, P, P],
    "opp_match_select_colmax_set": [P, P, P, P, P, I, I, I, I, F, I, F, P, P, P, P, P, P, P, P, I, P, P, P],
    "opp_fine_gather_set": [P, P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, P, P, P],
    "opp_conv_win": [P, P, P, P, P, P, I, P, I, I, I, I, I, I, I, I, I, I, F, I, P],
    "opp_fine_attention": [P, P, I, I, F, I, P, P],
    "opp_fine_match": [P, P, P, P, P, P, I, F, P, P],
    "opp_linear_act_f16_dyn": [P, I, P, I, P, P, L, P, I, I, I, I, I, P],
    "opp_linear_ln_dyn": [P, I, P, I, P, P, P, F, P, P, P, L, P, I, I, I, P],
    "opp_match_select_2d": [P, P, P, P, P, I, I, I, I, I, F, I, F, P, P, P, P, P, P, P, P, P],
    "opp_fine_gather_2d": [P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, P],
    "opp_seq_attention": [P, P, P, I, I, I, F, I, P],
    "opp_fine_match_2d": [P, P, P, P, P, P, I, I, F, P],
    "opp_pnp_ransac": [P, P, P, I, P, I, F, F, I, ctypes.c_uint, I, P, P, P, P, P],
    "opp_pnp_ransac_colmap": [P, P, P, I, P, I, F, I, ctypes.c_uint, I, P, P, P, P, P],
    "opp_pose_metrics": [P, I, P, P, P, P, I, P, L, P, P, P],
    "opp_crop_resize_u8": [P, I, I, I, P, P, I, I, P, P],
    "opp_coarse_focal_stats": [P, P, P, I, I, I, I, F, P, P, P, P],
    "opp_coarse_focal_fwd": [P, P, P, P, P, I, P, I, I, I, I, F, F, F, F, F] + [P] * 10,
    "opp_coarse_focal_bwd": [P] * 9 + [I, P, I, I, I, I, F, F, F, P, P, P],
    "opp_gt_index": [P, P, P, I, I, I, I, P, P, P, P, P],
    "opp_coarse_focal_fwd_sparse": [P] * 7 + [I, I, I, I, F, F, F, F, F] + [P] * 10,
    "opp_coarse_focal_bwd_sparse": [P] * 13 + [I, I, I, I, F, F, F, P, P, P],
    "opp_fine_supervision": [P, P, P, P, I, I, I, I, P, P, P, I, I, I, I, I, P, P, P],
    "opp_fine_train_gather": [P] * 5 + [I] * 7 + [P, I, P],
    "opp_fine_train_gather_bwd": [P, I, P, P] + [I] * 6 + [P, P],
    "opp_fine_train_linear": [P, I, P, I, I, I, I, P, I, I, P, I, P, I, P],
    "opp_fine_train_wgrad": [P, I, P, I, I, I, I, P, P, I, P],
    "opp_fine_train_ln": [P, I, P, P, P, I, P, I, P, I, P],
    "opp_fine_train_ln_bwd": [P, I, P, P, P, I, P, I, I, P, P, I, P],
    "opp_fine_train_attention": [P, P, I, I, F, P],
    "opp_fine_train_attention_bwd": [P, P, P, I, I, F, P],
    "opp_fine_train_match": [P, I, P, P],
    "opp_fine_train_match_bwd": [P, P, I, P, P],
    "opp_coarse_tf_kv": [P, I, P, I, I, P, P, P, P],
    "opp_coarse_tf_attn": [P, I, P, I, I, P, P, F, F, P, I, P],
    "opp_coarse_tf_attn_bwd_q": [P, I, P, I, I, P, P, F, F, P, I, P, I, P, P, P, P],
    "opp_coarse_tf_attn_bwd_kv": [P, I, P, I, I, P, P, P, I, P],
    "opp_coarse_tf_ln": [P, I, P, P, P, I, P, I, P, I, P],
    "opp_coarse_tf_ln_bwd": [P, I, P, P, P, I, P, I, I, P, P, I, P],
    "opp_backbone_train_conv": [P, P, I, I, I, I, I, I, I, P, P],
    "opp_backbone_train_conv_dgrad": [P, P, I, I, I, I, I, I, I, P, I, P],
    "opp_backbone_train_conv_wgrad": [P, P, I, I, I, I, I, I, I, I, I, P, P, I, P],
    "opp_backbone_train_bn_stats": [P, I, I, I, F, P, P, P, P, P, F, P],
    "opp_backbone_train_bn_act": [P, I, I, I, P, P, P, P, P, I, P, P],
    "opp_backbone_train_bn_act_bwd": [P, P, P, I, I, I, P, P, P, I, I, P, P, P, P, P],
    "opp_backbone_train_up2x_add": [P, P, I, I, I, I, P, P],
    "opp_backbone_train_up2x_bwd": [P, I, I, I, I, P, I, P],
    "opp_kpt_train_fwd": [P, P, P, P, P, I, I, P],
    "opp_kpt_train_bwd": [P, P, P, P, I, I, I, I, P, P, I, P],
    "opp_homography_warp_f32": [P, P, I, I, I, P, P],
    "opp_train_gt_build": [P, P, L, P, P, L, P, P, I, I, I, I, I, I, P, P, P, P, P, P, P, P],
    "opp_train_gt_compact": [P, P, L, P, I, I, L, P, P, P, P, P, P],
    "opp_sfm_points_emit": [P, L, P, P, I, P, P, P],
    "opp_sfm_points_segments": [P, L, P, P, P, P],
    "opp_sfm_points_sums": [P, P, P, P, I, I, P, P, P, P, P],
    "opp_sfm_points_image_key": [P, P, I, P, P],
    "opp_sfm_points_rank": [P, P, P, P, P, I, P, P, P, P],
    "opp_sfm_points_remap": [P, L, P, P, I, P, P, P, P, P, P],
    "opp_fine_gather_2d_images": [P, P, P, P, P, P, I, I, I, I, I, I, I, P],
    "opp_sample_feature": [P, P, P, I, L, I, I, I, I, P, I, P, P],
    "opp_sfm_refine_lookup": [P, P, L, P, L, P, P],
    "opp_sfm_refine_aggregate": [P, P, P, P, I, I, P, P, I, P, P, P, P, P],
}
PLAIN = {"opp_version": ([], c_int), "opp_num_sms": ([], c_int), "opp_sim_tiles": ([I], c_int),
         "opp_kv_chunks": ([I], c_int),
         "opp_kv_chunks_b": ([I, I], c_int),
         "opp_conv_win_pitch": ([I], c_int),
         "opp_coarse_focal_blocks": ([I], c_int),
         "opp_fine_train_groups": ([I], c_int),
         "opp_coarse_tf_chunks": ([I], c_int),
         "opp_backbone_train_wgrad_group": ([], c_int),
         "opp_backbone_train_bn_parts": ([I, I], c_int),
         "opp_kpt_train_group": ([], c_int),
         "opp_kpt_train_params": ([], c_int),
         "opp_kpt_train_pack_size": ([], c_int),
         "opp_train_batch_pack_size": ([], c_int),
         "opp_sfm_points_segments_scratch": ([L], c_int),
         "opp_pose_metrics_scratch_bytes": ([I, I], c_longlong),
         "opp_last_error": ([], ctypes.c_char_p)}


def load():
    """Load the shared library (once). Raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a). There is no CPU/PyTorch fallback for this path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        _sig(getattr(lib, name), argtypes)
    for name, (argtypes, restype) in PLAIN.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    _lib = lib
    return lib


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


# kernels launched per entry point (bench.py reports the per-step total as gpu_launches)
KERNELS_PER_CALL = {"opp_match_select_colmax": 3, "opp_match_select_colmax_set": 3,
                    "opp_pose_metrics": 3,
                    "opp_coarse_focal_stats": 2, "opp_coarse_focal_fwd": 3, "opp_coarse_focal_bwd": 2,
                    "opp_gt_index": 5, "opp_coarse_focal_fwd_sparse": 3, "opp_coarse_focal_bwd_sparse": 2,
                    "opp_fine_train_wgrad": 2, "opp_fine_train_ln_bwd": 2,
                    "opp_coarse_tf_kv": 2, "opp_coarse_tf_attn_bwd_q": 2, "opp_coarse_tf_ln_bwd": 2,
                    "opp_backbone_train_conv_wgrad": 2,
                    "opp_backbone_train_bn_stats": 2,
                    "opp_backbone_train_bn_act_bwd": 3, "opp_kpt_train_bwd": 2,
                    "opp_train_gt_build": 3, "opp_sfm_points_segments": 3}
LAUNCHES = 0
_PROFILE = None


def call(name, *args):
    global LAUNCHES
    lib = load()
    if _PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.opp_last_error()
        raise RuntimeError(f"{name} failed (status {rc}): {msg.decode() if msg else ''}")
    LAUNCHES += KERNELS_PER_CALL.get(name, 1)
    if _PROFILE is not None:
        e1.record()
        _PROFILE.append((name, e0, e1))


def profile_ops(fn, out):
    """Run fn() once with CUDA events around every C-ABI call and print per-entry-point totals."""
    global _PROFILE
    _PROFILE = []
    fn()
    torch.cuda.synchronize()
    rows, _PROFILE_local = {}, _PROFILE
    _PROFILE = None
    for name, e0, e1 in _PROFILE_local:
        ms = e0.elapsed_time(e1)
        n, t = rows.get(name, (0, 0.0))
        rows[name] = (n + 1, t + ms)
    total = sum(t for _, t in rows.values())
    for name, (n, t) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        print(f"{name:24s} calls={n:4d} total={t:9.3f} ms  {100 * t / total:5.1f}%", file=out)
    print(f"{'sum':24s} {'':10s} total={total:9.3f} ms", file=out)
    return rows
