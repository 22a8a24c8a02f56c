/* opp_b200.h — C ABI of libopp_b200.so: the H100 (sm_90a) kernels behind the OnePose++ 2D-3D
 * coarse-to-fine matcher, `OnePosePlus_model.forward` (reference:
 * src/models/OnePosePlus/OnePosePlusModel.py:96-201).
 *
 * The reference has no FFI on this path: every stage is a PyTorch library call.  The entry
 * points below are what a binding for this path would bind — one per reference stage — and each
 * one cites the reference code it replaces.  `onepose_plus_plus_b200/_lib.py` is the ctypes
 * binding; INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host; fp16 buffers are `void*`
 *   - no allocation and no synchronisation inside; work is enqueued on `stream`
 *   - return 0 on success, non-zero on error; opp_last_error() describes the last failure of the
 *     calling thread
 *   - feature maps are NHWC fp16 with the channel count padded to a multiple of 16
 *     (196 -> 208); token tensors are [batch][tokens][channels]
 *   - `split`: every fp16 tensor that feeds a tensor-core GEMM is stored as two planes along its
 *     channel axis, row = [hi(C) | lo(C)] with hi = fp16(x), lo = fp16(x - hi); GEMMs then issue
 *     hi*hi + hi*lo + lo*hi into one fp32 accumulator (fp32-grade result, parity mode).  With
 *     split = 0 rows are plain fp16 [C] (2^-11 operands; does not meet the 1e-3 parity bar).
 *     All `ld`/channel counts below are per plane; split = 1 doubles the row length.
 */
#ifndef OPP_B200_H_
#define OPP_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef void* opp_stream_t; /* cudaStream_t */

int opp_version(void);
const char* opp_last_error(void);
int opp_num_sms(void);


/* ------------------------------------------------------------------------------------------
 * Backbone — ResNetFPN_8_2.forward (backbone/resnet.py:141-164), BatchNorm folded on the host;
 * every convolution runs on the wgmma engine, the two bilinear x2 upsample-adds of the FPN are
 * epilogues of the lateral 1x1 convolutions
 * ---------------------------------------------------------------------------------------- */

/* conv1 on the tensor-core engine: im2col of the 7x7 stride-2 pad-3 windows (resnet.py:101-103).
 * a_out fp16 [B*H/2*W/2][planes*64]: row = (49 taps, 1.0, 14 zeros) of one output pixel, so that
 * opp_linear_act_f16(a_out, k0 = 64, w = [c_out][planes*64] holding (49 folded-BN taps, folded
 * bias, zeros), act = ReLU) yields the NHWC map [B][H/2][W/2][planes*c_out] of
 * relu(bn1(conv1(x))) (resnet.py:143).  image: fp32 [B][1][H][W] in [0,1], or (image_u8 != 0)
 * uint8 with x = u8 / 255 folded in (the host-side division of data_io.py:107). */
int opp_conv1_im2col(const void* image, int image_u8, void* a_out, int batch, int h, int w, int split,
                     opp_stream_t stream);

/* 3x3 (pad 1) or 1x1 (pad 0) convolution, stride 1 or 2, as a wgmma implicit GEMM
 * (resnet.py:10-17 conv1x1/conv3x3; BasicBlock resnet.py:36-45; FPN heads resnet.py:109-124).
 *   in    NHWC fp16 [B][in_h][in_w][c_in_pad]
 *   w     fp16 [c_out_pad][planes][ksize*ksize][c_in_pad]   (BN-folded, zero in the padding)
 *   bias  fp32 [c_out_pad]
 *   resid NHWC fp16 [B][out_h][out_w][c_out_pad] added before the activation, or NULL
 *   act   0 none, 1 ReLU, 2 LeakyReLU(slope)
 *   out   NHWC fp16 [B][out_h][out_w][c_out_pad], or NULL when only tokens are wanted
 *   tok/pe: when tok != NULL also writes  out + pe  as coarse tokens
 *          [B][out_h*out_w][planes*c_out_pad]; pe is fp32 [out_h*out_w][c_out_pad]
 *          (PositionEncodingSine.forward position_encoding.py:37-42 + the 'n c h w -> n (h w) c'
 *          rearrange OnePosePlusModel.py:137-142)
 *   up:    when up != NULL the epilogue adds  bilinear_x2(up), align_corners=True  (FPN top-down
 *          merge, resnet.py:149-157: F.interpolate(..., scale_factor=2, mode="bilinear",
 *          align_corners=True) + lateral conv); up is NHWC fp16 [B][out_h/2][out_w/2][c_out_pad] */
int opp_conv2d_nhwc(const void* in, const void* w, const float* bias, const void* resid,
                    void* out, int batch, int in_h, int in_w, int c_in_pad, int c_out_pad,
                    int ksize, int stride, int act, float slope, void* tok, const float* pe,
                    const void* up, int split, opp_stream_t stream);

/* The same 3x3 / stride 1 / pad 1 convolution evaluated only on a win x win window around each
 * coarse match (win = 7 or 5).  The fine branch of the FPN (resnet.py:155-157 layer1_outconv2) is
 * read only inside the 5x5 window of each match (fine_preprocess.py:40-47: unfold, then keep the
 * matched cells), so for few matches the two half-resolution convolutions run on those windows
 * alone: conv A on 7x7 (what conv B's 5x5 outputs need), conv B on 5x5; values are those of the
 * dense convolution at the same positions.
 *   out   fp16 [matches][win][8][planes*c_out_pad] (compact windows; column 7 of a row is padding;
 *         positions outside the image are written as zeros = the padding the next conv must see)
 *   j_ids != NULL (with b_ids): `in` is the dense NHWC map [batch][in_h][in_w][planes*c_in_pad];
 *         window m starts at (x, y) = (stride * cx + org, stride * cy + org), (cy, cx) = divmod(j_ids[m], wc)
 *   j_ids == NULL: `in` is the compact output [matches][win + 2][8][planes*c_in_pad] of a previous
 *         call; output (ly, lx) reads input rows ly..ly+2, columns lx..lx+2
 *   count: NULL = `matches` is exact; else the capacity, the real count is read on the device */
int opp_conv_win_pitch(int win);   /* row pitch P of the output windows: out is [matches][win][P][planes*c_out_pad] */
int opp_conv_win(const void* in, const void* w, const float* bias, void* out, const long long* b_ids,
                 const long long* j_ids, int matches, const int* count, int batch, int in_h, int in_w,
                 int c_in_pad, int c_out_pad, int win, int wc, int stride, int org, int act,
                 float slope, int split, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * 3D keypoint encoding — normalize_3d_keypoints (utils/normalize.py:16-26) +
 * KeypointEncoding_linear.forward (utils/position_encoding.py:54-60)
 * ---------------------------------------------------------------------------------------- */

/* stats fp32 [B][4] = (mean x, mean y, mean z, 0.6 * max extent of batch element 0) */
int opp_kpt_stats(const float* kpts, float* stats, int batch, int n, opp_stream_t stream);

/* tokens = desc^T + MLP(normalised kpts); MLP = Linear,IN,ReLU x3 + Linear with per-point
 * instance norm over channels (eps 1e-5).  wN_t are the transposed weights [in][out].
 * kpts fp32 [B][N][3]; desc fp32 [B][256][N]; tok fp16 [B][N][planes*256] */
int opp_kpt_encode(const float* kpts, const float* stats, const float* desc, const float* w1_t,
                   const float* b1, const float* w2_t, const float* b2, const float* w3_t,
                   const float* b3, const float* w4_t, const float* b4, void* tok, int batch, int n,
                   int split, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Transformer — LoFTREncoderLayer.forward (loftr_module/transformer.py:65-94) and
 * LinearAttention.forward (loftr_module/linear_attention.py:29-61), wgmma GEMMs
 * ---------------------------------------------------------------------------------------- */

/* out[rows][n] = act(concat_K(a0[rows][k0], a1[rows][k1]) @ w[n][k0+k1]^T), fp16 in/out.
 * act 0 none, 1 ReLU, 2 elu(x)+1, applied to output columns < act_cols.
 * Used for [k_proj;v_proj] (transformer.py:78-79 + linear_attention.py:46), mlp.0 + ReLU
 * (transformer.py:41-45,91) and the fine-level q/k/v projections. a1 may be NULL (k1 = 0). */
int opp_linear_act_f16(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                       long long rows, int n, int act, int act_cols, int split,
                       opp_stream_t stream);

/* Batched form: a0 / a1 / out are [batches][rows][..]; with a0_shared != 0 the first operand is
 * [1][rows][k0] — one object's tokens shared by every image of the batch (the 3D side of the
 * first cross layer, whose x is image-independent: transformer.py:148-159) — and is read once.
 * row_mask (uint8 [batches*rows], or NULL): rows whose mask is 0 are written as zeros — padded
 * source positions of query_image_mask (linear_attention.py:51-53: K and V are multiplied by kv_mask). */
int opp_linear_act_f16_b(const void* a0, int k0, int a0_shared, const void* a1, int k1, const void* w,
                         void* out, int batches, long long rows, int n, int act, int act_cols,
                         int split, const unsigned char* row_mask, opp_stream_t stream);

/* Same GEMM with split (hi|lo) operands but a single-plane fp16 output [rows][n]: for the K'/V rows
 * of the linear-attention state, whose consumer sums over thousands of rows. */
int opp_linear_act_f16_out1(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                            long long rows, int n, int act, int act_cols, const unsigned char* row_mask,
                            opp_stream_t stream);

/* opp_linear_act_f16 / opp_linear_ln with a device-side row count: rows = *count * rows_per_count
 * (clamped to cap_rows, the size the operands were allocated for). */
int opp_linear_act_f16_dyn(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                           long long cap_rows, const int* count, int rows_per_count, int n, int act,
                           int act_cols, int split, opp_stream_t stream);
int opp_linear_ln_dyn(const void* a0, int k0, const void* a1, int k1, const void* w, const float* gamma,
                      const float* beta, float eps, const void* resid, void* out16, float* out32,
                      long long cap_rows, const int* count, int rows_per_count, int n, int split,
                      opp_stream_t stream);

/* q_proj + feature map + normaliser (transformer.py:77, linear_attention.py:45,58):
 * out = Q * v_len / (Q . ksum_head + eps), Q = elu(x @ wq^T) + 1, heads of 32 channels.
 * x fp16 [B][rows][256] (or [1][rows][256] with x_shared != 0); ksum fp32 [B][256];
 * out fp16 [B][rows][256]; row_mask uint8 [B*rows] or NULL: Q = 0 on padded query positions
 * (linear_attention.py:49-50) */
int opp_linear_q_f16(const void* x, const void* wq, const float* ksum, void* out, int batches,
                     int rows, int d_model, float v_len, float eps, int split, int x_shared,
                     const unsigned char* row_mask, opp_stream_t stream);

/* y = LayerNorm(concat_K(a0,a1) @ w^T) [+ resid]  (transformer.py:85-94).
 * w fp16 [n][planes*k] or, when w_batched, [B][n][planes*k] (the per-image
 * blockdiag(KV) @ merge^T  matrix).  resid / out16 fp16 [B*rows][planes*n]; out32 fp32
 * [B*rows][n]; either output may be NULL.  resid_shared != 0: resid is [1][rows][planes*n]. */
int opp_linear_ln(const void* a0, int k0, const void* a1, int k1, const void* w, int w_batched,
                  const float* gamma, const float* beta, float eps, const void* resid,
                  int resid_shared, void* out16, float* out32, int batches, long long rows, int n,
                  int split, opp_stream_t stream);

/* FullAttention.forward (linear_attention.py:64-95): out = softmax(Q K^T / sqrt(head_dim)) V per
 * head; `attention: "full"` in the transformer config (no shipped configuration selects it).
 * q fp16 [B][l][planes*heads*head_dim] = q_proj(x); kv fp16 [B][s][planes*2*heads*head_dim] =
 * (k_proj(source) | v_proj(source)); out like q.  head_dim 32 (coarse) or 16 (fine). */
int opp_full_attention(const void* q, const void* kv, void* out, int batch, int l, int s, int heads,
                       int head_dim, int split, opp_stream_t stream);

/* Source side state of linear attention (linear_attention.py:55-57):
 * kv16 fp16 [B][S][2d] (one plane in both operand modes) holds K' = elu(k)+1 in columns [0,d) and
 * V in [d,2d).
 * part fp32 [B][chunks][H][33][32], chunks = opp_kv_chunks_b(S, B): per-chunk sum_s K'^T V (rows
 * 0..31) and sum_s K' (row 32) for each of the H = d/32 heads.  opp_kv_partial picks the chunk length
 * from (S, B) — 256 tokens, 128 when that would leave fewer than 64 CTAs — and opp_kv_finalize must
 * be given the matching chunk count: opp_kv_chunks_b(S, B).  opp_kv_chunks(S) = the 256-token count
 * (what large batches use), kept for callers that size buffers once. */
int opp_kv_chunks(int s);
int opp_kv_chunks_b(int s, int batch);
int opp_kv_partial(const void* kv16, float* part, int batch, int s, int d, opp_stream_t stream);

/* Reduces the chunk partials, scales KV by 1/v_len and folds the merge projection
 * (transformer.py:85): mt[b][c][h*32+dd] = sum_v merge_w[c][h*32+v] * KV[b][h][dd][v] / v_len.
 * merge_w fp32 [d][d]; mt fp16 [B][d][planes*d]; ksum fp32 [B][d]. */
int opp_kv_finalize(const float* part, const float* merge_w, void* mt, float* ksum, int batch,
                    int chunks, int d, float v_len, int split, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Coarse matching — CoarseMatching.forward / get_coarse_match
 * (utils/coarse_matching.py:76-123,125-242)
 * ---------------------------------------------------------------------------------------- */

int opp_sim_tiles(int cols); /* column tiles used by the two calls below */

/* lse[r] = logsumexp over tiles */
int opp_lse_finalize(const float* part_m, const float* part_s, float* lse, long long rows,
                     int tiles, opp_stream_t stream);

/* Dual-softmax statistics of sim = scale * a @ b^T in one GEMM pass, rows = 3D points.
 * a fp16 [B][rows][planes*k], b fp16 [B][cols][planes*k].  Row side: part_m/part_s fp32
 * [B*rows][opp_sim_tiles(cols)] = per-row partial (max, sum exp) over each column tile, merged by
 * opp_lse_finalize.  Column side: col_m/col_s fp32 [B][ceil(rows/32)][cols] = per 32-row group
 * (max, sum exp(x - max)) of every column; opp_lse_col_finalize merges the groups into
 * lse[b][s] = logsumexp_l sim[b, l, s].
 * col_mask (uint8 [B][cols] or NULL) = query_image_mask at coarse resolution: masked columns get
 * sim - 1e9 (coarse_matching.py:108-114), i.e. they drop out of every row's softmax, and
 * opp_lse_col_finalize writes lse = +inf for them so that conf is exactly 0 there. */
int opp_sim_lse_cols(const void* a, const void* b, float* part_m, float* part_s, float* col_m,
                     float* col_s, int batches, int rows, int cols, int k, float scale, int split,
                     const unsigned char* col_mask, opp_stream_t stream);
int opp_lse_col_finalize(const float* col_m, const float* col_s, float* lse, int batches, int groups,
                         int cols, const unsigned char* col_mask, opp_stream_t stream);

/* conf = exp((2 sim - lse_pt) - lse_px) (coarse_matching.py:115), rows = 3D points: per-row per-tile
 * (max, first argmax) into part_val/part_idx [B*rows][opp_sim_tiles(cols)], merged by
 * opp_best_finalize; conf (or NULL) fp32 [B*rows][cols] is data["conf_matrix"].  The column maxima
 * are folded into the same pass: colmax uint32 [B][cols] receives the float bits of
 * max_l conf[b, l, s] (zeroed inside, then atomicMax per 32-row group; conf >= 0 so the bits order
 * like the values). */
int opp_sim_conf_colmax(const void* a, const void* b, const float* lse_own, const float* lse_other,
                        float* conf, float* part_val, int* part_idx, unsigned* colmax, int batches,
                        int rows, int cols, int k, float scale, int split, opp_stream_t stream);

/* Bank sets (several objects in one forward, rows = the 3D points of each frame's object padded to
 * a common count): the two calls above with row_count int32 [B] (or NULL = the calls above).
 * Rows l >= row_count[b] are not rows of the matrix: they drop out of the column statistics and of
 * colmax, and conf stores 0 for them.  Their row partials (part_m / part_s, part_val / part_idx) are
 * not meaningful.  A 32-row group with no row below the count leaves (col_m, col_s) = (-inf, 0),
 * which opp_lse_col_finalize skips.  col_mask and row_count cannot be combined. */
int opp_sim_lse_cols_rows(const void* a, const void* b, float* part_m, float* part_s, float* col_m,
                          float* col_s, int batches, int rows, int cols, int k, float scale, int split,
                          const unsigned char* col_mask, const int* row_count, opp_stream_t stream);
int opp_sim_conf_colmax_rows(const void* a, const void* b, const float* lse_own, const float* lse_other,
                             float* conf, float* part_val, int* part_idx, unsigned* colmax, int batches,
                             int rows, int cols, int k, float scale, int split, const int* row_count,
                             opp_stream_t stream);

/* best[r] = max over tiles (ties -> lowest index) */
int opp_best_finalize(const float* part_val, const int* part_idx, float* best_val, int* best_idx,
                      long long rows, int tiles, opp_stream_t stream);

/* Threshold + top/left border + mutual nearest neighbour + ordered compaction
 * (coarse_matching.py:142-172, 223-239).  The mutual test is on values (coarse_matching.py:157-165
 * compares conf == conf.max(dim) the same way): row l keeps its argmax cell j iff pt_val[b][l] has
 * the same float bits as colmax[b][j] (from opp_sim_conf_colmax), so every row of an exact tie is
 * kept and the capacity of every output is batch*l.
 *   pt_val/pt_idx [B][l]: row maxima of conf;  colmax uint32 [B][s]: column maxima of conf
 *   kpts fp32 [B][l][3]; img_scale fp32 [B][2] = (h_scale, w_scale) or NULL
 *   scratch int32 [ceil(B*l/1024) + 2]
 *   bank_shared != 0: one object for the whole batch, kpts is [1][l][3] (no per-image copies)
 * Outputs (ascending (b, i) order): b_ids/i_ids/j_ids int64, mconf fp32, mkpts3d fp32 [.][3],
 * mkpts_c fp32 [.][2]; count_out int32 [1] = number of matches. */
int opp_match_select_colmax(const float* pt_val, const int* pt_idx, const unsigned* colmax,
                            const float* kpts, const float* img_scale, int batch, int l, int hc,
                            int wc, float thr, int border, float cell, int* scratch,
                            long long* b_ids, long long* i_ids, long long* j_ids, float* mconf,
                            float* mkpts3d, float* mkpts_c, int* count_out, int bank_shared,
                            opp_stream_t stream);

/* opp_match_select_colmax for a bank set: kpts fp32 [K][l][3] is read at bank_of_batch[b] (int32 [B],
 * entries in [0, K)), and rows i >= row_count[b] (int32 [B]) never match.  Both NULL = the call
 * above; one without the other is an error.  The capacity stays batch*l. */
int opp_match_select_colmax_set(const float* pt_val, const int* pt_idx, const unsigned* colmax,
                                const float* kpts, const float* img_scale, int batch, int l, int hc,
                                int wc, float thr, int border, float cell, int* scratch,
                                long long* b_ids, long long* i_ids, long long* j_ids, float* mconf,
                                float* mkpts3d, float* mkpts_c, int* count_out, int bank_shared,
                                const int* bank_of_batch, const int* row_count, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fine level — FinePreprocess (loftr_module/fine_preprocess.py:32-55), loftr_fine,
 * FineMatching (utils/fine_matching.py:28-110)
 * ---------------------------------------------------------------------------------------- */

/* Every fine-level entry point takes `count_dev`: NULL = `m` is the exact number of matches (known
 * on the host); otherwise `m` is the CAPACITY the buffers were sized for and the kernels read the
 * real match count from *count_dev (int32, device; written by the opp_match_select_* calls), so the whole
 * forward can be enqueued / captured in a CUDA graph without the host learning M first (the
 * reference synchronises in torch.where: coarse_matching.py:170). */

/* For match m: row 26m = descriptors3d_db[b, :, i]; rows 26m+1+ww = the 5x5 window (ww = ky*5+kx)
 * of the fine map centred on fine pixel (stride*jy, stride*jx), zero outside the map.
 * fine NHWC fp16 [B][hf][wf][planes*128]; desc3d fp32 [B][128][n];
 * x32 fp32 [26 M][128] (may be NULL) / x16 fp16 [26 M][planes*128];
 * bank_shared != 0: desc3d is [1][128][n], shared by every batch element;
 * windows != 0: `fine` is not the dense map but the compact per-match windows written by
 * opp_conv_win (win = 5): fp16 [M][5][8][planes*128] */
int opp_fine_gather(const void* fine, const float* desc3d, const long long* b_ids,
                    const long long* i_ids, const long long* j_ids, float* x32, void* x16, int m,
                    int hf, int wf, int wc, int stride, int n, int split, int bank_shared,
                    int windows, const int* count_dev, opp_stream_t stream);

/* opp_fine_gather for a bank set: desc3d fp32 [K][128][n] is read at bank_of_batch[b] (int32 [B]);
 * NULL = the call above. */
int opp_fine_gather_set(const void* fine, const float* desc3d, const long long* b_ids,
                        const long long* i_ids, const long long* j_ids, float* x32, void* x16, int m,
                        int hf, int wf, int wc, int stride, int n, int split, int bank_shared,
                        int windows, const int* count_dev, const int* bank_of_batch, opp_stream_t stream);

/* Linear attention for the 1 + 25 tokens of each match (linear_attention.py:29-61 with
 * L,S in {1,25}).  qkv fp16 [26 M][planes*384] = (elu(q)+1 | elu(k)+1 | v), 8 heads of 16.
 * cross = 0: self layer (each sequence attends to itself); 1: cross layer, both directions from
 * the pre-update tensors (transformer.py:154-159).  msg fp16 [26 M][planes*128] */
int opp_fine_attention(const void* qkv, void* msg, int m, int cross, float eps, int split,
                       const int* count_dev, opp_stream_t stream);

/* Correlation softmax + expectation + std (fine_matching.py:78-94) and sub-pixel coordinates
 * (fine_matching.py:96-110).  x32 fp32 [26 M][128]; img_scale fp32 [B][2] or NULL;
 * expec_f fp32 [M][3]; mkpts_f fp32 [M][2] */
int opp_fine_match(const float* x32, const float* mkpts_c, const long long* b_ids,
                   const float* img_scale, float* expec_f, float* mkpts_f, int m, float fine_scale,
                   const int* count_dev, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * LoFTR 2D-2D matcher (SURVEY §8 f3) — LoFTR_for_OnePose_Plus.forward
 * (src/KeypointFreeSfM/loftr_for_sfm/loftr.py:35-127; modules of submodules/LoFTR/src/loftr).
 * Backbone, transformer layers and dual-softmax passes are the entry points above; these four
 * are what differs from the 2D-3D matcher.
 * ---------------------------------------------------------------------------------------- */

/* LoFTR get_coarse_match (utils/coarse_matching.py:133-259, inference): threshold, `border` cells
 * removed on ALL sides of BOTH grids (:9-28), mutual nearest neighbour by value (rowmax == colmax),
 * ordered compaction.  pt_val/pt_idx [B][h0*w0] row maxima / argmax over image 1's cells, colmax
 * [B][h1*w1] (from opp_sim_conf_colmax).  scale0/scale1 fp32 [B][2] or NULL multiply (x, y) as
 * given (:248-253).  Capacity of the outputs: B*h0*w0.  scratch int32 [ceil(B*h0*w0/1024) + 2]. */
int opp_match_select_2d(const float* pt_val, const int* pt_idx, const unsigned* colmax, const float* scale0,
                        const float* scale1, int batch, int h0, int w0, int h1, int w1, float thr,
                        int border, float cell, int* scratch, long long* b_ids, long long* i_ids,
                        long long* j_ids, float* mconf, float* mkpts0_c, float* mkpts1_c, int* count_out,
                        opp_stream_t stream);

/* LoFTR FinePreprocess (loftr_module/fine_preprocess.py:30-59, fine_concat_coarse_feat False):
 * window x window patches (zero outside the map) of both fine maps, sequence-major rows
 * (seq * m + match) * window^2 + ww; seq 0 = image 0 centred on cell i_ids, seq 1 = image 1 on j_ids.
 * fine0/fine1 NHWC fp16 [B][hf][wf][planes*128]; x16 fp16 [2*m*window^2][planes*128]. */
int opp_fine_gather_2d(const void* fine0, const void* fine1, const long long* b_ids, const long long* i_ids,
                       const long long* j_ids, void* x16, int m, int hf0, int wf0, int wc0, int hf1, int wf1,
                       int wc1, int stride, int window, int split, opp_stream_t stream);

/* opp_fine_gather_2d over one store of many images' fine maps, fine NHWC fp16 [N][hf][wf][planes*128]:
 * match m reads image img0[m]'s map for seq 0 and image img1[m]'s for seq 1 (both sides one size). */
int opp_fine_gather_2d_images(const void* fine, const long long* img0, const long long* img1, const long long* i_ids,
                              const long long* j_ids, void* x16, int m, int hf, int wf, int wc, int stride,
                              int window, int split, opp_stream_t stream);

/* LinearAttention.forward (linear_attention.py:29-61) between small token groups, 8 heads x 16:
 * group g: q fp16 [g][l][planes*128] = elu(q_proj x)+1, kv fp16 [g][s][planes*256] =
 * (elu(k_proj src)+1 | v_proj src); out like q. */
int opp_seq_attention(const void* q, const void* kv, void* out, int groups, int l, int s, float eps, int split,
                      opp_stream_t stream);

/* LoFTR FineMatching.forward (utils/fine_matching.py:17-74): x32 fp32 [2][m][window^2][128]
 * (sequence-major), centre token of seq 0 against seq 1; expec_f [m][3], mkpts1_f [m][2] =
 * mkpts1_c + coords * (window // 2) * fine_scale * scale1[b]. */
int opp_fine_match_2d(const float* x32, const float* mkpts1_c, const long long* b_ids, const float* scale1,
                      float* expec_f, float* mkpts1_f, int m, int window, float fine_scale,
                      opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Pose from the matches — ransac_PnP (src/utils/metric_utils.py:121-204: cv2.solvePnPRansac with
 * EPnP, iterationsCount 10000, reprojectionError `pnp_reprojection_error`, per frame on the CPU
 * after a D2H copy; callers: compute_query_pose_errors metric_utils.py:207-292, demo.py:132)
 * ---------------------------------------------------------------------------------------- */

/* Batched RANSAC-PnP, one CTA per image, consuming the matcher's output lists in place.
 *   pts3d fp32 [m][3] (mkpts_3d_db), pts2d fp32 [m][2] (mkpts_query_f), m_bids int64 [m] ascending
 *   (the matches of image b are the run m_bids == b); intrinsics fp32 [batch][3][3];
 *   scale: point-cloud rescale (3D points are multiplied by it, t is divided by it: metric_utils.py:179,193)
 *   reproj_thr: inlier threshold in pixels; hypotheses: P3P minimal samples per image;
 *   seed: RNG seed (counter based: results are reproducible and independent of scheduling);
 *   refine_rounds: local-optimisation rounds (Gauss-Newton on the inliers + inlier re-selection)
 * Outputs: poses fp32 [batch][3][4] = [R | t] (identity when the image fails), n_inliers int32
 * [batch], inlier_mask uint8 [m], status int32 [batch] (1 = pose found from >= 4 inliers). */
int opp_pnp_ransac(const float* pts3d, const float* pts2d, const long long* m_bids, int m,
                   const float* intrinsics, int batch, float scale, float reproj_thr, int hypotheses,
                   unsigned seed, int refine_rounds, float* poses, int* n_inliers,
                   unsigned char* inlier_mask, int* status, opp_stream_t stream);

/* The use_pycolmap_ransac branch of ransac_PnP (metric_utils.py:137-170:
 * pycolmap.absolute_pose_estimation on a SIMPLE_PINHOLE camera), batched like opp_pnp_ransac and
 * with the same inputs and outputs, except:
 *   camera: f = K[0][0], principal point (K[0][2], K[1][2]); K[1][1] and the skew are not read;
 *   no scale: the 3D points are used as given and t is in their units;
 *   max_error_px: inlier = squared pixel error <= max_error_px^2 and in front of the camera;
 *   support of a model = (inlier count, then the smaller sum of squared errors of the inliers);
 *   lo_rounds: LO-RANSAC rounds (least squares on the inliers, kept while the support improves);
 *   the pose is then refined on that fixed inlier set by minimising sum log(1 + |r_i|^2) over the
 *   pixel residuals r_i (Cauchy loss of scale 1 per point), at most 100 iterations;
 *   inlier_mask / n_inliers: the inliers of the RANSAC model, before that refinement.
 * A frame with fewer than 4 matches, no admissible hypothesis or fewer than 4 inliers gets the
 * identity pose, n_inliers 0, a zero mask and status 0. */
int opp_pnp_ransac_colmap(const float* pts3d, const float* pts2d, const long long* m_bids, int m,
                          const float* intrinsics, int batch, float max_error_px, int hypotheses,
                          unsigned seed, int lo_rounds, float* poses, int* n_inliers,
                          unsigned char* inlier_mask, int* status, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * LINEMOD pose metrics — add_metric / projection_2d_error (src/utils/metric_utils.py:31-88, per
 * frame on the CPU with a scipy cKDTree for ADD-S; caller: the eval_ADD_metric branch of
 * compute_query_pose_errors :233-289)
 * ---------------------------------------------------------------------------------------- */

/* ADD / ADD-S and proj2D of `batch` frames of one object model, three launches.
 *   verts fp32 [num_verts][3] (model points); pose_pred, pose_gt fp32 [batch][3][4] = [R | t]
 *   (pose_pred as opp_pnp_ransac writes it); intrinsics fp32 [batch][3][3] (the ORIGINAL K);
 *   symmetric uint8 [batch]; scratch: at least opp_pose_metrics_scratch_bytes(num_verts, batch)
 *   bytes, 8-byte aligned.
 * Outputs fp64 [batch]: add_dist = mean_j |pred_j - tgt_j| (symmetric = 0) or the ADD-S mean
 * nearest-neighbour distance mean_j min_i |pred_i - tgt_j| (symmetric = 1), with pred = R_p x + t_p,
 * tgt = R_g x + t_g; proj2d = mean_j |pi(pred_j) - pi(tgt_j)| px, pi(p) = (K p)_xy / (K p)_z with no
 * guard on z (non-finite values propagate).  Deterministic: no floating-point atomics. */
int opp_pose_metrics(const float* verts, int num_verts, const float* pose_pred, const float* pose_gt,
                     const float* intrinsics, const unsigned char* symmetric, int batch, void* scratch,
                     long long scratch_bytes, double* add_dist, double* proj2d, opp_stream_t stream);

/* Scratch bytes opp_pose_metrics needs for num_verts model points and `batch` frames (0 if either
 * is not positive). */
long long opp_pose_metrics_scratch_bytes(int num_verts, int batch);

/* ------------------------------------------------------------------------------------------
 * Tracking front end — LocalFeatureObjectDetector.crop_img_by_bbox / previous_pose_detect
 * (src/local_feature_object_detector/local_feature_2D_detector.py:133-159, 200-226: two
 * cv2.warpAffine(INTER_LINEAR) calls of data_utils.get_image_crop_resize :239-255 per frame)
 * ---------------------------------------------------------------------------------------- */

/* Per-frame parameters of opp_crop_resize_u8 (64 bytes, 8-byte aligned):
 *   m: the INVERSE of the forward affine matrix of the warp, as cv2.warpAffine inverts it (fp64,
 *      row-major 2x3: src = m * (x, y, 1));
 *   (x0, y0, w, h): the virtual source — pixel (u, v) of the source is frame[v + y0][u + x0] for
 *      0 <= u < w, 0 <= v < h and inside the frame, else 0. */
typedef struct opp_crop_params {
  double m[6];
  int x0, y0, w, h;
} opp_crop_params;

/* cv2.warpAffine(src, M, (out_w, out_h), flags=INTER_LINEAR) of uint8 single-channel images, bit for
 * bit (cv2's fixed-point coordinates and 2^15-scaled bilinear weights, BORDER_CONSTANT 0), with src =
 * the virtual source of params[b].  For the two warps of crop_img_by_bbox, (x0, y0, w, h) is the box
 * and m is the inverse of the second (resize) warp: the first warp is the integer shift the virtual
 * source applies.  For one plain warp of the frame, (x0, y0, w, h) = (0, 0, width, height).
 *   frames uint8 [batch][height][width]; params [batch]; out uint8 [batch][out_h][out_w];
 *   status int32 [batch] or NULL: 0 = ok, 1 = w or h < 1 (cv2 raises), 2 = w or h >= 32767 (cv2
 *   raises) or a box coordinate with |.| >= 2^20 (outside the int32 fixed-point range); the crop of
 *   such a frame is written as zeros.  The params live on the device (so that the call can be
 *   captured in a CUDA graph): they are checked there, not on the host. */
int opp_crop_resize_u8(const unsigned char* frames, int batch, int height, int width,
                       const opp_crop_params* params, unsigned char* out, int out_h, int out_w, int* status,
                       opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training, coarse level — Loss.compute_coarse_loss, focal branch (src/lightning_model/
 * losses.py:18-58) on the dual-softmax confidence, forward and backward, without the [B, L, S]
 * matrix (opp_train.cu has the formulas).
 * ---------------------------------------------------------------------------------------- */

/* Row blocks (CTAs per batch element) of both calls below for `rows` 3D points. */
int opp_coarse_focal_blocks(int rows);

/* Softmax statistics of sim = scale * a b^T, computed from the same fp32 sim the two calls below
 * recompute (one statistics pass + an in-order merge of the column partials).
 *   a fp32 [B][rows][k], b fp32 [B][cols][k] (k = 256); col_mask uint8 [B][cols] or NULL (masked
 *   columns drop out of every row's softmax).  part_c fp32 [B][opp_coarse_focal_blocks(rows)][cols][2]
 *   workspace.  st_rows fp32 [B][rows][2], st_cols fp32 [B][cols][2]: (m, log s) with m = max of sim
 *   and s = sum exp(sim - m) over the row / column, so logsumexp = m + log s. */
int opp_coarse_focal_stats(const float* a, const float* b, const unsigned char* col_mask, int batches, int rows,
                           int cols, int k, float scale, float* part_c, float* st_rows, float* st_cols,
                           opp_stream_t stream);

/* Loss and the backward's per-row / per-column sums.
 *   a, b, col_mask as above; st_rows / st_cols from opp_coarse_focal_stats on the same a, b;
 *   gt [B][rows][cols], gt_bytes 1 (bool / uint8) or 2 (int16): 1 positive, 0 negative, anything
 *   else neither.
 *   Workspace (nb = opp_coarse_focal_blocks(rows)): part_loss fp64 [B*nb][2], part_cnt int64
 *   [B*nb][2], part_r fp64 [B][rows][2], part_c fp64 [B][nb][cols][2].
 *   Outputs: loss fp32 [1]; counts int64 [2] = (npos, nneg); wts fp32 [2] = (pos_w / npos,
 *   neg_w / nneg), 0 for an empty class; r fp64 [B][rows], c fp64 [B][cols] = the weighted sums of
 *   c dloss/dc over each row / column.  Deterministic (fixed-order sums, no atomics). */
int opp_coarse_focal_fwd(const float* a, const float* b, const float* st_rows, const float* st_cols,
                         const void* gt, int gt_bytes, const unsigned char* col_mask, int batches, int rows,
                         int cols, int k, float scale, float alpha, float gamma, float pos_w, float neg_w,
                         double* part_loss, long long* part_cnt, double* part_r, double* part_c, float* loss,
                         long long* counts, float* wts, double* r, double* c, opp_stream_t stream);

/* d loss / d a and d loss / d b times grad[0] (a device scalar: no host synchronisation), from the
 * statistics and r / c / wts of opp_coarse_focal_fwd.  da fp32 [B][rows][k], db fp32 [B][cols][k]
 * (overwritten).  Deterministic. */
int opp_coarse_focal_bwd(const float* a, const float* b, const float* st_rows, const float* st_cols,
                         const double* r, const double* c, const float* wts, const float* grad, const void* gt,
                         int gt_bytes, const unsigned char* col_mask, int batches, int rows, int cols, int k,
                         float scale, float alpha, float gamma, float* da, float* db, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training, sparse ground truth — the positives of conf_matrix_gt as a list (b_ids, i_ids, j_ids
 * int64 [g], ascending in (b, i, j), no duplicates: the order of torch.where on the dense matrix)
 * with their fine locations fine_xy fp32 [g][2], instead of the [B, L, S] and [B, L, S, 2] tensors.
 * ---------------------------------------------------------------------------------------- */

/* Index of the list by 3D point and by query cell.
 *   row_ptr int32 [B*rows + 1]: entries of row b*rows + i are [row_ptr[r], row_ptr[r + 1]).
 *   col_ptr int32 [B*cols + 1], col_rows int32 [g]: the i of the entries of column b*cols + j,
 *   ascending, at [col_ptr[c], col_ptr[c + 1]).  fill int32 [B*cols]: workspace.
 *   Several j per i and several i per j are legal; entries out of range are left out of the column
 *   view.  The result does not depend on launch order (integer atomics hand out slots, each
 *   bucket is then sorted; one thread sorts one bucket by insertion, which is quadratic in the
 *   number of 3D points of one cell). */
int opp_gt_index(const long long* b_ids, const long long* i_ids, const long long* j_ids, int g, int batches,
                 int rows, int cols, int* row_ptr, int* col_ptr, int* col_rows, int* fill, opp_stream_t stream);

/* opp_coarse_focal_fwd / _bwd with the class of an element taken from the list: 1 for a listed
 * (b, i, j), 0 for every other element.  row_ptr / col_ptr / col_rows from opp_gt_index of the same
 * list.  The arithmetic is that of the dense entry points, instruction for instruction: every output
 * has the bits the dense call gives on the dense form of the list. */
int opp_coarse_focal_fwd_sparse(const float* a, const float* b, const float* st_rows, const float* st_cols,
                                const int* row_ptr, const long long* j_ids, const unsigned char* col_mask,
                                int batches, int rows, int cols, int k, float scale, float alpha, float gamma,
                                float pos_w, float neg_w, double* part_loss, long long* part_cnt, double* part_r,
                                double* part_c, float* loss, long long* counts, float* wts, double* r, double* c,
                                opp_stream_t stream);

int opp_coarse_focal_bwd_sparse(const float* a, const float* b, const float* st_rows, const float* st_cols,
                                const double* r, const double* c, const float* wts, const float* grad,
                                const int* row_ptr, const long long* j_ids, const int* col_ptr, const int* col_rows,
                                const unsigned char* col_mask, int batches, int rows, int cols, int k, float scale,
                                float alpha, float gamma, float* da, float* db, opp_stream_t stream);

/* fine_supervision (src/models/OnePosePlus/utils/fine_supervision.py) from the list: for each of
 * the m matches (m_b, m_i, m_j int64) the fine location of (b, i, j), (-50, -50) when it is not in
 * the list, minus the cell's origin (j % w_c, j / w_c) * coarse scale, over the fine scale and the
 * window radius.  resolution = (coarse_res, fine_res).  img_scale fp32 [B][2] (query_image_scale,
 * (h, w) order) multiplies both scales; with img_scale NULL the coarse scale is fine_res, as in the
 * reference.  out fp32 [m][2]: the bits PyTorch's fp32 evaluation of the reference gives on the device. */
int opp_fine_supervision(const long long* b_ids, const long long* i_ids, const long long* j_ids,
                         const float* fine_xy, int g, int batches, int rows, int cols, const long long* m_b,
                         const long long* m_i, const long long* m_j, int m, int w_c, int coarse_res, int fine_res,
                         int radius, const float* img_scale, float* out, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training, fine level (opp_train_fine.cu): window gather, the two fine LoFTR layers and the
 * heatmap expectation, forward and backward, fp32.  Match m owns the 26 token rows m*26 + t
 * (t = ky*5 + kx the window, 25 the 3D token).  No floating-point atomics: every result is
 * bit-reproducible.
 * ---------------------------------------------------------------------------------------- */

/* Row groups (partials) of opp_fine_train_wgrad / _ln_bwd for `rows` rows. */
int opp_fine_train_groups(int rows);

/* x[m*26 + t][0..127] (row stride ldx): the 5 x 5 window of F.unfold(feat, 5, padding 2, stride)
 * around cell j_ids[m] (cells (j / wc, j % wc)), zeros outside the map, then desc3d[b][:, i].
 * feat fp32 [B][128][hf][wf], desc3d fp32 [B][128][n3d]. */
int opp_fine_train_gather(const float* feat, const float* desc3d, const long long* b_ids, const long long* i_ids,
                          const long long* j_ids, int m, int hf, int wf, int hc, int wc, int n3d, int stride,
                          float* x, int ldx, opp_stream_t stream);

/* d feat [B][128][hf][wf] (overwritten) from the window rows' gradient dx, one thread per element:
 * the cells whose window covers it in raster order, each cell's matches in the order of
 * col_rows[col_ptr[b*hc*wc + j] ..) (opp_gt_index's column view of the matches). */
int opp_fine_train_gather_bwd(const float* dx, int ldx, const int* col_ptr, const int* col_rows, int batches,
                              int hf, int wf, int hc, int wc, int stride, float* dfeat, opp_stream_t stream);

/* c[r][0..n) = epi(a[r][0..k) . B): B(k, n) = w[n][k] when trans_w, else w[k][n].  epi 0 store,
 * 1 ReLU (trans_w), 2 zero where aux <= 0, 3 add aux and aux2 (either may be NULL); 2 and 3 need
 * !trans_w.  n % 64 == 0, k % 16 == 0, 16-byte aligned rows. */
int opp_fine_train_linear(const float* a, int lda, const float* w, int trans_w, int rows, int n, int k, float* c,
                          int ldc, int epi, const float* aux, int ldaux, const float* aux2, int ldaux2,
                          opp_stream_t stream);

/* dw[n][k] (+)= sum_r g[r][n] a[r][k]: part fp32 [groups][n][k] per group of rows, then summed in
 * group order.  n, k multiples of 64. */
int opp_fine_train_wgrad(const float* g, int ldg, const float* a, int lda, int rows, int n, int k, float* part,
                         float* dw, int accumulate, opp_stream_t stream);

/* LayerNorm over 128 channels (eps 1e-5): y = LN(x) * gamma + beta (+ resid); stats [rows][2] =
 * (mean, rstd). */
int opp_fine_train_ln(const float* x, int ldx, const float* gamma, const float* beta, const float* resid, int ldr,
                      float* y, int ldy, float* stats, int rows, opp_stream_t stream);

/* Its backward: dx (overwritten) and dgb [2][128] (+)= (dgamma, dbeta); part [groups][2][128]. */
int opp_fine_train_ln_bwd(const float* x, int ldx, const float* gamma, const float* stats, const float* dy, int lddy,
                          float* dx, int lddx, int rows, float* part, float* dgb, int accumulate,
                          opp_stream_t stream);

/* Linear attention of one fine layer: qkv [m*26][384] = (q | k | v), out [m*26][128].  cross 0:
 * the window attends to the window and the 3D token to itself; cross 1: each to the other. */
int opp_fine_train_attention(const float* qkv, float* out, int m, int cross, float eps, opp_stream_t stream);
int opp_fine_train_attention_bwd(const float* qkv, const float* dout, float* dqkv, int m, int cross, float eps,
                                 opp_stream_t stream);

/* Heatmap expectation of x [m*26][128] (the last layer's output): expec_f [m][3] = (x, y, std), and
 * its backward to dx [m*26][128] (overwritten). */
int opp_fine_train_match(const float* x, int m, float* expec_f, opp_stream_t stream);
int opp_fine_train_match_bwd(const float* x, const float* dexpec, int m, float* dx, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training, coarse transformer (opp_train_coarse_tf.cu): linear attention of the coarse LoFTR
 * layers (d = 256, 8 heads of 32) forward and backward, and LayerNorm over 256 channels, fp32.
 * A sequence is passed as its first row, the row stride and len = rows per batch element (rows
 * b*len + s); qkv rows are (q | k | v), 768 floats; masks are uint8 [batches*len] (1 = keep) or
 * NULL.  Per head: K = elu(k) + 1, KV = sum_s (K_s m_s) (v_s m_s / len), ksum = sum_s K_s m_s,
 * Q = (elu(q) + 1) m, out = (Q KV) v_len / (Q . ksum + eps).  Rows run in chunks
 * (opp_coarse_tf_chunks); partials are summed in chunk order: every result is bit-reproducible.
 * ---------------------------------------------------------------------------------------- */

/* Chunks of a sequence of `len` rows per batch element (partials per batch element). */
int opp_coarse_tf_chunks(int len);

/* Source state of a sequence: kv fp32 [batches][8][32][32], ksum [batches][8][32]; part fp32
 * [batches][chunks][8*32*32 + 8*32]. */
int opp_coarse_tf_kv(const float* qkv, int ld, const unsigned char* mask, int batches, int len, float* part,
                     float* kv, float* ksum, opp_stream_t stream);

/* The message of every query row: out [batches*len][256] (row stride ldo). */
int opp_coarse_tf_attn(const float* qkv, int ld, const unsigned char* q_mask, int batches, int len, const float* kv,
                       const float* ksum, float v_len, float eps, float* out, int ldo, opp_stream_t stream);

/* Backward, query rows: dqkv's q columns (overwritten) from dout, and the gradient of the source
 * state dkv [batches][8][32][32], dksum [batches][8][32]; part as for opp_coarse_tf_kv. */
int opp_coarse_tf_attn_bwd_q(const float* qkv, int ld, const unsigned char* q_mask, int batches, int len,
                             const float* kv, const float* ksum, float v_len, float eps, const float* dout, int lddo,
                             float* dqkv, int lddq, float* part, float* dkv, float* dksum, opp_stream_t stream);

/* Backward, source rows (v_len = len): dqkv's k and v columns (overwritten) from dkv / dksum. */
int opp_coarse_tf_attn_bwd_kv(const float* qkv, int ld, const unsigned char* mask, int batches, int len,
                              const float* dkv, const float* dksum, float* dqkv, int lddq, opp_stream_t stream);

/* LayerNorm over 256 channels, as opp_fine_train_ln / _ln_bwd (part [groups][2][256], dgb [2][256];
 * groups = opp_fine_train_groups(rows)). */
int opp_coarse_tf_ln(const float* x, int ldx, const float* gamma, const float* beta, const float* resid, int ldr,
                     float* y, int ldy, float* stats, int rows, opp_stream_t stream);
int opp_coarse_tf_ln_bwd(const float* x, int ldx, const float* gamma, const float* stats, const float* dy, int lddy,
                         float* dx, int lddx, int rows, float* part, float* dgb, int accumulate, opp_stream_t stream);


/* ------------------------------------------------------------------------------------------
 * Training, backbone (opp_train_backbone.cu): the ResNet-FPN's convolutions, batch-statistics
 * BatchNorm + activation (+ residual) and the FPN's bilinear x2 upsample-add, forward and backward.
 * The convolutions run on the tensor cores in 3xTF32: each operand is split into tf32 hi + lo and
 * every k8 step sums lo·hi, hi·lo and hi·hi in fp32, so each product is within 3.01·2^-22 |a b| of
 * a·b before the fp32 accumulation (DESIGN §7 f4).  The rest is fp32.  Maps are NCHW fp32; weights
 * [c_out][c_in][k][k]; k in {1, 3, 7}, stride in {1, 2}, pad = k / 2; (h, w) is the convolution's
 * input size.  Every sum runs in a fixed order without floating-point atomics: results are
 * bit-reproducible.
 * ---------------------------------------------------------------------------------------- */

/* Output pixels per weight-gradient partial; BatchNorm partials of a [batches][c][hw] map per channel. */
int opp_backbone_train_wgrad_group(void);
int opp_backbone_train_bn_parts(int batches, int hw);

/* y [batches][c_out][ho][wo] = conv(x, w). */
int opp_backbone_train_conv(const float* x, const float* w, int batches, int c_in, int h, int wd, int c_out, int ksize,
                            int stride, float* y, opp_stream_t stream);
/* dx [batches][c_in][h][w] (+)= the data gradient of dy [batches][c_out][ho][wo]. */
int opp_backbone_train_conv_dgrad(const float* dy, const float* w, int batches, int c_in, int h, int wd, int c_out,
                                  int ksize, int stride, float* dx, int accumulate, opp_stream_t stream);
/* dw (+)= the weight gradient summed over the output pixels [pix0, pix0 + npix) of the flat (b, oy, ox)
 * index; pix0 a multiple of the group; part fp32 [ceil(npix / group)][c_out * c_in * k * k]. */
int opp_backbone_train_conv_wgrad(const float* x, const float* dy, int batches, int c_in, int h, int wd, int c_out,
                                  int ksize, int stride, int pix0, int npix, float* part, float* dw, int accumulate,
                                  opp_stream_t stream);
/* mean / invstd [c] of x [batches][c][hw] over batches * hw values (biased variance); when
 * running_mean / running_var are given they are updated as F.batch_norm does (unbiased variance).
 * part fp64 [c][parts][2]. */
int opp_backbone_train_bn_stats(const float* x, int batches, int c, int hw, float eps, double* part, float* mean,
                                float* invstd, float* running_mean, float* running_var, float momentum,
                                opp_stream_t stream);
/* y = act(gamma (x - mean) invstd + beta [+ res]); act 0 none, 1 ReLU, 2 LeakyReLU(0.01). */
int opp_backbone_train_bn_act(const float* x, int batches, int c, int hw, const float* mean, const float* invstd,
                              const float* gamma, const float* beta, const float* res, int act, float* y,
                              opp_stream_t stream);
/* Backward of opp_backbone_train_bn_act given its output y (NULL for act 0): dz = dy act'(y);
 * dx = gamma invstd (dz - sum dz / n - xhat sum(dz xhat) / n) when batch_stats, else gamma invstd dz;
 * dres = dz (or NULL); dgb [2][c] = (dgamma, dbeta).  dx may alias dy.  part fp64 [c][parts * 2 + 1]. */
int opp_backbone_train_bn_act_bwd(const float* x, const float* y, const float* dy, int batches, int c, int hw,
                                  const float* mean, const float* invstd, const float* gamma, int act,
                                  int batch_stats, double* part, float* dx, float* dres, float* dgb,
                                  opp_stream_t stream);
/* out [batches][c][2h][2w] = lat + bilinear x2 (align_corners) of in [batches][c][h][w]; out may alias lat. */
int opp_backbone_train_up2x_add(const float* in, const float* lat, int batches, int c, int h, int w, float* out,
                                opp_stream_t stream);
/* din [batches][c][h][w] (+)= the upsample's backward of dout [batches][c][2h][2w]. */
int opp_backbone_train_up2x_bwd(const float* dout, int batches, int c, int h, int w, float* din, int accumulate,
                                opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training, keypoint encoder (opp_train_kpt.cu): KeypointEncoding_linear 3-32-64-128-256 with
 * per-point InstanceNorm (eps 1e-5) + ReLU after the hidden layers, forward and backward, fp32 on the
 * CUDA cores.  kpts fp32 [batch][n][3] with stats [batch][4] from opp_kpt_stats; rows are the flat
 * (b, n) index.  pack fp32 [opp_kpt_train_pack_size()]: W1t b1 W2t b2 W3t b3 W4t b4 (weights
 * transposed, [in][out]) then W2 W3 W4 ([out][in]).  dparams fp32 [opp_kpt_train_params()]: dW1 db1
 * dW2 db2 dW3 db3 dW4 db4 in nn.Linear's layouts.  No floating-point atomics: bit-reproducible.
 * ---------------------------------------------------------------------------------------- */

/* Rows per weight-gradient partial (a backward slice starts at a multiple); floats of dparams / pack. */
int opp_kpt_train_group(void);
int opp_kpt_train_params(void);
int opp_kpt_train_pack_size(void);

/* out fp32 [batch * n][256] = desc^T + MLP(normalised kpts); desc fp32 [batch][256][n]. */
int opp_kpt_train_fwd(const float* kpts, const float* stats, const float* desc, const float* pack, float* out,
                      int batch, int n, opp_stream_t stream);
/* dparams (+)= the parameter gradient of out for dout fp32 [batch * n][256], summed over the rows
 * [row0, row0 + nrows) (row0 a multiple of the group) by recomputing their forward; part fp32
 * [ceil(nrows / group)][opp_kpt_train_params()] holds one partial per group, summed in group order. */
int opp_kpt_train_bwd(const float* kpts, const float* stats, const float* dout, const float* pack, int batch, int n,
                      int row0, int nrows, float* part, float* dparams, int accumulate, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training batch (opp_train_batch.cu): the homography augmentation of the query images and the
 * ground-truth correspondences projected from the pose (OnePosePlusDataset.read_anno,
 * src/datasets/OnePosePlus_dataset.py:341-444), fp32 with one rounding per operation.  pack fp32
 * [B][opp_train_batch_pack_size()] holds each item's R, t, K, the point warp, the pixel
 * normalisation, the image warp and the warp flag (layout in opp_train_batch.cu).
 * ---------------------------------------------------------------------------------------- */

int opp_train_batch_pack_size(void);

/* out fp32 [B][h][w]: kornia homography_warp of img fp32 [B][h][w] for the items whose warp flag is
 * set (bilinear, zero padding, align_corners=False), a copy of img for the others. */
int opp_homography_warp_f32(const float* img, const float* pack, int batches, int h, int w, float* out,
                            opp_stream_t stream);

/* The correspondences of B items, flattened: assign int64 [2][n] (2D keypoint, 3D point), item b
 * owns [offsets[b], offsets[b + 1]) and the 2D keypoints [kp_offsets[b], kp_offsets[b + 1]) of
 * n_kp; kp3d fp32 [B][rows][3]; img_scale fp32 [B][2] (query_image_scale).  Projects, warps,
 * rounds to the 8-px grid, keeps the first correspondence per cell and the last writer per 2D
 * keypoint and writes key int64 [n] = ((b rows + i) cols + j) R + rank (INT64_MAX when dropped,
 * R = ((w - 1) / 8 + 1) ((h - 1) / 8 + 1)) with its fine location key_xy fp32 [n][2].  Scratch:
 * cell_owner int32 [B][R], kp_owner int32 [n_kp], rank_of int32 [n], fine fp32 [n][2].
 * status int32 [2]: [0] error bits (1 cell index == cols or < 0, 2 assign[0] outside the item's
 * keypoints, 4 assign[1] outside [0, rows)), [1] set by opp_train_gt_compact. */
int opp_train_gt_build(const float* kp3d, const long long* assign, long long n, const long long* offsets,
                       const long long* kp_offsets, long long n_kp, const float* pack, const float* img_scale,
                       int batches, int rows, int h, int w, int w_c, int cols, int* cell_owner, int* kp_owner,
                       int* rank_of, float* fine, long long* key, float* key_xy, int* status, opp_stream_t stream);

/* From the keys sorted ascending (perm = their positions in key_xy): the last entry of each
 * (b, i, j) = key / ranks, in order, into b_ids / i_ids / j_ids int64 [n] and fine_xy fp32 [n][2];
 * status[1] = the number written.  One CTA. */
int opp_train_gt_compact(const long long* sorted_key, const long long* perm, long long n, const float* key_xy,
                         int rows, int cols, long long ranks, long long* b_ids, long long* i_ids, long long* j_ids,
                         float* fine_xy, int* status, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Keypoint-free SfM coarse matching (opp_sfm_points.cu): the 2D keypoint merge of
 * points2D_worker / update_matches / transform_points2D (coarse_match_worker.py:81-175).  The raw
 * matches of P pairs are fp32 [M][5] (x0, y0, x1, y1, mconf); pair p owns [offsets[p],
 * offsets[p + 1]) and names the images pair_img int32 [P][2].  Keys are int64 image << 42 | x << 21 | y
 * of the truncated coordinates: the caller guarantees 0 <= x, y < 2^21, images <= 2^20, mconf >= 0.
 * ---------------------------------------------------------------------------------------- */

/* key int64 [2M], conf fp32 [2M]: both endpoints of every match at their appearance index
 * 2 offsets[p] + side * (offsets[p + 1] - offsets[p]) + m. */
int opp_sfm_points_emit(const float* matches, long long m, const long long* offsets, const int* pair_img,
                        int pairs, long long* key, float* conf, opp_stream_t stream);

/* Entries of block_scratch (int32) that opp_sfm_points_segments needs for n sorted keys. */
int opp_sfm_points_segments_scratch(long long n);

/* From the n keys sorted ascending: start int32 [groups + 1] = the first position of each run of
 * equal keys and n; *groups int32 = the number of runs. */
int opp_sfm_points_segments(const long long* sorted_key, long long n, int* block_scratch, int* start, int* groups,
                            opp_stream_t stream);

/* One thread per group: ukey int64 [G] its key, sum fp64 [G] the sequential sum of conf[perm[j]] over
 * its run, rank_key int64 [G] = -bits(sum), img_off int64 [images + 1] the first group of each image. */
int opp_sfm_points_sums(const long long* sorted_key, const long long* perm, const float* conf, const int* start,
                        int groups, int images, long long* ukey, double* sum, long long* rank_key,
                        long long* img_off, opp_stream_t stream);

/* img_key int64 [G] = the image of group perm1[q] (perm1: the stable sort of rank_key). */
int opp_sfm_points_image_key(const long long* ukey, const long long* perm1, int groups, long long* img_key,
                             opp_stream_t stream);

/* q-th keypoint in (image, descending sum, ascending (x, y)) order, g = perm1[perm2[q]]:
 * kpts fp32 [G][2] = (x, y), scores fp32 [G] = sum rounded to fp32, id_of int64 [G]: id_of[g] =
 * q - img_off[image]. */
int opp_sfm_points_rank(const long long* ukey, const double* sum, const long long* img_off, const long long* perm1,
                        const long long* perm2, int groups, float* kpts, float* scores, long long* id_of,
                        opp_stream_t stream);

/* idx int64 [M][2] = the keypoint ids of each match's two endpoints; status int32 [1] = 1 when an
 * endpoint is missing from its image's keys (written -1). */
int opp_sfm_points_remap(const float* matches, long long m, const long long* offsets, const int* pair_img,
                         int pairs, const long long* ukey, const long long* img_off, const long long* id_of,
                         long long* idx, int* status, opp_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Keypoint-free SfM refinement (opp_sfm_refine.cu): feature sampling at keypoints and the track
 * feature aggregation of feature_aggregation_and_update (post_optimization/feature_aggregation.py).
 * ---------------------------------------------------------------------------------------- */

/* sample_feature_from_featuremap (loftr_for_sfm/utils/sample_feature_from_featuremap.py) at n
 * keypoints kpts [n][2] (x, y; fp64 when kpts_f64, else fp32) of images img int64 [n] (NULL: image 0)
 * in map NHWC fp16 [N][hm][wm][planes*channels] (hi plane, then lo plane when split).  imghw fp32
 * [N][2] = (h, w) of each image in pixels times its scale.  grid_sample(align_corners=True, zeros
 * padding), nearest (round half to even) when `nearest`, else bilinear.  out fp32 [n][channels]. */
int opp_sample_feature(const void* map, const long long* img, const void* kpts, int kpts_f64, long long n, int hm,
                       int wm, int channels, int split, const float* imghw, int nearest, float* out,
                       opp_stream_t stream);

/* row int64 [q]: for each query key, perm[j] where sorted_key[j] is its only occurrence among the n
 * sorted keys; -1 when the key is absent, -2 when it occurs more than once. */
int opp_sfm_refine_lookup(const long long* sorted_key, const long long* perm, long long n, const long long* query,
                          long long q, long long* row, opp_stream_t stream);

/* Track t owns members [track_off[t], track_off[t + 1]) (at least one), member k reads row[k]:
 * mean_c fp32 [T][dc] = the fp32 sum of c0[row[k]] in member order divided by the count (np.mean
 * of the stacked rows), mean_f [T][df] the same over f0; ref_c fp32 [K][dc] = c1[row[k]], ref_f
 * [K][df] = f1[row[k]]. */
int opp_sfm_refine_aggregate(const float* c0, const float* c1, const float* f0, const float* f1, int dc, int df,
                             const long long* row, const long long* track_off, int tracks, float* mean_c,
                             float* mean_f, float* ref_c, float* ref_f, opp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OPP_B200_H_ */
