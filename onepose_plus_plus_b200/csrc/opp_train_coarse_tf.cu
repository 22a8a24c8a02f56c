// opp_train_coarse_tf.cu — the coarse LoFTR transformer of training on the device: linear attention
// forward and backward over the 2D and 3D token rows, and LayerNorm over 256 channels (DESIGN §7 f4).
// The projections, the merge and the MLP run on the fine level's token-row GEMMs
// (opp_fine_train_linear / _wgrad); train_coarse_tf.py drives the layers.
//
// Rows: one fp32 buffer holds both sequences, the 2D rows [0, B·S) and the 3D rows [B·S, B·S + B·N);
// a kernel is handed one sequence as (pointer to its first row, row stride, len = rows per batch
// element).  qkv rows are [q | k | v], 768 floats.  Per head h (32 channels) of batch element b:
//   K_s = elu(k_s) + 1, m_s the source row's mask (1 without a mask), n = len of the source (masked
//   rows included: v_len of linear_attention.py:29-61),
//   KV = sum_s (K_s m_s) ⊗ (v_s m_s / n),  ksum = sum_s K_s m_s,
//   Q_l = (elu(q_l) + 1) · m_l,  Z_l = 1 / (Q_l · ksum + eps),  out_l = (Q_l KV) Z_l n.
// Each warp owns one head; lane i owns channel h·32 + i of a row, and the other lanes' values come by
// shuffle.  Rows are taken in chunks of kChunk per CTA; the per-chunk partials of KV / ksum (forward)
// and dKV / dksum (backward) are summed in chunk order by coarse_state_merge_kernel.  No floating-point
// atomics: two calls give the same bits.
#include <cmath>
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"
#include "opp_train_rows.cuh"

namespace opp {
namespace {

constexpr int kC = 256;              // d_model
constexpr int kHd = 32;              // channels per head
constexpr int kHeads = kC / kHd;     // 8: one warp each
constexpr int kQkv = 3 * kC;         // q | k | v
constexpr int kChunk = 128;          // rows per CTA (and per partial)
constexpr int kKvSize = kHeads * kHd * kHd;       // KV of one batch element
constexpr int kState = kKvSize + kHeads * kHd;    // KV then ksum, per partial
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v + 1.f : expf(v); }

// part[b][chunk] = (KV [8][32][32], ksum [8][32]) of the chunk's source rows.
__global__ void __launch_bounds__(256) coarse_kv_kernel(const float* __restrict__ qkv, int ld,
                                                        const uint8_t* __restrict__ mask, int len,
                                                        float* __restrict__ part) {
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, h = threadIdx.x >> 5;
  const int s0 = chunk * kChunk, s1 = min(len, s0 + kChunk);
  const float n = (float)len;
  float acc[kHd] = {};
  float ks = 0.f;
  for (int s = s0; s < s1; ++s) {
    const size_t row = (size_t)b * len + s;
    const float m = mask ? (float)mask[row] : 1.f;
    const float* p = qkv + row * ld + h * kHd + lane;
    const float k = elu1(p[kC]) * m;
    const float v = p[2 * kC] * m / n;
    ks += k;
#pragma unroll
    for (int d = 0; d < kHd; ++d) acc[d] = fmaf(__shfl_sync(kFull, k, d), v, acc[d]);
  }
  float* out = part + ((size_t)b * gridDim.x + chunk) * kState;
#pragma unroll
  for (int d = 0; d < kHd; ++d) out[(h * kHd + d) * kHd + lane] = acc[d];
  out[kKvSize + h * kHd + lane] = ks;
}

// kv[b] / ksum[b] = sum over the chunks c (ascending) of part[b][c].
__global__ void __launch_bounds__(256) coarse_state_merge_kernel(const float* __restrict__ part, int chunks,
                                                                 float* __restrict__ kv, float* __restrict__ ksum) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (e >= kState) return;
  const float* p = part + (size_t)b * chunks * kState + e;
  float s = 0.f;
  for (int c = 0; c < chunks; ++c) s += p[(size_t)c * kState];
  if (e < kKvSize) kv[(size_t)b * kKvSize + e] = s;
  else ksum[b * kHeads * kHd + e - kKvSize] = s;
}

// out_l = (Q_l KV) Z_l n for the query rows of chunk blockIdx.x of batch element blockIdx.y.
__global__ void __launch_bounds__(256) coarse_attn_kernel(const float* __restrict__ qkv, int ld,
                                                          const uint8_t* __restrict__ q_mask, int len,
                                                          const float* __restrict__ kv,
                                                          const float* __restrict__ ksum, float v_len, float eps,
                                                          float* __restrict__ out, int ldo) {
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, h = threadIdx.x >> 5;
  const float* st = kv + (size_t)b * kKvSize + h * kHd * kHd;
  float kvc[kHd];   // KV[d][lane]
#pragma unroll
  for (int d = 0; d < kHd; ++d) kvc[d] = st[d * kHd + lane];
  const float ksl = ksum[(b * kHeads + h) * kHd + lane];
  const int l0 = chunk * kChunk, l1 = min(len, l0 + kChunk);
  for (int l = l0; l < l1; ++l) {
    const size_t row = (size_t)b * len + l;
    const float m = q_mask ? (float)q_mask[row] : 1.f;
    const float q = elu1(qkv[row * ld + h * kHd + lane]) * m;
    const float den = warp_sum(q * ksl);
    float num = 0.f;
#pragma unroll
    for (int d = 0; d < kHd; ++d) num = fmaf(__shfl_sync(kFull, q, d), kvc[d], num);
    const float z = 1.f / (den + eps);
    out[row * ldo + h * kHd + lane] = num * z * v_len;
  }
}

// Query pass of the backward.  With g = d out_l, A_l = Q_l KV:
//   dU_l = g Z_l n, dden_l = -n Z_l^2 (g · A_l), dQ_l = KV dU_l + ksum dden_l,
//   dq_l = dQ_l m_l elu'(q_l) (elu'(x) = 1 for x > 0, else exp(x)), written to dqkv's q columns;
//   part[b][chunk] = (sum_l Q_l ⊗ dU_l, sum_l Q_l dden_l) over the chunk's rows.
__global__ void __launch_bounds__(256) coarse_attn_bwd_q_kernel(const float* __restrict__ qkv, int ld,
                                                                const uint8_t* __restrict__ q_mask, int len,
                                                                const float* __restrict__ kv,
                                                                const float* __restrict__ ksum, float v_len,
                                                                float eps, const float* __restrict__ dout,
                                                                int lddo, float* __restrict__ dqkv, int lddq,
                                                                float* __restrict__ part) {
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, h = threadIdx.x >> 5;
  const float* st = kv + (size_t)b * kKvSize + h * kHd * kHd;
  float kvc[kHd], kvr[kHd], dkv[kHd];   // KV[d][lane], KV[lane][e], dKV[d][lane]
#pragma unroll
  for (int d = 0; d < kHd; ++d) kvc[d] = st[d * kHd + lane], kvr[d] = st[lane * kHd + d], dkv[d] = 0.f;
  const float ksl = ksum[(b * kHeads + h) * kHd + lane];
  float dks = 0.f;
  const int l0 = chunk * kChunk, l1 = min(len, l0 + kChunk);
  for (int l = l0; l < l1; ++l) {
    const size_t row = (size_t)b * len + l;
    const float m = q_mask ? (float)q_mask[row] : 1.f;
    const float qraw = qkv[row * ld + h * kHd + lane];
    const float qe = elu1(qraw), q = qe * m;
    const float den = warp_sum(q * ksl);
    float num = 0.f;
#pragma unroll
    for (int d = 0; d < kHd; ++d) num = fmaf(__shfl_sync(kFull, q, d), kvc[d], num);
    const float z = 1.f / (den + eps);
    const float g = dout[row * lddo + h * kHd + lane];
    const float du = g * z * v_len;
    const float dden = -v_len * z * z * warp_sum(g * num);
    float dq = ksl * dden;
#pragma unroll
    for (int e = 0; e < kHd; ++e) dq = fmaf(kvr[e], __shfl_sync(kFull, du, e), dq);
    dqkv[row * lddq + h * kHd + lane] = dq * m * (qraw > 0.f ? 1.f : qe);
#pragma unroll
    for (int d = 0; d < kHd; ++d) dkv[d] = fmaf(__shfl_sync(kFull, q, d), du, dkv[d]);
    dks = fmaf(q, dden, dks);
  }
  float* out = part + ((size_t)b * gridDim.x + chunk) * kState;
#pragma unroll
  for (int d = 0; d < kHd; ++d) out[(h * kHd + d) * kHd + lane] = dkv[d];
  out[kKvSize + h * kHd + lane] = dks;
}

// Source pass of the backward, to dqkv's k and v columns of the source rows:
//   dk_s = m_s (dKV v_s / n + dksum) elu'(k_s),  dv_s = (m_s / n) dKV^T K_s.
__global__ void __launch_bounds__(256) coarse_attn_bwd_kv_kernel(const float* __restrict__ qkv, int ld,
                                                                 const uint8_t* __restrict__ mask, int len,
                                                                 const float* __restrict__ dkv,
                                                                 const float* __restrict__ dksum,
                                                                 float* __restrict__ dqkv, int lddq) {
  const int chunk = blockIdx.x, b = blockIdx.y;
  const int lane = threadIdx.x & 31, h = threadIdx.x >> 5;
  const float* st = dkv + (size_t)b * kKvSize + h * kHd * kHd;
  float dkc[kHd], dkr[kHd];   // dKV[d][lane], dKV[lane][e]
#pragma unroll
  for (int d = 0; d < kHd; ++d) dkc[d] = st[d * kHd + lane], dkr[d] = st[lane * kHd + d];
  const float dksl = dksum[(b * kHeads + h) * kHd + lane];
  const float n = (float)len;
  const int s0 = chunk * kChunk, s1 = min(len, s0 + kChunk);
  for (int s = s0; s < s1; ++s) {
    const size_t row = (size_t)b * len + s;
    const float m = mask ? (float)mask[row] : 1.f;
    const float* p = qkv + row * ld + h * kHd + lane;
    const float kraw = p[kC], v = p[2 * kC];
    const float k = elu1(kraw);
    float t = 0.f, u = 0.f;
#pragma unroll
    for (int e = 0; e < kHd; ++e) t = fmaf(dkr[e], __shfl_sync(kFull, v, e), t);
#pragma unroll
    for (int d = 0; d < kHd; ++d) u = fmaf(dkc[d], __shfl_sync(kFull, k, d), u);
    float* dp = dqkv + row * lddq + h * kHd + lane;
    dp[kC] = m * (t / n + dksl) * (kraw > 0.f ? 1.f : k);
    dp[2 * kC] = m * u / n;
  }
}

bool aligned4(const void* p, int ld) { return ((uintptr_t)p & 15) == 0 && ld % 4 == 0; }

int chunks_of(int len) { return (len + kChunk - 1) / kChunk; }

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" {

int opp_coarse_tf_chunks(int len) { return chunks_of(len); }

int opp_coarse_tf_kv(const float* qkv, int ld, const unsigned char* mask, int batches, int len, float* part,
                     float* kv, float* ksum, opp_stream_t stream) {
  OPP_REQUIRE(batches > 0 && len > 0 && ld >= kQkv, "opp_coarse_tf_kv: batches %d, len %d, ld %d", batches, len, ld);
  OPP_REQUIRE(qkv && part && kv && ksum, "opp_coarse_tf_kv: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = chunks_of(len);
  coarse_kv_kernel<<<dim3(chunks, batches), 256, 0, st>>>(qkv, ld, mask, len, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  coarse_state_merge_kernel<<<dim3((kState + 255) / 256, batches), 256, 0, st>>>(part, chunks, kv, ksum);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_coarse_tf_attn(const float* qkv, int ld, const unsigned char* q_mask, int batches, int len, const float* kv,
                       const float* ksum, float v_len, float eps, float* out, int ldo, opp_stream_t stream) {
  OPP_REQUIRE(batches > 0 && len > 0 && ld >= kQkv && ldo >= kC, "opp_coarse_tf_attn: batches %d, len %d",
              batches, len);
  OPP_REQUIRE(qkv && kv && ksum && out, "opp_coarse_tf_attn: null pointer");
  coarse_attn_kernel<<<dim3(chunks_of(len), batches), 256, 0, (cudaStream_t)stream>>>(qkv, ld, q_mask, len, kv, ksum,
                                                                                      v_len, eps, out, ldo);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_coarse_tf_attn_bwd_q(const float* qkv, int ld, const unsigned char* q_mask, int batches, int len,
                             const float* kv, const float* ksum, float v_len, float eps, const float* dout, int lddo,
                             float* dqkv, int lddq, float* part, float* dkv, float* dksum, opp_stream_t stream) {
  OPP_REQUIRE(batches > 0 && len > 0 && ld >= kQkv && lddo >= kC && lddq >= kQkv,
              "opp_coarse_tf_attn_bwd_q: batches %d, len %d", batches, len);
  OPP_REQUIRE(qkv && kv && ksum && dout && dqkv && part && dkv && dksum, "opp_coarse_tf_attn_bwd_q: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = chunks_of(len);
  coarse_attn_bwd_q_kernel<<<dim3(chunks, batches), 256, 0, st>>>(qkv, ld, q_mask, len, kv, ksum, v_len, eps, dout,
                                                                  lddo, dqkv, lddq, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  coarse_state_merge_kernel<<<dim3((kState + 255) / 256, batches), 256, 0, st>>>(part, chunks, dkv, dksum);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_coarse_tf_attn_bwd_kv(const float* qkv, int ld, const unsigned char* mask, int batches, int len,
                              const float* dkv, const float* dksum, float* dqkv, int lddq, opp_stream_t stream) {
  OPP_REQUIRE(batches > 0 && len > 0 && ld >= kQkv && lddq >= kQkv, "opp_coarse_tf_attn_bwd_kv: batches %d, len %d",
              batches, len);
  OPP_REQUIRE(qkv && dkv && dksum && dqkv, "opp_coarse_tf_attn_bwd_kv: null pointer");
  coarse_attn_bwd_kv_kernel<<<dim3(chunks_of(len), batches), 256, 0, (cudaStream_t)stream>>>(qkv, ld, mask, len, dkv,
                                                                                             dksum, dqkv, lddq);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_coarse_tf_ln(const float* x, int ldx, const float* gamma, const float* beta, const float* resid, int ldr,
                     float* y, int ldy, float* stats, int rows, opp_stream_t stream) {
  OPP_REQUIRE(rows >= 0, "opp_coarse_tf_ln: rows %d", rows);
  if (rows == 0) return OPP_OK;
  OPP_REQUIRE(x && gamma && beta && y && stats && aligned4(x, ldx) && aligned4(y, ldy) &&
                  (!resid || aligned4(resid, ldr)),
              "opp_coarse_tf_ln: bad operand");
  train_ln_fwd_kernel<kC><<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, ldx, gamma, beta, resid, ldr, y, ldy,
                                                                            reinterpret_cast<float2*>(stats), rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_coarse_tf_ln_bwd(const float* x, int ldx, const float* gamma, const float* stats, const float* dy, int lddy,
                         float* dx, int lddx, int rows, float* part, float* dgb, int accumulate, opp_stream_t stream) {
  OPP_REQUIRE(rows > 0, "opp_coarse_tf_ln_bwd: rows %d", rows);
  OPP_REQUIRE(x && gamma && stats && dy && dx && part && dgb && aligned4(x, ldx) && aligned4(dy, lddy) &&
                  aligned4(dx, lddx),
              "opp_coarse_tf_ln_bwd: bad operand");
  const cudaStream_t st = (cudaStream_t)stream;
  const int groups = (rows + kGroupRows - 1) / kGroupRows;
  train_ln_bwd_kernel<kC><<<groups, 256, 0, st>>>(x, ldx, gamma, reinterpret_cast<const float2*>(stats), dy, lddy, dx,
                                                  lddx, part, rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  fine_reduce_kernel<<<(2 * kC + 255) / 256, 256, 0, st>>>(part, groups, 2 * kC, accumulate, dgb);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
