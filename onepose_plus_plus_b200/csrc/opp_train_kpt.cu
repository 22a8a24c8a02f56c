// opp_train_kpt.cu — the keypoint encoder of training on the device: KeypointEncoding_linear
// (utils/position_encoding.py:46-79, norm_method "instancenorm") forward and backward, fp32 on the CUDA
// cores (DESIGN §7 f4).
//
// Per point p (x0 = the normalised keypoint, opp_kpt_stats' statistics):
//   a_l = W_l z_{l-1} + b_l,   y_l = (a_l - mean(a_l)) r_l,   r_l = 1 / sqrt(var(a_l) + 1e-5),
//   z_l = relu(y_l)   for l = 1, 2, 3 (32, 64, 128 channels; z_0 = x0),
//   out = W_4 z_3 + b_4 + desc   (256 channels, written as fp32 rows [B*N][256]).
// Backward from g = d out:  dz_3 = W_4^T g;  per hidden layer dy = [y > 0] dz,
//   da = r (dy - mean(dy) - y mean(dy y)),  dz_{l-1} = W_l^T da;  dW_l = sum_p da ⊗ z_{l-1}, db_l = sum_p da.
//
// One CTA handles one tile of kG consecutive rows of the flat (b, n) index.  The backward recomputes
// the tile's forward with the same device code (so the ReLU masks are the forward's) and keeps every
// activation in shared memory: nothing per point is stored between the passes.  The tile is also the
// weight-gradient group: each CTA writes its tile's sums (over its kG points in order) to one partial,
// and kpt_reduce adds the partials in tile order.  No floating-point atomics: two calls give the same bits.
//
// pack (fp32, built by train_kpt.pack): W1ᵀ b1 W2ᵀ b2 W3ᵀ b3 W4ᵀ b4 (transposed [in][out] for the
// forward) then W2 W3 W4 ([out][in], nn.Linear's layout, for the data gradient).
// dparams: dW1 db1 dW2 db2 dW3 db3 dW4 db4 in nn.Linear's layouts (encoder.{0,3,6,9}.{weight,bias}).
#include <cmath>
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kG = 32;          // rows per tile = per weight-gradient partial
constexpr int kThreads = 256;
constexpr int C0 = 3, C1 = 32, C2 = 64, C3 = 128, C4 = 256;

// pack offsets
constexpr int kW1t = 0, kB1 = kW1t + C0 * C1, kW2t = kB1 + C1, kB2 = kW2t + C1 * C2, kW3t = kB2 + C2,
              kB3 = kW3t + C2 * C3, kW4t = kB3 + C3, kB4 = kW4t + C3 * C4, kW2 = kB4 + C4, kW3 = kW2 + C2 * C1,
              kW4 = kW3 + C3 * C2, kPack = kW4 + C4 * C3;
// gradient offsets (one partial)
constexpr int gW1 = 0, gB1 = gW1 + C1 * C0, gW2 = gB1 + C1, gB2 = gW2 + C2 * C1, gW3 = gB2 + C2,
              gB3 = gW3 + C3 * C2, gW4 = gB3 + C3, gB4 = gW4 + C4 * C3, kParams = gB4 + C4;
static_assert(kParams == 43584, "eight parameter tensors of the 3-32-64-128-256 encoder");

// shared memory (floats); every buffer starts on a 16-byte boundary
constexpr int sX0 = 0, sR = sX0 + kG * 4, sY1 = sR + kG * 4, sZ1 = sY1 + kG * C1, sY2 = sZ1 + kG * C1,
              sZ2 = sY2 + kG * C2, sY3 = sZ2 + kG * C2, sZ3 = sY3 + kG * C3, sBig = sZ3 + kG * C3;
constexpr int kLdOut = C4 + 1;                         // forward output tile, padded for the descriptor add
constexpr int kFwdSmem = (sBig + kG * kLdOut) * 4;
constexpr int sD3 = sBig + kG * C4, sD2 = sD3 + kG * C3;   // backward: g [kG][256], d3 (then d1), d2
constexpr int kBwdSmem = (sD2 + kG * C2) * 4;

// out[p][j] = bias[j] + sum_k in[p][k] m[k][j] for the kG points; m is [K][NOUT] in global memory
// (coalesced over j), in / out are [kG][K] / [kG][LDO] in shared memory.  bias may be null.
template <int K, int NOUT, int LDO = NOUT>
__device__ __forceinline__ void rows_gemm(const float* __restrict__ in_s, const float* __restrict__ m,
                                          const float* __restrict__ bias, float* __restrict__ out_s) {
  constexpr int NG = kThreads / NOUT, PPT = kG / NG;
  static_assert(NG * NOUT == kThreads && PPT * NG == kG, "thread mapping");
  const int j = threadIdx.x % NOUT, g = threadIdx.x / NOUT;
  const float b0 = bias ? bias[j] : 0.f;
  float acc[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) acc[i] = b0;
  if constexpr (K % 4 == 0) {
#pragma unroll 2
    for (int k = 0; k < K; k += 4) {
      const float w0 = __ldg(m + (k + 0) * NOUT + j), w1 = __ldg(m + (k + 1) * NOUT + j),
                  w2 = __ldg(m + (k + 2) * NOUT + j), w3 = __ldg(m + (k + 3) * NOUT + j);
#pragma unroll
      for (int i = 0; i < PPT; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(in_s + (g + NG * i) * K + k);
        acc[i] = fmaf(v.x, w0, acc[i]);
        acc[i] = fmaf(v.y, w1, acc[i]);
        acc[i] = fmaf(v.z, w2, acc[i]);
        acc[i] = fmaf(v.w, w3, acc[i]);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float w = __ldg(m + k * NOUT + j);
#pragma unroll
      for (int i = 0; i < PPT; ++i) acc[i] = fmaf(in_s[(g + NG * i) * K + k], w, acc[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < PPT; ++i) out_s[(g + NG * i) * LDO + j] = acc[i];
}

// InstanceNorm1d over the C features of each point (biased variance, eps 1e-5), then ReLU: y_s holds
// a on entry and y on exit, z_s = relu(y), r_s[p * 4 + layer] = 1 / sqrt(var + eps).  One warp per point.
template <int C>
__device__ __forceinline__ void inorm_relu(float* __restrict__ y_s, float* __restrict__ z_s,
                                           float* __restrict__ r_s, int layer) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int p = warp; p < kG; p += kThreads / 32) {
    float* row = y_s + p * C;
    float s = 0.f;
#pragma unroll
    for (int k = lane; k < C; k += 32) s += row[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int k = lane; k < C; k += 32) {
      const float d = row[k] - mean;
      q = fmaf(d, d, q);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float r = 1.f / sqrtf(q / (float)C + 1e-5f);
#pragma unroll
    for (int k = lane; k < C; k += 32) {
      const float y = (row[k] - mean) * r;
      row[k] = y;
      z_s[p * C + k] = fmaxf(y, 0.f);
    }
    if (lane == 0) r_s[p * 4 + layer] = r;
  }
}

// Backward of inorm_relu in place: d_s holds dz on entry and da on exit.
template <int C>
__device__ __forceinline__ void inorm_relu_bwd(const float* __restrict__ y_s, float* __restrict__ d_s,
                                               const float* __restrict__ r_s, int layer) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int p = warp; p < kG; p += kThreads / 32) {
    const float* y = y_s + p * C;
    float* d = d_s + p * C;
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = lane; k < C; k += 32) {
      const float dy = y[k] > 0.f ? d[k] : 0.f;
      s1 += dy;
      s2 = fmaf(dy, y[k], s2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 / (float)C, m2 = s2 / (float)C, r = r_s[p * 4 + layer];
#pragma unroll
    for (int k = lane; k < C; k += 32) {
      const float dy = y[k] > 0.f ? d[k] : 0.f;
      d[k] = r * (dy - m1 - y[k] * m2);
    }
  }
}

// One tile's weight-gradient partial of a layer: part[c * K + k] = sum_p d[p][c] z[p][k] and
// part[NOUT * K + c] = sum_p d[p][c], each summed over p = 0 .. kG-1 in order.
template <int NOUT, int K>
__device__ __forceinline__ void tile_wgrad(const float* __restrict__ d_s, const float* __restrict__ z_s,
                                           float* __restrict__ part) {
  constexpr int SL = kThreads / NOUT, KPS = K / SL;     // thread -> (c, slice of KPS k's)
  const int c = threadIdx.x % NOUT, sl = threadIdx.x / NOUT;
  if constexpr (KPS >= 4) {
    constexpr int KC = KPS < 32 ? KPS : 32;
#pragma unroll 1
    for (int k0 = sl * KPS; k0 < (sl + 1) * KPS; k0 += KC) {
      float acc[KC];
#pragma unroll
      for (int j = 0; j < KC; ++j) acc[j] = 0.f;
#pragma unroll 2
      for (int p = 0; p < kG; ++p) {
        const float d = d_s[p * NOUT + c];
#pragma unroll
        for (int j = 0; j < KC; j += 4) {
          const float4 z = *reinterpret_cast<const float4*>(z_s + p * K + k0 + j);
          acc[j] = fmaf(d, z.x, acc[j]);
          acc[j + 1] = fmaf(d, z.y, acc[j + 1]);
          acc[j + 2] = fmaf(d, z.z, acc[j + 2]);
          acc[j + 3] = fmaf(d, z.w, acc[j + 3]);
        }
      }
#pragma unroll
      for (int j = 0; j < KC; ++j) part[c * K + k0 + j] = acc[j];
    }
  } else {   // the first layer (K = 3): one element per thread
    for (int e = threadIdx.x; e < NOUT * K; e += kThreads) {
      const int cc = e / K, k = e - cc * K;
      float acc = 0.f;
      for (int p = 0; p < kG; ++p) acc = fmaf(d_s[p * NOUT + cc], z_s[p * K + k], acc);
      part[e] = acc;
    }
  }
  if (sl == 0) {
    float s = 0.f;
    for (int p = 0; p < kG; ++p) s += d_s[p * NOUT + c];
    part[NOUT * K + c] = s;
  }
}

// The three hidden layers of the tile starting at row r0 (count valid rows; the others run on x0 = 0).
__device__ __forceinline__ void tile_forward(float* __restrict__ s, const float* __restrict__ kpts,
                                             const float* __restrict__ stats, const float* __restrict__ pack,
                                             int n, int r0, int count) {
  if (threadIdx.x < kG * C0) {
    const int p = threadIdx.x / C0, a = threadIdx.x - p * C0;
    float v = 0.f;
    if (p < count) {
      const int row = r0 + p, b = row / n;
      v = (kpts[(long long)row * 3 + a] - stats[b * 4 + a]) / stats[b * 4 + 3];
    }
    s[sX0 + p * C0 + a] = v;
  }
  __syncthreads();
  rows_gemm<C0, C1>(s + sX0, pack + kW1t, pack + kB1, s + sY1);
  __syncthreads();
  inorm_relu<C1>(s + sY1, s + sZ1, s + sR, 0);
  __syncthreads();
  rows_gemm<C1, C2>(s + sZ1, pack + kW2t, pack + kB2, s + sY2);
  __syncthreads();
  inorm_relu<C2>(s + sY2, s + sZ2, s + sR, 1);
  __syncthreads();
  rows_gemm<C2, C3>(s + sZ2, pack + kW3t, pack + kB3, s + sY3);
  __syncthreads();
  inorm_relu<C3>(s + sY3, s + sZ3, s + sR, 2);
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) kpt_train_fwd_kernel(const float* __restrict__ kpts,
                                                                 const float* __restrict__ stats,
                                                                 const float* __restrict__ desc,
                                                                 const float* __restrict__ pack,
                                                                 float* __restrict__ out, int n, int rows) {
  extern __shared__ __align__(16) float smem[];
  const int r0 = blockIdx.x * kG, count = min(kG, rows - r0);
  tile_forward(smem, kpts, stats, pack, n, r0, count);
  float* o = smem + sBig;
  rows_gemm<C3, C4, kLdOut>(smem + sZ3, pack + kW4t, pack + kB4, o);
  __syncthreads();
  // + descriptors [B][256][N], read coalesced along n
  {
    const int p = threadIdx.x % kG;
    if (p < count) {
      const int row = r0 + p, b = row / n, m = row - b * n;
      const float* dp = desc + (long long)b * C4 * n + m;
      for (int c = threadIdx.x / kG; c < C4; c += kThreads / kG) o[p * kLdOut + c] += dp[(long long)c * n];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < count * C4; i += kThreads) {
    const int p = i / C4, c = i - p * C4;
    out[(long long)(r0 + p) * C4 + c] = o[p * kLdOut + c];
  }
}

__global__ void __launch_bounds__(kThreads) kpt_train_bwd_kernel(const float* __restrict__ kpts,
                                                                 const float* __restrict__ stats,
                                                                 const float* __restrict__ dout,
                                                                 const float* __restrict__ pack, int n,
                                                                 int row0, int row_end, float* __restrict__ part) {
  extern __shared__ __align__(16) float smem[];
  const int r0 = row0 + blockIdx.x * kG, count = min(kG, row_end - r0);
  tile_forward(smem, kpts, stats, pack, n, r0, count);
  float* g = smem + sBig;
  float* d3 = smem + sD3;
  float* d2 = smem + sD2;
  float* d1 = d3;                         // d3 is dead once dz2 and dW3 are done
  for (int i = threadIdx.x; i < kG * C4; i += kThreads) {
    const int p = i / C4;
    g[i] = p < count ? dout[(long long)r0 * C4 + i] : 0.f;
  }
  __syncthreads();
  float* pp = part + (size_t)blockIdx.x * kParams;
  tile_wgrad<C4, C3>(g, smem + sZ3, pp + gW4);
  rows_gemm<C4, C3>(g, pack + kW4, nullptr, d3);
  __syncthreads();
  inorm_relu_bwd<C3>(smem + sY3, d3, smem + sR, 2);
  __syncthreads();
  tile_wgrad<C3, C2>(d3, smem + sZ2, pp + gW3);
  rows_gemm<C3, C2>(d3, pack + kW3, nullptr, d2);
  __syncthreads();
  inorm_relu_bwd<C2>(smem + sY2, d2, smem + sR, 1);
  __syncthreads();
  tile_wgrad<C2, C1>(d2, smem + sZ1, pp + gW2);
  rows_gemm<C2, C1>(d2, pack + kW2, nullptr, d1);
  __syncthreads();
  inorm_relu_bwd<C1>(smem + sY1, d1, smem + sR, 0);
  __syncthreads();
  tile_wgrad<C1, C0>(d1, smem + sX0, pp + gW1);
}

__global__ void kpt_reduce_kernel(const float* __restrict__ part, int parts, int accumulate,
                                  float* __restrict__ dparams) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kParams) return;
  float s = accumulate ? dparams[i] : 0.f;
  for (int q = 0; q < parts; ++q) s += part[(size_t)q * kParams + i];
  dparams[i] = s;
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" {

int opp_kpt_train_group(void) { return kG; }

int opp_kpt_train_params(void) { return kParams; }

int opp_kpt_train_pack_size(void) { return kPack; }

int opp_kpt_train_fwd(const float* kpts, const float* stats, const float* desc, const float* pack, float* out,
                      int batch, int n, opp_stream_t stream) {
  OPP_REQUIRE(kpts && stats && desc && pack && out, "opp_kpt_train_fwd: null pointer");
  OPP_REQUIRE(batch > 0 && n > 0 && (long long)batch * n * C4 < (1LL << 31),
              "opp_kpt_train_fwd: batch %d x n %d", batch, n);
  const int rows = batch * n;
  OPP_CHECK_CUDA(cudaFuncSetAttribute(kpt_train_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kFwdSmem));
  kpt_train_fwd_kernel<<<(rows + kG - 1) / kG, kThreads, kFwdSmem, (cudaStream_t)stream>>>(kpts, stats, desc, pack,
                                                                                          out, n, rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_kpt_train_bwd(const float* kpts, const float* stats, const float* dout, const float* pack, int batch, int n,
                      int row0, int nrows, float* part, float* dparams, int accumulate, opp_stream_t stream) {
  OPP_REQUIRE(kpts && stats && dout && pack && part && dparams, "opp_kpt_train_bwd: null pointer");
  OPP_REQUIRE(batch > 0 && n > 0 && (long long)batch * n * C4 < (1LL << 31),
              "opp_kpt_train_bwd: batch %d x n %d", batch, n);
  const int rows = batch * n;
  OPP_REQUIRE(row0 >= 0 && nrows > 0 && row0 % kG == 0 && row0 + nrows <= rows,
              "opp_kpt_train_bwd: row slice [%d, %d) of %d", row0, row0 + nrows, rows);
  const int groups = (nrows + kG - 1) / kG;
  const cudaStream_t st = (cudaStream_t)stream;
  OPP_CHECK_CUDA(cudaFuncSetAttribute(kpt_train_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kBwdSmem));
  kpt_train_bwd_kernel<<<groups, kThreads, kBwdSmem, st>>>(kpts, stats, dout, pack, n, row0, row0 + nrows, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  kpt_reduce_kernel<<<(kParams + 255) / 256, 256, 0, st>>>(part, groups, accumulate, dparams);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
