// opp_train_rows.cuh — row kernels shared by the training stages (opp_train_fine.cu at 128 channels,
// opp_train_coarse_tf.cu at 256): LayerNorm forward and backward over C = 128·V channels, and the
// in-order sum of per-group partials.  One warp per row; lane l owns channels j·128 + 4l .. 4l + 3 for
// j < V, so every load is a coalesced float4.  Every reduction runs in a fixed order (no atomics).
#pragma once

#include <cmath>

namespace opp {
namespace {

constexpr int kGroupRows = 256;  // rows per partial of the weight / LayerNorm parameter gradients
constexpr float kLnEps = 1e-5f;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// out[e] (+)= sum_{g < groups} part[g][e], g ascending.
__global__ void __launch_bounds__(256) fine_reduce_kernel(const float* __restrict__ part, int groups, int size,
                                                          int accumulate, float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= size) return;
  float s = 0.f;
  for (int gi = 0; gi < groups; ++gi) s += part[(size_t)gi * size + e];
  out[e] = accumulate ? out[e] + s : s;
}

// y = (x - mean) · rstd · gamma + beta (+ resid); stats[r] = (mean, rstd).  8 rows per CTA.
template <int kC>
__global__ void __launch_bounds__(256) train_ln_fwd_kernel(const float* __restrict__ x, int ldx,
                                                           const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, const float* resid,
                                                           int ldr, float* y, int ldy, float2* __restrict__ stats,
                                                           int rows) {
  constexpr int kV = kC / 128;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float4 v[kV];
#pragma unroll
  for (int j = 0; j < kV; ++j) v[j] = *reinterpret_cast<const float4*>(x + (size_t)r * ldx + j * 128 + lane * 4);
  float s = v[0].x + v[0].y + v[0].z + v[0].w;
#pragma unroll
  for (int j = 1; j < kV; ++j) s += v[j].x + v[j].y + v[j].z + v[j].w;
  const float mean = warp_sum(s) * (1.f / kC);
  float d[kV][4];
#pragma unroll
  for (int j = 0; j < kV; ++j) d[j][0] = v[j].x - mean, d[j][1] = v[j].y - mean, d[j][2] = v[j].z - mean,
                               d[j][3] = v[j].w - mean;
  float q = d[0][0] * d[0][0] + d[0][1] * d[0][1] + d[0][2] * d[0][2] + d[0][3] * d[0][3];
#pragma unroll
  for (int j = 1; j < kV; ++j) q += d[j][0] * d[j][0] + d[j][1] * d[j][1] + d[j][2] * d[j][2] + d[j][3] * d[j][3];
  const float var = warp_sum(q) * (1.f / kC);
  const float rstd = rsqrtf(var + kLnEps);
#pragma unroll
  for (int j = 0; j < kV; ++j) {
    const float4 gm = *reinterpret_cast<const float4*>(gamma + j * 128 + lane * 4);
    const float4 bt = *reinterpret_cast<const float4*>(beta + j * 128 + lane * 4);
    float4 o = make_float4(d[j][0] * rstd * gm.x + bt.x, d[j][1] * rstd * gm.y + bt.y, d[j][2] * rstd * gm.z + bt.z,
                           d[j][3] * rstd * gm.w + bt.w);
    if (resid) {
      const float4 p = *reinterpret_cast<const float4*>(resid + (size_t)r * ldr + j * 128 + lane * 4);
      o.x += p.x, o.y += p.y, o.z += p.z, o.w += p.w;
    }
    *reinterpret_cast<float4*>(y + (size_t)r * ldy + j * 128 + lane * 4) = o;
  }
  if (lane == 0) stats[r] = make_float2(mean, rstd);
}

// dx = rstd (dxh - mean(dxh) - xh mean(dxh xh)), dxh = dy gamma, xh = (x - mean) rstd; the partial
// part[group][0 / 1][c] = sum over the group's rows of dy xh / dy (dgamma / dbeta).  8 warps per CTA,
// kGroupRows rows per CTA; the warps' sums are combined in warp order.
template <int kC>
__global__ void __launch_bounds__(256) train_ln_bwd_kernel(const float* __restrict__ x, int ldx,
                                                           const float* __restrict__ gamma,
                                                           const float2* __restrict__ stats,
                                                           const float* __restrict__ dy, int lddy,
                                                           float* __restrict__ dx, int lddx,
                                                           float* __restrict__ part, int rows) {
  constexpr int kV = kC / 128;
  constexpr int kLog = kC == 128 ? 7 : 8;
  static_assert(kC == 128 || kC == 256, "LayerNorm rows of 128 or 256 channels");
  __shared__ float red[8][2][kC];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int rb = blockIdx.x * kGroupRows, re = min(rows, rb + kGroupRows);
  float4 gm[kV];
#pragma unroll
  for (int j = 0; j < kV; ++j) gm[j] = *reinterpret_cast<const float4*>(gamma + j * 128 + lane * 4);
  float sg[kV][4] = {}, sb[kV][4] = {};
  for (int r = rb + wid; r < re; r += 8) {
    const float2 st = stats[r];
    float xh[kV][4], gg[kV][4], dxh[kV][4];
#pragma unroll
    for (int j = 0; j < kV; ++j) {
      const float4 v = *reinterpret_cast<const float4*>(x + (size_t)r * ldx + j * 128 + lane * 4);
      const float4 g = *reinterpret_cast<const float4*>(dy + (size_t)r * lddy + j * 128 + lane * 4);
      xh[j][0] = (v.x - st.x) * st.y, xh[j][1] = (v.y - st.x) * st.y, xh[j][2] = (v.z - st.x) * st.y,
      xh[j][3] = (v.w - st.x) * st.y;
      gg[j][0] = g.x, gg[j][1] = g.y, gg[j][2] = g.z, gg[j][3] = g.w;
      dxh[j][0] = g.x * gm[j].x, dxh[j][1] = g.y * gm[j].y, dxh[j][2] = g.z * gm[j].z, dxh[j][3] = g.w * gm[j].w;
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < kV; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        s1 += dxh[j][i], s2 += dxh[j][i] * xh[j][i];
        sg[j][i] = fmaf(gg[j][i], xh[j][i], sg[j][i]);
        sb[j][i] += gg[j][i];
      }
    const float m1 = warp_sum(s1) * (1.f / kC), m2 = warp_sum(s2) * (1.f / kC);
#pragma unroll
    for (int j = 0; j < kV; ++j) {
      float4 o;
      o.x = st.y * (dxh[j][0] - m1 - xh[j][0] * m2);
      o.y = st.y * (dxh[j][1] - m1 - xh[j][1] * m2);
      o.z = st.y * (dxh[j][2] - m1 - xh[j][2] * m2);
      o.w = st.y * (dxh[j][3] - m1 - xh[j][3] * m2);
      *reinterpret_cast<float4*>(dx + (size_t)r * lddx + j * 128 + lane * 4) = o;
    }
  }
#pragma unroll
  for (int j = 0; j < kV; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) red[wid][0][j * 128 + lane * 4 + i] = sg[j][i], red[wid][1][j * 128 + lane * 4 + i] = sb[j][i];
  __syncthreads();
#pragma unroll
  for (int p = 0; p < kV; ++p) {
    const int e = threadIdx.x + 256 * p;   // 0 .. 2·kC - 1 = (which, c)
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][e >> kLog][e & (kC - 1)];
    part[(size_t)blockIdx.x * 2 * kC + e] = s;
  }
}

}  // namespace
}  // namespace opp
