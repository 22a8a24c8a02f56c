// opp_train_fine.cu — the fine level of training on the device: window gather, the two fine LoFTR
// layers (self, cross; d = 128, 8 heads, linear attention) and the heatmap expectation, forward and
// backward (DESIGN §7 f4).
//
// Token rows: match m owns 26 consecutive fp32 rows, m·26 + t; t = ky·5 + kx (0..24) are the 5 x 5
// window of its query cell (F.unfold's order, padding 2, zeros outside the map), t = 25 is its 3D
// descriptor.  One weight set serves both sequences of a layer, so every projection, LayerNorm and
// MLP is one GEMM over all 26·M rows and its weight gradient is the sum over the 2D and the 3D rows.
// Only the attention core tells the two sequences apart (fine_attn_*: side 0 = the 25 window
// queries, side 1 = the 3D query; "self" reads keys from the query's own sequence, "cross" from the
// other one).
//
// Every reduction runs in a fixed order and no kernel uses floating-point atomics, so two calls give
// the same bits:
//   - weight gradients (fine_wgrad): rows are cut into groups of kGroupRows; each CTA sums one group
//     for one 64 x 64 tile of dW into a partial, and fine_reduce adds the partials in group order;
//   - LayerNorm dgamma / dbeta: the same, one partial per group of kGroupRows rows;
//   - d feat_f (fine_gather_bwd): one thread per fine pixel and channel sums the window gradients of
//     the matches whose window covers it — cells in raster order, the matches of a cell in ascending
//     order (the column view of opp_gt_index) — instead of scattering from the matches.
#include <cmath>
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"
#include "opp_train_rows.cuh"

namespace opp {
namespace {

constexpr int kTok = 26;        // 25 window tokens + the 3D token
constexpr int kWin = 25;
constexpr int kD = 128;         // d_model
constexpr int kHeadDim = 16;    // d_model / nhead

// ------------------------------------------------------------------------------------------------
// Gather: x[m·26 + t][0..127] (row stride ldx) from feat [B][128][Hf][Wf] and desc3d [B][128][N].
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) fine_gather_fwd_kernel(const float* __restrict__ feat,
                                                              const float* __restrict__ desc3d,
                                                              const long long* __restrict__ b_ids,
                                                              const long long* __restrict__ i_ids,
                                                              const long long* __restrict__ j_ids, int hf, int wf,
                                                              int wc, int n3d, int stride, float* __restrict__ x,
                                                              int ldx) {
  const int m = blockIdx.x, c = threadIdx.x;
  const long long b = b_ids[m], j = j_ids[m];
  const int y0 = (int)(j / wc) * stride - 2, x0 = (int)(j % wc) * stride - 2;
  const float* f = feat + ((size_t)b * kD + c) * hf * wf;
  float* out = x + (size_t)m * kTok * ldx + c;
#pragma unroll
  for (int ky = 0; ky < 5; ++ky) {
    const int y = y0 + ky;
#pragma unroll
    for (int kx = 0; kx < 5; ++kx) {
      const int xx = x0 + kx;
      const bool in = y >= 0 && y < hf && xx >= 0 && xx < wf;
      out[(size_t)(ky * 5 + kx) * ldx] = in ? f[(size_t)y * wf + xx] : 0.f;
    }
  }
  out[(size_t)kWin * ldx] = desc3d[((size_t)b * kD + c) * n3d + i_ids[m]];
}

// dfeat[b][c][y][x] = sum over the cells (cy, cx) whose window holds (y, x), in raster order, and over
// the matches of that cell (col_ptr / col_rows, ascending) of dx[m·26 + (y - cy·s + 2)·5 + x - cx·s + 2][c].
__global__ void __launch_bounds__(256) fine_gather_bwd_kernel(const float* __restrict__ dx, int ldx,
                                                              const int* __restrict__ col_ptr,
                                                              const int* __restrict__ col_rows, int batches, int hf,
                                                              int wf, int hc, int wc, int stride,
                                                              float* __restrict__ dfeat) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)batches * kD * hf * wf;
  if (idx >= total) return;
  const int xx = (int)(idx % wf);
  const int y = (int)((idx / wf) % hf);
  const int c = (int)((idx / ((long long)wf * hf)) % kD);
  const int b = (int)(idx / ((long long)wf * hf * kD));
  const int cy0 = y - 2 <= 0 ? 0 : (y - 2 + stride - 1) / stride, cy1 = min(hc - 1, (y + 2) / stride);
  const int cx0 = xx - 2 <= 0 ? 0 : (xx - 2 + stride - 1) / stride, cx1 = min(wc - 1, (xx + 2) / stride);
  float acc = 0.f;
  for (int cy = cy0; cy <= cy1; ++cy) {
    for (int cx = cx0; cx <= cx1; ++cx) {
      const int cell = (b * hc + cy) * wc + cx;
      const int t = (y - cy * stride + 2) * 5 + (xx - cx * stride + 2);
      for (int p = col_ptr[cell], e = col_ptr[cell + 1]; p < e; ++p)
        acc += dx[((size_t)col_rows[p] * kTok + t) * ldx + c];
    }
  }
  dfeat[idx] = acc;
}

// ------------------------------------------------------------------------------------------------
// Token-row GEMM, fp32: C[r][n] = epi(sum_k A[r][k] · B(k, n)), B(k, n) = W[n][k] (kTransW, the
// forward y = x W^T) or W[k][n] (the data gradient dx = dy W).  64 x 64 tile, K step 16, 256 threads,
// 4 x 4 outputs per thread.  n % 64 == 0, k % 16 == 0.
// ------------------------------------------------------------------------------------------------
enum FineEpi { kEpiStore = 0, kEpiRelu = 1, kEpiMask = 2, kEpiAdd = 3 };

template <bool kTransW, int kEpi>
__global__ void __launch_bounds__(256) fine_linear_kernel(const float* __restrict__ a, int lda,
                                                          const float* __restrict__ w, int rows, int n, int k,
                                                          float* c, int ldc, const float* aux, int ldaux,
                                                          const float* aux2, int ldaux2) {
  __shared__ float as[16][64 + 4];
  __shared__ float bs[16][64 + 4];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int r0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < k; k0 += 16) {
    {
      const int r = t >> 2, kq = (t & 3) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < rows) v = *reinterpret_cast<const float4*>(a + (size_t)(r0 + r) * lda + k0 + kq);
      as[kq][r] = v.x, as[kq + 1][r] = v.y, as[kq + 2][r] = v.z, as[kq + 3][r] = v.w;
      if (kTransW) {
        const float4 u = *reinterpret_cast<const float4*>(w + (size_t)(n0 + r) * k + k0 + kq);
        bs[kq][r] = u.x, bs[kq + 1][r] = u.y, bs[kq + 2][r] = u.z, bs[kq + 3][r] = u.w;
      } else {
        const int kk = t >> 4, nq = (t & 15) * 4;
        const float4 u = *reinterpret_cast<const float4*>(w + (size_t)(k0 + kk) * n + n0 + nq);
        bs[kk][nq] = u.x, bs[kk][nq + 1] = u.y, bs[kk][nq + 2] = u.z, bs[kk][nq + 3] = u.w;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = as[kk][ty + 16 * i], bv[i] = bs[kk][tx + 16 * i];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 16 * i;
    if (r >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = n0 + tx + 16 * j;
      float v = acc[i][j];
      if (kEpi == kEpiRelu) v = fmaxf(v, 0.f);
      if (kEpi == kEpiMask) v = aux[(size_t)r * ldaux + col] > 0.f ? v : 0.f;
      if (kEpi == kEpiAdd) {
        if (aux) v += aux[(size_t)r * ldaux + col];
        if (aux2) v += aux2[(size_t)r * ldaux2 + col];
      }
      c[(size_t)r * ldc + col] = v;
    }
  }
}

// Weight gradient partial: part[g][n][k] = sum over rows r of group g of G[r][n] · A[r][k].
__global__ void __launch_bounds__(256) fine_wgrad_kernel(const float* __restrict__ g, int ldg,
                                                         const float* __restrict__ a, int lda, int rows, int n,
                                                         int k, float* __restrict__ part) {
  __shared__ float gs[16][64 + 4];
  __shared__ float as[16][64 + 4];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int k0 = blockIdx.x * 64, n0 = blockIdx.y * 64, grp = blockIdx.z;
  const int rb = grp * kGroupRows, re = min(rows, rb + kGroupRows);
  float acc[4][4] = {};
  const int lr = t >> 4, lq = (t & 15) * 4;
  for (int r0 = rb; r0 < re; r0 += 16) {
    const int r = r0 + lr;
    float4 gv = make_float4(0.f, 0.f, 0.f, 0.f), av = gv;
    if (r < re) {
      gv = *reinterpret_cast<const float4*>(g + (size_t)r * ldg + n0 + lq);
      av = *reinterpret_cast<const float4*>(a + (size_t)r * lda + k0 + lq);
    }
    gs[lr][lq] = gv.x, gs[lr][lq + 1] = gv.y, gs[lr][lq + 2] = gv.z, gs[lr][lq + 3] = gv.w;
    as[lr][lq] = av.x, as[lr][lq + 1] = av.y, as[lr][lq + 2] = av.z, as[lr][lq + 3] = av.w;
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
      float gr[4], ar[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) gr[i] = gs[rr][ty + 16 * i], ar[i] = as[rr][tx + 16 * i];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gr[i], ar[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = part + (size_t)grp * n * k;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[(size_t)(n0 + ty + 16 * i) * k + k0 + tx + 16 * j] = acc[i][j];
}

// ------------------------------------------------------------------------------------------------
// Linear attention (linear_attention.py:29-61 as in train_path._linear_attention): per match and
// side, queries Q (25 window rows or the 3D row), keys / values of the source sequence (25 rows
// or 1), n = its length.  Qf = elu(q) + 1, Kf = elu(k) + 1, Vs = v / n, KV = Kf^T Vs, ksum = sum Kf,
// Z_l = 1 / (Qf_l . ksum + eps), out_l = (Qf_l KV) Z_l n — per head of 16 channels.
// qkv rows: [q | k | v] (384 floats); thread c = head·16 + lane16 owns channel c.
// ------------------------------------------------------------------------------------------------
struct AttnSets {
  int q0, nq, s0, ns;
};

__device__ __forceinline__ AttnSets attn_sets(int side, int cross) {
  // side 0: the 25 window queries; side 1: the 3D query.  self: keys of the own sequence.
  const int q0 = side ? kWin : 0, nq = side ? 1 : kWin;
  const bool src_win = cross ? side == 1 : side == 0;
  return AttnSets{q0, nq, src_win ? 0 : kWin, src_win ? kWin : 1};
}

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v + 1.f : expf(v); }

__global__ void __launch_bounds__(128) fine_attn_fwd_kernel(const float* __restrict__ qkv, float* __restrict__ out,
                                                            int cross, float eps) {
  __shared__ float qf[kWin][kD], kf[kWin][kD], vs[kWin][kD], ks[kD];
  const int m = blockIdx.x, c = threadIdx.x, h0 = c & ~(kHeadDim - 1);
  const AttnSets S = attn_sets(blockIdx.y, cross);
  const float* base = qkv + (size_t)m * kTok * 3 * kD;
  const float inv_n = 1.f / (float)S.ns, n = (float)S.ns;
  for (int l = 0; l < S.nq; ++l) qf[l][c] = elu1(base[(size_t)(S.q0 + l) * 3 * kD + c]);
  float ksum = 0.f;
  for (int s = 0; s < S.ns; ++s) {
    const float kv = elu1(base[(size_t)(S.s0 + s) * 3 * kD + kD + c]);
    kf[s][c] = kv;
    vs[s][c] = base[(size_t)(S.s0 + s) * 3 * kD + 2 * kD + c] * inv_n;
    ksum += kv;
  }
  ks[c] = ksum;
  __syncthreads();
  float kvcol[kHeadDim];   // KV[d][e] of this thread's e = c
#pragma unroll
  for (int d = 0; d < kHeadDim; ++d) {
    float acc = 0.f;
    for (int s = 0; s < S.ns; ++s) acc = fmaf(kf[s][h0 + d], vs[s][c], acc);
    kvcol[d] = acc;
  }
  for (int l = 0; l < S.nq; ++l) {
    float den = 0.f, num = 0.f;
#pragma unroll
    for (int d = 0; d < kHeadDim; ++d) {
      const float q = qf[l][h0 + d];
      den = fmaf(q, ks[h0 + d], den);
      num = fmaf(q, kvcol[d], num);
    }
    const float z = 1.f / (den + eps);
    out[((size_t)m * kTok + S.q0 + l) * kD + c] = num * z * n;
  }
}

// Backward of fine_attn_fwd: dqkv rows [dq | dk | dv].  With g = d out, A_l = Qf_l KV:
//   dA_l = n Z_l g_l, dden_l = -Z_l^2 n (g_l . A_l), dQf_l = KV dA_l + dden_l ksum,
//   dKV = sum_l Qf_l^T dA_l, dksum = sum_l dden_l Qf_l, dKf_s = dKV Vs_s + dksum, dv_s = (Kf_s dKV) / n,
//   elu'(x) = 1 for x > 0, else exp(x) = Qf (Kf).
// Dynamic shared memory: qf, kf, vs, ga [25][128] (ga holds g, then dA), ks [128], dden [25][8].
__global__ void __launch_bounds__(128) fine_attn_bwd_kernel(const float* __restrict__ qkv,
                                                            const float* __restrict__ dout,
                                                            float* __restrict__ dqkv, int cross, float eps) {
  extern __shared__ float smem[];
  float(*qf)[kD] = reinterpret_cast<float(*)[kD]>(smem);
  float(*kf)[kD] = qf + kWin;
  float(*vs)[kD] = kf + kWin;
  float(*ga)[kD] = vs + kWin;
  float* ks = smem + 4 * kWin * kD;
  float* dden = ks + kD;   // [25][8]
  const int m = blockIdx.x, c = threadIdx.x, h0 = c & ~(kHeadDim - 1), head = c / kHeadDim;
  const AttnSets S = attn_sets(blockIdx.y, cross);
  const float* base = qkv + (size_t)m * kTok * 3 * kD;
  float* dbase = dqkv + (size_t)m * kTok * 3 * kD;
  const float inv_n = 1.f / (float)S.ns, n = (float)S.ns;
  for (int l = 0; l < S.nq; ++l) {
    qf[l][c] = elu1(base[(size_t)(S.q0 + l) * 3 * kD + c]);
    ga[l][c] = dout[((size_t)m * kTok + S.q0 + l) * kD + c];
  }
  float ksum = 0.f;
  for (int s = 0; s < S.ns; ++s) {
    const float kv = elu1(base[(size_t)(S.s0 + s) * 3 * kD + kD + c]);
    kf[s][c] = kv;
    vs[s][c] = base[(size_t)(S.s0 + s) * 3 * kD + 2 * kD + c] * inv_n;
    ksum += kv;
  }
  ks[c] = ksum;
  __syncthreads();
  {
    float kvcol[kHeadDim];   // thread = column e = c
#pragma unroll
    for (int d = 0; d < kHeadDim; ++d) {
      float acc = 0.f;
      for (int s = 0; s < S.ns; ++s) acc = fmaf(kf[s][h0 + d], vs[s][c], acc);
      kvcol[d] = acc;
    }
    for (int l = 0; l < S.nq; ++l) {
      float den = 0.f, num = 0.f;
#pragma unroll
      for (int d = 0; d < kHeadDim; ++d) {
        const float q = qf[l][h0 + d];
        den = fmaf(q, ks[h0 + d], den);
        num = fmaf(q, kvcol[d], num);
      }
      const float z = 1.f / (den + eps);
      const float g = ga[l][c];
      float ga_sum = g * num;
#pragma unroll
      for (int o = kHeadDim / 2; o > 0; o >>= 1) ga_sum += __shfl_xor_sync(0xffffffffu, ga_sum, o);
      ga[l][c] = n * z * g;
      if ((c & (kHeadDim - 1)) == 0) dden[l * 8 + head] = -z * z * n * ga_sum;
    }
  }
  __syncthreads();
  float dks = 0.f;
  float dkvrow[kHeadDim];   // thread = row d = c: dKV[d][e]
  {
    float kvrow[kHeadDim];
#pragma unroll
    for (int e = 0; e < kHeadDim; ++e) {
      float acc = 0.f;
      for (int s = 0; s < S.ns; ++s) acc = fmaf(kf[s][c], vs[s][h0 + e], acc);
      kvrow[e] = acc;
      dkvrow[e] = 0.f;
    }
    const float kc = ks[c];
    for (int l = 0; l < S.nq; ++l) {
      const float q = qf[l][c], dd = dden[l * 8 + head];
      float dq = dd * kc;
#pragma unroll
      for (int e = 0; e < kHeadDim; ++e) {
        const float da = ga[l][h0 + e];
        dq = fmaf(da, kvrow[e], dq);
        dkvrow[e] = fmaf(q, da, dkvrow[e]);
      }
      dks = fmaf(dd, q, dks);
      dbase[(size_t)(S.q0 + l) * 3 * kD + c] = q > 1.f ? dq : dq * q;
    }
  }
  for (int s = 0; s < S.ns; ++s) {
    float dk = dks;
#pragma unroll
    for (int e = 0; e < kHeadDim; ++e) dk = fmaf(dkvrow[e], vs[s][h0 + e], dk);
    const float k = kf[s][c];
    dbase[(size_t)(S.s0 + s) * 3 * kD + kD + c] = k > 1.f ? dk : dk * k;
  }
  __syncthreads();   // qf is free: it holds dKV [128][16] from here on
  float* dkv = smem;
#pragma unroll
  for (int e = 0; e < kHeadDim; ++e) dkv[c * kHeadDim + e] = dkvrow[e];
  __syncthreads();
  for (int s = 0; s < S.ns; ++s) {
    float dv = 0.f;
#pragma unroll
    for (int d = 0; d < kHeadDim; ++d) dv = fmaf(kf[s][h0 + d], dkv[(h0 + d) * kHeadDim + (c & (kHeadDim - 1))], dv);
    dbase[(size_t)(S.s0 + s) * 3 * kD + 2 * kD + c] = dv * inv_n;
  }
}

constexpr int kAttnBwdSmem = (4 * kWin * kD + kD + kWin * 8) * (int)sizeof(float);

// ------------------------------------------------------------------------------------------------
// Heatmap expectation (fine_matching.py:28-110, s2d): sim_r = f3d . f2d_r / sqrt(128), heat =
// softmax_r, (x, y) = heat . grid, var = heat . grid^2 - (x, y)^2, std = sqrt(max(var_x, 1e-10)) +
// sqrt(max(var_y, 1e-10)).  One warp per match, 4 channels per lane; grid r -> (lin[r % 5], lin[r / 5]),
// lin = linspace(-1, 1, 5).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float grid_lin(int i) { return -1.f + 0.5f * (float)i; }

struct Heat {
  float p[kWin];
  float cx, cy, vx, vy;
};

__device__ __forceinline__ void heat_of(const float* __restrict__ x, int m, int lane, float4& f0, Heat& h) {
  const float* rows = x + (size_t)m * kTok * kD;
  f0 = *reinterpret_cast<const float4*>(rows + (size_t)kWin * kD + lane * 4);
  const float inv = 1.f / sqrtf((float)kD);
  float mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < kWin; ++r) {
    const float4 v = *reinterpret_cast<const float4*>(rows + (size_t)r * kD + lane * 4);
    h.p[r] = warp_sum(f0.x * v.x + f0.y * v.y + f0.z * v.z + f0.w * v.w) * inv;
    mx = fmaxf(mx, h.p[r]);
  }
  float sum = 0.f;
#pragma unroll
  for (int r = 0; r < kWin; ++r) h.p[r] = expf(h.p[r] - mx), sum += h.p[r];
  const float is = 1.f / sum;
  float cx = 0.f, cy = 0.f, sx = 0.f, sy = 0.f;
#pragma unroll
  for (int r = 0; r < kWin; ++r) {
    h.p[r] *= is;
    const float gx = grid_lin(r % 5), gy = grid_lin(r / 5);
    cx = fmaf(h.p[r], gx, cx), cy = fmaf(h.p[r], gy, cy);
    sx = fmaf(h.p[r], gx * gx, sx), sy = fmaf(h.p[r], gy * gy, sy);
  }
  h.cx = cx, h.cy = cy, h.vx = sx - cx * cx, h.vy = sy - cy * cy;
}

__global__ void __launch_bounds__(128) fine_match_fwd_kernel(const float* __restrict__ x, int m_count,
                                                             float* __restrict__ expec) {
  const int lane = threadIdx.x & 31, m = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (m >= m_count) return;
  float4 f0;
  Heat h;
  heat_of(x, m, lane, f0, h);
  if (lane == 0) {
    expec[3 * m] = h.cx;
    expec[3 * m + 1] = h.cy;
    expec[3 * m + 2] = sqrtf(fmaxf(h.vx, 1e-10f)) + sqrtf(fmaxf(h.vy, 1e-10f));
  }
}

// d expec -> d x (rows 0..24 and 25 of each match, overwritten).  clamp(var, min=1e-10) passes the
// gradient where var >= 1e-10 and 0 where the clamp is active (torch.clamp's backward).
__global__ void __launch_bounds__(128) fine_match_bwd_kernel(const float* __restrict__ x,
                                                             const float* __restrict__ dexpec, int m_count,
                                                             float* __restrict__ dx) {
  const int lane = threadIdx.x & 31, m = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (m >= m_count) return;
  float4 f0;
  Heat h;
  heat_of(x, m, lane, f0, h);
  const float gx = dexpec[3 * m], gy = dexpec[3 * m + 1], gs = dexpec[3 * m + 2];
  const float dvx = h.vx >= 1e-10f ? gs / (2.f * sqrtf(h.vx)) : 0.f;
  const float dvy = h.vy >= 1e-10f ? gs / (2.f * sqrtf(h.vy)) : 0.f;
  const float dcx = gx - 2.f * h.cx * dvx, dcy = gy - 2.f * h.cy * dvy;
  float dh[kWin], dot = 0.f;
#pragma unroll
  for (int r = 0; r < kWin; ++r) {
    const float px = grid_lin(r % 5), py = grid_lin(r / 5);
    dh[r] = dcx * px + dcy * py + dvx * px * px + dvy * py * py;
    dot = fmaf(h.p[r], dh[r], dot);
  }
  const float inv = 1.f / sqrtf((float)kD);
  const float* rows = x + (size_t)m * kTok * kD;
  float* drows = dx + (size_t)m * kTok * kD;
  float4 df0 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int r = 0; r < kWin; ++r) {
    const float ds = h.p[r] * (dh[r] - dot) * inv;
    const float4 v = *reinterpret_cast<const float4*>(rows + (size_t)r * kD + lane * 4);
    df0.x = fmaf(ds, v.x, df0.x), df0.y = fmaf(ds, v.y, df0.y), df0.z = fmaf(ds, v.z, df0.z),
    df0.w = fmaf(ds, v.w, df0.w);
    *reinterpret_cast<float4*>(drows + (size_t)r * kD + lane * 4) =
        make_float4(ds * f0.x, ds * f0.y, ds * f0.z, ds * f0.w);
  }
  *reinterpret_cast<float4*>(drows + (size_t)kWin * kD + lane * 4) = df0;
}

template <bool kTransW, int kEpi>
cudaError_t launch_linear(const float* a, int lda, const float* w, int rows, int n, int k, float* c, int ldc,
                          const float* aux, int ldaux, const float* aux2, int ldaux2, cudaStream_t st) {
  fine_linear_kernel<kTransW, kEpi><<<dim3((rows + 63) / 64, n / 64), 256, 0, st>>>(a, lda, w, rows, n, k, c, ldc,
                                                                                    aux, ldaux, aux2, ldaux2);
  return cudaGetLastError();
}

bool aligned4(const void* p, int ld) { return ((uintptr_t)p & 15) == 0 && ld % 4 == 0; }

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" {

int opp_fine_train_groups(int rows) { return (rows + kGroupRows - 1) / kGroupRows; }

int opp_fine_train_gather(const float* feat, const float* desc3d, const long long* b_ids, const long long* i_ids,
                          const long long* j_ids, int m, int hf, int wf, int hc, int wc, int n3d, int stride,
                          float* x, int ldx, opp_stream_t stream) {
  OPP_REQUIRE(m >= 0 && hf > 0 && wf > 0 && hc > 0 && wc > 0 && n3d > 0 && stride > 0 && ldx >= kD,
              "opp_fine_train_gather: bad geometry");
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(feat && desc3d && b_ids && i_ids && j_ids && x, "opp_fine_train_gather: null pointer");
  fine_gather_fwd_kernel<<<m, 128, 0, (cudaStream_t)stream>>>(feat, desc3d, b_ids, i_ids, j_ids, hf, wf, wc, n3d,
                                                              stride, x, ldx);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_gather_bwd(const float* dx, int ldx, const int* col_ptr, const int* col_rows, int batches,
                              int hf, int wf, int hc, int wc, int stride, float* dfeat, opp_stream_t stream) {
  OPP_REQUIRE(dx && col_ptr && dfeat && batches > 0 && hf > 0 && wf > 0 && hc > 0 && wc > 0 && stride > 0 &&
                  ldx >= kD,
              "opp_fine_train_gather_bwd: bad arguments");
  const long long total = (long long)batches * kD * hf * wf;
  fine_gather_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      dx, ldx, col_ptr, col_rows, batches, hf, wf, hc, wc, stride, dfeat);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_linear(const float* a, int lda, const float* w, int trans_w, int rows, int n, int k, float* c,
                          int ldc, int epi, const float* aux, int ldaux, const float* aux2, int ldaux2,
                          opp_stream_t stream) {
  OPP_REQUIRE(rows >= 0 && n > 0 && k > 0 && n % 64 == 0 && k % 16 == 0, "opp_fine_train_linear: shape %d x %d x %d",
              rows, n, k);
  if (rows == 0) return OPP_OK;
  OPP_REQUIRE(a && w && c && aligned4(a, lda) && aligned4(w, 4) && ldc >= n && lda >= k,
              "opp_fine_train_linear: null or misaligned operand");
  OPP_REQUIRE(epi != kEpiMask || aux, "opp_fine_train_linear: the mask epilogue needs aux");
  const cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaErrorInvalidValue;
  if (trans_w) {
    if (epi == kEpiStore) e = launch_linear<true, kEpiStore>(a, lda, w, rows, n, k, c, ldc, aux, ldaux, aux2, ldaux2, st);
    if (epi == kEpiRelu) e = launch_linear<true, kEpiRelu>(a, lda, w, rows, n, k, c, ldc, aux, ldaux, aux2, ldaux2, st);
  } else {
    if (epi == kEpiMask) e = launch_linear<false, kEpiMask>(a, lda, w, rows, n, k, c, ldc, aux, ldaux, aux2, ldaux2, st);
    if (epi == kEpiStore) e = launch_linear<false, kEpiStore>(a, lda, w, rows, n, k, c, ldc, aux, ldaux, aux2, ldaux2, st);
    if (epi == kEpiAdd) e = launch_linear<false, kEpiAdd>(a, lda, w, rows, n, k, c, ldc, aux, ldaux, aux2, ldaux2, st);
  }
  OPP_REQUIRE(e != cudaErrorInvalidValue, "opp_fine_train_linear: epilogue %d not built for trans_w=%d", epi, trans_w);
  OPP_CHECK_CUDA(e);
  return OPP_OK;
}

int opp_fine_train_wgrad(const float* g, int ldg, const float* a, int lda, int rows, int n, int k, float* part,
                         float* dw, int accumulate, opp_stream_t stream) {
  OPP_REQUIRE(rows > 0 && n % 64 == 0 && k % 64 == 0 && n > 0 && k > 0, "opp_fine_train_wgrad: shape %d x %d x %d",
              rows, n, k);
  OPP_REQUIRE(g && a && part && dw && aligned4(g, ldg) && aligned4(a, lda), "opp_fine_train_wgrad: bad operand");
  const cudaStream_t st = (cudaStream_t)stream;
  const int groups = opp_fine_train_groups(rows);
  fine_wgrad_kernel<<<dim3(k / 64, n / 64, groups), 256, 0, st>>>(g, ldg, a, lda, rows, n, k, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  fine_reduce_kernel<<<(n * k + 255) / 256, 256, 0, st>>>(part, groups, n * k, accumulate, dw);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_ln(const float* x, int ldx, const float* gamma, const float* beta, const float* resid, int ldr,
                      float* y, int ldy, float* stats, int rows, opp_stream_t stream) {
  OPP_REQUIRE(rows >= 0, "opp_fine_train_ln: rows %d", rows);
  if (rows == 0) return OPP_OK;
  OPP_REQUIRE(x && gamma && beta && y && stats && aligned4(x, ldx) && aligned4(y, ldy) &&
                  (!resid || aligned4(resid, ldr)),
              "opp_fine_train_ln: bad operand");
  train_ln_fwd_kernel<kD><<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, ldx, gamma, beta, resid, ldr, y, ldy,
                                                                      reinterpret_cast<float2*>(stats), rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_ln_bwd(const float* x, int ldx, const float* gamma, const float* stats, const float* dy, int lddy,
                          float* dx, int lddx, int rows, float* part, float* dgb, int accumulate,
                          opp_stream_t stream) {
  OPP_REQUIRE(rows > 0, "opp_fine_train_ln_bwd: rows %d", rows);
  OPP_REQUIRE(x && gamma && stats && dy && dx && part && dgb && aligned4(x, ldx) && aligned4(dy, lddy) &&
                  aligned4(dx, lddx),
              "opp_fine_train_ln_bwd: bad operand");
  const cudaStream_t st = (cudaStream_t)stream;
  const int groups = opp_fine_train_groups(rows);
  train_ln_bwd_kernel<kD><<<groups, 256, 0, st>>>(x, ldx, gamma, reinterpret_cast<const float2*>(stats), dy, lddy, dx,
                                             lddx, part, rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  fine_reduce_kernel<<<1, 256, 0, st>>>(part, groups, 2 * kD, accumulate, dgb);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_attention(const float* qkv, float* out, int m, int cross, float eps, opp_stream_t stream) {
  OPP_REQUIRE(m >= 0, "opp_fine_train_attention: m %d", m);
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(qkv && out, "opp_fine_train_attention: null pointer");
  fine_attn_fwd_kernel<<<dim3(m, 2), 128, 0, (cudaStream_t)stream>>>(qkv, out, cross, eps);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_attention_bwd(const float* qkv, const float* dout, float* dqkv, int m, int cross, float eps,
                                 opp_stream_t stream) {
  OPP_REQUIRE(m >= 0, "opp_fine_train_attention_bwd: m %d", m);
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(qkv && dout && dqkv, "opp_fine_train_attention_bwd: null pointer");
  OPP_CHECK_CUDA(cudaFuncSetAttribute(fine_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kAttnBwdSmem));
  fine_attn_bwd_kernel<<<dim3(m, 2), 128, kAttnBwdSmem, (cudaStream_t)stream>>>(qkv, dout, dqkv, cross, eps);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_match(const float* x, int m, float* expec_f, opp_stream_t stream) {
  OPP_REQUIRE(m >= 0, "opp_fine_train_match: m %d", m);
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(x && expec_f && aligned4(x, 4), "opp_fine_train_match: bad operand");
  fine_match_fwd_kernel<<<(m + 3) / 4, 128, 0, (cudaStream_t)stream>>>(x, m, expec_f);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_train_match_bwd(const float* x, const float* dexpec, int m, float* dx, opp_stream_t stream) {
  OPP_REQUIRE(m >= 0, "opp_fine_train_match_bwd: m %d", m);
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(x && dexpec && dx && aligned4(x, 4) && aligned4(dx, 4), "opp_fine_train_match_bwd: bad operand");
  fine_match_bwd_kernel<<<(m + 3) / 4, 128, 0, (cudaStream_t)stream>>>(x, dexpec, m, dx);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
