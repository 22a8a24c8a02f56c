// opp_train.cu — coarse supervision of training on the device: the dual-softmax focal loss
// (Loss.compute_coarse_loss, src/lightning_model/losses.py:18-58, focal branch) and its backward to
// the two feature sets, without ever writing the [B, L, S] confidence matrix (DESIGN §7 f4).
//
//   sim = s A B^T (A [B][L][256] 3D features, B [B][S][256] 2D features), p = softmax over L,
//   q = softmax over S, c = p q.
//   Loss: c~ = clamp(c, 1e-6, 1 - 1e-6); gt == 1 -> -a (1 - c~)^g log c~, gt == 0 -> -(1 - a) c~^g
//   log(1 - c~), any other value -> nothing; loss = pos_w mean(pos) + neg_w mean(neg).
//   Backward: w = pos_w / npos or neg_w / nneg, gc = w c dl/dc (0 where the clamp is active),
//   R_i = sum_j gc_ij, C_j = sum_i gc_ij, dsim = go (2 gc - p C - q R), dA = s dsim B, dB = s dsim^T A.
//   Masked query columns (query_image_mask) have c = p = q = 0 and dsim = 0.
//   The ground truth is the dense [B, L, S] class matrix or, in the _sparse entry points, the sorted
//   list of its positives (opp_gt_index); the arithmetic is the same instructions either way.  The
//   fine level's ground truth offsets (fine_supervision) are looked up in the same list.
//
// One kernel shape serves every pass: a CTA keeps 64 "own" feature rows in shared memory and
// streams the other side in 64-row tiles; each tile's 64 x 64 block of sim is recomputed in fp32
// registers (CUDA-core FMA, K = 256, the same instruction sequence in every pass, so every pass sees
// the same sim bits), and
//   - statistics (own = 3D points): per row and per column the softmax statistics as a pair
//     (m, log s) — m = the max of sim, s = sum exp(sim - m) — rows complete per CTA, columns as
//     per-CTA partials merged in order by a second kernel;
//   - forward (own = 3D points): loss sums (fp64) and counts per CTA, R complete per row (pos and neg
//     halves), C partial per (CTA, column) — pos / neg kept apart because the weights pos_w / npos,
//     neg_w / nneg are only known after the pass;
//   - backward (own = 3D points, then own = query cells): dsim staged in shared memory, then
//     d_own += dsim . Y_tile on the same resident tile.
// log p = (sim - m) - log s keeps full fp32 accuracy when sim is the maximum itself (the exponent of
// a confident match is formed from differences of the same sim bits), and 1 - c = -expm1(log p +
// log q) is formed without cancellation: the focal terms near c = 1 depend on it as 1 / (1 - c).
// Every sum runs in a fixed order (no atomics), so results are bit-reproducible.
#include <cmath>
#include <cstdint>
#include <type_traits>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kFT = 64;            // own rows per CTA = other rows per streamed tile
constexpr int kFK = 256;           // feature width (coarse d_model)
constexpr int kFP = kFT + 4;       // shared pitch (floats) of the [k][row] tiles: float4-aligned
constexpr int kFThreads = 256;
constexpr size_t kFSmem = (2 * (size_t)kFK * kFP + (size_t)kFT * kFP + 6 * kFT) * sizeof(float) +
                          2 * kFT * sizeof(double);
constexpr size_t kFSmemSparse = kFSmem + kFT * sizeof(unsigned long long);   // + the tile's class bits

enum FocalPass { kStats = 0, kFwd = 1, kBwd = 2 };

struct FocalCfg {
  float alpha, gamma;
};

// loss term (on the clamped c) and c * dloss/dc (0 where the clamp is active), unweighted.
// om = 1 - c computed without cancellation.  cls: 1 positive, 0 negative, -1 neither.
__device__ __forceinline__ void focal_term(float c, float om, int cls, FocalCfg f, float& loss, float& gc) {
  const float lo = 1e-6f;
  const bool low = c < lo, high = om < 1e-6f;     // c > 1 - 1e-6
  const float ct = low ? lo : (high ? 1.f - 1e-6f : c);
  const float omt = low ? 1.f - lo : (high ? 1e-6f : om);
  const bool pass = !low && !high;
  loss = 0.f;
  gc = 0.f;
  if (cls == 1) {
    const float lg = logf(ct), omg = powf(omt, f.gamma);
    loss = -f.alpha * omg * lg;
    if (pass) gc = f.alpha * (f.gamma * ct * powf(omt, f.gamma - 1.f) * lg - omg);
  } else if (cls == 0) {
    const float l1 = logf(omt), cg = powf(ct, f.gamma);
    loss = -(1.f - f.alpha) * cg * l1;
    if (pass) gc = (1.f - f.alpha) * (-f.gamma * cg * l1 + cg * ct / omt);
  }
}

__device__ __forceinline__ int gt_class(const void* gt, int gt_bytes, long long idx) {
  const int v = gt_bytes == 2 ? (int)static_cast<const short*>(gt)[idx]
                              : (int)static_cast<const unsigned char*>(gt)[idx];
  return v == 1 ? 1 : (v == 0 ? 0 : -1);
}

// The ground truth of a launch.  Dense: the [B][L][S] class matrix.  Sparse: the positives as a
// list — per own row a bucket [ptr[r], ptr[r + 1]) of `ids`, ascending along the streamed side
// (own = 3D points: ptr = row_ptr, ids = the list's int64 j_ids; own = query cells: ptr = col_ptr,
// ids = int32 col_rows of opp_gt_index); every element outside the list is a negative.
typedef const void* __restrict__ DenseGt;
struct SparseGt {
  const int* ptr;
  const void* ids;
};

// running (max, sum exp(x - max)); m = -inf, s = 0 is the empty set
__device__ __forceinline__ void lse_add(float& m, float& s, float x) {
  if (x > m) {
    s = s * expf(m - x) + 1.f;
    m = x;
  } else {
    s += expf(x - m);
  }
}

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m == -INFINITY) {
    m = m2;
    s = s2;
    return;
  }
  const float mm = fmaxf(m, m2);
  s = s * expf(m - mm) + s2 * expf(m2 - mm);
  m = mm;
}

// rows [r0, r0 + 64) of x [n][256] -> xs[k][row] (zero past n)
__device__ __forceinline__ void load_tile_t(float* xs, const float* __restrict__ x, int r0, int n) {
  for (int idx = threadIdx.x; idx < kFT * (kFK / 4); idx += kFThreads) {
    const int row = idx % kFT, k4 = idx / kFT;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + row < n) v = *reinterpret_cast<const float4*>(x + (long long)(r0 + row) * kFK + 4 * k4);
    xs[(4 * k4 + 0) * kFP + row] = v.x;
    xs[(4 * k4 + 1) * kFP + row] = v.y;
    xs[(4 * k4 + 2) * kFP + row] = v.z;
    xs[(4 * k4 + 3) * kFP + row] = v.w;
  }
}

// kPass kStats / kFwd (own = rows = 3D points) or kBwd (own = rows when kOwnRows, else query cells).
// grid (ceil(n_own / 64), B).  st_own / st_oth: (m, log s) statistics of the own / other side (the
// softmax of an own row runs over the other side).  gt [B][L][S] (1 or 2 bytes), col_mask [B][S] or NULL.
// kSparse: gt is a SparseGt; per tile, thread r < 64 writes the 64 class bits of own row r from its
// bucket, which it walks once over the whole launch (the streamed index only grows).
template <int kPass, bool kOwnRows, bool kSparse>
__global__ void __launch_bounds__(kFThreads, 1)
coarse_focal_kernel(const float* __restrict__ own, const float* __restrict__ oth,
                    const float2* __restrict__ st_own, const float2* __restrict__ st_oth,
                    const double* __restrict__ stat_own, const double* __restrict__ stat_oth,
                    const float* __restrict__ wts, const float* __restrict__ grad,
                    typename std::conditional<kSparse, SparseGt, DenseGt>::type gt, int gt_bytes,
                    const unsigned char* __restrict__ col_mask, int n_own, int n_oth, float scale, FocalCfg f,
                    double* __restrict__ part_loss, long long* __restrict__ part_cnt,
                    void* __restrict__ part_r_, void* __restrict__ part_c_, float* __restrict__ d_own) {
  static_assert(kPass == kBwd || kOwnRows, "statistics and forward run with the 3D points as own rows");
  static_assert(kPass != kStats || !kSparse, "the statistics read no ground truth");
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;                          // [256][kFP] own rows, transposed
  float* ys = xs + kFK * kFP;                // [256][kFP] other tile, transposed
  float* ds = ys + kFK * kFP;                // [64][kFP] dsim (backward) / reduction scratch
  float* s_m_own = ds + kFT * kFP;           // [64] statistics of the own rows: max
  float* s_l_own = s_m_own + kFT;            // [64] log sum
  float* s_m_oth = s_l_own + kFT;            // [64]
  float* s_l_oth = s_m_oth + kFT;            // [64]
  float* s_mask_own = s_l_oth + kFT;         // [64] 1 = column kept (own = query cells)
  float* s_mask_oth = s_mask_own + kFT;      // [64]
  double* s_stat_own = reinterpret_cast<double*>(s_mask_oth + kFT);   // [64] R or C of the own rows (bwd)
  double* s_stat_oth = s_stat_own + kFT;     // [64]
  unsigned long long* s_bits = reinterpret_cast<unsigned long long*>(s_stat_oth + kFT);   // [64] (kSparse)
  // statistics: part_r = (m, log s) per row, part_c = (m, s) per (CTA, column), fp32;
  // forward: part_r = (pos, neg) R per row, part_c = (pos, neg) C per (CTA, column), fp64
  float2* st_part_r = static_cast<float2*>(part_r_);
  float2* st_part_c = static_cast<float2*>(part_c_);
  double2* fw_part_r = static_cast<double2*>(part_r_);
  double2* fw_part_c = static_cast<double2*>(part_c_);

  const int b = blockIdx.y, blk = blockIdx.x, o0 = blk * kFT;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  const int L = kOwnRows ? n_own : n_oth, S = kOwnRows ? n_oth : n_own;
  own += (long long)b * n_own * kFK;
  oth += (long long)b * n_oth * kFK;
  const unsigned char* mask = col_mask ? col_mask + (long long)b * S : nullptr;
  const long long gt0 = (long long)b * L * S;

  load_tile_t(xs, own, o0, n_own);
  if (tid < kFT) {
    const int o = o0 + tid;
    const bool in = o < n_own;
    const float2 st = (kPass != kStats && in) ? st_own[(long long)b * n_own + o] : make_float2(0.f, 0.f);
    s_m_own[tid] = st.x;
    s_l_own[tid] = st.y;
    s_stat_own[tid] = (kPass == kBwd && in) ? stat_own[(long long)b * n_own + o] : 0.0;
    s_mask_own[tid] = (kOwnRows || !mask || (in && mask[o])) ? 1.f : 0.f;
  }
  // sparse ground truth: the unread rest [cur, end) of own row tid's bucket (threads tid < 64)
  int cur = 0, end = 0;
  if constexpr (kSparse) {
    if (tid < kFT && o0 + tid < n_own) {
      cur = gt.ptr[(long long)b * n_own + o0 + tid];
      end = gt.ptr[(long long)b * n_own + o0 + tid + 1];
    }
  }
  float go = 0.f, wpos = 0.f, wneg = 0.f;
  if (kPass == kBwd) {
    go = grad[0];
    wpos = wts[0];
    wneg = wts[1];
  }

  // statistics accumulators (own rows 4 ty + a over this thread's columns)
  float rm[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, rsum[4] = {0.f, 0.f, 0.f, 0.f};
  // forward accumulators
  double lsum_pos = 0.0, lsum_neg = 0.0;
  long long npos = 0, nneg = 0;
  double rp[4] = {0.0, 0.0, 0.0, 0.0}, rn[4] = {0.0, 0.0, 0.0, 0.0};
  // backward accumulators: d_own rows ty2 + 8 n, k = tx2 + 32 m
  float acc2[8][8];
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int m = 0; m < 8; ++m) acc2[n][m] = 0.f;
  const int tx2 = tid % 32, ty2 = tid / 32;

  const int tiles = (n_oth + kFT - 1) / kFT;
  for (int t = 0; t < tiles; ++t) {
    const int t0 = t * kFT;
    __syncthreads();   // previous tile's readers of ys / ds are done
    load_tile_t(ys, oth, t0, n_oth);
    if (tid < kFT) {
      const int o = t0 + tid;
      const bool in = o < n_oth;
      const float2 st = (kPass != kStats && in) ? st_oth[(long long)b * n_oth + o] : make_float2(0.f, 0.f);
      s_m_oth[tid] = st.x;
      s_l_oth[tid] = st.y;
      s_stat_oth[tid] = (kPass == kBwd && in) ? stat_oth[(long long)b * n_oth + o] : 0.0;
      s_mask_oth[tid] = (!kOwnRows || !mask || (in && mask[o])) ? 1.f : 0.f;
      if constexpr (kSparse) {
        unsigned long long bits = 0;
        for (; cur < end; ++cur) {
          const long long id = kOwnRows ? static_cast<const long long*>(gt.ids)[cur]
                                        : (long long)static_cast<const int*>(gt.ids)[cur];
          if (id >= t0 + kFT) break;
          if (id >= t0) bits |= 1ull << (int)(id - t0);
        }
        s_bits[tid] = bits;
      }
    }
    __syncthreads();

    // sim block: own rows 4 ty + a, other rows 4 tx + c
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
#pragma unroll 8
    for (int k = 0; k < kFK; ++k) {
      const float4 xv = *reinterpret_cast<const float4*>(xs + k * kFP + 4 * ty);
      const float4 yv = *reinterpret_cast<const float4*>(ys + k * kFP + 4 * tx);
      const float xa[4] = {xv.x, xv.y, xv.z, xv.w}, yc[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(xa[a], yc[c], acc[a][c]);
    }

    if (kPass == kStats) {
      float cm[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int ro = 4 * ty + a;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int rc = 4 * tx + c;
          if (o0 + ro >= n_own || t0 + rc >= n_oth) continue;
          const float sim = __fmul_rn(scale, acc[a][c]);   // no contraction: the same bits in every pass
          lse_add(cm[c], cs[c], sim);                       // column softmax: over every row
          if (s_mask_oth[rc] != 0.f) lse_add(rm[a], rsum[a], sim);   // row softmax: kept columns only
        }
      }
      float2* cst = reinterpret_cast<float2*>(ds);   // [16][64]
#pragma unroll
      for (int c = 0; c < 4; ++c) cst[ty * kFT + 4 * tx + c] = make_float2(cm[c], cs[c]);
      __syncthreads();
      if (tid < kFT && t0 + tid < n_oth) {
        float m = -INFINITY, s = 0.f;
        for (int y = 0; y < 16; ++y) lse_merge(m, s, cst[y * kFT + tid].x, cst[y * kFT + tid].y);
        st_part_c[((long long)b * gridDim.x + blk) * n_oth + t0 + tid] = make_float2(m, s);
      }
      continue;
    }

    double cp[4] = {0.0, 0.0, 0.0, 0.0}, cn[4] = {0.0, 0.0, 0.0, 0.0};
    float dsv[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int ro = 4 * ty + a, o = o0 + ro;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int rc = 4 * tx + c, j = t0 + rc;
        dsv[a][c] = 0.f;
        if (o >= n_own || j >= n_oth) continue;
        const float sim = __fmul_rn(scale, acc[a][c]);   // no contraction: the same bits in every pass
        const bool kept = s_mask_own[ro] != 0.f && s_mask_oth[rc] != 0.f;
        // log of the softmax over the other side (statistics of the own row) and over the own side
        const float lp_row = kept ? (sim - s_m_own[ro]) - s_l_own[ro] : -INFINITY;
        const float lp_col = kept ? (sim - s_m_oth[rc]) - s_l_oth[rc] : -INFINITY;
        const float p_row = expf(lp_row), p_col = expf(lp_col);
        const float conf = p_row * p_col;
        const float om = kept ? -expm1f(lp_row + lp_col) : 1.f;
        int cls;
        if constexpr (kSparse) {
          cls = (int)((s_bits[ro] >> rc) & 1ull);
        } else {
          const long long gi = kOwnRows ? gt0 + (long long)o * S + j : gt0 + (long long)j * S + o;
          cls = gt_class(gt, gt_bytes, gi);
        }
        float l, gc;
        focal_term(conf, om, cls, f, l, gc);
        if (kPass == kFwd) {
          if (cls == 1) {
            lsum_pos += (double)l;
            ++npos;
            rp[a] += gc;
            cp[c] += gc;
          } else if (cls == 0) {
            lsum_neg += (double)l;
            ++nneg;
            rn[a] += gc;
            cn[c] += gc;
          }
        } else {
          // 2 gc - p C - q R = gc (1 - p) + gc (1 - q) - p (C - gc) - q (R - gc): for a confident
          // element C and R are dominated by its own gc ~ 1 / (1 - c), and the direct form would
          // cancel terms of that size; R, C are fp64 sums of the same fp32 gc bits, so C - gc is exact
          if (kept) {
            const double w = cls == 1 ? wpos : (cls == 0 ? wneg : 0.f);
            const double g = w * (double)gc;
            const double d = g * (double)(-expm1f(lp_col)) + g * (double)(-expm1f(lp_row)) -
                             (double)p_col * (s_stat_oth[rc] - g) - (double)p_row * (s_stat_own[ro] - g);
            dsv[a][c] = go * (float)d;
          }
        }
      }
    }

    if (kPass == kFwd) {
      // C partial of this CTA for the tile's columns: sum over the 64 own rows, ty in order
      double2* cs = reinterpret_cast<double2*>(ds);   // [16][64]
#pragma unroll
      for (int c = 0; c < 4; ++c) cs[ty * kFT + 4 * tx + c] = make_double2(cp[c], cn[c]);
      __syncthreads();
      if (tid < kFT && t0 + tid < n_oth) {
        double2 s = make_double2(0.0, 0.0);
        for (int y = 0; y < 16; ++y) {
          s.x += cs[y * kFT + tid].x;
          s.y += cs[y * kFT + tid].y;
        }
        fw_part_c[((long long)b * gridDim.x + blk) * n_oth + t0 + tid] = s;
      }
    } else {
#pragma unroll
      for (int a = 0; a < 4; ++a)
        *reinterpret_cast<float4*>(ds + (4 * ty + a) * kFP + 4 * tx) =
            make_float4(dsv[a][0], dsv[a][1], dsv[a][2], dsv[a][3]);
      __syncthreads();
      // d_own[r][k] += sum_c dsim[r][c] * Y[c][k]
#pragma unroll 2
      for (int c4 = 0; c4 < kFT / 4; ++c4) {
        float4 yv[8], dv[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) yv[m] = *reinterpret_cast<const float4*>(ys + (tx2 + 32 * m) * kFP + 4 * c4);
#pragma unroll
        for (int n = 0; n < 8; ++n) dv[n] = *reinterpret_cast<const float4*>(ds + (ty2 + 8 * n) * kFP + 4 * c4);
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
          for (int m = 0; m < 8; ++m) {
            float s = acc2[n][m];
            s = fmaf(dv[n].x, yv[m].x, s);
            s = fmaf(dv[n].y, yv[m].y, s);
            s = fmaf(dv[n].z, yv[m].z, s);
            s = fmaf(dv[n].w, yv[m].w, s);
            acc2[n][m] = s;
          }
      }
    }
  }

  if (kPass == kStats) {
    __syncthreads();
    float2* rs = reinterpret_cast<float2*>(ds);   // [64][16]
#pragma unroll
    for (int a = 0; a < 4; ++a) rs[(4 * ty + a) * 16 + tx] = make_float2(rm[a], rsum[a]);
    __syncthreads();
    if (tid < kFT && o0 + tid < n_own) {
      float m = -INFINITY, s = 0.f;
      for (int x = 0; x < 16; ++x) lse_merge(m, s, rs[tid * 16 + x].x, rs[tid * 16 + x].y);
      st_part_r[(long long)b * n_own + o0 + tid] = make_float2(m, logf(s));
    }
  } else if (kPass == kFwd) {
    __syncthreads();
    // R per own row: sum over tx in order
    double2* rs = reinterpret_cast<double2*>(ds);   // [64][16]
#pragma unroll
    for (int a = 0; a < 4; ++a) rs[(4 * ty + a) * 16 + tx] = make_double2(rp[a], rn[a]);
    __syncthreads();
    if (tid < kFT && o0 + tid < n_own) {
      double2 s = make_double2(0.0, 0.0);
      for (int x = 0; x < 16; ++x) {
        s.x += rs[tid * 16 + x].x;
        s.y += rs[tid * 16 + x].y;
      }
      fw_part_r[(long long)b * n_own + o0 + tid] = s;
    }
    __syncthreads();
    // loss sums and counts of the CTA: fixed tree over the 256 threads
    double* dl = reinterpret_cast<double*>(ds);              // [2][256]
    long long* dc = reinterpret_cast<long long*>(dl + 2 * kFThreads);   // [2][256]
    dl[tid] = lsum_pos;
    dl[kFThreads + tid] = lsum_neg;
    dc[tid] = npos;
    dc[kFThreads + tid] = nneg;
    __syncthreads();
    for (int h = kFThreads / 2; h > 0; h >>= 1) {
      if (tid < h) {
        dl[tid] += dl[tid + h];
        dl[kFThreads + tid] += dl[kFThreads + tid + h];
        dc[tid] += dc[tid + h];
        dc[kFThreads + tid] += dc[kFThreads + tid + h];
      }
      __syncthreads();
    }
    if (tid == 0) {
      const long long p = (long long)b * gridDim.x + blk;
      part_loss[2 * p] = dl[0];
      part_loss[2 * p + 1] = dl[kFThreads];
      part_cnt[2 * p] = dc[0];
      part_cnt[2 * p + 1] = dc[kFThreads];
    }
  } else {
    float* out = d_own + (long long)b * n_own * kFK;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int o = o0 + ty2 + 8 * n;
      if (o < n_own)
#pragma unroll
        for (int m = 0; m < 8; ++m) out[(long long)o * kFK + tx2 + 32 * m] = scale * acc2[n][m];
    }
  }
}

// column statistics: merge the per-CTA (max, sum) partials in block order -> (m, log s)
__global__ void coarse_focal_colstats_kernel(const float2* __restrict__ part_c, int batches, int cols, int blocks,
                                             float2* __restrict__ st_cols) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (long long)batches * cols) return;
  const long long b = q / cols, s = q % cols;
  float m = -INFINITY, sum = 0.f;
  for (int k = 0; k < blocks; ++k) {
    const float2 v = part_c[((long long)b * blocks + k) * cols + s];
    lse_merge(m, sum, v.x, v.y);
  }
  st_cols[q] = make_float2(m, logf(sum));
}

// One CTA: the loss and the per-class weights from the per-CTA partials, in a fixed order (fp64).
__global__ void __launch_bounds__(256)
coarse_focal_scalar_kernel(const double* __restrict__ part_loss, const long long* __restrict__ part_cnt,
                           int parts, float pos_w, float neg_w, float* __restrict__ loss,
                           long long* __restrict__ counts, float* __restrict__ wts) {
  __shared__ double sl[2][256];
  __shared__ long long sc[2][256];
  const int tid = threadIdx.x;
  double lp = 0.0, ln = 0.0;
  long long cp = 0, cn = 0;
  for (int i = tid; i < parts; i += 256) {
    lp += part_loss[2 * i];
    ln += part_loss[2 * i + 1];
    cp += part_cnt[2 * i];
    cn += part_cnt[2 * i + 1];
  }
  sl[0][tid] = lp;
  sl[1][tid] = ln;
  sc[0][tid] = cp;
  sc[1][tid] = cn;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (tid < h) {
      sl[0][tid] += sl[0][tid + h];
      sl[1][tid] += sl[1][tid + h];
      sc[0][tid] += sc[0][tid + h];
      sc[1][tid] += sc[1][tid + h];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const long long np = sc[0][0], nn = sc[1][0];
    // losses.py:44-53: an empty class drops out; both empty is the mean of nothing (NaN)
    double l;
    if (np == 0 && nn == 0) l = __longlong_as_double(0x7ff8000000000000LL);
    else l = (np ? (double)pos_w * sl[0][0] / (double)np : 0.0) + (nn ? (double)neg_w * sl[1][0] / (double)nn : 0.0);
    loss[0] = (float)l;
    counts[0] = np;
    counts[1] = nn;
    wts[0] = np ? (float)((double)pos_w / (double)np) : 0.f;
    wts[1] = nn ? (float)((double)neg_w / (double)nn) : 0.f;
  }
}

// R[b][l] = wpos Rp + wneg Rn; C[b][s] = wpos sum_blk Cp + wneg sum_blk Cn (blocks in order), fp64
__global__ void coarse_focal_rc_kernel(const double2* __restrict__ part_r, const double2* __restrict__ part_c,
                                       const float* __restrict__ wts, int batches, int rows, int cols,
                                       int blocks, double* __restrict__ r, double* __restrict__ c) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nr = (long long)batches * rows, nc = (long long)batches * cols;
  const double wp = wts[0], wn = wts[1];
  if (i < nr) {
    const double2 v = part_r[i];
    r[i] = wp * v.x + wn * v.y;
  } else if (i < nr + nc) {
    const long long q = i - nr, b = q / cols, s = q % cols;
    double sp = 0.0, sn = 0.0;
    for (int k = 0; k < blocks; ++k) {
      const double2 v = part_c[((long long)b * blocks + k) * cols + s];
      sp += v.x;
      sn += v.y;
    }
    c[q] = wp * sp + wn * sn;
  }
}

template <int kPass, bool kOwnRows, bool kSparse>
cudaError_t launch_focal(dim3 grid, cudaStream_t st, const float* own, const float* oth, const float2* st_own,
                         const float2* st_oth, const double* stat_own, const double* stat_oth,
                         const float* wts, const float* grad,
                         typename std::conditional<kSparse, SparseGt, const void*>::type gt, int gt_bytes,
                         const unsigned char* mask, int n_own, int n_oth, float scale, FocalCfg f, double* pl,
                         long long* pc, void* pr, void* pcc, float* d_own) {
  auto kern = coarse_focal_kernel<kPass, kOwnRows, kSparse>;
  constexpr size_t smem = kSparse ? kFSmemSparse : kFSmem;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, kFThreads, smem, st>>>(own, oth, st_own, st_oth, stat_own, stat_oth, wts, grad, gt, gt_bytes, mask,
                                      n_own, n_oth, scale, f, pl, pc, pr, pcc, d_own);
  return cudaGetLastError();
}

// ---- sparse ground truth: the positives as a list sorted by (b, i, j) ----------------------------

// row_ptr[r] = first entry whose row b L + i is >= r (r = 0 .. B L): one thread per row
__global__ void gt_row_ptr_kernel(const long long* __restrict__ b_ids, const long long* __restrict__ i_ids, int g,
                                  int rows, long long n_rows, int* __restrict__ row_ptr) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_rows) return;
  int lo = 0, hi = g;
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (b_ids[mid] * rows + i_ids[mid] < r) lo = mid + 1;
    else hi = mid;
  }
  row_ptr[r] = lo;
}

__device__ __forceinline__ bool gt_in_range(long long b, long long i, long long j, int batches, int rows, int cols) {
  return b >= 0 && b < batches && i >= 0 && i < rows && j >= 0 && j < cols;
}

// col_ptr[1 + b S + j] += 1 per entry (col_ptr zeroed before)
__global__ void gt_col_count_kernel(const long long* __restrict__ b_ids, const long long* __restrict__ i_ids,
                                    const long long* __restrict__ j_ids, int g, int batches, int rows, int cols,
                                    int* __restrict__ col_ptr) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g || !gt_in_range(b_ids[e], i_ids[e], j_ids[e], batches, rows, cols)) return;
  atomicAdd(col_ptr + 1 + b_ids[e] * cols + j_ids[e], 1);
}

// in-place inclusive scan of x[0 .. n) by one CTA, 1024 elements per round with a running carry
__global__ void __launch_bounds__(1024) gt_scan_kernel(int* __restrict__ x, long long n) {
  __shared__ int warp_sum[32];
  __shared__ int carry_s;
  const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (long long base = 0; base < n; base += 1024) {
    const long long idx = base + tid;
    int v = idx < n ? x[idx] : 0;
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, d);
      if (lane >= d) v += u;
    }
    if (lane == 31) warp_sum[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sum[lane];
      for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w += u;
      }
      warp_sum[lane] = w;
    }
    __syncthreads();
    const int carry = carry_s;
    v += carry + (warp ? warp_sum[warp - 1] : 0);
    if (idx < n) x[idx] = v;
    __syncthreads();
    if (tid == 1023) carry_s = v;
    __syncthreads();
  }
}

// col_rows[col_ptr[c] + slot] = i, slot handed out by an integer atomic (fill zeroed before); the
// order inside a bucket is settled by gt_col_sort_kernel
__global__ void gt_col_scatter_kernel(const long long* __restrict__ b_ids, const long long* __restrict__ i_ids,
                                      const long long* __restrict__ j_ids, int g, int batches, int rows, int cols,
                                      const int* __restrict__ col_ptr, int* __restrict__ fill,
                                      int* __restrict__ col_rows) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g || !gt_in_range(b_ids[e], i_ids[e], j_ids[e], batches, rows, cols)) return;
  const long long c = b_ids[e] * cols + j_ids[e];
  col_rows[col_ptr[c] + atomicAdd(fill + c, 1)] = (int)i_ids[e];
}

// each column's bucket ascending in i (insertion sort, one thread per column: a bucket holds the 3D
// points of one query cell, a handful at most), so the result does not depend on the scatter's order
__global__ void gt_col_sort_kernel(const int* __restrict__ col_ptr, long long n_cols, int* __restrict__ col_rows) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  const int lo = col_ptr[c], hi = col_ptr[c + 1];
  for (int x = lo + 1; x < hi; ++x) {
    const int v = col_rows[x];
    int y = x - 1;
    for (; y >= lo && col_rows[y] > v; --y) col_rows[y + 1] = col_rows[y];
    col_rows[y + 1] = v;
  }
}

// fine_supervision (src/models/OnePosePlus/utils/fine_supervision.py:18-28) for one match per
// thread: (b, i, j) looked up in the sorted list -> its fine location, or (-50, -50) when it is not
// ground truth.  Every operation is a separately rounded fp32 one in the reference's order; the
// scalar divisions are multiplications by the fp32 reciprocal, as PyTorch evaluates tensor / scalar
// on the device.
__global__ void fine_supervision_kernel(const long long* __restrict__ gb, const long long* __restrict__ gi,
                                        const long long* __restrict__ gj, const float* __restrict__ fine_xy, int g,
                                        const long long* __restrict__ mb, const long long* __restrict__ mi,
                                        const long long* __restrict__ mj, int m, int w_c, int coarse_res,
                                        int fine_res, float inv_fine, float inv_radius,
                                        const float* __restrict__ img_scale, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const long long b = mb[t], i = mi[t], j = mj[t];
  int lo = 0, hi = g;
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    const long long b2 = gb[mid], i2 = gi[mid];
    const bool less = b2 != b ? b2 < b : (i2 != i ? i2 < i : gj[mid] < j);
    if (less) lo = mid + 1;
    else hi = mid;
  }
  float x = -50.f, y = -50.f;
  if (lo < g && gb[lo] == b && gi[lo] == i && gj[lo] == j) {
    x = fine_xy[2 * lo];
    y = fine_xy[2 * lo + 1];
  }
  const long long jx = j % w_c, jy = j / w_c;
  float ex, ey;
  if (img_scale) {
    // (x, y) scales = query_image_scale[b][[1, 0]]
    const float sx = img_scale[2 * b + 1], sy = img_scale[2 * b];
    const float qx = __fmul_rn((float)jx, __fmul_rn((float)coarse_res, sx));
    const float qy = __fmul_rn((float)jy, __fmul_rn((float)coarse_res, sy));
    ex = __fdiv_rn(__fsub_rn(x, qx), __fmul_rn((float)fine_res, sx));
    ey = __fdiv_rn(__fsub_rn(y, qy), __fmul_rn((float)fine_res, sy));
  } else {
    // fine_supervision.py:18: without query_image_scale the coarse scale is the fine one
    ex = __fmul_rn(__fsub_rn(x, (float)(jx * fine_res)), inv_fine);
    ey = __fmul_rn(__fsub_rn(y, (float)(jy * fine_res)), inv_fine);
  }
  out[2 * t] = __fmul_rn(ex, inv_radius);
  out[2 * t + 1] = __fmul_rn(ey, inv_radius);
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" int opp_coarse_focal_blocks(int rows) { return (rows + kFT - 1) / kFT; }

#define OPP_FOCAL_SHAPE(name)                                                                               \
  OPP_REQUIRE(a && b, name ": null pointer");                                                              \
  OPP_REQUIRE(batches > 0 && batches <= 65535 && rows > 0 && cols > 0, name ": bad shape B=%d L=%d S=%d",  \
              batches, rows, cols);                                                                        \
  OPP_REQUIRE(k == kFK, name ": feature width %d (built for %d)", k, kFK);                                 \
  OPP_REQUIRE(((uintptr_t)a & 15) == 0 && ((uintptr_t)b & 15) == 0, name ": features must be 16-byte aligned")

#define OPP_FOCAL_CHECKS(name)                                                                              \
  OPP_FOCAL_SHAPE(name);                                                                                   \
  OPP_REQUIRE(st_rows && st_cols && gt, name ": null pointer");                                            \
  OPP_REQUIRE(gt_bytes == 1 || gt_bytes == 2, name ": gt element size %d (bool / uint8 / int16)", gt_bytes)

extern "C" int opp_coarse_focal_stats(const float* a, const float* b, const unsigned char* col_mask, int batches,
                                      int rows, int cols, int k, float scale, float* part_c, float* st_rows,
                                      float* st_cols, opp_stream_t stream) {
  OPP_FOCAL_SHAPE("opp_coarse_focal_stats");
  OPP_REQUIRE(part_c && st_rows && st_cols, "opp_coarse_focal_stats: null output");
  const cudaStream_t st = (cudaStream_t)stream;
  const int blocks = opp_coarse_focal_blocks(rows);
  OPP_CHECK_CUDA((launch_focal<kStats, true, false>(dim3(blocks, batches), st, a, b, nullptr, nullptr, nullptr, nullptr,
                                             nullptr, nullptr, nullptr, 1, col_mask, rows, cols, scale,
                                             FocalCfg{0.f, 0.f}, nullptr, nullptr, st_rows, part_c, nullptr)));
  const long long n = (long long)batches * cols;
  coarse_focal_colstats_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const float2*>(part_c), batches, cols, blocks, reinterpret_cast<float2*>(st_cols));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_coarse_focal_fwd(const float* a, const float* b, const float* st_rows, const float* st_cols,
                                    const void* gt, int gt_bytes, const unsigned char* col_mask, int batches,
                                    int rows, int cols, int k, float scale, float alpha, float gamma, float pos_w,
                                    float neg_w, double* part_loss, long long* part_cnt, double* part_r,
                                    double* part_c, float* loss, long long* counts, float* wts, double* r, double* c,
                                    opp_stream_t stream) {
  OPP_FOCAL_CHECKS("opp_coarse_focal_fwd");
  OPP_REQUIRE(part_loss && part_cnt && part_r && part_c && loss && counts && wts && r && c,
              "opp_coarse_focal_fwd: null output");
  const cudaStream_t st = (cudaStream_t)stream;
  const int blocks = opp_coarse_focal_blocks(rows);
  const FocalCfg f{alpha, gamma};
  OPP_CHECK_CUDA((launch_focal<kFwd, true, false>(dim3(blocks, batches), st, a, b, reinterpret_cast<const float2*>(st_rows),
                                           reinterpret_cast<const float2*>(st_cols), nullptr, nullptr, nullptr,
                                           nullptr, gt, gt_bytes, col_mask, rows, cols, scale, f, part_loss,
                                           part_cnt, part_r, part_c, nullptr)));
  coarse_focal_scalar_kernel<<<1, 256, 0, st>>>(part_loss, part_cnt, batches * blocks, pos_w, neg_w, loss, counts,
                                               wts);
  OPP_CHECK_CUDA(cudaGetLastError());
  const long long n = (long long)batches * (rows + cols);
  coarse_focal_rc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const double2*>(part_r), reinterpret_cast<const double2*>(part_c), wts, batches, rows, cols,
      blocks, r, c);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_coarse_focal_bwd(const float* a, const float* b, const float* st_rows, const float* st_cols,
                                    const double* r, const double* c, const float* wts, const float* grad,
                                    const void* gt, int gt_bytes, const unsigned char* col_mask, int batches,
                                    int rows, int cols, int k, float scale, float alpha, float gamma, float* da,
                                    float* db, opp_stream_t stream) {
  OPP_FOCAL_CHECKS("opp_coarse_focal_bwd");
  OPP_REQUIRE(r && c && wts && grad && da && db, "opp_coarse_focal_bwd: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const FocalCfg f{alpha, gamma};
  const float2* sr = reinterpret_cast<const float2*>(st_rows);
  const float2* sc = reinterpret_cast<const float2*>(st_cols);
  OPP_CHECK_CUDA((launch_focal<kBwd, true, false>(dim3(opp_coarse_focal_blocks(rows), batches), st, a, b, sr, sc, r, c,
                                           wts, grad, gt, gt_bytes, col_mask, rows, cols, scale, f, nullptr, nullptr,
                                           nullptr, nullptr, da)));
  OPP_CHECK_CUDA((launch_focal<kBwd, false, false>(dim3(opp_coarse_focal_blocks(cols), batches), st, b, a, sc, sr, c, r,
                                            wts, grad, gt, gt_bytes, col_mask, cols, rows, scale, f, nullptr,
                                            nullptr, nullptr, nullptr, db)));
  return OPP_OK;
}

#define OPP_GT_LIST(name)                                                                                   \
  OPP_REQUIRE(g >= 0 && (g == 0 || (b_ids && i_ids && j_ids)), name ": bad list (g=%d)", g);                \
  OPP_REQUIRE(batches > 0 && rows > 0 && cols > 0 && (long long)batches * rows < INT32_MAX &&               \
                  (long long)batches * cols < INT32_MAX,                                                    \
              name ": bad shape B=%d L=%d S=%d", batches, rows, cols)

extern "C" int opp_gt_index(const long long* b_ids, const long long* i_ids, const long long* j_ids, int g,
                            int batches, int rows, int cols, int* row_ptr, int* col_ptr, int* col_rows, int* fill,
                            opp_stream_t stream) {
  OPP_GT_LIST("opp_gt_index");
  OPP_REQUIRE(row_ptr && col_ptr && fill && (g == 0 || col_rows), "opp_gt_index: null output");
  const cudaStream_t st = (cudaStream_t)stream;
  const long long n_rows = (long long)batches * rows, n_cols = (long long)batches * cols;
  gt_row_ptr_kernel<<<(unsigned)((n_rows + 256) / 256), 256, 0, st>>>(b_ids, i_ids, g, rows, n_rows, row_ptr);
  OPP_CHECK_CUDA(cudaGetLastError());
  OPP_CHECK_CUDA(cudaMemsetAsync(col_ptr, 0, (n_cols + 1) * sizeof(int), st));
  if (g == 0) return OPP_OK;
  OPP_CHECK_CUDA(cudaMemsetAsync(fill, 0, n_cols * sizeof(int), st));
  const unsigned eb = (unsigned)((g + 255) / 256);
  gt_col_count_kernel<<<eb, 256, 0, st>>>(b_ids, i_ids, j_ids, g, batches, rows, cols, col_ptr);
  OPP_CHECK_CUDA(cudaGetLastError());
  gt_scan_kernel<<<1, 1024, 0, st>>>(col_ptr, n_cols + 1);
  OPP_CHECK_CUDA(cudaGetLastError());
  gt_col_scatter_kernel<<<eb, 256, 0, st>>>(b_ids, i_ids, j_ids, g, batches, rows, cols, col_ptr, fill, col_rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  gt_col_sort_kernel<<<(unsigned)((n_cols + 255) / 256), 256, 0, st>>>(col_ptr, n_cols, col_rows);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_coarse_focal_fwd_sparse(const float* a, const float* b, const float* st_rows,
                                           const float* st_cols, const int* row_ptr, const long long* j_ids,
                                           const unsigned char* col_mask, int batches, int rows, int cols, int k,
                                           float scale, float alpha, float gamma, float pos_w, float neg_w,
                                           double* part_loss, long long* part_cnt, double* part_r, double* part_c,
                                           float* loss, long long* counts, float* wts, double* r, double* c,
                                           opp_stream_t stream) {
  OPP_FOCAL_SHAPE("opp_coarse_focal_fwd_sparse");
  OPP_REQUIRE(st_rows && st_cols && row_ptr, "opp_coarse_focal_fwd_sparse: null pointer");
  OPP_REQUIRE(part_loss && part_cnt && part_r && part_c && loss && counts && wts && r && c,
              "opp_coarse_focal_fwd_sparse: null output");
  const cudaStream_t st = (cudaStream_t)stream;
  const int blocks = opp_coarse_focal_blocks(rows);
  const FocalCfg f{alpha, gamma};
  OPP_CHECK_CUDA((launch_focal<kFwd, true, true>(dim3(blocks, batches), st, a, b,
                                                 reinterpret_cast<const float2*>(st_rows),
                                                 reinterpret_cast<const float2*>(st_cols), nullptr, nullptr, nullptr,
                                                 nullptr, SparseGt{row_ptr, j_ids}, 0, col_mask, rows, cols, scale, f,
                                                 part_loss, part_cnt, part_r, part_c, nullptr)));
  coarse_focal_scalar_kernel<<<1, 256, 0, st>>>(part_loss, part_cnt, batches * blocks, pos_w, neg_w, loss, counts,
                                               wts);
  OPP_CHECK_CUDA(cudaGetLastError());
  const long long n = (long long)batches * (rows + cols);
  coarse_focal_rc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const double2*>(part_r), reinterpret_cast<const double2*>(part_c), wts, batches, rows, cols,
      blocks, r, c);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_coarse_focal_bwd_sparse(const float* a, const float* b, const float* st_rows,
                                           const float* st_cols, const double* r, const double* c, const float* wts,
                                           const float* grad, const int* row_ptr, const long long* j_ids,
                                           const int* col_ptr, const int* col_rows, const unsigned char* col_mask,
                                           int batches, int rows, int cols, int k, float scale, float alpha,
                                           float gamma, float* da, float* db, opp_stream_t stream) {
  OPP_FOCAL_SHAPE("opp_coarse_focal_bwd_sparse");
  OPP_REQUIRE(st_rows && st_cols && row_ptr && col_ptr, "opp_coarse_focal_bwd_sparse: null pointer");
  OPP_REQUIRE(r && c && wts && grad && da && db, "opp_coarse_focal_bwd_sparse: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const FocalCfg f{alpha, gamma};
  const float2* sr = reinterpret_cast<const float2*>(st_rows);
  const float2* sc = reinterpret_cast<const float2*>(st_cols);
  OPP_CHECK_CUDA((launch_focal<kBwd, true, true>(dim3(opp_coarse_focal_blocks(rows), batches), st, a, b, sr, sc, r, c,
                                                 wts, grad, SparseGt{row_ptr, j_ids}, 0, col_mask, rows, cols, scale,
                                                 f, nullptr, nullptr, nullptr, nullptr, da)));
  OPP_CHECK_CUDA((launch_focal<kBwd, false, true>(dim3(opp_coarse_focal_blocks(cols), batches), st, b, a, sc, sr, c,
                                                  r, wts, grad, SparseGt{col_ptr, col_rows}, 0, col_mask, cols, rows,
                                                  scale, f, nullptr, nullptr, nullptr, nullptr, db)));
  return OPP_OK;
}

extern "C" int opp_fine_supervision(const long long* b_ids, const long long* i_ids, const long long* j_ids,
                                    const float* fine_xy, int g, int batches, int rows, int cols,
                                    const long long* m_b, const long long* m_i, const long long* m_j, int m, int w_c,
                                    int coarse_res, int fine_res, int radius, const float* img_scale, float* out,
                                    opp_stream_t stream) {
  OPP_GT_LIST("opp_fine_supervision");
  OPP_REQUIRE(g == 0 || fine_xy, "opp_fine_supervision: null fine_xy");
  OPP_REQUIRE(m >= 0 && (m == 0 || (m_b && m_i && m_j && out)), "opp_fine_supervision: bad matches (m=%d)", m);
  OPP_REQUIRE(w_c > 0 && cols % w_c == 0 && coarse_res > 0 && fine_res > 0 && radius > 0,
              "opp_fine_supervision: bad geometry w_c=%d S=%d resolution=(%d, %d) radius=%d", w_c, cols, coarse_res,
              fine_res, radius);
  if (m == 0) return OPP_OK;
  fine_supervision_kernel<<<(unsigned)((m + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      b_ids, i_ids, j_ids, fine_xy, g, m_b, m_i, m_j, m, w_c, coarse_res, fine_res, 1.f / (float)fine_res,
      1.f / (float)radius, img_scale, out);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
