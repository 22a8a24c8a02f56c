// opp_train_backbone.cu — the ResNet-FPN backbone of training on the device: convolution forward,
// data gradient and weight gradient on the tensor cores in 3xTF32, batch-statistics BatchNorm with its
// activation and residual, and the FPN's bilinear x2 upsample-add, forward and backward (DESIGN §7 f4).
//
// Activations are NCHW fp32.  Weights are [C_out][C_in][k][k] (nn.Conv2d's layout), pad = k / 2.
// The three convolution passes are one implicit GEMM with operands gathered straight from the maps:
//   forward  out[p][co]     = sum_{ci,tap} x(p, ci, tap)  W[co][ci][tap]     M = output pixels, N = c_out
//   dgrad    dx[q][ci]      = sum_{co,tap} dy(q, co, tap) W[co][ci][tap]     M = input pixels,  N = c_in
//   wgrad    dW[co][ci,tap] = sum_p        dy[p][co]      x(p, ci, tap)      M = c_out, N = c_in·k², K = pixels
// where x(p, ci, tap) is the input the tap reads for output pixel p (0 outside the map) and
// dy(q, co, tap) the output-gradient pixel whose tap reads input pixel q: for stride 2 a tap
// contributes only where (i + pad - k_y) is even and (i + pad - k_y) / 2 is in range.
//
// Each gathered value v is split into tf32 hi = rna(v) and lo = rna(v - hi), and every k8 step issues
// three wgmma m64n64k8 tf32 MMAs into one fp32 accumulator, always in the order lo·hi, hi·lo, hi·hi
// (the lo·lo term, |lo·lo| <= 2^-22 |a·b|, is dropped).  The accumulator restarts at every 32-wide K
// chunk and its sum is added to an fp32 register total, in chunk order.
//
// CTA: 256 threads = two warpgroups, a 128 x 64 tile of C (each warpgroup 64 rows), K in chunks of 32.
// Every thread gathers: a chunk's A (128 rows) and B (64 rows) go to registers, are split, and are
// stored as four K-major planes (A hi, A lo, B hi, B lo; rows of 32 tf32 = 128 B, 128-byte swizzle)
// into one of two ring stages.  The gather of chunk k + 1 runs while the MMAs of chunk k are in flight.
//
// Every reduction runs in a fixed order and no kernel uses floating-point atomics, so two calls give
// the same bits:
//   - wgrad: output pixels are cut into groups of kWgradGroup; each CTA sums one group for one tile of
//     dW into a partial, and bb_reduce adds the partials in group order;
//   - BatchNorm statistics and dgamma / dbeta: fp64 partials per (image, chunk of kBnChunk pixels) of a
//     channel, merged per channel in that order;
//   - the upsample backward gathers, for each input pixel, the output pixels that read it.
#include <cmath>
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kBM = 128, kBN = 64, kBK = 32, kThreads = 256;
constexpr int kWgradGroup = 2048;                          // output pixels per wgrad partial
constexpr int kPlaneA = kBM * kBK * 4, kPlaneB = kBN * kBK * 4;
constexpr int kStage = 2 * kPlaneA + 2 * kPlaneB;          // A hi, A lo, B hi, B lo: 48 KiB
constexpr int kSmem = 2 * kStage + 1024;                   // two stages + 1024-byte alignment slack
constexpr int kBnChunk = 4096;                             // pixels per BatchNorm partial
constexpr float kLeakySlope = 0.01f;

enum { kFwd = 0, kDgrad = 1, kWgrad = 2 };
enum { kActNone = 0, kActRelu = 1, kActLeaky = 2 };

struct ConvGeo {
  int batches, c_in, h, w, c_out, ho, wo, stride, pad;
};


__device__ __forceinline__ uint32_t tf32_rna(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}

// byte offset of (row, 16-byte column chunk) in a K-major plane of 128-byte rows, 128-byte swizzle
__device__ __forceinline__ uint32_t swz(int row, int chunk) {
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// four consecutive K values of one row, split into hi and lo, into the hi plane and the lo plane
__device__ __forceinline__ void store_split4(uint32_t hi_plane, uint32_t lo_plane, uint32_t off, const float* v) {
  uint4 h, l;
  h.x = tf32_rna(v[0]), h.y = tf32_rna(v[1]), h.z = tf32_rna(v[2]), h.w = tf32_rna(v[3]);
  l.x = tf32_rna(v[0] - __uint_as_float(h.x)), l.y = tf32_rna(v[1] - __uint_as_float(h.y));
  l.z = tf32_rna(v[2] - __uint_as_float(h.z)), l.w = tf32_rna(v[3] - __uint_as_float(h.w));
  sts128(hi_plane + off, h);
  sts128(lo_plane + off, l);
}

#define OPP_WG_ACC8(i)                                                                              \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]),    \
      "+f"(d[i + 6]), "+f"(d[i + 7])
// d = A B^T (+ d when accumulate) for one m64n64k8 tf32 step, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc,
                                                    int accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n\t"
      "}\n"
      : OPP_WG_ACC8(0), OPP_WG_ACC8(8), OPP_WG_ACC8(16), OPP_WG_ACC8(24)
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}
#undef OPP_WG_ACC8

// One CTA: a kBM x kBN tile of C = A B^T over K [k_begin, k_end).
//   kFwd:   C -> y (NCHW);  kDgrad: C -> dx (NCHW, += when accumulate);  kWgrad: C -> part[blockIdx.z]
// Gather mapping per chunk:
//   kFwd / kDgrad A: row m = tid % 128 (consecutive pixels across a warp), K quads tid / 128 + 2 i;
//   B (all modes) and kWgrad A: K quad tid % 8, rows tid / 8 + 32 i (128 contiguous bytes per row).
template <int MODE, int KS>
__global__ void __launch_bounds__(kThreads, 2) bb_conv_kernel(const float* __restrict__ x,
                                                                 const float* __restrict__ wt,
                                                                 const float* __restrict__ dy, ConvGeo g, int pix0,
                                                                 int npix, int accumulate, float* __restrict__ out) {
  constexpr int KK = KS * KS;
  constexpr int kAQ = 4, kBQ = 2;                          // quads of 4 values per thread: A, B
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x;
  const int hw = g.h * g.w, howo = g.ho * g.wo;
  int M, N, k_begin, k_end;
  if constexpr (MODE == kFwd) {
    M = g.batches * howo, N = g.c_out, k_begin = 0, k_end = g.c_in * KK;
  } else if constexpr (MODE == kDgrad) {
    M = g.batches * hw, N = g.c_in, k_begin = 0, k_end = g.c_out * KK;
  } else {
    M = g.c_out, N = g.c_in * KK;
    k_begin = pix0 + blockIdx.z * kWgradGroup;
    k_end = min(k_begin + kWgradGroup, pix0 + npix);
  }
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const int q = tid & 7;                                   // K quad of the row-per-8-threads loads

  // loader state ----------------------------------------------------------------------------------
  int a_b = 0, a_y = 0, a_x = 0;
  bool a_ok = false;
  if constexpr (MODE != kWgrad) {
    const int m = m0 + (tid & (kBM - 1));
    a_ok = m < M;
    const int pw = MODE == kFwd ? g.wo : g.w, ph = MODE == kFwd ? g.ho : g.h;
    const int mm = a_ok ? m : 0;
    a_b = mm / (pw * ph);
    const int p = mm - a_b * pw * ph;
    a_y = p / pw;
    a_x = p - a_y * pw;
  }
  int bw_ci[kBQ], bw_ky[kBQ], bw_kx[kBQ];                  // kWgrad B rows: (ci, tap) of n
  if constexpr (MODE == kWgrad) {
#pragma unroll
    for (int i = 0; i < kBQ; ++i) {
      const int n = n0 + (tid >> 3) + 32 * i;
      const int ci = n / KK, tap = n - ci * KK;
      bw_ci[i] = n < N ? ci : -1;
      bw_ky[i] = tap / KS;
      bw_kx[i] = tap - (tap / KS) * KS;
    }
  }

  float ra[kAQ][4], rb[kBQ][4];
  auto load = [&](int kc) {
    if constexpr (MODE == kFwd || MODE == kDgrad) {
#pragma unroll
      for (int i = 0; i < kAQ; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = kc + 4 * ((tid >> 7) + 2 * i) + e;
          float v = 0.f;
          if (a_ok && k < k_end) {
            const int c = k / KK, tap = k - c * KK, ky = tap / KS, kx = tap - ky * KS;
            if constexpr (MODE == kFwd) {
              const int iy = a_y * g.stride - g.pad + ky, ix = a_x * g.stride - g.pad + kx;
              if (iy >= 0 && iy < g.h && ix >= 0 && ix < g.w) v = x[((size_t)a_b * g.c_in + c) * hw + iy * g.w + ix];
            } else {
              const int ty = a_y + g.pad - ky, tx = a_x + g.pad - kx;
              if (ty >= 0 && tx >= 0 && ty % g.stride == 0 && tx % g.stride == 0) {
                const int oy = ty / g.stride, ox = tx / g.stride;
                if (oy < g.ho && ox < g.wo) v = dy[((size_t)a_b * g.c_out + c) * howo + oy * g.wo + ox];
              }
            }
          }
          ra[i][e] = v;
        }
#pragma unroll
      for (int i = 0; i < kBQ; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int k = kc + 4 * q + e, n = n0 + (tid >> 3) + 32 * i;
          float v = 0.f;
          if (n < N && k < k_end) {
            if constexpr (MODE == kFwd) {
              v = wt[n * k_end + k];                      // < 2^31 (conv_geo)
            } else {
              const int co = k / KK, tap = k - co * KK;
              v = wt[((size_t)co * g.c_in + n) * KK + tap];
            }
          }
          rb[i][e] = v;
        }
    } else {
      // the four output pixels of this thread's quad, shared by its A and B rows
      int pb[4], pp[4], py[4], px[4];
      bool pok[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = kc + 4 * q + e;
        pok[e] = k < k_end;
        pb[e] = pok[e] ? k / howo : 0;
        pp[e] = pok[e] ? k - pb[e] * howo : 0;
        py[e] = pp[e] / g.wo;
        px[e] = pp[e] - py[e] * g.wo;
      }
#pragma unroll
      for (int i = 0; i < kAQ; ++i) {
        const int m = m0 + (tid >> 3) + 32 * i;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          ra[i][e] = (pok[e] && m < M) ? dy[((size_t)pb[e] * g.c_out + m) * howo + pp[e]] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < kBQ; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = 0.f;
          if (pok[e] && bw_ci[i] >= 0) {
            const int iy = py[e] * g.stride - g.pad + bw_ky[i], ix = px[e] * g.stride - g.pad + bw_kx[i];
            if (iy >= 0 && iy < g.h && ix >= 0 && ix < g.w)
              v = x[((size_t)pb[e] * g.c_in + bw_ci[i]) * hw + iy * g.w + ix];
          }
          rb[i][e] = v;
        }
    }
  };
  auto store = [&](int s) {
    const uint32_t a_hi = base + s * kStage, a_lo = a_hi + kPlaneA;
    const uint32_t b_hi = a_lo + kPlaneA, b_lo = b_hi + kPlaneB;
#pragma unroll
    for (int i = 0; i < kAQ; ++i) {
      const uint32_t off = MODE == kWgrad ? swz((tid >> 3) + 32 * i, q) : swz(tid & (kBM - 1), (tid >> 7) + 2 * i);
      store_split4(a_hi, a_lo, off, ra[i]);
    }
#pragma unroll
    for (int i = 0; i < kBQ; ++i) store_split4(b_hi, b_lo, swz((tid >> 3) + 32 * i, q), rb[i]);
    fence_proxy_async_smem();                            // generic stores -> the MMAs' async-proxy reads
  };

  // main loop -------------------------------------------------------------------------------------
  // The wgmma accumulator rounds toward zero once per instruction (DESIGN §3), a bias that grows with
  // the number of accumulating MMAs.  So each chunk's 12 MMAs start from zero in acc, and the chunk sum
  // is added to tot with an IEEE fp32 add: one round-to-nearest add per 32 K values.
  const int wg = tid >> 7;
  float acc[32], tot[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) tot[i] = 0.f;
  int s = 0;
  load(k_begin);
  store(0);
  __syncthreads();
  for (int kc = k_begin; kc < k_end; kc += kBK) {
    const bool more = kc + kBK < k_end;
    const uint32_t a_hi = base + s * kStage + wg * (kPlaneA / 2), a_lo = a_hi + kPlaneA;
    const uint32_t b_hi = base + s * kStage + 2 * kPlaneA, b_lo = b_hi + kPlaneB;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBK / 8; ++kk) {
      const uint32_t o = kk * 32;                        // one k8 step: 32 bytes along the row
      wgmma_m64n64k8_tf32(acc, make_kmajor_sw128_desc(a_lo + o), make_kmajor_sw128_desc(b_hi + o), kk);
      wgmma_m64n64k8_tf32(acc, make_kmajor_sw128_desc(a_hi + o), make_kmajor_sw128_desc(b_lo + o), 1);
      wgmma_m64n64k8_tf32(acc, make_kmajor_sw128_desc(a_hi + o), make_kmajor_sw128_desc(b_hi + o), 1);
    }
    wgmma_commit();
    if (more) {
      load(kc + kBK);                                    // the other stage was released by the last wait
      store(s ^ 1);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) tot[i] += acc[i];
    __syncthreads();
    s ^= 1;
  }

  // epilogue: accumulator element 4 j + 2 h + c is row r0 + 8 h, column 8 j + c0 + c --------------------
  const int warp = (tid >> 5) & 3, lane = tid & 31;
  const int r0 = m0 + 64 * wg + 16 * warp + (lane >> 2), c0 = n0 + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r0 + 8 * h;
    if (m >= M) continue;
    if constexpr (MODE == kWgrad) {
      float* o = out + (size_t)blockIdx.z * M * N + (size_t)m * N;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int n = c0 + 8 * j + c;
          if (n < N) o[n] = tot[4 * j + 2 * h + c];
        }
    } else {
      const int plane = MODE == kFwd ? howo : hw;
      const int b = m / plane, p = m - b * plane;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int n = c0 + 8 * j + c;
          if (n >= N) continue;
          float* o = out + ((size_t)b * N + n) * plane + p;
          const float v = tot[4 * j + 2 * h + c];
          *o = (MODE == kDgrad && accumulate) ? *o + v : v;
        }
    }
  }
}

// dw[i] (+)= sum over the partials in order.
__global__ void bb_reduce_kernel(const float* __restrict__ part, int parts, int n, int accumulate,
                                 float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = accumulate ? dw[i] : 0.f;
  for (int p = 0; p < parts; ++p) s += part[(size_t)p * n + i];
  dw[i] = s;
}

// ------------------------------------------------------------------------------------------------
// BatchNorm.  Partials: part[c][b * chunks + chunk][2] (fp64) over kBnChunk pixels of one plane.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double2 block_sum2(double a, double b) {
  __shared__ double red[2][kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[0][w] = a, red[1][w] = b;
  __syncthreads();
  double sa = 0.0, sb = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < kThreads / 32; ++i) sa += red[0][i], sb += red[1][i];
  return make_double2(sa, sb);
}

// grid (chunks, batches, c): sum x and x^2
__global__ void __launch_bounds__(kThreads) bb_bn_stats_part_kernel(const float* __restrict__ x, int c, int hw,
                                                                    double* __restrict__ part) {
  const int chunk = blockIdx.x, b = blockIdx.y, ch = blockIdx.z;
  const float* p = x + ((size_t)b * c + ch) * hw;
  const int e0 = chunk * kBnChunk, e1 = min(e0 + kBnChunk, hw);
  double s = 0.0, ss = 0.0;
  for (int e = e0 + threadIdx.x; e < e1; e += kThreads) {
    const double v = p[e];
    s += v;
    ss += v * v;
  }
  const double2 r = block_sum2(s, ss);
  if (threadIdx.x == 0) {
    double* o = part + ((size_t)ch * gridDim.y * gridDim.x + (size_t)b * gridDim.x + chunk) * 2;
    o[0] = r.x, o[1] = r.y;
  }
}

__global__ void bb_bn_stats_merge_kernel(const double* __restrict__ part, int c, int parts, long long n, float eps,
                                         float* __restrict__ mean, float* __restrict__ invstd,
                                         float* __restrict__ running_mean, float* __restrict__ running_var,
                                         float momentum) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double s = 0.0, ss = 0.0;
  for (int q = 0; q < parts; ++q) s += part[((size_t)ch * parts + q) * 2], ss += part[((size_t)ch * parts + q) * 2 + 1];
  const double mu = s / (double)n;
  const double var = fmax(ss / (double)n - mu * mu, 0.0);
  mean[ch] = (float)mu;
  invstd[ch] = (float)(1.0 / sqrt(var + (double)eps));
  if (running_mean) {
    const double m = momentum;
    running_mean[ch] = (float)((1.0 - m) * running_mean[ch] + m * mu);
    running_var[ch] = (float)((1.0 - m) * running_var[ch] + m * var * (double)n / (double)(n - 1));
  }
}

__device__ __forceinline__ float act_grad(int act, const float* y, size_t i) {
  if (act == kActNone) return 1.f;
  return y[i] > 0.f ? 1.f : (act == kActLeaky ? kLeakySlope : 0.f);
}

// y = act(gamma (x - mean) invstd + beta [+ res]); y may alias x or res
__global__ void bb_bn_act_kernel(const float* x, int c, int hw, long long total, const float* __restrict__ mean,
                                 const float* __restrict__ invstd, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, const float* res, int act, float* y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)((i / hw) % c);
  float z = fmaf(gamma[ch], (x[i] - mean[ch]) * invstd[ch], beta[ch]);
  if (res) z += res[i];
  if (act == kActRelu) z = fmaxf(z, 0.f);
  if (act == kActLeaky) z = z > 0.f ? z : z * kLeakySlope;
  y[i] = z;
}

// grid (chunks, batches, c): sum dz and dz·xhat, dz = dy·act'(y)
__global__ void __launch_bounds__(kThreads) bb_bn_bwd_part_kernel(const float* __restrict__ x,
                                                                  const float* __restrict__ y,
                                                                  const float* __restrict__ dy, int c, int hw,
                                                                  const float* __restrict__ mean,
                                                                  const float* __restrict__ invstd, int act,
                                                                  double* __restrict__ part) {
  const int chunk = blockIdx.x, b = blockIdx.y, ch = blockIdx.z;
  const size_t base = ((size_t)b * c + ch) * hw;
  const int e0 = chunk * kBnChunk, e1 = min(e0 + kBnChunk, hw);
  const float mu = mean[ch], r = invstd[ch];
  double s = 0.0, sx = 0.0;
  for (int e = e0 + threadIdx.x; e < e1; e += kThreads) {
    const float dz = dy[base + e] * act_grad(act, y, base + e);
    s += dz;
    sx += (double)dz * (double)((x[base + e] - mu) * r);
  }
  const double2 t = block_sum2(s, sx);
  if (threadIdx.x == 0) {
    double* o = part + ((size_t)ch * gridDim.y * gridDim.x + (size_t)b * gridDim.x + chunk) * 2;
    o[0] = t.x, o[1] = t.y;
  }
}

// dgb[0][c] = dgamma = sum dz·xhat, dgb[1][c] = dbeta = sum dz; coef[c] = (sum dz / n, sum dz·xhat / n)
__global__ void bb_bn_bwd_merge_kernel(const double* __restrict__ part, int c, int parts, long long n,
                                       float* __restrict__ dgb, float* __restrict__ coef) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  if (ch >= c) return;
  double s = 0.0, sx = 0.0;
  for (int q = 0; q < parts; ++q) s += part[((size_t)ch * parts + q) * 2], sx += part[((size_t)ch * parts + q) * 2 + 1];
  dgb[ch] = (float)sx;
  dgb[c + ch] = (float)s;
  coef[2 * ch] = (float)(s / (double)n);
  coef[2 * ch + 1] = (float)(sx / (double)n);
}

// dx = gamma invstd (dz - sum dz / n - xhat sum(dz xhat) / n) (batch statistics) or gamma invstd dz;
// dres = dz.  dx may alias dy.
__global__ void bb_bn_bwd_dx_kernel(const float* x, const float* y, const float* dy, int c, int hw, long long total,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ gamma, const float* __restrict__ coef, int act,
                                    int batch_stats, float* dx, float* dres) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)((i / hw) % c);
  const float dz = dy[i] * act_grad(act, y, i);
  const float r = invstd[ch];
  float g = dz;
  if (batch_stats) g = dz - coef[2 * ch] - (x[i] - mean[ch]) * r * coef[2 * ch + 1];
  if (dres) dres[i] = dz;
  dx[i] = gamma[ch] * r * g;
}

// ------------------------------------------------------------------------------------------------
// Bilinear x2 upsample, align_corners=True, with ATen's fp32 source index:
// scale = (in - 1) / (out - 1), src = scale·dst, i0 = (int)src, i1 = i0 + (i0 < in - 1), l = src - i0.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void up_src(int dst, int n_in, float scale, int& i0, int& i1, float& l1) {
  const float src = scale * (float)dst;
  i0 = (int)src;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = src - (float)i0;
}

__device__ __forceinline__ float up_scale(int n_in) { return n_in > 1 ? (float)(n_in - 1) / (float)(2 * n_in - 1) : 0.f; }

// out[b][c][Y][X] = lat + up(in); in [B][C][h][w], lat / out [B][C][2h][2w]; out may alias lat
__global__ void bb_up2x_add_kernel(const float* __restrict__ in, const float* lat, int h, int w, long long total,
                                   float* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int W2 = 2 * w, H2 = 2 * h;
  const int X = (int)(i % W2), Y = (int)((i / W2) % H2);
  const long long bc = i / ((long long)W2 * H2);
  int y0, y1, x0, x1;
  float ly, lx;
  up_src(Y, h, up_scale(h), y0, y1, ly);
  up_src(X, w, up_scale(w), x0, x1, lx);
  const float* p = in + bc * h * w;
  const float v = (1.f - ly) * ((1.f - lx) * p[y0 * w + x0] + lx * p[y0 * w + x1]) +
                  ly * ((1.f - lx) * p[y1 * w + x0] + lx * p[y1 * w + x1]);
  out[i] = lat[i] + v;
}

// The weight with which output position d (along one axis) reads input position i: 0 unless i is one of
// d's two source positions; both when i0 == i1 (the last input position).
__device__ __forceinline__ float up_weight(int d, int i, int n_in, float scale) {
  int i0, i1;
  float l1;
  up_src(d, n_in, scale, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}

// din[b][c][y][x] (+)= sum over the output pixels that read it of weight·dout.  1/scale > 2 bounds the
// output positions that read input position i to [2i - 2, 2i + 3]; the scan covers [2i - 3, 2i + 4].
__global__ void bb_up2x_bwd_kernel(const float* __restrict__ dout, int h, int w, long long total, int accumulate,
                                   float* __restrict__ din) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int xx = (int)(i % w), yy = (int)((i / w) % h);
  const long long bc = i / ((long long)w * h);
  const float sy = up_scale(h), sx = up_scale(w);
  const int y_lo = max(0, 2 * yy - 3), y_hi = min(2 * h - 1, 2 * yy + 4);
  const int x_lo = max(0, 2 * xx - 3), x_hi = min(2 * w - 1, 2 * xx + 4);
  const float* d = dout + bc * 4 * h * w;
  float acc = 0.f;
  for (int oy = y_lo; oy <= y_hi; ++oy) {
    const float wy = up_weight(oy, yy, h, sy);
    if (wy == 0.f) continue;
    float row = 0.f;
    for (int ox = x_lo; ox <= x_hi; ++ox) {
      const float wx = up_weight(ox, xx, w, sx);
      if (wx != 0.f) row += wx * d[oy * 2 * w + ox];
    }
    acc += wy * row;
  }
  din[i] = accumulate ? din[i] + acc : acc;
}

int conv_geo(int batches, int c_in, int h, int w, int c_out, int ksize, int stride, ConvGeo& g) {
  OPP_REQUIRE(batches > 0 && c_in > 0 && h > 0 && w > 0 && c_out > 0, "opp_backbone_train_conv*: bad shape");
  OPP_REQUIRE(ksize == 1 || ksize == 3 || ksize == 7, "opp_backbone_train_conv*: kernel size %d not built", ksize);
  OPP_REQUIRE(stride == 1 || stride == 2, "opp_backbone_train_conv*: stride %d not built", stride);
  g.batches = batches, g.c_in = c_in, g.h = h, g.w = w, g.c_out = c_out, g.stride = stride, g.pad = ksize / 2;
  g.ho = (h + 2 * g.pad - ksize) / stride + 1;
  g.wo = (w + 2 * g.pad - ksize) / stride + 1;
  const long long big = (long long)batches * (c_in > c_out ? c_in : c_out) * h * w;
  OPP_REQUIRE(big < (1LL << 31) && (long long)c_in * ksize * ksize * c_out < (1LL << 31),
              "opp_backbone_train_conv*: tensor too large");
  return OPP_OK;
}

template <int MODE, int KS>
cudaError_t launch_ks(dim3 grid, cudaStream_t st, const float* x, const float* w, const float* dy, const ConvGeo& g,
                      int pix0, int npix, int accumulate, float* out) {
  static const cudaError_t attr =
      cudaFuncSetAttribute(bb_conv_kernel<MODE, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  if (attr != cudaSuccess) return attr;
  bb_conv_kernel<MODE, KS><<<grid, kThreads, kSmem, st>>>(x, w, dy, g, pix0, npix, accumulate, out);
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_conv(int ksize, dim3 grid, cudaStream_t st, const float* x, const float* w, const float* dy,
                        const ConvGeo& g, int pix0, int npix, int accumulate, float* out) {
  if (ksize == 1) return launch_ks<MODE, 1>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
  if (ksize == 3) return launch_ks<MODE, 3>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
  return launch_ks<MODE, 7>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
}

int bn_parts(int batches, int hw) { return batches * ((hw + kBnChunk - 1) / kBnChunk); }

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" {

int opp_backbone_train_wgrad_group(void) { return kWgradGroup; }

int opp_backbone_train_bn_parts(int batches, int hw) { return bn_parts(batches, hw); }

int opp_backbone_train_conv(const float* x, const float* w, int batches, int c_in, int h, int wd, int c_out, int ksize,
                            int stride, float* y, opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(x && w && y, "opp_backbone_train_conv: null pointer");
  const int M = batches * g.ho * g.wo;
  const dim3 grid((c_out + kBN - 1) / kBN, (M + kBM - 1) / kBM);
  OPP_CHECK_CUDA(launch_conv<kFwd>(ksize, grid, (cudaStream_t)stream, x, w, nullptr, g, 0, 0, 0, y));
  return OPP_OK;
}

int opp_backbone_train_conv_dgrad(const float* dy, const float* w, int batches, int c_in, int h, int wd, int c_out,
                                  int ksize, int stride, float* dx, int accumulate, opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(dy && w && dx, "opp_backbone_train_conv_dgrad: null pointer");
  const int M = batches * h * wd;
  const dim3 grid((c_in + kBN - 1) / kBN, (M + kBM - 1) / kBM);
  OPP_CHECK_CUDA(launch_conv<kDgrad>(ksize, grid, (cudaStream_t)stream, nullptr, w, dy, g, 0, 0, accumulate, dx));
  return OPP_OK;
}

int opp_backbone_train_conv_wgrad(const float* x, const float* dy, int batches, int c_in, int h, int wd, int c_out,
                                  int ksize, int stride, int pix0, int npix, float* part, float* dw, int accumulate,
                                  opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(x && dy && part && dw, "opp_backbone_train_conv_wgrad: null pointer");
  const int pixels = batches * g.ho * g.wo;
  OPP_REQUIRE(pix0 >= 0 && npix > 0 && pix0 % kWgradGroup == 0 && pix0 + npix <= pixels,
              "opp_backbone_train_conv_wgrad: pixel slice [%d, %d) of %d", pix0, pix0 + npix, pixels);
  const int groups = (npix + kWgradGroup - 1) / kWgradGroup;
  const int N = c_in * ksize * ksize;
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((N + kBN - 1) / kBN, (c_out + kBM - 1) / kBM, groups);
  OPP_CHECK_CUDA(launch_conv<kWgrad>(ksize, grid, st, x, nullptr, dy, g, pix0, npix, 0, part));
  bb_reduce_kernel<<<(c_out * N + 255) / 256, 256, 0, st>>>(part, groups, c_out * N, accumulate, dw);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_backbone_train_bn_stats(const float* x, int batches, int c, int hw, float eps, double* part, float* mean,
                                float* invstd, float* running_mean, float* running_var, float momentum,
                                opp_stream_t stream) {
  OPP_REQUIRE(x && part && mean && invstd && batches > 0 && c > 0 && hw > 0, "opp_backbone_train_bn_stats: bad arguments");
  OPP_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "opp_backbone_train_bn_stats: running_mean and "
              "running_var go together");
  const long long n = (long long)batches * hw;
  OPP_REQUIRE(!running_mean || n > 1, "opp_backbone_train_bn_stats: the running variance needs more than 1 value");
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = (hw + kBnChunk - 1) / kBnChunk;
  bb_bn_stats_part_kernel<<<dim3(chunks, batches, c), kThreads, 0, st>>>(x, c, hw, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  bb_bn_stats_merge_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, c, bn_parts(batches, hw), n, eps, mean, invstd,
                                                          running_mean, running_var, momentum);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_backbone_train_bn_act(const float* x, int batches, int c, int hw, const float* mean, const float* invstd,
                              const float* gamma, const float* beta, const float* res, int act, float* y,
                              opp_stream_t stream) {
  OPP_REQUIRE(x && mean && invstd && gamma && beta && y && batches > 0 && c > 0 && hw > 0 && act >= 0 && act <= 2,
              "opp_backbone_train_bn_act: bad arguments");
  const long long total = (long long)batches * c * hw;
  bb_bn_act_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, c, hw, total, mean, invstd,
                                                                                      gamma, beta, res, act, y);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_backbone_train_bn_act_bwd(const float* x, const float* y, const float* dy, int batches, int c, int hw,
                                  const float* mean, const float* invstd, const float* gamma, int act,
                                  int batch_stats, double* part, float* dx, float* dres, float* dgb,
                                  opp_stream_t stream) {
  OPP_REQUIRE(x && dy && mean && invstd && gamma && part && dx && dgb && batches > 0 && c > 0 && hw > 0 &&
                  act >= 0 && act <= 2 && (act == kActNone || y),
              "opp_backbone_train_bn_act_bwd: bad arguments");
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = (hw + kBnChunk - 1) / kBnChunk, parts = bn_parts(batches, hw);
  const long long n = (long long)batches * hw, total = n * c;
  float* coef = reinterpret_cast<float*>(part + (size_t)c * parts * 2);      // [c][2] after the partials
  bb_bn_bwd_part_kernel<<<dim3(chunks, batches, c), kThreads, 0, st>>>(x, y, dy, c, hw, mean, invstd, act, part);
  OPP_CHECK_CUDA(cudaGetLastError());
  bb_bn_bwd_merge_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, c, parts, n, dgb, coef);
  OPP_CHECK_CUDA(cudaGetLastError());
  bb_bn_bwd_dx_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, dy, c, hw, total, mean, invstd, gamma,
                                                                      coef, act, batch_stats, dx, dres);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_backbone_train_up2x_add(const float* in, const float* lat, int batches, int c, int h, int w, float* out,
                                opp_stream_t stream) {
  OPP_REQUIRE(in && lat && out && batches > 0 && c > 0 && h > 0 && w > 0, "opp_backbone_train_up2x_add: bad arguments");
  const long long total = (long long)batches * c * 4 * h * w;
  bb_up2x_add_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, lat, h, w, total, out);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_backbone_train_up2x_bwd(const float* dout, int batches, int c, int h, int w, float* din, int accumulate,
                                opp_stream_t stream) {
  OPP_REQUIRE(dout && din && batches > 0 && c > 0 && h > 0 && w > 0, "opp_backbone_train_up2x_bwd: bad arguments");
  const long long total = (long long)batches * c * h * w;
  bb_up2x_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dout, h, w, total,
                                                                                       accumulate, din);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
