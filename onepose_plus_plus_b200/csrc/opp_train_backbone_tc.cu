// opp_train_backbone_tc.cu — the backbone's convolution forward, data gradient and weight gradient on
// the tensor cores in 3xTF32 (model.backbone_train_mode "tf32x3", DESIGN §7 f4).
//
// The three passes are the implicit GEMMs of opp_train_backbone.cu, with the same gather rules:
//   forward  out[p][co]     = sum_{ci,tap} x(p, ci, tap)  W[co][ci][tap]     M = output pixels, N = c_out
//   dgrad    dx[q][ci]      = sum_{co,tap} dy(q, co, tap) W[co][ci][tap]     M = input pixels,  N = c_in
//   wgrad    dW[co][ci,tap] = sum_p        dy[p][co]      x(p, ci, tap)      M = c_out, N = c_in·k², K = pixels
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
// wgrad sums output pixels in groups of kWgradGroup (as opp_train_backbone.cu): each CTA writes one
// partial, and a reduce adds the partials in group order.  No floating-point atomics: two calls give
// the same bits.
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

enum { kFwd = 0, kDgrad = 1, kWgrad = 2 };

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
__global__ void __launch_bounds__(kThreads, 2) bb_tc_conv_kernel(const float* __restrict__ x,
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
__global__ void bb_tc_reduce_kernel(const float* __restrict__ part, int parts, int n, int accumulate,
                                    float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = accumulate ? dw[i] : 0.f;
  for (int p = 0; p < parts; ++p) s += part[(size_t)p * n + i];
  dw[i] = s;
}

int conv_geo(int batches, int c_in, int h, int w, int c_out, int ksize, int stride, ConvGeo& g) {
  OPP_REQUIRE(batches > 0 && c_in > 0 && h > 0 && w > 0 && c_out > 0, "opp_backbone_train_conv*_tf32x3: bad shape");
  OPP_REQUIRE(ksize == 1 || ksize == 3 || ksize == 7, "opp_backbone_train_conv*_tf32x3: kernel size %d not built",
              ksize);
  OPP_REQUIRE(stride == 1 || stride == 2, "opp_backbone_train_conv*_tf32x3: stride %d not built", stride);
  g.batches = batches, g.c_in = c_in, g.h = h, g.w = w, g.c_out = c_out, g.stride = stride, g.pad = ksize / 2;
  g.ho = (h + 2 * g.pad - ksize) / stride + 1;
  g.wo = (w + 2 * g.pad - ksize) / stride + 1;
  const long long big = (long long)batches * (c_in > c_out ? c_in : c_out) * h * w;
  OPP_REQUIRE(big < (1LL << 31) && (long long)c_in * ksize * ksize * c_out < (1LL << 31),
              "opp_backbone_train_conv*_tf32x3: tensor too large");
  return OPP_OK;
}

template <int MODE, int KS>
cudaError_t launch_ks(dim3 grid, cudaStream_t st, const float* x, const float* w, const float* dy, const ConvGeo& g,
                      int pix0, int npix, int accumulate, float* out) {
  static const cudaError_t attr =
      cudaFuncSetAttribute(bb_tc_conv_kernel<MODE, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  if (attr != cudaSuccess) return attr;
  bb_tc_conv_kernel<MODE, KS><<<grid, kThreads, kSmem, st>>>(x, w, dy, g, pix0, npix, accumulate, out);
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_conv(int ksize, dim3 grid, cudaStream_t st, const float* x, const float* w, const float* dy,
                        const ConvGeo& g, int pix0, int npix, int accumulate, float* out) {
  if (ksize == 1) return launch_ks<MODE, 1>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
  if (ksize == 3) return launch_ks<MODE, 3>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
  return launch_ks<MODE, 7>(grid, st, x, w, dy, g, pix0, npix, accumulate, out);
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" {

int opp_backbone_train_conv_tf32x3(const float* x, const float* w, int batches, int c_in, int h, int wd, int c_out,
                                   int ksize, int stride, float* y, opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(x && w && y, "opp_backbone_train_conv_tf32x3: null pointer");
  const int M = batches * g.ho * g.wo;
  const dim3 grid((c_out + kBN - 1) / kBN, (M + kBM - 1) / kBM);
  OPP_CHECK_CUDA(launch_conv<kFwd>(ksize, grid, (cudaStream_t)stream, x, w, nullptr, g, 0, 0, 0, y));
  return OPP_OK;
}

int opp_backbone_train_conv_dgrad_tf32x3(const float* dy, const float* w, int batches, int c_in, int h, int wd,
                                         int c_out, int ksize, int stride, float* dx, int accumulate,
                                         opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(dy && w && dx, "opp_backbone_train_conv_dgrad_tf32x3: null pointer");
  const int M = batches * h * wd;
  const dim3 grid((c_in + kBN - 1) / kBN, (M + kBM - 1) / kBM);
  OPP_CHECK_CUDA(launch_conv<kDgrad>(ksize, grid, (cudaStream_t)stream, nullptr, w, dy, g, 0, 0, accumulate, dx));
  return OPP_OK;
}

int opp_backbone_train_conv_wgrad_tf32x3(const float* x, const float* dy, int batches, int c_in, int h, int wd,
                                         int c_out, int ksize, int stride, int pix0, int npix, float* part,
                                         float* dw, int accumulate, opp_stream_t stream) {
  ConvGeo g;
  if (int e = conv_geo(batches, c_in, h, wd, c_out, ksize, stride, g)) return e;
  OPP_REQUIRE(x && dy && part && dw, "opp_backbone_train_conv_wgrad_tf32x3: null pointer");
  const int pixels = batches * g.ho * g.wo;
  OPP_REQUIRE(pix0 >= 0 && npix > 0 && pix0 % kWgradGroup == 0 && pix0 + npix <= pixels,
              "opp_backbone_train_conv_wgrad_tf32x3: pixel slice [%d, %d) of %d", pix0, pix0 + npix, pixels);
  const int groups = (npix + kWgradGroup - 1) / kWgradGroup;
  const int N = c_in * ksize * ksize;
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((N + kBN - 1) / kBN, (c_out + kBM - 1) / kBM, groups);
  OPP_CHECK_CUDA(launch_conv<kWgrad>(ksize, grid, st, x, nullptr, dy, g, pix0, npix, 0, part));
  bb_tc_reduce_kernel<<<(c_out * N + 255) / 256, 256, 0, st>>>(part, groups, c_out * N, accumulate, dw);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
