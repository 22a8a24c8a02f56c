// opp_sfm_refine.cu — the device parts of the keypoint-free SfM refinement that the reference runs in
// Python (src/KeypointFreeSfM/loftr_for_sfm/utils/sample_feature_from_featuremap.py and
// src/KeypointFreeSfM/post_optimization/feature_aggregation.py:10-180).
//
//   sample     sample_feature_from_featuremap at keypoints: coord_normalization in the keypoints'
//              own type (fp32 or fp64: (k - 0.5) + 0.5, / (size - 1), * 2 - 1), rounded to fp32,
//              then grid_sample(align_corners=True, zeros padding) in fp32: un-normalise to
//              (g + 1) * ((n - 1) / 2), then nearest (round half to even) or bilinear with the four
//              weights (1-n)(1-w), (1-n)w, n(1-w), nw summed nw, ne, sw, se.  Every operation is
//              one IEEE rounding (no FMA contraction).  Taps outside the map read 0.  The map is the
//              engine's NHWC fp16 store, hi plane then lo plane when split: value = hi + lo in fp32.
//   lookup     (pair, mkpts0_idx) -> row: a binary search of each query key in the sorted row keys
//              (torch.sort outside this file), -1 when absent, -2 when the key repeats.
//   aggregate  one CTA per track: the rows of its members summed in fp32 in member order, then
//              divided by the count (np.mean(axis=0) of float32 rows, bit for bit), and the other
//              side's row of every member copied out.
// No floating-point atomics: two runs give the same bits.
#include <cstdint>

#include <cuda_fp16.h>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kThreads = 128;
constexpr int kLookupThreads = 256;

__device__ __forceinline__ float map_at(const __half* px, int c, int lo_off) {
  float v = __half2float(px[c]);
  if (lo_off) v = __fadd_rn(v, __half2float(px[lo_off + c]));
  return v;
}

template <typename T>
__device__ __forceinline__ float normalise(T k, float size) {
  // coord_normalization(k, h, w): (k - 1/2 + 0.5) / (size - 1) * 2 - 1 in k's type, then .float()
  const T r = (T)(size - 1.0f);
  T v;
  if constexpr (sizeof(T) == 8) {
    v = __dadd_rn(__dsub_rn(k, 0.5), 0.5);
    v = __ddiv_rn(v, r);
    v = __dsub_rn(__dmul_rn(v, 2.0), 1.0);
    return __double2float_rn(v);
  } else {
    v = __fadd_rn(__fsub_rn(k, 0.5f), 0.5f);
    v = __fdiv_rn(v, r);
    return __fsub_rn(__fmul_rn(v, 2.0f), 1.0f);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
sample_kernel(const __half* __restrict__ map, const long long* __restrict__ img, const T* __restrict__ kpts,
              const float* __restrict__ imghw, int hm, int wm, int channels, int lo_off, int nearest,
              float* __restrict__ out) {
  const long long p = blockIdx.x;
  const long long b = img ? img[p] : 0;
  const float gx = normalise<T>(kpts[2 * p], imghw[2 * b + 1]);
  const float gy = normalise<T>(kpts[2 * p + 1], imghw[2 * b]);
  const float ix = __fmul_rn(__fadd_rn(gx, 1.0f), (float)(wm - 1) * 0.5f);
  const float iy = __fmul_rn(__fadd_rn(gy, 1.0f), (float)(hm - 1) * 0.5f);
  const int ld = lo_off ? 2 * channels : channels;
  const __half* base = map + b * hm * (long long)wm * ld;
  float* o = out + p * channels;
  if (nearest) {
    const float xr = rintf(ix), yr = rintf(iy);
    const bool in = xr >= 0.f && xr <= (float)(wm - 1) && yr >= 0.f && yr <= (float)(hm - 1);
    const __half* px = in ? base + ((long long)yr * wm + (long long)xr) * ld : nullptr;
    for (int c = threadIdx.x; c < channels; c += kThreads) o[c] = in ? map_at(px, c, lo_off) : 0.f;
    return;
  }
  const float xw = floorf(ix), yn = floorf(iy);
  const float w = __fsub_rn(ix, xw), e = __fsub_rn(1.0f, w);
  const float n = __fsub_rn(iy, yn), s = __fsub_rn(1.0f, n);
  const float wnw = __fmul_rn(s, e), wne = __fmul_rn(s, w), wsw = __fmul_rn(n, e), wse = __fmul_rn(n, w);
  const bool xin0 = xw > -1.f && xw < (float)wm, xin1 = xw + 1.f > -1.f && xw + 1.f < (float)wm;
  const bool yin0 = yn > -1.f && yn < (float)hm, yin1 = yn + 1.f > -1.f && yn + 1.f < (float)hm;
  const long long x0 = xin0 || xin1 ? (long long)xw : 0, y0 = yin0 || yin1 ? (long long)yn : 0;
  const __half* pnw = base + (y0 * wm + x0) * ld;
  const __half* pne = pnw + ld;
  const __half* psw = pnw + (long long)wm * ld;
  const __half* pse = psw + ld;
  for (int c = threadIdx.x; c < channels; c += kThreads) {
    const float vnw = yin0 && xin0 ? map_at(pnw, c, lo_off) : 0.f;
    const float vne = yin0 && xin1 ? map_at(pne, c, lo_off) : 0.f;
    const float vsw = yin1 && xin0 ? map_at(psw, c, lo_off) : 0.f;
    const float vse = yin1 && xin1 ? map_at(pse, c, lo_off) : 0.f;
    float acc = __fadd_rn(__fmul_rn(vnw, wnw), __fmul_rn(vne, wne));
    acc = __fadd_rn(acc, __fmul_rn(vsw, wsw));
    o[c] = __fadd_rn(acc, __fmul_rn(vse, wse));
  }
}

__global__ void __launch_bounds__(kLookupThreads)
lookup_kernel(const long long* __restrict__ sorted_key, const long long* __restrict__ perm, long long n,
              const long long* __restrict__ query, long long q, long long* __restrict__ row) {
  const long long t = (long long)blockIdx.x * kLookupThreads + threadIdx.x;
  if (t >= q) return;
  const long long k = query[t];
  long long lo = 0, hi = n;            // the first sorted key >= k
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (sorted_key[mid] < k) lo = mid + 1; else hi = mid;
  }
  long long r = -1;
  if (lo < n && sorted_key[lo] == k) r = (lo + 1 < n && sorted_key[lo + 1] == k) ? -2 : perm[lo];
  row[t] = r;
}

__global__ void __launch_bounds__(kThreads)
aggregate_kernel(const float* __restrict__ c0, const float* __restrict__ c1, const float* __restrict__ f0,
                 const float* __restrict__ f1, int dc, int df, const long long* __restrict__ row,
                 const long long* __restrict__ track_off, float* __restrict__ mean_c, float* __restrict__ mean_f,
                 float* __restrict__ ref_c, float* __restrict__ ref_f) {
  const long long t = blockIdx.x;
  const long long s = track_off[t], e = track_off[t + 1];
  const float cnt = (float)(e - s);
  for (int c = threadIdx.x; c < dc; c += kThreads) {
    float acc = c0[row[s] * dc + c];
    ref_c[s * dc + c] = c1[row[s] * dc + c];
    for (long long k = s + 1; k < e; ++k) {
      acc = __fadd_rn(acc, c0[row[k] * dc + c]);
      ref_c[k * dc + c] = c1[row[k] * dc + c];
    }
    mean_c[t * dc + c] = __fdiv_rn(acc, cnt);
  }
  for (int c = threadIdx.x; c < df; c += kThreads) {
    float acc = f0[row[s] * df + c];
    ref_f[s * df + c] = f1[row[s] * df + c];
    for (long long k = s + 1; k < e; ++k) {
      acc = __fadd_rn(acc, f0[row[k] * df + c]);
      ref_f[k * df + c] = f1[row[k] * df + c];
    }
    mean_f[t * df + c] = __fdiv_rn(acc, cnt);
  }
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" int opp_sample_feature(const void* map, const long long* img, const void* kpts, int kpts_f64, long long n,
                                  int hm, int wm, int channels, int split, const float* imghw, int nearest,
                                  float* out, opp_stream_t stream) {
  if (n == 0) return OPP_OK;
  OPP_REQUIRE(n > 0 && n < INT32_MAX && hm > 0 && wm > 0 && channels > 0 && channels <= 1024,
              "opp_sample_feature: bad shape n=%lld map %dx%dx%d", n, hm, wm, channels);
  OPP_REQUIRE(map && kpts && imghw && out, "opp_sample_feature: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const int lo_off = split ? channels : 0;
  if (kpts_f64)
    sample_kernel<double><<<(unsigned)n, kThreads, 0, st>>>((const __half*)map, img, (const double*)kpts, imghw, hm,
                                                           wm, channels, lo_off, nearest, out);
  else
    sample_kernel<float><<<(unsigned)n, kThreads, 0, st>>>((const __half*)map, img, (const float*)kpts, imghw, hm,
                                                          wm, channels, lo_off, nearest, out);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_refine_lookup(const long long* sorted_key, const long long* perm, long long n,
                                     const long long* query, long long q, long long* row, opp_stream_t stream) {
  if (q == 0) return OPP_OK;
  OPP_REQUIRE(n > 0 && q > 0, "opp_sfm_refine_lookup: bad shape n=%lld q=%lld", n, q);
  OPP_REQUIRE(sorted_key && perm && query && row, "opp_sfm_refine_lookup: null pointer");
  lookup_kernel<<<(unsigned)((q + kLookupThreads - 1) / kLookupThreads), kLookupThreads, 0, (cudaStream_t)stream>>>(
      sorted_key, perm, n, query, q, row);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_refine_aggregate(const float* c0, const float* c1, const float* f0, const float* f1, int dc,
                                        int df, const long long* row, const long long* track_off, int tracks,
                                        float* mean_c, float* mean_f, float* ref_c, float* ref_f,
                                        opp_stream_t stream) {
  if (tracks == 0) return OPP_OK;
  OPP_REQUIRE(tracks > 0 && dc > 0 && df > 0, "opp_sfm_refine_aggregate: bad shape T=%d dc=%d df=%d", tracks, dc, df);
  OPP_REQUIRE(c0 && c1 && f0 && f1 && row && track_off && mean_c && mean_f && ref_c && ref_f,
              "opp_sfm_refine_aggregate: null pointer");
  aggregate_kernel<<<(unsigned)tracks, kThreads, 0, (cudaStream_t)stream>>>(c0, c1, f0, f1, dc, df, row, track_off,
                                                                           mean_c, mean_f, ref_c, ref_f);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
