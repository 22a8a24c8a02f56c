// opp_sfm_points.cu — the 2D keypoint merge of the keypoint-free SfM coarse matching on the device
// (reference: points2D_worker / agg_groupby_2d(..., agg="sum") / update_matches / transform_points2D,
// src/KeypointFreeSfM/coarse_match/coarse_match_worker.py:81-175 and coarse_match/utils.py:5-60).
//
// Input: the raw matches of P pairs flattened, fp32 [M][5] = (x0, y0, x1, y1, mconf), pair p owns
// [offsets[p], offsets[p + 1]) and names the images pair_img[p][0], pair_img[p][1].
//
//   emit      one thread per match writes its two endpoints at their appearance index
//             a = 2 offsets[p] + side * M_p + m: pair position, then side, then match — the order in
//             which Match2Pts2D concatenates an image's observations (a pair that names one image
//             twice lists side 0 before side 1).  key = image << 42 | x << 21 | y with (x, y) truncated
//             toward zero (.astype(int)); the host checks 0 <= x, y < 2^21 and images <= 2^20.
//   sort      a stable device sort of the keys (torch.sort, outside this file) keeps each group in
//             appearance order.
//   segments  head flags, per-CTA counts, one CTA's scan of the counts, then the heads' positions.
//   sums      one thread per group sums its confidences in fp64 in sorted order — np.bincount's
//             sequential sum, bit for bit — and writes the descending-sum rank key -bits(sum)
//             (sums are >= 0, so the bits order like the values) and the groups' image offsets.
//   rank      after two stable sorts (rank key, then image id; outside this file) an image's groups
//             are in descending-sum order with ties in np.unique's ascending (x, y) order, which is
//             where Python's stable sorted(reverse=True) leaves them.  Writes keypoints / scores
//             fp32 in id order and the group -> id map.
//   remap     one thread per match finds its two keys in their images' unique keys (binary search)
//             and writes [id0, id1].
// No floating-point atomics: two runs give the same bits.
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kXYBits = 21;
constexpr int kImageShift = 2 * kXYBits;
constexpr long long kXYMask = (1ll << kXYBits) - 1;

__device__ __forceinline__ int pair_of(const long long* offsets, int pairs, long long t) {
  int lo = 0, hi = pairs - 1;          // the last pair whose range starts at or before t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ long long pack_key(int image, float x, float y) {
  return ((long long)image << kImageShift) | ((long long)__float2int_rz(x) << kXYBits) | (long long)__float2int_rz(y);
}

__global__ void __launch_bounds__(kThreads)
emit_kernel(const float* __restrict__ matches, long long m, const long long* __restrict__ offsets,
            const int* __restrict__ pair_img, int pairs, long long* __restrict__ key, float* __restrict__ conf) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= m) return;
  const int p = pair_of(offsets, pairs, t);
  const long long o = offsets[p], mp = offsets[p + 1] - o;
  const float* r = matches + t * 5;
  const long long a0 = 2 * o + (t - o), a1 = a0 + mp;
  key[a0] = pack_key(pair_img[2 * p], r[0], r[1]);
  key[a1] = pack_key(pair_img[2 * p + 1], r[2], r[3]);
  conf[a0] = r[4];
  conf[a1] = r[4];
}

__device__ __forceinline__ bool is_head(const long long* sorted_key, long long n, long long j) {
  return j < n && (j == 0 || sorted_key[j] != sorted_key[j - 1]);
}

__global__ void __launch_bounds__(kScanThreads)
head_count_kernel(const long long* __restrict__ sorted_key, long long n, int* __restrict__ block_count) {
  const long long j = (long long)blockIdx.x * kScanThreads + threadIdx.x;
  const int c = __syncthreads_count(is_head(sorted_key, n, j));
  if (threadIdx.x == 0) block_count[blockIdx.x] = c;
}

// Block-wide exclusive prefix of one flag per thread; *total receives the CTA's sum.
__device__ __forceinline__ int block_exclusive(int v, int* warp_sum, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) warp_sum[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = warp_sum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    warp_sum[lane] = w;
  }
  __syncthreads();
  const int before = (wid ? warp_sum[wid - 1] : 0) + inc - v;
  *total = warp_sum[kScanThreads / 32 - 1];
  __syncthreads();
  return before;
}

// One CTA: block_count -> exclusive offsets in place; start[groups] = n, *groups_out = groups.
__global__ void __launch_bounds__(kScanThreads)
scan_counts_kernel(int* __restrict__ block_count, int blocks, long long n, int* __restrict__ start,
                   int* __restrict__ groups_out) {
  __shared__ int warp_sum[kScanThreads / 32];
  int base = 0;
  for (int b0 = 0; b0 < blocks; b0 += kScanThreads) {
    const int b = b0 + threadIdx.x;
    const int v = b < blocks ? block_count[b] : 0;
    int total;
    const int before = block_exclusive(v, warp_sum, &total);
    if (b < blocks) block_count[b] = base + before;
    base += total;
  }
  if (threadIdx.x == 0) {
    start[base] = (int)n;
    *groups_out = base;
  }
}

__global__ void __launch_bounds__(kScanThreads)
head_write_kernel(const long long* __restrict__ sorted_key, long long n, const int* __restrict__ block_base,
                  int* __restrict__ start) {
  __shared__ int warp_sum[kScanThreads / 32];
  const long long j = (long long)blockIdx.x * kScanThreads + threadIdx.x;
  const bool h = is_head(sorted_key, n, j);
  int total;
  const int before = block_exclusive(h ? 1 : 0, warp_sum, &total);
  if (h) start[block_base[blockIdx.x] + before] = (int)j;
}

__global__ void __launch_bounds__(kThreads)
sums_kernel(const long long* __restrict__ sorted_key, const long long* __restrict__ perm,
            const float* __restrict__ conf, const int* __restrict__ start, int groups, int images,
            long long* __restrict__ ukey, double* __restrict__ sum, long long* __restrict__ rank_key,
            long long* __restrict__ img_off) {
  const int g = blockIdx.x * kThreads + threadIdx.x;
  if (g >= groups) return;
  const int s = start[g], e = start[g + 1];
  double acc = 0.0;
  for (int j = s; j < e; ++j) acc += (double)conf[perm[j]];
  const long long k = sorted_key[s];
  ukey[g] = k;
  sum[g] = acc;
  rank_key[g] = -__double_as_longlong(acc);
  const int img = (int)(k >> kImageShift);
  const int prev = g ? (int)(sorted_key[start[g - 1]] >> kImageShift) : -1;
  for (int i = prev + 1; i <= img; ++i) img_off[i] = g;     // images without a group start here too
  if (g == groups - 1)
    for (int i = img + 1; i <= images; ++i) img_off[i] = groups;
}

__global__ void __launch_bounds__(kThreads)
image_key_kernel(const long long* __restrict__ ukey, const long long* __restrict__ perm1, int groups,
                 long long* __restrict__ img_key) {
  const int q = blockIdx.x * kThreads + threadIdx.x;
  if (q < groups) img_key[q] = ukey[perm1[q]] >> kImageShift;
}

__global__ void __launch_bounds__(kThreads)
rank_kernel(const long long* __restrict__ ukey, const double* __restrict__ sum, const long long* __restrict__ img_off,
            const long long* __restrict__ perm1, const long long* __restrict__ perm2, int groups,
            float2* __restrict__ kpts, float* __restrict__ scores, long long* __restrict__ id_of) {
  const int q = blockIdx.x * kThreads + threadIdx.x;
  if (q >= groups) return;
  const long long g = perm1[perm2[q]];
  const long long k = ukey[g];
  kpts[q] = make_float2((float)((k >> kXYBits) & kXYMask), (float)(k & kXYMask));
  scores[q] = __double2float_rn(sum[g]);
  id_of[g] = q - img_off[k >> kImageShift];
}

__device__ __forceinline__ long long find_id(const long long* ukey, const long long* img_off,
                                             const long long* id_of, long long k, int* status) {
  const int img = (int)(k >> kImageShift);
  long long lo = img_off[img], hi = img_off[img + 1] - 1;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (ukey[mid] < k) lo = mid + 1; else hi = mid;
  }
  if (lo > hi || ukey[lo] != k) {
    atomicOr(status, 1);
    return -1;
  }
  return id_of[lo];
}

__global__ void __launch_bounds__(kThreads)
remap_kernel(const float* __restrict__ matches, long long m, const long long* __restrict__ offsets,
             const int* __restrict__ pair_img, int pairs, const long long* __restrict__ ukey,
             const long long* __restrict__ img_off, const long long* __restrict__ id_of,
             longlong2* __restrict__ idx, int* __restrict__ status) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= m) return;
  const int p = pair_of(offsets, pairs, t);
  const float* r = matches + t * 5;
  const long long id0 = find_id(ukey, img_off, id_of, pack_key(pair_img[2 * p], r[0], r[1]), status);
  const long long id1 = find_id(ukey, img_off, id_of, pack_key(pair_img[2 * p + 1], r[2], r[3]), status);
  idx[t] = make_longlong2(id0, id1);
}

unsigned blocks_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" int opp_sfm_points_emit(const float* matches, long long m, const long long* offsets, const int* pair_img,
                                   int pairs, long long* key, float* conf, opp_stream_t stream) {
  OPP_REQUIRE(m > 0 && 2 * m < INT32_MAX && pairs > 0, "opp_sfm_points_emit: bad shape M=%lld P=%d", m, pairs);
  OPP_REQUIRE(matches && offsets && pair_img && key && conf, "opp_sfm_points_emit: null pointer");
  emit_kernel<<<blocks_of(m, kThreads), kThreads, 0, (cudaStream_t)stream>>>(matches, m, offsets, pair_img, pairs,
                                                                               key, conf);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_points_segments_scratch(long long n) { return (int)blocks_of(n, kScanThreads); }

extern "C" int opp_sfm_points_segments(const long long* sorted_key, long long n, int* block_scratch, int* start,
                                       int* groups, opp_stream_t stream) {
  OPP_REQUIRE(n > 0 && n < INT32_MAX, "opp_sfm_points_segments: bad length %lld", n);
  OPP_REQUIRE(sorted_key && block_scratch && start && groups, "opp_sfm_points_segments: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = blocks_of(n, kScanThreads);
  head_count_kernel<<<blocks, kScanThreads, 0, st>>>(sorted_key, n, block_scratch);
  OPP_CHECK_CUDA(cudaGetLastError());
  scan_counts_kernel<<<1, kScanThreads, 0, st>>>(block_scratch, (int)blocks, n, start, groups);
  OPP_CHECK_CUDA(cudaGetLastError());
  head_write_kernel<<<blocks, kScanThreads, 0, st>>>(sorted_key, n, block_scratch, start);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_points_sums(const long long* sorted_key, const long long* perm, const float* conf,
                                   const int* start, int groups, int images, long long* ukey, double* sum,
                                   long long* rank_key, long long* img_off, opp_stream_t stream) {
  OPP_REQUIRE(groups > 0 && images > 0 && images <= (1 << 20), "opp_sfm_points_sums: bad shape G=%d I=%d", groups,
              images);
  OPP_REQUIRE(sorted_key && perm && conf && start && ukey && sum && rank_key && img_off,
              "opp_sfm_points_sums: null pointer");
  sums_kernel<<<blocks_of(groups, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      sorted_key, perm, conf, start, groups, images, ukey, sum, rank_key, img_off);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_points_image_key(const long long* ukey, const long long* perm1, int groups, long long* img_key,
                                        opp_stream_t stream) {
  OPP_REQUIRE(groups > 0, "opp_sfm_points_image_key: bad shape G=%d", groups);
  OPP_REQUIRE(ukey && perm1 && img_key, "opp_sfm_points_image_key: null pointer");
  image_key_kernel<<<blocks_of(groups, kThreads), kThreads, 0, (cudaStream_t)stream>>>(ukey, perm1, groups, img_key);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_points_rank(const long long* ukey, const double* sum, const long long* img_off,
                                   const long long* perm1, const long long* perm2, int groups, float* kpts,
                                   float* scores, long long* id_of, opp_stream_t stream) {
  OPP_REQUIRE(groups > 0, "opp_sfm_points_rank: bad shape G=%d", groups);
  OPP_REQUIRE(ukey && sum && img_off && perm1 && perm2 && kpts && scores && id_of, "opp_sfm_points_rank: null pointer");
  rank_kernel<<<blocks_of(groups, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      ukey, sum, img_off, perm1, perm2, groups, reinterpret_cast<float2*>(kpts), scores, id_of);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_sfm_points_remap(const float* matches, long long m, const long long* offsets, const int* pair_img,
                                    int pairs, const long long* ukey, const long long* img_off,
                                    const long long* id_of, long long* idx, int* status, opp_stream_t stream) {
  OPP_REQUIRE(m > 0 && 2 * m < INT32_MAX && pairs > 0, "opp_sfm_points_remap: bad shape M=%lld P=%d", m, pairs);
  OPP_REQUIRE(matches && offsets && pair_img && ukey && img_off && id_of && idx && status,
              "opp_sfm_points_remap: null pointer");
  const cudaStream_t st = (cudaStream_t)stream;
  OPP_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  remap_kernel<<<blocks_of(m, kThreads), kThreads, 0, st>>>(matches, m, offsets, pair_img, pairs, ukey, img_off,
                                                            id_of, reinterpret_cast<longlong2*>(idx), status);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
