// opp_train_batch.cu — the training batch's homography augmentation and its ground-truth
// correspondences, built on the device from the pose (reference: OnePosePlusDataset.read_anno,
// src/datasets/OnePosePlus_dataset.py:341-444, and build_assignmatrix :174-236).
//
// Arithmetic.  fp32, one rounding per operation in the order written below: every product, sum and
// quotient is an explicit __fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn (no FMA contraction) and
// every rounding to the 8-px grid is rintf (half to even, as torch.round and np.round).
// oracle/train_batch.py restates the same operations in NumPy, so the two agree bit for bit.
//
// Per-item parameters (pack fp32 [B][kPack], built on the host from the item's pose, K_crop and
// sampled homography H, 3x3 matrices row-major):
//   R [0, 9), t [9, 12), K [12, 21)    pose_gt[:3, :3], pose_gt[:3, 3], K_crop, as fp32
//   M [21, 30)                         normal_transform_pixel(h, w)^-1 . normalize_homography(H)
//   N [30, 34)                         normal_transform_pixel(h, w): N00, N02, N11, N12
//   A [34, 43)                         normalize_homography(H)^-1 (the image warp's src <- dst)
//   [43]                               1 when the item is warped
//
// Ground truth, one thread per correspondence c (all items flattened, item b owns
// [offsets[b], offsets[b + 1])):
//   project  x = K (R X + t), (x0, x1) / (x2 + 1e-6)  (:342-354); warped items: the point normalised
//            by N, mapped by M, divided by its third coordinate, dropped outside [0, w-1] x [0, h-1]
//            (:372-400).  Round to the 8-px grid, drop cells outside the image (:411-424); the cell
//            (cx, cy) = rint(x / 8) has rank cx * ncy + cy — np.unique's lexicographic row order.
//            cell_owner[b][rank] = atomicMin(c): the first correspondence of the cell survives (:426).
//   survive  each survivor: kp_owner[b][assign0] = atomicMax(rank).  The reference writes the
//            survivors in rank order, so the last writer of a 2D keypoint is its largest rank (:431-433).
//   emit     each survivor reads back its keypoint's stored cell and fine location (those of the
//            winning rank), applies i < L, j = rint(cell / scale * 0.125) and the j > S drop (:195-228),
//            and writes key = ((b L + i) S + j) R + rank (R = ncx * ncy; dropped: INT64_MAX).
// A device sort of the keys (torch.sort, outside this file) orders the list by (b, i, j) with the
// rank as tie-break; opp_train_gt_compact keeps the last entry of each (b, i, j) — a cell written
// twice keeps the later location, as the matrix assignment of :230-231 does.
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kPack = 44;
constexpr int kWarpTx = 32, kWarpTy = 8;
constexpr int kGtThreads = 256;
constexpr int kCompactThreads = 1024;
constexpr long long kDropped = INT64_MAX;

// status bits (status[0]); status[1] = list length
constexpr int kErrCell = 1, kErrAssign2d = 2, kErrAssign3d = 4;

__device__ __forceinline__ float mad3(float a0, float x, float a1, float y, float a2, float z) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, x), __fmul_rn(a1, y)), __fmul_rn(a2, z));
}

// torch.linspace(-1, 1, n)[i]: start + step * i below the halfway index, end - step * (n - 1 - i) above
__device__ __forceinline__ float linspace_pm1(int i, int n) {
  const float step = __fdiv_rn(2.f, (float)(n - 1));
  return i < n / 2 ? __fadd_rn(-1.f, __fmul_rn(step, (float)i)) : __fsub_rn(1.f, __fmul_rn(step, (float)(n - 1 - i)));
}

__device__ __forceinline__ int item_of(const long long* offsets, int batches, long long c) {
  int lo = 0, hi = batches - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= c) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// kornia homography_warp(img, A, (h, w)): grid = meshgrid(linspace(-1, 1)), src = A . (gx, gy, 1),
// (x, y) * (1 / z) (z kept when |z| <= 1e-8), then grid_sample bilinear, zeros, align_corners=False:
// ix = (x + 1) * (w / 2) - 0.5, weights from ix - floor(ix), taps outside the image read 0.
__global__ void __launch_bounds__(kWarpTx * kWarpTy)
homography_warp_kernel(const float* __restrict__ img, const float* __restrict__ pack, int h, int w,
                       float* __restrict__ out) {
  const int u = blockIdx.x * kWarpTx + threadIdx.x, v = blockIdx.y * kWarpTy + threadIdx.y, b = blockIdx.z;
  if (u >= w || v >= h) return;
  const float* p = pack + (size_t)b * kPack;
  const float* src = img + (size_t)b * h * w;
  float val;
  if (p[43] == 0.f) {
    val = src[(size_t)v * w + u];
  } else {
    const float* A = p + 34;
    const float gx = linspace_pm1(u, w), gy = linspace_pm1(v, h);
    const float sx = mad3(A[0], gx, A[1], gy, A[2], 1.f);
    const float sy = mad3(A[3], gx, A[4], gy, A[5], 1.f);
    const float sz = mad3(A[6], gx, A[7], gy, A[8], 1.f);
    const float s = fabsf(sz) > 1e-8f ? __fdiv_rn(1.f, sz) : 1.f;
    const float ix = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(s, sx), 1.f), 0.5f * (float)w), 0.5f);
    const float iy = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(s, sy), 1.f), 0.5f * (float)h), 0.5f);
    val = 0.f;
    // beyond [-1, w] x [-1, h] every tap is outside (and NaN fails the test): 0
    if (ix > -1.f && ix < (float)w && iy > -1.f && iy < (float)h) {
      const float fx = floorf(ix), fy = floorf(iy);
      const int x0 = (int)fx, y0 = (int)fy;
      const float wx = __fsub_rn(ix, fx), ex = __fsub_rn(1.f, wx);
      const float ny = __fsub_rn(iy, fy), sy_ = __fsub_rn(1.f, ny);
      const bool xin0 = x0 >= 0, xin1 = x0 + 1 < w, yin0 = y0 >= 0, yin1 = y0 + 1 < h;
      const float v00 = (xin0 && yin0) ? src[(size_t)y0 * w + x0] : 0.f;
      const float v01 = (xin1 && yin0) ? src[(size_t)y0 * w + x0 + 1] : 0.f;
      const float v10 = (xin0 && yin1) ? src[(size_t)(y0 + 1) * w + x0] : 0.f;
      const float v11 = (xin1 && yin1) ? src[(size_t)(y0 + 1) * w + x0 + 1] : 0.f;
      val = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(sy_, ex), v00), __fmul_rn(__fmul_rn(sy_, wx), v01)),
                                __fmul_rn(__fmul_rn(ny, ex), v10)),
                      __fmul_rn(__fmul_rn(ny, wx), v11));
    }
  }
  out[((size_t)b * h + v) * w + u] = val;
}

struct GtGeom {
  int batches, rows, h, w, w_c, cols, ncx, ncy;
};

__global__ void __launch_bounds__(kGtThreads)
gt_project_kernel(const float* __restrict__ kp3d, const long long* __restrict__ assign, long long n,
                  const long long* __restrict__ offsets, const long long* __restrict__ kp_offsets,
                  const float* __restrict__ pack, GtGeom g, int* __restrict__ cell_owner, int* __restrict__ rank_of,
                  float2* __restrict__ fine, int* __restrict__ status) {
  const long long c = (long long)blockIdx.x * kGtThreads + threadIdx.x;
  if (c >= n) return;
  rank_of[c] = -1;
  const int b = item_of(offsets, g.batches, c);
  const long long a0 = assign[c], a1 = assign[n + c];
  const long long n2d = kp_offsets[b + 1] - kp_offsets[b];
  if (a0 < 0 || a0 >= n2d) { atomicOr(status, kErrAssign2d); return; }
  if (a1 < 0 || a1 >= g.rows) { atomicOr(status, kErrAssign3d); return; }
  const float* p = pack + (size_t)b * kPack;
  const float* X = kp3d + ((size_t)b * g.rows + a1) * 3;
  const float* R = p;
  const float* t = p + 9;
  const float* K = p + 12;
  float cam[3], q[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) cam[r] = __fadd_rn(mad3(R[3 * r], X[0], R[3 * r + 1], X[1], R[3 * r + 2], X[2]), t[r]);
#pragma unroll
  for (int r = 0; r < 3; ++r) q[r] = mad3(K[3 * r], cam[0], K[3 * r + 1], cam[1], K[3 * r + 2], cam[2]);
  const float zd = __fadd_rn(q[2], 1e-6f);
  float x = __fdiv_rn(q[0], zd), y = __fdiv_rn(q[1], zd);
  if (p[43] != 0.f) {
    const float* M = p + 21;
    const float xn = __fadd_rn(__fmul_rn(p[30], x), p[31]);
    const float yn = __fadd_rn(__fmul_rn(p[32], y), p[33]);
    const float w0 = mad3(M[0], xn, M[1], yn, M[2], 1.f);
    const float w1 = mad3(M[3], xn, M[4], yn, M[5], 1.f);
    const float w2 = mad3(M[6], xn, M[7], yn, M[8], 1.f);
    x = __fdiv_rn(w0, w2);
    y = __fdiv_rn(w1, w2);
    // :393-400 keeps 0 <= x <= w-1, 0 <= y <= h-1 (a NaN fails every comparison there and is kept;
    // it has no cell, so it is dropped below)
    if (x < 0.f || x > (float)(g.w - 1) || y < 0.f || y > (float)(g.h - 1)) return;
  }
  const float cx = rintf(__fmul_rn(x, 0.125f)), cy = rintf(__fmul_rn(y, 0.125f));
  const float rx = __fmul_rn(cx, 8.f), ry = __fmul_rn(cy, 8.f);
  if (!(rx >= 0.f && rx <= (float)(g.w - 1) && ry >= 0.f && ry <= (float)(g.h - 1))) return;
  const int rank = (int)cx * g.ncy + (int)cy;
  rank_of[c] = rank;
  fine[c] = make_float2(x, y);
  atomicMin(cell_owner + (size_t)b * g.ncx * g.ncy + rank, (int)(c - offsets[b]));
}

__device__ __forceinline__ bool survivor(const int* cell_owner, const long long* offsets, const GtGeom& g, int b,
                                         long long c, int rank) {
  return rank >= 0 && cell_owner[(size_t)b * g.ncx * g.ncy + rank] == (int)(c - offsets[b]);
}

__global__ void __launch_bounds__(kGtThreads)
gt_survive_kernel(const long long* __restrict__ assign, long long n, const long long* __restrict__ offsets,
                  const long long* __restrict__ kp_offsets, GtGeom g, const int* __restrict__ cell_owner,
                  const int* __restrict__ rank_of, int* __restrict__ kp_owner) {
  const long long c = (long long)blockIdx.x * kGtThreads + threadIdx.x;
  if (c >= n) return;
  const int rank = rank_of[c];
  const int b = item_of(offsets, g.batches, c);
  if (!survivor(cell_owner, offsets, g, b, c, rank)) return;
  atomicMax(kp_owner + kp_offsets[b] + assign[c], rank);
}

__global__ void __launch_bounds__(kGtThreads)
gt_emit_kernel(const long long* __restrict__ assign, long long n, const long long* __restrict__ offsets,
               const long long* __restrict__ kp_offsets, const float* __restrict__ img_scale, GtGeom g,
               const int* __restrict__ cell_owner, const int* __restrict__ rank_of, const int* __restrict__ kp_owner,
               const float2* __restrict__ fine, long long* __restrict__ key, float2* __restrict__ key_xy,
               int* __restrict__ status) {
  const long long c = (long long)blockIdx.x * kGtThreads + threadIdx.x;
  if (c >= n) return;
  key[c] = kDropped;
  const int rank = rank_of[c];
  const int b = item_of(offsets, g.batches, c);
  if (!survivor(cell_owner, offsets, g, b, c, rank)) return;
  const long long i = assign[n + c];
  if (i >= g.rows) return;                                   // :195-196
  const int won = kp_owner[kp_offsets[b] + assign[c]];       // the stored keypoint (:200, :202)
  const long long cw = offsets[b] + cell_owner[(size_t)b * g.ncx * g.ncy + won];
  const float px = __fmul_rn((float)(won / g.ncy), 8.f), py = __fmul_rn((float)(won % g.ncy), 8.f);
  // query_img_scale[[1, 0]] = (w scale, h scale); * coarse_scale; round (:205-212)
  const float jx = rintf(__fmul_rn(__fdiv_rn(px, img_scale[2 * b + 1]), 0.125f));
  const float jy = rintf(__fmul_rn(__fdiv_rn(py, img_scale[2 * b]), 0.125f));
  const float jf = __fadd_rn(__fmul_rn(jy, (float)g.w_c), jx);  // :219-223, .long() truncates
  if (!(jf > -9.2e18f && jf < 9.2e18f)) { atomicOr(status, kErrCell); return; }
  const long long j = (long long)jf;
  if (j > g.cols) return;                                    // :225-228
  if (j == g.cols || j < 0) { atomicOr(status, kErrCell); return; }
  key[c] = (((long long)b * g.rows + i) * g.cols + j) * (long long)(g.ncx * g.ncy) + rank;
  key_xy[c] = fine[cw];
}

// One CTA: walks the sorted keys in chunks of 1024, keeps the last entry of each (b, i, j) and
// writes the kept entries in order (block-wide exclusive scan of the keep flags).
__global__ void __launch_bounds__(kCompactThreads)
gt_compact_kernel(const long long* __restrict__ sorted_key, const long long* __restrict__ perm, long long n,
                  const float2* __restrict__ key_xy, int rows, int cols, long long ranks,
                  long long* __restrict__ b_ids, long long* __restrict__ i_ids, long long* __restrict__ j_ids,
                  float2* __restrict__ fine_xy, int* __restrict__ status) {
  __shared__ int warp_sum[kCompactThreads / 32];
  __shared__ long long base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) base = 0;
  __syncthreads();
  for (long long c0 = 0; c0 < n; c0 += kCompactThreads) {
    const long long p = c0 + tid;
    bool keep = false;
    long long k = kDropped;
    if (p < n) {
      k = sorted_key[p];
      if (k != kDropped) {
        const long long nk = p + 1 < n ? sorted_key[p + 1] : kDropped;
        keep = nk == kDropped || nk / ranks != k / ranks;
      }
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_sum[wid] = __popc(ballot);
    __syncthreads();
    if (wid == 0) {
      int v = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      warp_sum[lane] = v;                                   // inclusive
    }
    __syncthreads();
    const long long before = base + (wid ? warp_sum[wid - 1] : 0) + __popc(ballot & ((1u << lane) - 1u));
    if (keep) {
      const long long cell = k / ranks;
      j_ids[before] = cell % cols;
      i_ids[before] = (cell / cols) % rows;
      b_ids[before] = cell / ((long long)cols * rows);
      fine_xy[before] = key_xy[perm[p]];
    }
    __syncthreads();
    if (tid == 0) base += warp_sum[kCompactThreads / 32 - 1];
    __syncthreads();
  }
  if (tid == 0) status[1] = (int)base;
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" int opp_train_batch_pack_size(void) { return kPack; }

extern "C" int opp_homography_warp_f32(const float* img, const float* pack, int batches, int h, int w, float* out,
                                       opp_stream_t stream) {
  OPP_REQUIRE(img && pack && out, "opp_homography_warp_f32: null pointer");
  OPP_REQUIRE(batches > 0 && batches <= 65535 && h > 1 && w > 1 && (long long)h * w < INT32_MAX,
              "opp_homography_warp_f32: bad shape B=%d h=%d w=%d", batches, h, w);
  const dim3 grid((unsigned)((w + kWarpTx - 1) / kWarpTx), (unsigned)((h + kWarpTy - 1) / kWarpTy), (unsigned)batches);
  homography_warp_kernel<<<grid, dim3(kWarpTx, kWarpTy), 0, (cudaStream_t)stream>>>(img, pack, h, w, out);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_train_gt_build(const float* kp3d, const long long* assign, long long n, const long long* offsets,
                                  const long long* kp_offsets, long long n_kp, const float* pack,
                                  const float* img_scale, int batches, int rows, int h, int w, int w_c, int cols,
                                  int* cell_owner, int* kp_owner, int* rank_of, float* fine, long long* key,
                                  float* key_xy, int* status, opp_stream_t stream) {
  OPP_REQUIRE(batches > 0 && rows > 0 && h > 0 && w > 0 && w_c > 0 && cols > 0 && n >= 0 && n < INT32_MAX &&
                  n_kp >= 0 && n_kp < INT32_MAX,
              "opp_train_gt_build: bad shape B=%d L=%d h=%d w=%d w_c=%d S=%d n=%lld", batches, rows, h, w, w_c, cols,
              n);
  OPP_REQUIRE(offsets && kp_offsets && pack && img_scale && status && cell_owner,
              "opp_train_gt_build: null pointer");
  OPP_REQUIRE(n == 0 || (kp3d && assign && rank_of && fine && key && key_xy && (n_kp == 0 || kp_owner)),
              "opp_train_gt_build: null pointer");
  const GtGeom g{batches, rows, h, w, w_c, cols, (w - 1) / 8 + 1, (h - 1) / 8 + 1};
  const long long ranks = (long long)g.ncx * g.ncy;
  OPP_REQUIRE((double)batches * rows * cols * ranks < 9.0e18, "opp_train_gt_build: B L S R overflows the int64 key");
  const cudaStream_t st = (cudaStream_t)stream;
  OPP_CHECK_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(int), st));
  if (n == 0) return OPP_OK;
  OPP_CHECK_CUDA(cudaMemsetAsync(cell_owner, 0x7f, (size_t)batches * ranks * sizeof(int), st));
  if (n_kp) OPP_CHECK_CUDA(cudaMemsetAsync(kp_owner, 0xff, (size_t)n_kp * sizeof(int), st));
  const unsigned blocks = (unsigned)((n + kGtThreads - 1) / kGtThreads);
  gt_project_kernel<<<blocks, kGtThreads, 0, st>>>(kp3d, assign, n, offsets, kp_offsets, pack, g, cell_owner, rank_of,
                                                   reinterpret_cast<float2*>(fine), status);
  OPP_CHECK_CUDA(cudaGetLastError());
  gt_survive_kernel<<<blocks, kGtThreads, 0, st>>>(assign, n, offsets, kp_offsets, g, cell_owner, rank_of, kp_owner);
  OPP_CHECK_CUDA(cudaGetLastError());
  gt_emit_kernel<<<blocks, kGtThreads, 0, st>>>(assign, n, offsets, kp_offsets, img_scale, g, cell_owner, rank_of,
                                                kp_owner, reinterpret_cast<const float2*>(fine), key,
                                                reinterpret_cast<float2*>(key_xy), status);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_train_gt_compact(const long long* sorted_key, const long long* perm, long long n,
                                    const float* key_xy, int rows, int cols, long long ranks, long long* b_ids,
                                    long long* i_ids, long long* j_ids, float* fine_xy, int* status,
                                    opp_stream_t stream) {
  OPP_REQUIRE(n >= 0 && n < INT32_MAX && rows > 0 && cols > 0 && ranks > 0, "opp_train_gt_compact: bad shape");
  OPP_REQUIRE(status && (n == 0 || (sorted_key && perm && key_xy && b_ids && i_ids && j_ids && fine_xy)),
              "opp_train_gt_compact: null pointer");
  gt_compact_kernel<<<1, kCompactThreads, 0, (cudaStream_t)stream>>>(
      sorted_key, perm, n, reinterpret_cast<const float2*>(key_xy), rows, cols, ranks, b_ids, i_ids, j_ids,
      reinterpret_cast<float2*>(fine_xy), status);
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
