// opp_metrics.cu — LINEMOD pose metrics on the device: ADD, ADD-S and proj2D for a batch of frames
// of one object model (reference: src/utils/metric_utils.py:31-88 `projection_2d_error` /
// `add_metric`, called per frame from `compute_query_pose_errors` :233-289 after the D2H copy of
// the pose; ADD-S there is a scipy cKDTree built on the predicted points and queried with the
// target points).
//
// Three launches, all reading the poses where opp_pnp_ransac left them:
//   1. pointwise (frame x 256-vertex tile): ADD and proj2D terms in fp64, literally
//      pred = R_p x + t_p, tgt = R_g x + t_g, |pred - tgt| and |pi(pred) - pi(tgt)| with
//      pi(p) = (K p)_xy / (K p)_z (no guard: IEEE inf / nan carry through as in numpy); one fp64
//      partial sum per tile and term; the per-target minima of symmetric frames are set to +inf.
//   2. nearest neighbour (frame x target tile x predicted-point split), symmetric frames only:
//      min_i |pred_i - tgt_j|^2 for every target j.  Rotation preserves distance, so this runs in
//      model coordinates, |dR x_i + dt - x_j| with dR = R_g^T R_p, dt = R_g^T (t_p - t_g) formed in
//      fp64: no cancellation against the metre-scale translation, and the inner loop can be fp32 in
//      the direct-difference form (|a|^2 + |b|^2 - 2ab would cancel for near neighbours).  Splits
//      of the predicted points combine with atomicMin on the bit pattern of the non-negative fp32
//      squared distance: min is exact and order-independent.
//   3. finalize (one CTA per frame): fixed-order fp64 sums of the tile partials, or of the square
//      roots of the minima, divided by V.
// No floating-point atomics anywhere: two identical calls give bit-identical results.
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {

int num_sms();

namespace {

constexpr int kMetThreads = 256;
constexpr int kNnPerThread = 2;                          // targets held in registers per thread
constexpr int kNnTile = kMetThreads * kNnPerThread;      // targets per CTA
constexpr int kNnChunk = kMetThreads;                    // predicted points staged per pass
constexpr int kNnMinSplit = 512;                         // predicted points per split, at least
constexpr unsigned kInfBits = 0x7f800000u;               // +inf as fp32

int pointwise_tiles(int verts) { return (verts + kMetThreads - 1) / kMetThreads; }

// dR = R_g^T R_p, dt = R_g^T (t_p - t_g):  pred_i - tgt_j = R_g (dR x_i + dt - x_j)
__device__ void frame_delta(const float* __restrict__ P, const float* __restrict__ G, double* dR, double* dt) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
      dR[r * 3 + c] = (double)G[r] * P[c] + (double)G[4 + r] * P[4 + c] + (double)G[8 + r] * P[8 + c];
    dt[r] = (double)G[r] * ((double)P[3] - G[3]) + (double)G[4 + r] * ((double)P[7] - G[7]) +
            (double)G[8 + r] * ((double)P[11] - G[11]);
  }
}

// sum of (a, b) over the CTA in a fixed order (shuffle tree, then the warps in index order)
__device__ void block_sum2(double& a, double& b, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[warp] = a;
    red[kMetThreads / 32 + warp] = b;
  }
  __syncthreads();
  a = 0.0;
  b = 0.0;
#pragma unroll
  for (int w = 0; w < kMetThreads / 32; ++w) {
    a += red[w];
    b += red[kMetThreads / 32 + w];
  }
}

__device__ __forceinline__ void project(const float* K, const double* p, double& u, double& v) {
  const double x = (double)K[0] * p[0] + (double)K[1] * p[1] + (double)K[2] * p[2];
  const double y = (double)K[3] * p[0] + (double)K[4] * p[1] + (double)K[5] * p[2];
  const double w = (double)K[6] * p[0] + (double)K[7] * p[1] + (double)K[8] * p[2];
  u = x / w;
  v = y / w;
}

__global__ void __launch_bounds__(kMetThreads)
pose_metrics_pointwise_kernel(const float* __restrict__ verts, int V, const float* __restrict__ pose_pred,
                              const float* __restrict__ pose_gt, const float* __restrict__ Kmat,
                              const unsigned char* __restrict__ symmetric, double* __restrict__ partial,
                              unsigned* __restrict__ minbits) {
  pdl_sync();
  __shared__ double red[2 * kMetThreads / 32];
  const int b = blockIdx.y, j = blockIdx.x * kMetThreads + threadIdx.x;
  double add = 0.0, prj = 0.0;
  if (j < V) {
    const float* P = pose_pred + b * 12;
    const float* G = pose_gt + b * 12;
    const double x[3] = {(double)verts[j * 3], (double)verts[j * 3 + 1], (double)verts[j * 3 + 2]};
    double pr[3], tg[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      pr[r] = (double)P[r * 4] * x[0] + (double)P[r * 4 + 1] * x[1] + (double)P[r * 4 + 2] * x[2] + P[r * 4 + 3];
      tg[r] = (double)G[r * 4] * x[0] + (double)G[r * 4 + 1] * x[1] + (double)G[r * 4 + 2] * x[2] + G[r * 4 + 3];
    }
    const double dx = pr[0] - tg[0], dy = pr[1] - tg[1], dz = pr[2] - tg[2];
    add = sqrt(dx * dx + dy * dy + dz * dz);
    double up, vp, ug, vg;
    project(Kmat + b * 9, pr, up, vp);
    project(Kmat + b * 9, tg, ug, vg);
    const double du = up - ug, dv = vp - vg;
    prj = sqrt(du * du + dv * dv);
    if (symmetric[b]) minbits[(long long)b * V + j] = kInfBits;
  }
  block_sum2(add, prj, red);
  if (threadIdx.x == 0) {
    double* out = partial + ((long long)b * gridDim.x + blockIdx.x) * 2;
    out[0] = add;
    out[1] = prj;
  }
}

__global__ void __launch_bounds__(kMetThreads)
pose_metrics_nn_kernel(const float* __restrict__ verts, int V, const float* __restrict__ pose_pred,
                       const float* __restrict__ pose_gt, const unsigned char* __restrict__ symmetric,
                       int splits, unsigned* __restrict__ minbits) {
  pdl_sync();
  const int b = blockIdx.y;
  if (!symmetric[b]) return;
  __shared__ float4 sp[kNnChunk];
  __shared__ double delta[12];
  const int tid = threadIdx.x;
  const int tile = blockIdx.x / splits, split = blockIdx.x % splits;
  if (tid == 0) frame_delta(pose_pred + b * 12, pose_gt + b * 12, delta, delta + 9);
  float tx[kNnPerThread], ty[kNnPerThread], tz[kNnPerThread], best[kNnPerThread];
#pragma unroll
  for (int k = 0; k < kNnPerThread; ++k) {
    const int j = tile * kNnTile + k * kMetThreads + tid;
    const bool ok = j < V;
    tx[k] = ok ? verts[j * 3] : 0.f;
    ty[k] = ok ? verts[j * 3 + 1] : 0.f;
    tz[k] = ok ? verts[j * 3 + 2] : 0.f;
    best[k] = __uint_as_float(kInfBits);
  }
  const int per = (V + splits - 1) / splits;
  const int lo = split * per, hi = min(V, lo + per);
  for (int base = lo; base < hi; base += kNnChunk) {
    __syncthreads();   // delta written / previous chunk consumed
    const int i = base + tid;
    float4 p = make_float4(__uint_as_float(kInfBits), __uint_as_float(kInfBits), __uint_as_float(kInfBits), 0.f);
    if (i < hi) {   // dR x_i + dt, fp64 then rounded once; padding rows sit at +inf (never the min)
      const double x0 = verts[i * 3], x1 = verts[i * 3 + 1], x2 = verts[i * 3 + 2];
      p.x = (float)(delta[0] * x0 + delta[1] * x1 + delta[2] * x2 + delta[9]);
      p.y = (float)(delta[3] * x0 + delta[4] * x1 + delta[5] * x2 + delta[10]);
      p.z = (float)(delta[6] * x0 + delta[7] * x1 + delta[8] * x2 + delta[11]);
    }
    sp[tid] = p;
    __syncthreads();
#pragma unroll 8
    for (int q = 0; q < kNnChunk; ++q) {
      const float4 s = sp[q];
#pragma unroll
      for (int k = 0; k < kNnPerThread; ++k) {
        const float dx = s.x - tx[k], dy = s.y - ty[k], dz = s.z - tz[k];
        best[k] = fminf(best[k], dx * dx + dy * dy + dz * dz);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kNnPerThread; ++k) {
    const int j = tile * kNnTile + k * kMetThreads + tid;
    if (j < V) atomicMin(minbits + (long long)b * V + j, __float_as_uint(best[k]));
  }
}

__global__ void __launch_bounds__(kMetThreads)
pose_metrics_finalize_kernel(int V, int tiles, const unsigned char* __restrict__ symmetric,
                             const double* __restrict__ partial, const unsigned* __restrict__ minbits,
                             double* __restrict__ add_dist, double* __restrict__ proj2d) {
  pdl_sync();
  __shared__ double red[2 * kMetThreads / 32];
  const int b = blockIdx.x;
  double add = 0.0, prj = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kMetThreads) {
    add += partial[((long long)b * tiles + t) * 2];
    prj += partial[((long long)b * tiles + t) * 2 + 1];
  }
  if (symmetric[b]) {
    add = 0.0;
    for (int j = threadIdx.x; j < V; j += kMetThreads)
      add += sqrt((double)__uint_as_float(minbits[(long long)b * V + j]));
  }
  block_sum2(add, prj, red);
  if (threadIdx.x == 0) {
    add_dist[b] = add / V;
    proj2d[b] = prj / V;
  }
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" long long opp_pose_metrics_scratch_bytes(int verts, int batch) {
  if (verts <= 0 || batch <= 0) return 0;
  return (long long)batch * pointwise_tiles(verts) * 2 * (long long)sizeof(double) +
         (long long)batch * verts * (long long)sizeof(unsigned);
}

extern "C" int opp_pose_metrics(const float* verts, int num_verts, const float* pose_pred, const float* pose_gt,
                                const float* intrinsics, const unsigned char* symmetric, int batch,
                                void* scratch, long long scratch_bytes, double* add_dist, double* proj2d,
                                opp_stream_t stream) {
  OPP_REQUIRE(verts && pose_pred && pose_gt && intrinsics && symmetric && scratch && add_dist && proj2d,
              "null pointer");
  OPP_REQUIRE(num_verts > 0 && num_verts <= (1 << 26), "opp_pose_metrics: num_verts %d out of range", num_verts);
  OPP_REQUIRE(batch > 0 && batch <= 65535, "opp_pose_metrics: batch %d out of range", batch);
  OPP_REQUIRE(scratch_bytes >= opp_pose_metrics_scratch_bytes(num_verts, batch),
              "opp_pose_metrics: scratch of %lld bytes, need %lld", scratch_bytes,
              opp_pose_metrics_scratch_bytes(num_verts, batch));
  OPP_REQUIRE(((uintptr_t)scratch & 7) == 0, "opp_pose_metrics: scratch must be 8-byte aligned");
  const int tiles = pointwise_tiles(num_verts);
  double* partial = static_cast<double*>(scratch);
  unsigned* minbits = reinterpret_cast<unsigned*>(partial + (long long)batch * tiles * 2);
  const cudaStream_t st = (cudaStream_t)stream;
  OPP_CHECK_CUDA(launch_pdl(pose_metrics_pointwise_kernel, dim3(tiles, batch), dim3(kMetThreads), 0, st, verts,
                            num_verts, pose_pred, pose_gt, intrinsics, symmetric, partial, minbits));
  // Fill the GPU at batch 1, where a frame has only V / 512 target tiles: split the predicted points
  // across CTAs until there are 8 CTAs per SM (the kernel was sized for symmetric frames; the others
  // exit at once), keeping every split >= kNnMinSplit points so that the atomics stay rare.
  const int nn_tiles = (num_verts + kNnTile - 1) / kNnTile;
  const long long want = 8LL * num_sms();
  const long long have = (long long)nn_tiles * batch;
  int splits = (int)((want + have - 1) / have);
  splits = max(1, min(splits, (num_verts + kNnMinSplit - 1) / kNnMinSplit));
  OPP_CHECK_CUDA(launch_pdl(pose_metrics_nn_kernel, dim3(nn_tiles * splits, batch), dim3(kMetThreads), 0, st,
                            verts, num_verts, pose_pred, pose_gt, symmetric, splits, minbits));
  OPP_CHECK_CUDA(launch_pdl(pose_metrics_finalize_kernel, dim3(batch), dim3(kMetThreads), 0, st, num_verts, tiles,
                            symmetric, partial, minbits, add_dist, proj2d));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
