// opp_image.cu — the demo's bbox crop of uint8 frames on the device (reference:
// LocalFeatureObjectDetector.crop_img_by_bbox, src/local_feature_object_detector/
// local_feature_2D_detector.py:133-159: two cv2.warpAffine(INTER_LINEAR) calls through
// data_utils.get_image_crop_resize :239-255 — the box at native scale, then a resize to crop x crop).
//
// Exactness.  cv2 warps uint8 images with a fixed-point scheme (imgwarp.cpp, warpAffine +
// remapBilinear), restated here with no floating-point freedom left:
//   m = cv2's inverse of the forward matrix (fp64, computed on the host the way warpAffine does);
//   adelta[x] = rint(m0 * x * 1024), bdelta[x] = rint(m3 * x * 1024);
//   X0[y] = rint((m1 * y + m2) * 1024) + 16, Y0[y] = rint((m4 * y + m5) * 1024) + 16;
//   X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5: tap (X >> 5, Y >> 5), fractions a = X & 31, b = Y & 31;
//   out = (sum_taps v * w + 2^14) >> 15 with w = 32 (32 - a)(32 - b), 32 a (32 - b), ... and v = 0
//   for a tap outside the source (BORDER_CONSTANT 0).
// Every fp64 product and sum is issued with an explicit _rn intrinsic (no FMA contraction) and every
// rint is __double2int_rn (cvRound: round half to even), so the integers equal cv2's.
//
// One stage.  The first warp of crop_img_by_bbox maps the box [x0, y0, x0 + w, y0 + h] to a w x h
// image at scale 1: an integer shift (the host checks this on the fixed-point parameters), so that
// image is frame[v + y0][u + x0], 0 outside the frame.  The kernel therefore runs only the second
// warp, over a VIRTUAL source of w x h pixels: the frame shifted by (x0, y0), zero outside the
// frame and zero outside [0, w) x [0, h).  The intermediate image is never written.
//
// Layout: one CTA per 128 x 8 output tile per frame, 4 horizontally adjacent pixels per thread
// (one 32-bit store); the 4 taps of a pixel are plain loads that hit L1/L2 (a 512^2 crop of a box
// reads at most the box's bytes).
#include <cstdint>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
namespace {

constexpr int kCropTx = 32, kCropTy = 8;   // threads per CTA (x, y)
constexpr int kCropPx = 4;                 // output pixels per thread along x
constexpr int kCoordLimit = 1 << 20;       // |box coordinate| bound: keeps every fixed-point sum in int32
constexpr int kShrtMax = 32767;            // cv2 remap: source and destination sides < SHRT_MAX

__device__ __forceinline__ int sat_short(int v) { return max(-32768, min(32767, v)); }

__global__ void __launch_bounds__(kCropTx * kCropTy)
crop_resize_u8_kernel(const unsigned char* __restrict__ frames, int H, int W,
                      const opp_crop_params* __restrict__ params, unsigned char* __restrict__ out, int out_h,
                      int out_w, int* __restrict__ status) {
  pdl_sync();
  const int b = blockIdx.z;
  const opp_crop_params p = params[b];
  const long long plane = (long long)out_h * out_w;
  unsigned char* dst = out + b * plane;
  const int y = blockIdx.y * kCropTy + threadIdx.y;
  const int xb = (blockIdx.x * kCropTx + threadIdx.x) * kCropPx;
  int st = 0;
  if (p.w < 1 || p.h < 1) st = 1;   // cv2 raises: empty destination of the first warp
  else if (p.w >= kShrtMax || p.h >= kShrtMax || abs(p.x0) >= kCoordLimit || abs(p.y0) >= kCoordLimit ||
           abs(p.x0 + p.w) >= kCoordLimit || abs(p.y0 + p.h) >= kCoordLimit)
    st = 2;
  if (status != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0)
    status[b] = st;
  if (y >= out_h || xb >= out_w) return;
  unsigned char v[kCropPx] = {0, 0, 0, 0};
  if (st == 0) {
    const unsigned char* src = frames + (long long)b * H * W;
    const double yd = (double)y;
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.m[1], yd), p.m[2]), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(p.m[4], yd), p.m[5]), 1024.0)) + 16;
#pragma unroll
    for (int k = 0; k < kCropPx; ++k) {
      const double xd = (double)(xb + k);
      const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(p.m[0], xd), 1024.0))) >> 5;
      const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(p.m[3], xd), 1024.0))) >> 5;
      const int sx = sat_short(X >> 5), sy = sat_short(Y >> 5);
      const int a = X & 31, bb = Y & 31;
      int acc = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int u = sx + (t & 1), r = sy + (t >> 1);
        const int fx = u + p.x0, fy = r + p.y0;
        const bool in = u >= 0 && u < p.w && r >= 0 && r < p.h && fx >= 0 && fx < W && fy >= 0 && fy < H;
        const int wx = (t & 1) ? a : 32 - a, wy = (t >> 1) ? bb : 32 - bb;
        if (in) acc += (int)__ldg(src + (long long)fy * W + fx) * (wx * wy * 32);
      }
      v[k] = (unsigned char)min(255, (acc + (1 << 14)) >> 15);
    }
  }
  unsigned char* row = dst + (long long)y * out_w;
  if ((out_w & 3) == 0 && xb + kCropPx <= out_w) {
    *reinterpret_cast<uchar4*>(row + xb) = make_uchar4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int k = 0; k < kCropPx; ++k)
      if (xb + k < out_w) row[xb + k] = v[k];
  }
}

}  // namespace
}  // namespace opp

using namespace opp;

extern "C" int opp_crop_resize_u8(const unsigned char* frames, int batch, int height, int width,
                                  const opp_crop_params* params, unsigned char* out, int out_h, int out_w,
                                  int* status, opp_stream_t stream) {
  OPP_REQUIRE(frames && params && out, "opp_crop_resize_u8: null pointer");
  OPP_REQUIRE(batch > 0 && batch <= 65535, "opp_crop_resize_u8: batch %d out of range", batch);
  OPP_REQUIRE(height > 0 && width > 0 && height < kShrtMax && width < kShrtMax,
              "opp_crop_resize_u8: frame %dx%d out of range (cv2 needs both sides in [1, 32766])", height, width);
  OPP_REQUIRE(out_h > 0 && out_w > 0 && out_h < kShrtMax && out_w < kShrtMax,
              "opp_crop_resize_u8: output %dx%d out of range", out_h, out_w);
  OPP_REQUIRE(((uintptr_t)params & 7) == 0, "opp_crop_resize_u8: params must be 8-byte aligned");
  OPP_REQUIRE((out_w & 3) != 0 || ((uintptr_t)out & 3) == 0, "opp_crop_resize_u8: out must be 4-byte aligned");
  const dim3 grid((out_w + kCropTx * kCropPx - 1) / (kCropTx * kCropPx), (out_h + kCropTy - 1) / kCropTy, batch);
  OPP_CHECK_CUDA(launch_pdl(crop_resize_u8_kernel, grid, dim3(kCropTx, kCropTy), 0, (cudaStream_t)stream, frames,
                            height, width, params, out, out_h, out_w, status));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
