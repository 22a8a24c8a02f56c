// opp_pnp.cu — batched RANSAC-PnP on the device: the consumer of the matcher's output
// (reference: src/utils/metric_utils.py:121-204 `ransac_PnP` = cv2.solvePnPRansac(EPnP, 10000
// iterations, reprojectionError) per frame on the CPU after a D2H sync; called per frame from
// `compute_query_pose_errors` :207-292 and demo.py:132).
//
// One CTA per query image.  The matches of image b are the contiguous run of `m_bids == b` in the
// match lists (the matcher emits them in ascending (b, i) order).  Per image:
//   1. hypotheses: every thread draws 4 distinct matches (counter-based hash RNG), solves P3P on the
//      first three (Grunert's quartic in the depth ratio, closed-form Ferrari roots + Newton
//      polish, pose from the two triangle frames) and keeps the root that best reprojects the 4th;
//   2. scoring: reprojection error of every match under the hypothesis, inlier = err < thr and in
//      front of the camera; block-wide argmax of the inlier count (ties -> lowest hypothesis id, so
//      the result does not depend on scheduling);
//   3. refinement (local optimisation): Gauss-Newton / LM on the 6-DoF pose over the current
//      inliers (normal equations accumulated by the whole CTA, 6x6 Cholesky by one thread),
//      inlier set re-evaluated between rounds.  The optimum of the reprojection error over the
//      inliers is what cv2's iterative refinement converges to as well, which is what the parity
//      test compares against.
// All geometry runs in fp64 (a few MFLOP per image); inputs / outputs are fp32.
// The same kernel, instantiated for PnpSolver::kColmap (opp_pnp_ransac_colmap), is the reference's
// use_pycolmap_ransac branch (metric_utils.py:137-170); see pnp_ransac_kernel.
#include <cstdint>
#include <cstdio>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {

struct Pose {
  double R[9];
  double t[3];
};

__device__ __forceinline__ uint32_t pnp_hash(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

__host__ __device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
__host__ __device__ __forceinline__ double dot3(const double* a, const double* b) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}
__host__ __device__ __forceinline__ bool normalize3(double* a) {
  const double n = sqrt(dot3(a, a));
  if (!(n > 1e-300)) return false;
  a[0] /= n;
  a[1] /= n;
  a[2] /= n;
  return true;
}

// largest real root of x^3 + a2 x^2 + a1 x + a0
__host__ __device__ double cubic_largest_real(double a2, double a1, double a0) {
  const double p = a1 - a2 * a2 / 3.0;
  const double q = 2.0 * a2 * a2 * a2 / 27.0 - a2 * a1 / 3.0 + a0;
  const double disc = q * q / 4.0 + p * p * p / 27.0;
  double y;
  if (disc > 0.0) {
    const double sq = sqrt(disc);
    y = cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq);
  } else if (p < 0.0) {
    const double r = sqrt(-p / 3.0);
    double c = -q / 2.0 / (r * r * r);
    c = fmin(1.0, fmax(-1.0, c));
    y = 2.0 * r * cos(acos(c) / 3.0);
  } else {
    y = 0.0;
  }
  return y - a2 / 3.0;
}

// real roots of A4 x^4 + ... + A0 (Ferrari), each polished with Newton steps; returns the count
__host__ __device__ int solve_quartic(double A4, double A3, double A2, double A1, double A0, double* roots) {
  if (!(fabs(A4) > 1e-14)) return 0;
  const double b = A3 / A4, c = A2 / A4, d = A1 / A4, e = A0 / A4;
  const double p = c - 3.0 * b * b / 8.0;
  const double q = d - b * c / 2.0 + b * b * b / 8.0;
  const double r = e - b * d / 4.0 + b * b * c / 16.0 - 3.0 * b * b * b * b / 256.0;
  int n = 0;
  double y[4];
  const double m = cubic_largest_real(p, p * p / 4.0 - r, -q * q / 8.0);
  if (m > 1e-14) {
    const double s = sqrt(2.0 * m);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const double sg = k == 0 ? 1.0 : -1.0;
      const double B = sg * s, C = p / 2.0 + m - sg * q / (2.0 * s);
      const double D = B * B - 4.0 * C;
      if (D >= 0.0) {
        const double sd = sqrt(D);
        y[n++] = (-B + sd) / 2.0;
        y[n++] = (-B - sd) / 2.0;
      } else if (D > -1e-9 * fmax(1.0, B * B)) {
        y[n++] = -B / 2.0;
      }
    }
  } else {
    const double D = p * p / 4.0 - r;   // biquadratic y^4 + p y^2 + r
    if (D >= 0.0) {
      const double sd = sqrt(D);
      const double z0 = -p / 2.0 + sd, z1 = -p / 2.0 - sd;
      if (z0 >= 0.0) {
        y[n++] = sqrt(z0);
        y[n++] = -sqrt(z0);
      }
      if (z1 >= 0.0 && n <= 2) {
        y[n++] = sqrt(z1);
        y[n++] = -sqrt(z1);
      }
    }
  }
  for (int i = 0; i < n; ++i) {
    double x = y[i] - b / 4.0;
#pragma unroll
    for (int it = 0; it < 3; ++it) {
      const double f = (((x + b) * x + c) * x + d) * x + e;
      const double fp = ((4.0 * x + 3.0 * b) * x + 2.0 * c) * x + d;
      if (fabs(fp) > 1e-300) x -= f / fp;
    }
    roots[i] = x;
  }
  return n;
}

// orthonormal frame of a triangle: columns e1 = (Q1-Q0)^, e3 = (e1 x (Q2-Q0))^, e2 = e3 x e1
__host__ __device__ bool tri_frame(const double* Q0, const double* Q1, const double* Q2, double* F) {
  double e1[3] = {Q1[0] - Q0[0], Q1[1] - Q0[1], Q1[2] - Q0[2]};
  double w[3] = {Q2[0] - Q0[0], Q2[1] - Q0[1], Q2[2] - Q0[2]};
  double e3[3], e2[3];
  if (!normalize3(e1)) return false;
  cross3(e1, w, e3);
  if (!normalize3(e3)) return false;
  cross3(e3, e1, e2);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    F[k * 3 + 0] = e1[k];
    F[k * 3 + 1] = e2[k];
    F[k * 3 + 2] = e3[k];
  }
  return true;
}

// P3P (Grunert 1841 as restated by Haralick et al. 1994): world points P[3], unit bearings f[3].
// Calls `visit(pose)` for every admissible solution.
template <class V>
__host__ __device__ void p3p_grunert(const double (*P)[3], const double (*f)[3], V&& visit) {
  double d12[3], d02[3], d01[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    d12[k] = P[1][k] - P[2][k];
    d02[k] = P[0][k] - P[2][k];
    d01[k] = P[0][k] - P[1][k];
  }
  const double a2 = dot3(d12, d12), b2 = dot3(d02, d02), c2 = dot3(d01, d01);
  if (!(a2 > 1e-20 && b2 > 1e-20 && c2 > 1e-20)) return;
  const double ca = dot3(f[1], f[2]), cb = dot3(f[0], f[2]), cg = dot3(f[0], f[1]);
  const double q = (a2 - c2) / b2, ac = (a2 + c2) / b2;
  const double A4 = (q - 1.0) * (q - 1.0) - 4.0 * c2 / b2 * ca * ca;
  const double A3 = 4.0 * (q * (1.0 - q) * cb - (1.0 - ac) * ca * cg + 2.0 * c2 / b2 * ca * ca * cb);
  const double A2 = 2.0 * (q * q - 1.0 + 2.0 * q * q * cb * cb + 2.0 * ((b2 - c2) / b2) * ca * ca -
                           4.0 * ac * ca * cb * cg + 2.0 * ((b2 - a2) / b2) * cg * cg);
  const double A1 = 4.0 * (-q * (1.0 + q) * cb + 2.0 * a2 / b2 * cg * cg * cb - (1.0 - ac) * ca * cg);
  const double A0 = (1.0 + q) * (1.0 + q) - 4.0 * a2 / b2 * cg * cg;
  double roots[4];
  const int n = solve_quartic(A4, A3, A2, A1, A0, roots);
  double Fw[9];
  if (!tri_frame(P[0], P[1], P[2], Fw)) return;
  for (int i = 0; i < n; ++i) {
    const double v = roots[i];
    if (!(v > 0.0) || !isfinite(v)) continue;
    const double den = 2.0 * (cg - v * ca);
    if (!(fabs(den) > 1e-12)) continue;
    const double u = ((q - 1.0) * v * v - 2.0 * q * cb * v + 1.0 + q) / den;
    if (!(u > 0.0)) continue;
    const double s1sq = b2 / (1.0 + v * v - 2.0 * v * cb);
    if (!(s1sq > 0.0)) continue;
    const double s1 = sqrt(s1sq);
    double X[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      X[0][k] = s1 * f[0][k];
      X[1][k] = u * s1 * f[1][k];
      X[2][k] = v * s1 * f[2][k];
    }
    double Fc[9];
    if (!tri_frame(X[0], X[1], X[2], Fc)) continue;
    Pose ps;
    // R = Fc * Fw^T
#pragma unroll
    for (int r_ = 0; r_ < 3; ++r_)
#pragma unroll
      for (int c_ = 0; c_ < 3; ++c_)
        ps.R[r_ * 3 + c_] = Fc[r_ * 3 + 0] * Fw[c_ * 3 + 0] + Fc[r_ * 3 + 1] * Fw[c_ * 3 + 1] +
                            Fc[r_ * 3 + 2] * Fw[c_ * 3 + 2];
#pragma unroll
    for (int k = 0; k < 3; ++k)
      ps.t[k] = X[0][k] - (ps.R[k * 3] * P[0][0] + ps.R[k * 3 + 1] * P[0][1] + ps.R[k * 3 + 2] * P[0][2]);
    visit(ps);
  }
}

struct Cam {
  double fx, fy, cx, cy, skew;
};

// squared reprojection error (pixels^2) of world point p against pixel (u, v); +inf behind the camera
__device__ __forceinline__ double reproj_err2(const Pose& ps, const Cam& cam, const double* p, double u,
                                              double v) {
  const double x = ps.R[0] * p[0] + ps.R[1] * p[1] + ps.R[2] * p[2] + ps.t[0];
  const double y = ps.R[3] * p[0] + ps.R[4] * p[1] + ps.R[5] * p[2] + ps.t[1];
  const double z = ps.R[6] * p[0] + ps.R[7] * p[1] + ps.R[8] * p[2] + ps.t[2];
  if (!(z > 1e-9)) return INFINITY;
  const double xn = x / z, yn = y / z;
  const double du = cam.fx * xn + cam.skew * yn + cam.cx - u;
  const double dv = cam.fy * yn + cam.cy - v;
  return du * du + dv * dv;
}

constexpr int kPnpThreads = 256;

__device__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < kPnpThreads / 32; ++w) s += red[w];
  return s;
}

// Adds the Gauss-Newton terms of match (p, u, v) at pose `ps` to acc[27]: the upper triangle of
// J^T J, then J^T r, with r the pixel residual and J its derivative in (w, t) of the update
// R <- exp([w]x) R, t <- t + dt.  A point behind the camera adds nothing.  kCauchy weights the
// terms by w = 1 / (1 + |r|^2), the IRLS weight of the per-point loss log(1 + |r|^2), and adds
// that loss to *cost (+inf behind the camera, so that a step moving an inlier there is refused).
template <bool kCauchy>
__device__ __forceinline__ void gn_terms(const Pose& ps, const Cam& cam, const double* p, double u, double v,
                                         double* acc, double* cost) {
  const double Y0 = ps.R[0] * p[0] + ps.R[1] * p[1] + ps.R[2] * p[2];
  const double Y1 = ps.R[3] * p[0] + ps.R[4] * p[1] + ps.R[5] * p[2];
  const double Y2 = ps.R[6] * p[0] + ps.R[7] * p[1] + ps.R[8] * p[2];
  const double x = Y0 + ps.t[0], y = Y1 + ps.t[1], z = Y2 + ps.t[2];
  if (!(z > 1e-9)) {
    if constexpr (kCauchy) *cost = INFINITY;
    return;
  }
  const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
  double ru = cam.fx * xn + cam.skew * yn + cam.cx - u;
  double rv = cam.fy * yn + cam.cy - v;
  // d(u)/dXc, d(v)/dXc
  const double gu[3] = {cam.fx * iz, cam.skew * iz, -(cam.fx * xn + cam.skew * yn) * iz};
  const double gv[3] = {0.0, cam.fy * iz, -cam.fy * yn * iz};
  // Xc = exp(w) Y + t  ->  dXc/dw = -[Y]x ; J row = (g x ... ) : g^T (-[Y]x) = (Y x g)^T
  const double Yv[3] = {Y0, Y1, Y2};
  double ju[6], jv[6];
  cross3(Yv, gu, ju);
  cross3(Yv, gv, jv);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ju[3 + k] = gu[k];
    jv[3 + k] = gv[k];
  }
  if constexpr (kCauchy) {
    const double s = ru * ru + rv * rv;
    *cost += log1p(s);
    const double sw = sqrt(1.0 / (1.0 + s));   // rows scaled by sqrt(w): J^T w J, J^T w r
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      ju[k] *= sw;
      jv[k] *= sw;
    }
    ru *= sw;
    rv *= sw;
  }
  int o = 0;
#pragma unroll
  for (int r_ = 0; r_ < 6; ++r_) {
#pragma unroll
    for (int c_ = r_; c_ < 6; ++c_) acc[o++] += ju[r_] * ju[c_] + jv[r_] * jv[c_];
  }
#pragma unroll
  for (int r_ = 0; r_ < 6; ++r_) acc[21 + r_] += ju[r_] * ru + jv[r_] * rv;
}

// Solves (H + damping diag H) d = -g by Cholesky, H and g packed in Hs as gn_terms accumulates
// them.  Returns false when the damped H is not positive definite.
__device__ __forceinline__ bool solve_damped(const double* Hs, double damping, double* d) {
  double H[6][6], g[6], L[6][6];
  int o = 0;
  for (int r_ = 0; r_ < 6; ++r_)
    for (int c_ = r_; c_ < 6; ++c_) {
      H[r_][c_] = Hs[o];
      H[c_][r_] = Hs[o];
      ++o;
    }
  for (int r_ = 0; r_ < 6; ++r_) {
    g[r_] = Hs[21 + r_];
    H[r_][r_] *= 1.0 + damping;
  }
  bool okc = true;
  for (int r_ = 0; r_ < 6 && okc; ++r_)
    for (int c_ = 0; c_ <= r_; ++c_) {
      double s = H[r_][c_];
      for (int k = 0; k < c_; ++k) s -= L[r_][k] * L[c_][k];
      if (r_ == c_) {
        if (!(s > 1e-300)) {
          okc = false;
          break;
        }
        L[r_][r_] = sqrt(s);
      } else {
        L[r_][c_] = s / L[c_][c_];
      }
    }
  if (okc) {
    double yv[6];
    for (int r_ = 0; r_ < 6; ++r_) {
      double s = -g[r_];
      for (int k = 0; k < r_; ++k) s -= L[r_][k] * yv[k];
      yv[r_] = s / L[r_][r_];
    }
    for (int r_ = 5; r_ >= 0; --r_) {
      double s = yv[r_];
      for (int k = r_ + 1; k < 6; ++k) s -= L[k][r_] * d[k];
      d[r_] = s / L[r_][r_];
    }
  }
  return okc;
}

// to = (exp([d0 d1 d2]x) from.R, from.t + (d3, d4, d5)) (Rodrigues); `to` may be `from`
__device__ __forceinline__ void apply_step(const Pose& from, const double* d, Pose& to) {
  const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  double E[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (th > 1e-16) {
    const double kx = d[0] / th, ky = d[1] / th, kz = d[2] / th;
    const double sn = sin(th), cs = 1.0 - cos(th);
    const double Kx[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
    double K2[9];
    for (int r_ = 0; r_ < 3; ++r_)
      for (int c_ = 0; c_ < 3; ++c_)
        K2[r_ * 3 + c_] = Kx[r_ * 3] * Kx[c_] + Kx[r_ * 3 + 1] * Kx[3 + c_] + Kx[r_ * 3 + 2] * Kx[6 + c_];
    for (int k = 0; k < 9; ++k) E[k] += sn * Kx[k] + cs * K2[k];
  }
  double Rn[9];
  for (int r_ = 0; r_ < 3; ++r_)
    for (int c_ = 0; c_ < 3; ++c_)
      Rn[r_ * 3 + c_] = E[r_ * 3] * from.R[c_] + E[r_ * 3 + 1] * from.R[3 + c_] + E[r_ * 3 + 2] * from.R[6 + c_];
  for (int k = 0; k < 9; ++k) to.R[k] = Rn[k];
  for (int k = 0; k < 3; ++k) to.t[k] = from.t[k] + d[3 + k];
}

// Least squares of the reprojection error over the matches with mask[i] set: up to 10 Gauss-Newton
// steps (normal equations reduced by the CTA, solved by thread 0) from `cur`.  Every thread calls
// it; on return `cur` and the shared `sh_pose` hold the result.
template <class Load>
__device__ __forceinline__ void least_squares_on_mask(Pose& cur, Pose& sh_pose, const Cam& cam, const Load& load_pt,
                                                      const unsigned char* mask, int n, double* red, double* Hs,
                                                      int& flag) {
  const int tid = threadIdx.x;
  for (int it = 0; it < 10; ++it) {
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) acc[k] = 0.0;
    for (int i = tid; i < n; i += kPnpThreads) {
      if (!mask[i]) continue;
      double p[3], u, v;
      load_pt(i, p, u, v);
      gn_terms<false>(cur, cam, p, u, v, acc, nullptr);
    }
    for (int k = 0; k < 27; ++k) {
      const double s = block_sum(acc[k], red);
      if (tid == 0) Hs[k] = s;
    }
    __syncthreads();
    if (tid == 0) {
      double d[6];
      double step = 0.0;
      const bool okc = solve_damped(Hs, 1e-9, d);
      if (okc) {
        apply_step(sh_pose, d, sh_pose);
        for (int k = 0; k < 6; ++k) step = fmax(step, fabs(d[k]));
      }
      flag = (!okc || step < 1e-12) ? 1 : 0;
    }
    __syncthreads();
    cur = sh_pose;
    const int stop = flag;
    __syncthreads();
    if (stop) break;
  }
}

// Support of a model in the COLMAP mode: inlier count, then the smaller sum of squared errors of
// the inliers, then the lower hypothesis id (so that the winner does not depend on scheduling).
struct Support {
  int count;
  double sse;
  unsigned h;
};
__device__ __forceinline__ bool better(const Support& a, const Support& b) {
  return a.count > b.count || (a.count == b.count && (a.sse < b.sse || (a.sse == b.sse && a.h < b.h)));
}

// kOpenCv: cv2.solvePnPRansac as the reference's default branch calls it (full K, err < thr, the
//   3D points multiplied by `scale`), then `refine_rounds` rounds of least squares on the inliers
//   with the inlier set re-evaluated between rounds.
// kColmap: pycolmap.absolute_pose_estimation as the reference's use_pycolmap_ransac branch calls it
//   (metric_utils.py:137-170): SIMPLE_PINHOLE camera (f = K[0][0], fy and skew ignored), inlier =
//   err <= thr and in front, support = (count, smaller SSE); LO-RANSAC: least squares on the
//   winner's inliers, kept while the support improves, for at most `refine_rounds` rounds; then the
//   pose is refined on that fixed inlier set with the Cauchy loss sum log(1 + |r_i|^2) per point
//   (IRLS Levenberg-Marquardt).  The mask is the RANSAC model's inlier set, before that refinement.
enum class PnpSolver { kOpenCv, kColmap };

template <PnpSolver kSolver>
__global__ void __launch_bounds__(kPnpThreads)
pnp_ransac_kernel(const float* __restrict__ pts3d, const float* __restrict__ pts2d,
                  const long long* __restrict__ m_bids, int M, const float* __restrict__ Kmat,
                  float scale, float thr, int n_hyp, unsigned seed, int refine_rounds,
                  float* __restrict__ pose_out, int* __restrict__ n_inl_out,
                  unsigned char* __restrict__ inl_mask, int* __restrict__ status_out) {
  constexpr bool kColmap = kSolver == PnpSolver::kColmap;
  pdl_sync();
  __shared__ int seg[2];
  __shared__ unsigned long long best_key[kPnpThreads / 32];
  __shared__ Pose best_pose;
  __shared__ double red[kPnpThreads / 32];
  __shared__ double Hs[27];
  __shared__ int flag;
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  // [lo, hi) = run of matches with m_bids == b (lower bounds of b and b + 1)
  if (tid < 2) {
    const long long key = b + tid;
    int lo = 0, hi = M;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (m_bids[mid] < key) lo = mid + 1; else hi = mid;
    }
    seg[tid] = lo;
  }
  __syncthreads();
  const int lo = seg[0], n = seg[1] - seg[0];
  const float* K = Kmat + b * 9;
  Cam cam{(double)K[0], (double)K[4], (double)K[2], (double)K[5], (double)K[1]};
  if constexpr (kColmap) cam = Cam{(double)K[0], (double)K[0], (double)K[2], (double)K[5], 0.0};
  const double thr2 = (double)thr * (double)thr;
  float* pose = pose_out + b * 12;
  auto fail = [&]() {
    if (tid < 12) pose[tid] = (tid == 0 || tid == 5 || tid == 10) ? 1.f : 0.f;
    if (tid == 0) {
      n_inl_out[b] = 0;
      status_out[b] = 0;
    }
    for (int i = tid; i < n; i += kPnpThreads) inl_mask[lo + i] = 0;
  };
  if (n < 4) {
    fail();
    return;
  }
  auto load_pt = [&](int i, double* p, double& u, double& v) {
    const float* q = pts3d + (long long)(lo + i) * 3;
    p[0] = (double)q[0] * scale;
    p[1] = (double)q[1] * scale;
    p[2] = (double)q[2] * scale;
    u = pts2d[(long long)(lo + i) * 2];
    v = pts2d[(long long)(lo + i) * 2 + 1];
  };

  // ---------------------------------------------------------------- 1+2: hypotheses and scoring
  int my_count = -1;
  double my_sse = INFINITY;
  unsigned my_h = 0xffffffffu;
  Pose my_pose;
  for (int h = tid; h < n_hyp; h += kPnpThreads) {
    int idx[4];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int pick = -1;
      for (int attempt = 0; attempt < 8 && pick < 0; ++attempt) {
        const uint32_t r = pnp_hash(seed ^ pnp_hash((uint32_t)b * 0x9E3779B9u + (uint32_t)h) ^
                                    ((uint32_t)(j * 8 + attempt + 1) * 0x85EBCA6Bu));
        const int cand = (int)(((unsigned long long)r * (unsigned long long)n) >> 32);
        bool dup = false;
        for (int k = 0; k < j; ++k) dup |= idx[k] == cand;
        if (!dup) pick = cand;
      }
      if (pick < 0) ok = false;
      idx[j] = pick < 0 ? 0 : pick;
    }
    if (!ok) continue;
    double P[3][3], f[3][3], p4[3], u4, v4;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double u, v;
      load_pt(idx[j], P[j], u, v);
      const double yn = (v - cam.cy) / cam.fy;
      const double xn = (u - cam.cx - cam.skew * yn) / cam.fx;
      f[j][0] = xn;
      f[j][1] = yn;
      f[j][2] = 1.0;
      normalize3(f[j]);
    }
    load_pt(idx[3], p4, u4, v4);
    Pose cand;
    double cand_err = INFINITY;
    p3p_grunert(P, f, [&](const Pose& ps) {
      const double e = reproj_err2(ps, cam, p4, u4, v4);
      if (e < cand_err) {
        cand_err = e;
        cand = ps;
      }
    });
    if (!(cand_err < INFINITY)) continue;
    int count = 0;
    double sse = 0.0;
    for (int i = 0; i < n; ++i) {
      double p[3], u, v;
      load_pt(i, p, u, v);
      const double e = reproj_err2(cand, cam, p, u, v);
      if constexpr (kColmap) {
        if (e <= thr2) {
          ++count;
          sse += e;
        }
      } else {
        count += e < thr2 ? 1 : 0;
      }
    }
    // strided h is increasing: the first best stays (lowest id on ties)
    if (count > my_count || (kColmap && count == my_count && sse < my_sse)) {
      my_count = count;
      my_sse = sse;
      my_h = (unsigned)h;
      my_pose = cand;
    }
  }
  if constexpr (kColmap) {
    // block argmax of the support (count, smaller sse, lower h)
    __shared__ Support w_best[kPnpThreads / 32];
    Support s{my_count, my_sse, my_h};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const Support other{__shfl_xor_sync(0xffffffffu, s.count, o), __shfl_xor_sync(0xffffffffu, s.sse, o),
                          __shfl_xor_sync(0xffffffffu, s.h, o)};
      if (better(other, s)) s = other;
    }
    if ((tid & 31) == 0) w_best[tid >> 5] = s;
    __syncthreads();
    Support best = w_best[0];
#pragma unroll
    for (int w = 1; w < kPnpThreads / 32; ++w)
      if (better(w_best[w], best)) best = w_best[w];
    if (best.count < 0) {   // no admissible hypothesis at all
      fail();
      return;
    }
    if (my_count >= 0 && my_h == best.h) best_pose = my_pose;   // h is unique
  } else {
    // block argmax of (count, lowest h)
    unsigned long long key = my_count < 0 ? 0ull
                                          : (((unsigned long long)(unsigned)my_count + 1ull) << 32) |
                                                (unsigned long long)(0xffffffffu - my_h);
    unsigned long long wkey = key;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, wkey, o);
      wkey = other > wkey ? other : wkey;
    }
    if ((tid & 31) == 0) best_key[tid >> 5] = wkey;
    __syncthreads();
    unsigned long long bkey = 0;
#pragma unroll
    for (int w = 0; w < kPnpThreads / 32; ++w) bkey = best_key[w] > bkey ? best_key[w] : bkey;
    if (bkey == 0ull) {   // no admissible hypothesis at all
      fail();
      return;
    }
    if (key == bkey) best_pose = my_pose;   // keys are unique (h is)
  }
  __syncthreads();
  Pose cur = best_pose;
  unsigned char* mask = inl_mask + lo;

  int n_inl = 0;
  if constexpr (kColmap) {
    // ---------------------------------------------------------------- 3: local optimisation
    // support of `ps` over the CTA (fixed-order sums), its inlier set written to the mask
    auto score = [&](const Pose& ps, int& cnt_out, double& sse_out) {
      int cnt = 0;
      double sse = 0.0;
      for (int i = tid; i < n; i += kPnpThreads) {
        double p[3], u, v;
        load_pt(i, p, u, v);
        const double e = reproj_err2(ps, cam, p, u, v);
        const unsigned char in = e <= thr2 ? 1 : 0;
        mask[i] = in;
        cnt += in;
        sse += in ? e : 0.0;
      }
      cnt_out = (int)(block_sum((double)cnt, red) + 0.5);
      sse_out = block_sum(sse, red);
    };
    double sse;
    score(cur, n_inl, sse);
    for (int round = 0; round < refine_rounds && n_inl >= 4; ++round) {
      __syncthreads();   // mask written by other threads is read below
      const Pose prev = cur;
      least_squares_on_mask(cur, best_pose, cam, load_pt, mask, n, red, Hs, flag);
      int cnt2;
      double sse2;
      score(cur, cnt2, sse2);
      if (cnt2 > n_inl || (cnt2 == n_inl && sse2 < sse)) {
        n_inl = cnt2;
        sse = sse2;
      } else {   // not better: back to the previous model and its inlier set
        cur = prev;
        score(cur, n_inl, sse);
        break;
      }
    }
    if (n_inl < 4) {
      fail();
      return;
    }
    // ---------------------------------------------------------------- 4: Cauchy refinement
    // weighted normal equations and cost sum log(1 + |r|^2) over the inliers at `ps` -> out[28]
    __shared__ double Hc[2][28];
    auto cauchy_terms = [&](const Pose& ps, double* out) {
      double acc[27], cost = 0.0;
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = 0.0;
      for (int i = tid; i < n; i += kPnpThreads) {
        if (!mask[i]) continue;
        double p[3], u, v;
        load_pt(i, p, u, v);
        gn_terms<true>(ps, cam, p, u, v, acc, &cost);
      }
      for (int k = 0; k < 27; ++k) {
        const double s = block_sum(acc[k], red);
        if (tid == 0) out[k] = s;
      }
      const double c = block_sum(cost, red);
      if (tid == 0) out[27] = c;
      __syncthreads();
    };
    __syncthreads();   // mask written by other threads is read below
    int buf = 0;
    cauchy_terms(cur, Hc[buf]);
    double cost = Hc[buf][27];
    double lambda = 1e-4;   // Levenberg-Marquardt damping, relative to diag H
    for (int it = 0; it < 100; ++it) {
      if (tid == 0) {
        double d[6];
        double step = 0.0;
        const bool okc = solve_damped(Hc[buf], lambda, d);
        if (okc) {
          apply_step(cur, d, best_pose);
          for (int k = 0; k < 6; ++k) step = fmax(step, fabs(d[k]));
        }
        flag = (!okc || step < 1e-12) ? 1 : 0;
      }
      __syncthreads();
      if (flag) break;
      const Pose trial = best_pose;
      cauchy_terms(trial, Hc[buf ^ 1]);
      const double c_new = Hc[buf ^ 1][27];
      if (c_new < cost) {   // accept; the normal equations at the new pose are already there
        const double rel = (cost - c_new) / cost;
        cur = trial;
        cost = c_new;
        buf ^= 1;
        lambda = fmax(lambda * 0.1, 1e-12);
        if (rel < 1e-12) break;
      } else {
        lambda *= 10.0;
        if (lambda > 1e12) break;
      }
    }
  } else {
    // ---------------------------------------------------------------- 3: refinement on the inliers
    for (int round = 0; round <= refine_rounds; ++round) {
      // inlier set under the current pose
      int cnt = 0;
      for (int i = tid; i < n; i += kPnpThreads) {
        double p[3], u, v;
        load_pt(i, p, u, v);
        const unsigned char in = reproj_err2(cur, cam, p, u, v) < thr2 ? 1 : 0;
        inl_mask[lo + i] = in;
        cnt += in;
      }
      n_inl = (int)(block_sum((double)cnt, red) + 0.5);
      if (round == refine_rounds || n_inl < 4) break;
      __syncthreads();   // inl_mask written by other threads is read below
      for (int it = 0; it < 10; ++it) {
        double acc[27];
  #pragma unroll
        for (int k = 0; k < 27; ++k) acc[k] = 0.0;
        for (int i = tid; i < n; i += kPnpThreads) {
          if (!inl_mask[lo + i]) continue;
          double p[3], u, v;
          load_pt(i, p, u, v);
          const double Y0 = cur.R[0] * p[0] + cur.R[1] * p[1] + cur.R[2] * p[2];
          const double Y1 = cur.R[3] * p[0] + cur.R[4] * p[1] + cur.R[5] * p[2];
          const double Y2 = cur.R[6] * p[0] + cur.R[7] * p[1] + cur.R[8] * p[2];
          const double x = Y0 + cur.t[0], y = Y1 + cur.t[1], z = Y2 + cur.t[2];
          if (!(z > 1e-9)) continue;
          const double iz = 1.0 / z, xn = x * iz, yn = y * iz;
          const double ru = cam.fx * xn + cam.skew * yn + cam.cx - u;
          const double rv = cam.fy * yn + cam.cy - v;
          // d(u)/dXc, d(v)/dXc
          const double gu[3] = {cam.fx * iz, cam.skew * iz, -(cam.fx * xn + cam.skew * yn) * iz};
          const double gv[3] = {0.0, cam.fy * iz, -cam.fy * yn * iz};
          // Xc = exp(w) Y + t  ->  dXc/dw = -[Y]x ; J row = (g x ... ) : g^T (-[Y]x) = (Y x g)^T
          const double Yv[3] = {Y0, Y1, Y2};
          double ju[6], jv[6];
          cross3(Yv, gu, ju);
          cross3(Yv, gv, jv);
  #pragma unroll
          for (int k = 0; k < 3; ++k) {
            ju[3 + k] = gu[k];
            jv[3 + k] = gv[k];
          }
          int o = 0;
  #pragma unroll
          for (int r_ = 0; r_ < 6; ++r_) {
  #pragma unroll
            for (int c_ = r_; c_ < 6; ++c_) acc[o++] += ju[r_] * ju[c_] + jv[r_] * jv[c_];
          }
  #pragma unroll
          for (int r_ = 0; r_ < 6; ++r_) acc[21 + r_] += ju[r_] * ru + jv[r_] * rv;
        }
        for (int k = 0; k < 27; ++k) {
          const double s = block_sum(acc[k], red);
          if (tid == 0) Hs[k] = s;
        }
        __syncthreads();
        if (tid == 0) {
          // solve (H + lambda diag H) d = -g by Cholesky
          double H[6][6], g[6], L[6][6], d[6];
          int o = 0;
          for (int r_ = 0; r_ < 6; ++r_)
            for (int c_ = r_; c_ < 6; ++c_) {
              H[r_][c_] = Hs[o];
              H[c_][r_] = Hs[o];
              ++o;
            }
          for (int r_ = 0; r_ < 6; ++r_) {
            g[r_] = Hs[21 + r_];
            H[r_][r_] *= 1.0 + 1e-9;
          }
          bool okc = true;
          for (int r_ = 0; r_ < 6 && okc; ++r_)
            for (int c_ = 0; c_ <= r_; ++c_) {
              double s = H[r_][c_];
              for (int k = 0; k < c_; ++k) s -= L[r_][k] * L[c_][k];
              if (r_ == c_) {
                if (!(s > 1e-300)) {
                  okc = false;
                  break;
                }
                L[r_][r_] = sqrt(s);
              } else {
                L[r_][c_] = s / L[c_][c_];
              }
            }
          double step = 0.0;
          if (okc) {
            double yv[6];
            for (int r_ = 0; r_ < 6; ++r_) {
              double s = -g[r_];
              for (int k = 0; k < r_; ++k) s -= L[r_][k] * yv[k];
              yv[r_] = s / L[r_][r_];
            }
            for (int r_ = 5; r_ >= 0; --r_) {
              double s = yv[r_];
              for (int k = r_ + 1; k < 6; ++k) s -= L[k][r_] * d[k];
              d[r_] = s / L[r_][r_];
            }
            // R <- exp(w) R (Rodrigues), t <- t + dt
            const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            double E[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
            if (th > 1e-16) {
              const double kx = d[0] / th, ky = d[1] / th, kz = d[2] / th;
              const double sn = sin(th), cs = 1.0 - cos(th);
              const double Kx[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
              double K2[9];
              for (int r_ = 0; r_ < 3; ++r_)
                for (int c_ = 0; c_ < 3; ++c_)
                  K2[r_ * 3 + c_] = Kx[r_ * 3] * Kx[c_] + Kx[r_ * 3 + 1] * Kx[3 + c_] + Kx[r_ * 3 + 2] * Kx[6 + c_];
              for (int k = 0; k < 9; ++k) E[k] += sn * Kx[k] + cs * K2[k];
            }
            double Rn[9];
            for (int r_ = 0; r_ < 3; ++r_)
              for (int c_ = 0; c_ < 3; ++c_)
                Rn[r_ * 3 + c_] = E[r_ * 3] * best_pose.R[c_] + E[r_ * 3 + 1] * best_pose.R[3 + c_] +
                                  E[r_ * 3 + 2] * best_pose.R[6 + c_];
            for (int k = 0; k < 9; ++k) best_pose.R[k] = Rn[k];
            for (int k = 0; k < 3; ++k) best_pose.t[k] += d[3 + k];
            for (int k = 0; k < 6; ++k) step = fmax(step, fabs(d[k]));
          }
          flag = (!okc || step < 1e-12) ? 1 : 0;
        }
        __syncthreads();
        cur = best_pose;
        const int stop = flag;
        __syncthreads();
        if (stop) break;
      }
    }
  }
  if (tid < 9) pose[(tid / 3) * 4 + tid % 3] = (float)cur.R[tid];
  if (tid < 3) pose[tid * 4 + 3] = (float)(cur.t[tid] / (double)scale);
  if (tid == 0) {
    n_inl_out[b] = n_inl;
    status_out[b] = n_inl >= 4 ? 1 : 0;
  }
}

}  // namespace opp

using namespace opp;

extern "C" int opp_pnp_ransac(const float* pts3d, const float* pts2d, const long long* m_bids, int m,
                              const float* intrinsics, int batch, float scale, float reproj_thr,
                              int hypotheses, unsigned seed, int refine_rounds, float* poses,
                              int* n_inliers, unsigned char* inlier_mask, int* status,
                              opp_stream_t stream) {
  OPP_REQUIRE(intrinsics && poses && n_inliers && status, "null pointer");
  OPP_REQUIRE(m == 0 || (pts3d && pts2d && m_bids && inlier_mask), "null match lists");
  OPP_REQUIRE(batch > 0 && hypotheses > 0 && scale > 0.f && reproj_thr > 0.f && refine_rounds >= 0,
              "bad pnp arguments");
  OPP_CHECK_CUDA(opp::launch_pdl(pnp_ransac_kernel<PnpSolver::kOpenCv>, dim3(batch), dim3(kPnpThreads), 0,
      (cudaStream_t)stream, pts3d, pts2d, m_bids, m, intrinsics, scale, reproj_thr, hypotheses, seed,
      refine_rounds, poses, n_inliers, inlier_mask, status));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

extern "C" int opp_pnp_ransac_colmap(const float* pts3d, const float* pts2d, const long long* m_bids, int m,
                                     const float* intrinsics, int batch, float max_error_px, int hypotheses,
                                     unsigned seed, int lo_rounds, float* poses, int* n_inliers,
                                     unsigned char* inlier_mask, int* status, opp_stream_t stream) {
  OPP_REQUIRE(intrinsics && poses && n_inliers && status, "null pointer");
  OPP_REQUIRE(m == 0 || (pts3d && pts2d && m_bids && inlier_mask), "null match lists");
  OPP_REQUIRE(batch > 0 && hypotheses > 0 && max_error_px > 0.f && lo_rounds >= 0, "bad pnp arguments");
  // the points are used as given (scale 1): pycolmap's call has no rescale
  OPP_CHECK_CUDA(opp::launch_pdl(pnp_ransac_kernel<PnpSolver::kColmap>, dim3(batch), dim3(kPnpThreads), 0,
      (cudaStream_t)stream, pts3d, pts2d, m_bids, m, intrinsics, 1.0f, max_error_px, hypotheses, seed,
      lo_rounds, poses, n_inliers, inlier_mask, status));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}
