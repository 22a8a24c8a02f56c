// opp_stages.cu — the bandwidth / latency bound stages of the 2D-3D matcher that are not GEMMs:
// first 7x7 conv (C_in = 1), bilinear x2 upsample + add, 3D keypoint encoding MLP, the
// linear-attention KV state, dual-softmax finalisers, mutual-NN selection + ordered compaction,
// fine-window gather, per-match linear attention and the correlation soft-argmax.
// Each kernel cites the reference code it replaces (paths relative to zju3dv/OnePose_Plus_Plus).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/opp_b200.h"
#include "opp_common.cuh"

namespace opp {
int num_sms();

constexpr int kC1Tile = 16;  // 16x16 output pixels per CTA of the conv1 im2col

// =============================================================================================
// conv1 as a tensor-core GEMM (backbone/resnet.py:101-103,143): the 7x7 stride-2 pad-3 window of
// every output pixel is written as one GEMM row  A[pixel][64] = (49 taps, 1.0, 0 x 14)  in fp16
// planes; the weight matrix W[c][64] = (49 folded-BN taps, folded bias, 0 x 14) then gives
// conv + bias as ONE 64-wide K chunk of the wgmma engine (opp_linear_act_f16 with ReLU), whose
// row-major output [pixel][planes*C] IS the NHWC feature map.  This kernel is the im2col: pure
// streaming (reads the image through a shared-memory patch, writes 128 B per pixel and plane,
// fully coalesced).  IMG_U8: the image is uint8 and  x = u8 / 255  (data_io.py:34-68 does the
// division on the host; folding it here lets callers upload 1 B instead of 4 B per pixel).
// =============================================================================================
template <bool IMG_U8>
__global__ void __launch_bounds__(256) conv1_im2col_kernel(const void* __restrict__ img_v,
                                                           __half* __restrict__ a_out, int H, int W,
                                                           int lo_off) {
  pdl_sync();
  constexpr int P = 2 * kC1Tile + 5;   // 37 x 37 input patch of a 16 x 16 output tile
  __shared__ float p_s[P * P];
  const int b = blockIdx.z;
  const int oy0 = blockIdx.y * kC1Tile, ox0 = blockIdx.x * kC1Tile;
  const int OH = H / 2, OW = W / 2;
  const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
  for (int i = threadIdx.x; i < P * P; i += 256) {
    const int py = i / P, px = i - py * P;
    const int y = iy0 + py, x = ix0 + px;
    float v = 0.f;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const long long o = ((long long)b * H + y) * W + x;
      if (IMG_U8) v = (float)reinterpret_cast<const uint8_t*>(img_v)[o] / 255.f;
      else v = reinterpret_cast<const float*>(img_v)[o];
    }
    p_s[i] = v;
  }
  __syncthreads();
  // thread -> (pixel, 8-column group): 8 consecutive lanes write one pixel's 128 B plane row
  const int g = threadIdx.x & 7;
  const int ld = lo_off ? 128 : 64;
#pragma unroll 1
  for (int pp = threadIdx.x >> 3; pp < kC1Tile * kC1Tile; pp += 32) {
    const int ly = pp / kC1Tile, lx = pp - ly * kC1Tile;
    const int oy = oy0 + ly, ox = ox0 + lx;
    if (oy >= OH || ox >= OW) continue;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = g * 8 + j;
      const int ky = col / 7, kx = col - ky * 7;
      v[j] = col < 49 ? p_s[(2 * ly + ky) * P + 2 * lx + kx] : (col == 49 ? 1.f : 0.f);
    }
    store_split8(a_out + (((long long)b * OH + oy) * OW + ox) * ld, g * 8, v, lo_off ? 64 : 0);
  }
}

// =============================================================================================
// 3D keypoint normalisation statistics   (utils/normalize.py:16-26)
// stats[b] = (mean xyz over points of batch b, 0.6 * max extent of batch element 0)
// =============================================================================================
__global__ void __launch_bounds__(256) kpt_stats_kernel(const float* __restrict__ kpts,
                                                        float* __restrict__ stats, int n) {
  pdl_sync();
  __shared__ float red[9][256];
  const int b = blockIdx.x;
  const float* k0 = kpts;                        // batch element 0 for the extents
  const float* kb = kpts + (long long)b * n * 3;
  float s[3] = {0.f, 0.f, 0.f}, mn[3] = {INFINITY, INFINITY, INFINITY},
        mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = threadIdx.x; i < n; i += 256) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      s[a] += kb[i * 3 + a];
      const float v = k0[i * 3 + a];
      mn[a] = fminf(mn[a], v);
      mx[a] = fmaxf(mx[a], v);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    red[a][threadIdx.x] = s[a];
    red[3 + a][threadIdx.x] = mn[a];
    red[6 + a][threadIdx.x] = mx[a];
  }
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        red[a][threadIdx.x] += red[a][threadIdx.x + st];
        red[3 + a][threadIdx.x] = fminf(red[3 + a][threadIdx.x], red[3 + a][threadIdx.x + st]);
        red[6 + a][threadIdx.x] = fmaxf(red[6 + a][threadIdx.x], red[6 + a][threadIdx.x + st]);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float ext = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      stats[b * 4 + a] = red[a][0] / (float)n;
      ext = fmaxf(ext, red[6 + a][0] - red[3 + a][0]);
    }
    stats[b * 4 + 3] = ext * 0.6f;
  }
}

// =============================================================================================
// KeypointEncoding_linear   (utils/position_encoding.py:46-79 with norm_method "instancenorm":
// InstanceNorm1d on [B, N, C] normalises over the C features of each point, biased variance,
// eps 1e-5, no affine), then  tokens = descriptors^T + encoding.
// 32 points per CTA; activations ping-pong through shared memory; weights read transposed.
// =============================================================================================
constexpr int kKeP = 16;

template <int CIN, int COUT>
__device__ __forceinline__ void kpt_layer(const float* __restrict__ in_s,  // [kKeP][CIN]
                                          float* __restrict__ out_s,       // [kKeP][COUT+1]
                                          const float* __restrict__ w_t,   // [CIN][COUT]
                                          const float* __restrict__ bias, bool norm_relu) {
  // thread -> output channel c = tid % COUT, point group g = tid / COUT
  constexpr int PG = 256 / COUT > 0 ? 256 / COUT : 1;          // point groups in flight
  constexpr int CPT = COUT > 256 ? COUT / 256 : 1;             // channels per thread (COUT<=256)
  static_assert(CPT == 1, "COUT <= 256");
  const int c = threadIdx.x % COUT;
  const int g = threadIdx.x / COUT;
  if (g < PG) {
    for (int p = g; p < kKeP; p += PG) {
      float acc = bias[c];
      for (int k = 0; k < CIN; ++k) acc = fmaf(in_s[p * CIN + k], w_t[k * COUT + c], acc);
      out_s[p * (COUT + 1) + c] = acc;
    }
  }
  __syncthreads();
  if (norm_relu) {
    // one warp per point at a time: mean / biased variance over COUT channels
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int p = warp; p < kKeP; p += 8) {
      float* row = out_s + p * (COUT + 1);
      float s = 0.f;
      for (int k = lane; k < COUT; k += 32) s += row[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s / (float)COUT;
      float q = 0.f;
      for (int k = lane; k < COUT; k += 32) {
        const float d = row[k] - mean;
        q = fmaf(d, d, q);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = 1.f / sqrtf(q / (float)COUT + 1e-5f);
      for (int k = lane; k < COUT; k += 32) row[k] = fmaxf((row[k] - mean) * rstd, 0.f);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
kpt_encode_kernel(const float* __restrict__ kpts, const float* __restrict__ stats,
                  const float* __restrict__ desc, const float* __restrict__ w1_t,
                  const float* __restrict__ b1, const float* __restrict__ w2_t,
                  const float* __restrict__ b2, const float* __restrict__ w3_t,
                  const float* __restrict__ b3, const float* __restrict__ w4_t,
                  const float* __restrict__ b4, __half* __restrict__ tok, int n, int lo_off) {
  pdl_sync();
  __shared__ float buf_a[kKeP * 129];   // holds [P][3], [P][64+1] ... reused
  __shared__ float buf_b[kKeP * 257];
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * kKeP;
  const float cx = stats[b * 4 + 0], cy = stats[b * 4 + 1], cz = stats[b * 4 + 2];
  const float sc = stats[b * 4 + 3];
  // normalised keypoints -> buf_b as [P][3]
  if (threadIdx.x < kKeP * 3) {
    const int p = threadIdx.x / 3, a = threadIdx.x % 3;
    const int gp = p0 + p;
    float v = 0.f;
    if (gp < n) {
      const float c = a == 0 ? cx : (a == 1 ? cy : cz);
      v = (kpts[((long long)b * n + gp) * 3 + a] - c) / sc;
    }
    buf_b[p * 3 + a] = v;
  }
  __syncthreads();
  // layer outputs are stored with row stride COUT+1; the next layer reads with stride CIN, so
  // compact in place between layers.
  kpt_layer<3, 32>(buf_b, buf_a, w1_t, b1, true);     // buf_a [P][33]
  for (int i = threadIdx.x; i < kKeP * 32; i += 256) buf_b[i] = buf_a[(i / 32) * 33 + (i % 32)];
  __syncthreads();
  kpt_layer<32, 64>(buf_b, buf_a, w2_t, b2, true);    // buf_a [P][65]
  for (int i = threadIdx.x; i < kKeP * 64; i += 256) buf_b[i] = buf_a[(i / 64) * 65 + (i % 64)];
  __syncthreads();
  kpt_layer<64, 128>(buf_b, buf_a, w3_t, b3, true);   // buf_a [P][129]
  __syncthreads();
  // last layer reads buf_a with stride 129
  {
    const int c = threadIdx.x;  // 256 output channels
    for (int p = 0; p < kKeP; ++p) {
      float acc = b4[c];
      const float* row = buf_a + p * 129;
      for (int k = 0; k < 128; ++k) acc = fmaf(row[k], w4_t[k * 256 + c], acc);
      buf_b[p * 257 + c] = acc;
    }
  }
  __syncthreads();
  // add descriptors (read [B][256][N] coalesced along n), then write token-major
  {
    const int pl = threadIdx.x % kKeP, cgp = threadIdx.x / kKeP;  // 256/kKeP channel groups
    const int gp = p0 + pl;
    if (gp < n)
      for (int c = cgp; c < 256; c += 256 / kKeP)
        buf_b[pl * 257 + c] += desc[((long long)b * 256 + c) * n + gp];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kKeP * 256; i += 256) {
    const int p = i / 256, c = i % 256;
    const int gp = p0 + p;
    if (gp < n)
      store_split1(tok + ((long long)b * n + gp) * (lo_off ? 512 : 256), c, buf_b[p * 257 + c], lo_off);
  }
}

// =============================================================================================
// Linear-attention source state   (loftr_module/linear_attention.py:55-57)
// part[b][chunk][h][d][v] = sum_{s in chunk} K'[s,h,d] V[s,h,v];  row d = 32 holds sum_s K'[s,h,:]
// =============================================================================================
constexpr int kKvChunk = 256;   // tokens per CTA (128 -> 256: half the partial-state traffic of kv_finalize)

// ---------------------------------------------------------------------------------------------
// Per head the state is a 32x32 GEMM over the tokens of the chunk, KV[d][v] = sum_t K'[t][d] V[t][v]:
// M = d, N = v, K = token.  The tile is far too small for the wgmma engine (M = 128 would compute 8x the
// needed head blocks and wants token-major operands transposed), so each warp (= head) runs
// mma.sync m16n8k16 on fragments fetched with ldmatrix.trans straight from the token-major rows:
// the kernel is a pure stream over kv16 (1 KB per token: one fp16 plane, whatever the operand mode
// of the projections) and should sit on the HBM roofline instead of the shared-memory/FMA issue
// limit of the SIMT version.
//   ksum:  one extra n-tile whose B fragment is the constant 1.0 (no loads): C[d][*] = sum_t K'[t][d]
// Rows are staged by cp.async (16 B, zero-filled past the end of the sequence) into a 3-stage
// ring of 16-token slabs; the 16 B row padding makes the 8 row addresses of every ldmatrix 8x8
// block fall into distinct bank groups.
// ---------------------------------------------------------------------------------------------
constexpr int kKvmTok = 16;     // tokens per pipeline stage = one k16 MMA step
constexpr int kKvmStages = 3;
constexpr int kKvmRowB = 1024;  // [K'(256) V(256)] fp16
constexpr int kKvmStride = kKvmRowB + 16;
constexpr int kKvmSmem = kKvmStages * kKvmTok * kKvmStride;

__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                          uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
      "{%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(256) kv_partial_mma_kernel(const __half* __restrict__ kv16,
                                                             float* __restrict__ part, int S,
                                                             int kv_chunk) {
  pdl_sync();
  extern __shared__ __align__(16) uint8_t kvm_smem[];
  constexpr int kStageB = kKvmTok * kKvmStride;
  constexpr int kUnitsPerRow = kKvmRowB / 16;
  constexpr int kUnits = kKvmTok * kUnitsPerRow;   // 16-byte units per stage
  const int chunk = blockIdx.x, b = blockIdx.y, chunks = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s0 = chunk * kv_chunk;
  const int cnt = min(kv_chunk, S - s0);
  const int nsteps = (cnt + kKvmTok - 1) / kKvmTok;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(kv16) + ((long long)b * S + s0) * kKvmRowB;
  const uint32_t sbase = smem_u32(kvm_smem);

  auto load_stage = [&](int step) {
    if (step < nsteps) {
      const uint32_t st = sbase + (step % kKvmStages) * kStageB;
      const int t0 = step * kKvmTok;
#pragma unroll
      for (int j = 0; j < kUnits / 256; ++j) {
        const int u = threadIdx.x + j * 256;
        const int t = u / kUnitsPerRow, o = (u % kUnitsPerRow) * 16;
        const bool ok = t0 + t < cnt;
        cp_async16_zfill(st + t * kKvmStride + o, src + (long long)(ok ? t0 + t : 0) * kKvmRowB + o,
                         ok ? 16 : 0);
      }
    }
    cp_async_commit();   // an empty group keeps the wait_group arithmetic uniform
  };

  float acc[2][4][4], ks[2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) ks[mt][i] = 0.f;
  }
  // ldmatrix row addresses of this lane: matrix q = lane / 8, row r = lane % 8
  const int q = lane >> 3, r = lane & 7;
  //   A (K', M = d): q -> (token half q >> 1, d half q & 1)
  const uint32_t a_off = (uint32_t)(((q >> 1) * 8 + r) * kKvmStride + (warp * 32 + (q & 1) * 8) * 2);
  //   B (V, N = v):  q -> (token half q & 1, n-tile q >> 1 of the pair)
  const uint32_t b_off = (uint32_t)(((q & 1) * 8 + r) * kKvmStride + (256 + warp * 32 + (q >> 1) * 8) * 2);
  const uint32_t ones = 0x3C003C00u;   // half2(1, 1)

  load_stage(0);
  load_stage(1);
  for (int step = 0; step < nsteps; ++step) {
    load_stage(step + 2);
    cp_async_wait<2>();
    __syncthreads();
    const uint32_t st = sbase + (step % kKvmStages) * kStageB;
    uint32_t ah[2][4], bh[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) ldsm_x4_trans(ah[mt], st + a_off + mt * 32);
#pragma unroll
    for (int np = 0; np < 2; ++np) ldsm_x4_trans(bh[np], st + b_off + np * 32);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int np = nt >> 1, o = (nt & 1) * 2;
        mma_16816(acc[mt][nt], ah[mt], bh[np][o], bh[np][o + 1]);
      }
      mma_16816(ks[mt], ah[mt], ones, ones);
    }
    __syncthreads();   // the slab is refilled by the load issued at the top of the next iteration
  }
  cp_async_wait<0>();
  // C fragment: c0,c1 = (row g, cols 2tg, 2tg+1), c2,c3 = (row g + 8, same cols)
  const int g = lane >> 2, tg = lane & 3;
  float* dst = part + ((((long long)b * chunks + chunk) * 8 + warp) * 33) * 32;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      *reinterpret_cast<float2*>(dst + (mt * 16 + g) * 32 + nt * 8 + 2 * tg) =
          make_float2(acc[mt][nt][0], acc[mt][nt][1]);
      *reinterpret_cast<float2*>(dst + (mt * 16 + g + 8) * 32 + nt * 8 + 2 * tg) =
          make_float2(acc[mt][nt][2], acc[mt][nt][3]);
    }
    if (tg == 0) {
      dst[32 * 32 + mt * 16 + g] = ks[mt][0];
      dst[32 * 32 + mt * 16 + g + 8] = ks[mt][2];
    }
  }
}

// mt[b][c][h*32+dd] = sum_v merge_w[c][h*32+v] * KV[b][h][dd][v] / v_len ; ksum[b][h*32+dd]
// (transformer.py:85 `merge` folded into the per-image KV state)
__global__ void __launch_bounds__(1024) kv_finalize_kernel(const float* __restrict__ part,
                                                          const float* __restrict__ merge_w,
                                                          __half* __restrict__ mt,
                                                          float* __restrict__ ksum, int chunks,
                                                          int d, float inv_vlen, int lo_off) {
  pdl_sync();
  __shared__ float kv_s[33][33];
  const int h = blockIdx.x, b = blockIdx.y, H = gridDim.x;
  // chunk partials are 33.8 KB apart: keep 8 loads in flight per element (a plain loop serialised
  // ~40 DRAM/L2 round trips per thread and made this tiny kernel cost as much as a GEMM)
  const long long cstride = (long long)H * 33 * 32;
  const float* pbase = part + (((long long)b * chunks) * H + h) * 33 * 32;
  for (int i = threadIdx.x; i < 33 * 32; i += 1024) {   // 1024 threads: one pass for 1056 elements
    float acc8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int c = 0;
    for (; c + 8 <= chunks; c += 8) {
#pragma unroll
      for (int u = 0; u < 8; ++u) acc8[u] += pbase[(c + u) * cstride + i];
    }
    for (; c < chunks; ++c) acc8[0] += pbase[c * cstride + i];
    kv_s[i / 32][i % 32] = ((acc8[0] + acc8[1]) + (acc8[2] + acc8[3])) + ((acc8[4] + acc8[5]) + (acc8[6] + acc8[7]));
  }
  __syncthreads();
  if (threadIdx.x < 32) ksum[(long long)b * d + h * 32 + threadIdx.x] = kv_s[32][threadIdx.x];
  // thread (c, g): output row c of the merge-folded state, columns h*32 + 8g .. +7
  {
    const int c = threadIdx.x & 255, g = threadIdx.x >> 8;
    if (c < d) {
      float w[32];
      const float4* wp = reinterpret_cast<const float4*>(merge_w + (long long)c * d + h * 32);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 t = wp[q];
        w[4 * q] = t.x;
        w[4 * q + 1] = t.y;
        w[4 * q + 2] = t.z;
        w[4 * q + 3] = t.w;
      }
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float sacc = 0.f;
#pragma unroll
        for (int v = 0; v < 32; ++v) sacc = fmaf(w[v], kv_s[g * 8 + j][v], sacc);
        o[j] = sacc * inv_vlen;
      }
      store_split8(mt + ((long long)b * d + c) * (lo_off ? 2 * d : d), h * 32 + g * 8, o, lo_off);
    }
  }
}

// =============================================================================================
// dual-softmax finalisers   (utils/coarse_matching.py:115,157-165)
// =============================================================================================
__global__ void lse_finalize_kernel(const float* __restrict__ pm, const float* __restrict__ ps,
                                    float* __restrict__ lse, long long rows, int tiles) {
  pdl_sync();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float m = -INFINITY;
  for (int t = 0; t < tiles; ++t) m = fmaxf(m, pm[r * tiles + t]);
  float s = 0.f;
  for (int t = 0; t < tiles; ++t) s += ps[r * tiles + t] * expf(pm[r * tiles + t] - m);
  lse[r] = m + logf(s);
}

// column side of opp_sim_lse_cols: lse[b][s] = logsumexp over the row groups of (col_m, col_s).
// Block = 32 columns x kLseColSlices group slices (coalesced 128 B rows; that many independent load
// chains per column instead of one thread walking all ~150 groups: the first form took 63 us for
// ONE image, 8 slices 22 us), merged through shared memory.
constexpr int kLseColSlices = 32;
__global__ void __launch_bounds__(32 * kLseColSlices) lse_col_finalize_kernel(const float* __restrict__ cm,
                                                               const float* __restrict__ cs,
                                                               float* __restrict__ lse, int batches,
                                                               int groups, int cols,
                                                               const unsigned char* __restrict__ col_mask) {
  pdl_sync();
  __shared__ float m_s[kLseColSlices][32], s_s[kLseColSlices][32];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int sidx = blockIdx.x * 32 + lane;
  float m = -INFINITY, sum = 0.f;
  if (sidx < cols) {
    const float* pm = cm + (long long)b * groups * cols + sidx;
    const float* ps = cs + (long long)b * groups * cols + sidx;
    for (int g = slice; g < groups; g += kLseColSlices) {
      const float pg = pm[(long long)g * cols];
      if (pg == -INFINITY) continue;
      const float sg = ps[(long long)g * cols];
      if (pg > m) {
        sum = sum * expf(m - pg) + sg;
        m = pg;
      } else {
        sum += sg * expf(pg - m);
      }
    }
  }
  m_s[slice][lane] = m;
  s_s[slice][lane] = sum;
  __syncthreads();
  if (slice == 0 && sidx < cols) {
    const long long idx = (long long)b * cols + sidx;
    if (col_mask && col_mask[idx] == 0) {
      // padded query cell: every sim of this column is -1e9, so conf = 0 whatever the row
      // (coarse_matching.py:108-115); +inf makes exp((2 sim - lse_pt) - lse_px) exactly 0
      lse[idx] = INFINITY;
      return;
    }
    float mm = -INFINITY;
#pragma unroll
    for (int k = 0; k < kLseColSlices; ++k) mm = fmaxf(mm, m_s[k][lane]);
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < kLseColSlices; ++k)
      if (m_s[k][lane] != -INFINITY) tot += s_s[k][lane] * expf(m_s[k][lane] - mm);
    lse[idx] = mm + logf(tot);
  }
}

__global__ void best_finalize_kernel(const float* __restrict__ pv, const int* __restrict__ pi,
                                     float* __restrict__ bv, int* __restrict__ bi, long long rows,
                                     int tiles) {
  pdl_sync();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float best = pv[r * tiles];
  int idx = pi[r * tiles];
  for (int t = 1; t < tiles; ++t) {
    const float v = pv[r * tiles + t];
    const int vi = pi[r * tiles + t];
    if (v > best || (v == best && vi < idx)) {   // ties -> lowest index, whatever the slot order
      best = v;
      idx = vi;
    }
  }
  bv[r] = best;
  bi[r] = idx;
}

// =============================================================================================
// match selection + ordered compaction   (utils/coarse_matching.py:142-172, 223-239)
//   keep (b, l) iff conf_max > thr, argmax cell j not in the top/left border (mask_border only
//   clears rows < b and cols < b: coarse_matching.py:10-20), and l is a column maximum of j.
// =============================================================================================
// The mutual test is expressed on values: row i keeps its argmax cell j iff its
// row maximum IS the column maximum of j (colmax holds the float bits written by EpiConfCol from
// the very same conf values, so the comparison is exact; coarse_matching.py:157-165 compares
// conf == conf.max(dim) the same way, so every row of an exact tie is kept).
// kRows (bank sets): rows i >= row_count[b] are the padding of the frame's object and never match.
template <bool kRows = false>
__device__ __forceinline__ bool match_flag_colmax(const float* pt_val, const int* pt_idx,
                                                  const unsigned* colmax, long long r, int l, int s,
                                                  int wc, float thr, int border,
                                                  const int* row_count = nullptr) {
  if constexpr (kRows) {
    const long long b = r / l;
    if (r - b * l >= row_count[b]) return false;
  }
  const float v = pt_val[r];
  if (!(v > thr)) return false;
  const int j = pt_idx[r];
  const int jy = j / wc, jx = j - jy * wc;
  if (jy < border || jx < border) return false;
  const long long b = r / l;
  return colmax[b * s + j] == __float_as_uint(v);
}

template <bool kRows>
__global__ void __launch_bounds__(1024) match_count_colmax_kernel(const float* pt_val,
                                                                  const int* pt_idx,
                                                                  const unsigned* colmax,
                                                                  long long rows, int l, int s, int wc,
                                                                  float thr, int border,
                                                                  int* block_counts,
                                                                  const int* row_count) {
  pdl_sync();
  const long long r = (long long)blockIdx.x * 1024 + threadIdx.x;
  const bool f = r < rows && match_flag_colmax<kRows>(pt_val, pt_idx, colmax, r, l, s, wc, thr, border,
                                                      row_count);
  const int c = __syncthreads_count(f);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// single block: exclusive scan of block_counts in place; total -> counts[nblocks] and count_out
__global__ void __launch_bounds__(1024) match_scan_kernel(int* counts, int nblocks,
                                                          int* count_out) {
  pdl_sync();
  __shared__ int warp_sums[32];
  __shared__ int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nblocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nblocks ? counts[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = warp_sums[threadIdx.x];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, w, o);
        if (threadIdx.x >= o) w += y;
      }
      warp_sums[threadIdx.x] = w;
    }
    __syncthreads();
    const int warp_off = (threadIdx.x >> 5) > 0 ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
    const int incl = x + warp_off + carry_s;
    if (i < nblocks) counts[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[nblocks] = carry_s;
    *count_out = carry_s;
  }
}

// kSet (bank sets): kpts is [K][l][3], read at bank_of_batch[b]; rows past row_count[b] are skipped
template <bool kSet>
__global__ void __launch_bounds__(1024)
match_scatter_colmax_kernel(const float* pt_val, const int* pt_idx, const unsigned* px_idx, const float* kpts,
                     const float* img_scale, long long rows, int l, int s, int wc, float thr,
                     int border, float cell, const int* block_offsets, long long* b_ids,
                     long long* i_ids, long long* j_ids, float* mconf, float* mkpts3d,
                     float* mkpts_c, int kpts_shared, const int* bank_of_batch, const int* row_count) {
  pdl_sync();
  __shared__ int warp_sums[32];
  const long long r = (long long)blockIdx.x * 1024 + threadIdx.x;
  const bool f = r < rows && match_flag_colmax<kSet>(pt_val, pt_idx, px_idx, r, l, s, wc, thr, border,
                                                     row_count);
  const unsigned ballot = __ballot_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_sums[warp] = __popc(ballot);
  __syncthreads();
  if (warp == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  if (!f) return;
  const int pos = block_offsets[blockIdx.x] + (warp > 0 ? warp_sums[warp - 1] : 0) +
                  __popc(ballot & ((1u << lane) - 1u));
  const long long b = r / l;
  const int i = (int)(r - b * l);
  const int j = pt_idx[r];
  b_ids[pos] = b;
  i_ids[pos] = i;
  j_ids[pos] = j;
  mconf[pos] = pt_val[r];
  long long kb = kpts_shared ? 0 : b;
  if constexpr (kSet) kb = bank_of_batch[b];
  const float* kp = kpts + (kb * l + i) * 3;
  mkpts3d[pos * 3 + 0] = kp[0];
  mkpts3d[pos * 3 + 1] = kp[1];
  mkpts3d[pos * 3 + 2] = kp[2];
  // coarse_matching.py:223-229: [j % w, j // w] * (scale * query_image_scale[b][[1, 0]])
  float sx = cell, sy = cell;
  if (img_scale) {
    sx = cell * img_scale[b * 2 + 1];
    sy = cell * img_scale[b * 2 + 0];
  }
  mkpts_c[pos * 2 + 0] = (float)(j % wc) * sx;
  mkpts_c[pos * 2 + 1] = (float)(j / wc) * sy;
}

// =============================================================================================
// fine window gather   (loftr_module/fine_preprocess.py:41-55)
// =============================================================================================
// kSet (bank sets): desc3d is [K][128][n], read at the frame's object bank_of_batch[b]
template <bool kSet>
__global__ void __launch_bounds__(128) fine_gather_kernel(
    const __half* __restrict__ fine, const float* __restrict__ desc3d,
    const long long* __restrict__ b_ids, const long long* __restrict__ i_ids,
    const long long* __restrict__ j_ids, float* __restrict__ x32, __half* __restrict__ x16, int hf,
    int wf, int wc, int stride, int n, int lo_off, int desc_shared, int windows,
    const int* __restrict__ count_dev, const int* __restrict__ bank_of_batch) {
  pdl_sync();
  const int m = blockIdx.x, c = threadIdx.x;
  if (count_dev && m >= *count_dev) return;   // launched at capacity, match count on the device
  const long long b = b_ids[m], i = i_ids[m], j = j_ids[m];
  const int jy = (int)(j / wc), jx = (int)(j - (long long)jy * wc);
  const long long row0 = (long long)m * 26;
  const int ld = lo_off ? 256 : 128;
  long long db = desc_shared ? 0 : b;
  if constexpr (kSet) db = bank_of_batch[b];
  const float d = desc3d[(db * 128 + c) * n + i];
  if (x32) x32[row0 * 128 + c] = d;
  store_split1(x16 + row0 * ld, c, d, lo_off);
  // windows (= row pitch P, opp_conv_win_pitch): `fine` holds the compact per-match windows of opp_conv_win, [m][5][P][ld]
  const __half* fb = windows ? fine + (long long)m * 5 * windows * ld : fine + b * hf * wf * ld;
  // all 25 window loads in flight before the first store (one block per match: the dependent
  // load -> store pairs of the rolled loop were 25 serial round trips)
  float v[25];
#pragma unroll
  for (int ww = 0; ww < 25; ++ww) {
    const int y = jy * stride + ww / 5 - 2, x = jx * stride + ww % 5 - 2;
    v[ww] = 0.f;
    if (y >= 0 && y < hf && x >= 0 && x < wf)
      v[ww] = load_split1(fb + (windows ? (long long)((ww / 5) * windows + ww % 5) : (long long)y * wf + x) * ld, c, lo_off);
  }
#pragma unroll
  for (int ww = 0; ww < 25; ++ww) {
    if (x32) x32[(row0 + 1 + ww) * 128 + c] = v[ww];
    store_split1(x16 + (row0 + 1 + ww) * ld, c, v[ww], lo_off);
  }
}

// =============================================================================================
// per-match linear attention, 1 + 25 tokens, 8 heads x 16   (linear_attention.py:29-61)
// The v/v_length ... * v_length pair of the reference cancels exactly and is omitted.
// =============================================================================================
__global__ void __launch_bounds__(128) fine_attention_kernel(const __half* __restrict__ qkv,
                                                             __half* __restrict__ msg, int cross,
                                                             float eps, int lo_off_in,
                                                             int lo_off_out,
                                                             const int* __restrict__ count_dev) {
  pdl_sync();
  if (count_dev && (int)blockIdx.x >= *count_dev) return;
  // Rows are fetched with 16-byte global loads, operands every lane of a head shares are read as
  // float4 broadcasts, and the window state column each thread owns stays in registers (32-bit
  // shared loads of shared values and re-reading the state from shared memory made the kernel
  // bound by shared-memory instructions).
  __shared__ __align__(16) float q_s[26][128];
  __shared__ __align__(16) float k_s[26][128];
  __shared__ __align__(16) float v_s[26][128];
  __shared__ __align__(16) float ks2[128];
  const int m = blockIdx.x, c = threadIdx.x;
  const int ldi = lo_off_in ? 768 : 384;
  const __half* src = qkv + (long long)m * 26 * ldi;
  for (int i = c; i < 26 * 48; i += 128) {
    const int t = i / 48, sg = i - t * 48;
    float f[8];
    load_split8(src + (long long)t * ldi, sg * 8, f, lo_off_in);
    const int col = sg * 8;   // 0..383: q | k | v, 128 each
    float* dstrow = col < 128 ? &q_s[t][col] : (col < 256 ? &k_s[t][col - 128] : &v_s[t][col - 256]);
    reinterpret_cast<float4*>(dstrow)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(dstrow)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  __syncthreads();
  const int h = c >> 4;
  // window state: thread (h, v) owns column v of head h:  col[dd] = sum_t K'[t, h, dd] V[t, h, v]
  float col[16];
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) col[dd] = 0.f;
  float ksum_c = 0.f;  // thread c also owns ks2[c]
  for (int t = 1; t < 26; ++t) {
    const float vv = v_s[t][c];
    const float4* kr = reinterpret_cast<const float4*>(&k_s[t][h * 16]);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 k4 = kr[g];
      col[4 * g + 0] = fmaf(k4.x, vv, col[4 * g + 0]);
      col[4 * g + 1] = fmaf(k4.y, vv, col[4 * g + 1]);
      col[4 * g + 2] = fmaf(k4.z, vv, col[4 * g + 2]);
      col[4 * g + 3] = fmaf(k4.w, vv, col[4 * g + 3]);
    }
    ksum_c += k_s[t][c];
  }
  ks2[c] = ksum_c;
  __syncthreads();
  float ksw[16], k0[16];   // window Ksum and the 3D token's K' of this head
  {
    const float4* a = reinterpret_cast<const float4*>(&ks2[h * 16]);
    const float4* b = reinterpret_cast<const float4*>(&k_s[0][h * 16]);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 x = a[g], y = b[g];
      ksw[4 * g] = x.x; ksw[4 * g + 1] = x.y; ksw[4 * g + 2] = x.z; ksw[4 * g + 3] = x.w;
      k0[4 * g] = y.x; k0[4 * g + 1] = y.y; k0[4 * g + 2] = y.z; k0[4 * g + 3] = y.w;
    }
  }
  const float v0 = v_s[0][c];
  float o[26];
#pragma unroll
  for (int t = 0; t < 26; ++t) {
    // which source state does token t read?  self: own sequence; cross: the other one
    const bool use_window = cross ? (t == 0) : (t > 0);
    const float4* qr = reinterpret_cast<const float4*>(&q_s[t][h * 16]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 q4 = qr[g];
      const float qv[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (use_window) {
          num = fmaf(qv[j], col[4 * g + j], num);
          den = fmaf(qv[j], ksw[4 * g + j], den);
        } else {   // source is the single 3D token (row 0): KV = k0^T v0, Ksum = k0
          den = fmaf(qv[j], k0[4 * g + j], den);
        }
      }
    }
    if (!use_window) num = den * v0;
    o[t] = num / (den + eps);
  }
  __syncthreads();   // every read of q_s is done: reuse it as the output tile
#pragma unroll
  for (int t = 0; t < 26; ++t) q_s[t][c] = o[t];
  __syncthreads();
  const int ldo = lo_off_out ? 256 : 128;
  __half* dst = msg + (long long)m * 26 * ldo;
  for (int i = c; i < 26 * 16; i += 128) {
    const int t = i >> 4, sg = i & 15;
    float f[8];
    const float4 a = reinterpret_cast<const float4*>(&q_s[t][sg * 8])[0];
    const float4 b = reinterpret_cast<const float4*>(&q_s[t][sg * 8])[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
    f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    store_split8(dst + (long long)t * ldo, sg * 8, f, lo_off_out);
  }
}

// =============================================================================================
// FullAttention.forward   (loftr_module/linear_attention.py:64-95): softmax(Q K^T / sqrt(D)) V per
// head.  Selected by `attention: "full"` in the transformer config — never by a shipped
// configuration (cold path), so this is a plain fp32 SIMT kernel: one thread per query row with an
// online softmax over 64-key tiles staged in shared memory; no S x L matrix is materialised.
//   q   fp16 [B][L][planes*(H*D)]           (q_proj output)
//   kv  fp16 [B][S][planes*(2*H*D)]         (k_proj | v_proj outputs)
//   out fp16 [B][L][planes*(H*D)]
// =============================================================================================
constexpr int kFaKeys = 64;

template <int D>
__global__ void __launch_bounds__(128) full_attention_kernel(const __half* __restrict__ q,
                                                             const __half* __restrict__ kv,
                                                             __half* __restrict__ out, int L, int S,
                                                             int heads, int lo_q, int lo_kv) {
  pdl_sync();
  __shared__ __align__(16) float k_s[kFaKeys][D];
  __shared__ __align__(16) float v_s[kFaKeys][D];
  const int b = blockIdx.z, h = blockIdx.y;
  const int row = blockIdx.x * 128 + threadIdx.x;
  const int dm = heads * D;
  const int ldq = lo_q ? 2 * dm : dm, ldk = lo_kv ? 4 * dm : 2 * dm;
  const float temp = rsqrtf((float)D);
  float qr[D], acc[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    acc[d] = 0.f;
    qr[d] = 0.f;
  }
  if (row < L) {
    const __half* qp = q + ((long long)b * L + row) * ldq + h * D;
#pragma unroll
    for (int d = 0; d < D; d += 8) load_split8(qp, d, qr + d, lo_q);
  }
  float m = -INFINITY, l = 0.f;
  for (int s0 = 0; s0 < S; s0 += kFaKeys) {
    __syncthreads();
    for (int i = threadIdx.x; i < kFaKeys * (D / 8) * 2; i += 128) {
      const int which = i / (kFaKeys * (D / 8));          // 0 = K, 1 = V
      const int r = (i / (D / 8)) % kFaKeys, g = i % (D / 8);
      float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (s0 + r < S)
        load_split8(kv + ((long long)b * S + s0 + r) * ldk + which * dm + h * D, g * 8, f, lo_kv);
      float* dst = which ? &v_s[r][g * 8] : &k_s[r][g * 8];
      reinterpret_cast<float4*>(dst)[0] = make_float4(f[0], f[1], f[2], f[3]);
      reinterpret_cast<float4*>(dst)[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
    const int cnt = min(kFaKeys, S - s0);
    for (int j = 0; j < cnt; ++j) {
      float sc = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) sc = fmaf(qr[d], k_s[j][d], sc);
      sc *= temp;
      const float mn = fmaxf(m, sc);
      const float corr = expf(m - mn), pj = expf(sc - mn);
      l = l * corr + pj;
#pragma unroll
      for (int d = 0; d < D; ++d) acc[d] = fmaf(pj, v_s[j][d], acc[d] * corr);
      m = mn;
    }
  }
  if (row < L) {
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < D; ++d) acc[d] *= inv;
    __half* op = out + ((long long)b * L + row) * ldq + h * D;
#pragma unroll
    for (int d = 0; d < D; d += 8) store_split8(op, d, acc + d, lo_q);
  }
}

// =============================================================================================
// fine matching   (utils/fine_matching.py:78-110): one warp per match
// =============================================================================================
__global__ void __launch_bounds__(128) fine_match_kernel(
    const float* __restrict__ x32, const float* __restrict__ mkpts_c,
    const long long* __restrict__ b_ids, const float* __restrict__ img_scale,
    float* __restrict__ expec_f, float* __restrict__ mkpts_f, int M, float fine_scale,
    const int* __restrict__ count_dev) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  if (m >= M || (count_dev && m >= *count_dev)) return;
  const float* f0 = x32 + (long long)m * 26 * 128;
  const float4 a = reinterpret_cast<const float4*>(f0)[lane];
  float my_sim = -INFINITY;
  for (int r = 0; r < 25; ++r) {
    const float4 w = reinterpret_cast<const float4*>(f0 + (1 + r) * 128)[lane];
    float d = a.x * w.x + a.y * w.y + a.z * w.z + a.w * w.w;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == r) my_sim = d * 0.08838834764831845f;  // 1/sqrt(128)
  }
  float mx = my_sim;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float e = lane < 25 ? expf(my_sim - mx) : 0.f;
  float sum = e;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float p = e / sum;
  // grid: linspace(-1, 1, 5), x fastest (kornia create_meshgrid + spatial_expectation2d)
  const float gx = lane < 25 ? -1.f + 0.5f * (float)(lane % 5) : 0.f;
  const float gy = lane < 25 ? -1.f + 0.5f * (float)(lane / 5) : 0.f;
  float ex = gx * p, ey = gy * p, exx = gx * gx * p, eyy = gy * gy * p;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ex += __shfl_xor_sync(0xffffffffu, ex, o);
    ey += __shfl_xor_sync(0xffffffffu, ey, o);
    exx += __shfl_xor_sync(0xffffffffu, exx, o);
    eyy += __shfl_xor_sync(0xffffffffu, eyy, o);
  }
  if (lane == 0) {
    const float vx = exx - ex * ex, vy = eyy - ey * ey;
    const float sd = sqrtf(fmaxf(vx, 1e-10f)) + sqrtf(fmaxf(vy, 1e-10f));
    expec_f[m * 3 + 0] = ex;
    expec_f[m * 3 + 1] = ey;
    expec_f[m * 3 + 2] = sd;
    float sx = fine_scale, sy = fine_scale;
    if (img_scale) {
      const long long b = b_ids[m];
      sx = fine_scale * img_scale[b * 2 + 1];
      sy = fine_scale * img_scale[b * 2 + 0];
    }
    // fine_matching.py:104-105: mkpts_query_c + coords * (W // 2) * scale
    mkpts_f[m * 2 + 0] = mkpts_c[m * 2 + 0] + ex * 2.f * sx;
    mkpts_f[m * 2 + 1] = mkpts_c[m * 2 + 1] + ey * 2.f * sy;
  }
}

// =============================================================================================
// LoFTR 2D-2D matcher (SURVEY §8 f3): LoFTR_for_OnePose_Plus.forward
// (src/KeypointFreeSfM/loftr_for_sfm/loftr.py:35-127 on submodules/LoFTR/src/loftr).  The backbone,
// the coarse transformer layers and the dual-softmax passes are the engine's; the kernels below are
// what differs from the 2D-3D matcher: symmetric border + two image grids in the match selection,
// W x W windows from BOTH fine maps, linear attention between two token groups, and the centre
// token of image 0's window correlated with image 1's window.
// =============================================================================================

// keep (b, i) iff conf_max > thr, i and its argmax j are >= border cells away from ALL four sides of
// their grids (LoFTR utils/coarse_matching.py:9-28,197-203) and i is the column maximum of j
__device__ __forceinline__ bool match_flag_2d(const float* pt_val, const int* pt_idx,
                                              const unsigned* colmax, long long r, int l, int s,
                                              int h0, int w0, int h1, int w1, float thr, int border) {
  const float v = pt_val[r];
  if (!(v > thr)) return false;
  const int j = pt_idx[r];
  const long long b = r / l;
  const int i = (int)(r - b * l);
  const int iy = i / w0, ix = i - iy * w0, jy = j / w1, jx = j - jy * w1;
  if (iy < border || ix < border || iy >= h0 - border || ix >= w0 - border) return false;
  if (jy < border || jx < border || jy >= h1 - border || jx >= w1 - border) return false;
  return colmax[b * s + j] == __float_as_uint(v);
}

__global__ void __launch_bounds__(1024) match_count_2d_kernel(const float* pt_val, const int* pt_idx,
                                                              const unsigned* colmax, long long rows,
                                                              int l, int s, int h0, int w0, int h1,
                                                              int w1, float thr, int border,
                                                              int* block_counts) {
  pdl_sync();
  const long long r = (long long)blockIdx.x * 1024 + threadIdx.x;
  const bool f = r < rows && match_flag_2d(pt_val, pt_idx, colmax, r, l, s, h0, w0, h1, w1, thr, border);
  const int c = __syncthreads_count(f);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

__global__ void __launch_bounds__(1024)
match_scatter_2d_kernel(const float* pt_val, const int* pt_idx, const unsigned* colmax,
                        const float* scale0, const float* scale1, long long rows, int l, int s, int h0,
                        int w0, int h1, int w1, float thr, int border, float cell,
                        const int* block_offsets, long long* b_ids, long long* i_ids, long long* j_ids,
                        float* mconf, float* mk0, float* mk1) {
  pdl_sync();
  __shared__ int warp_sums[32];
  const long long r = (long long)blockIdx.x * 1024 + threadIdx.x;
  const bool f = r < rows && match_flag_2d(pt_val, pt_idx, colmax, r, l, s, h0, w0, h1, w1, thr, border);
  const unsigned ballot = __ballot_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_sums[warp] = __popc(ballot);
  __syncthreads();
  if (warp == 0) {
    int w = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  if (!f) return;
  const int pos = block_offsets[blockIdx.x] + (warp > 0 ? warp_sums[warp - 1] : 0) +
                  __popc(ballot & ((1u << lane) - 1u));
  const long long b = r / l;
  const int i = (int)(r - b * l);
  const int j = pt_idx[r];
  b_ids[pos] = b;
  i_ids[pos] = i;
  j_ids[pos] = j;
  mconf[pos] = pt_val[r];
  // LoFTR coarse_matching.py:248-253: [idx % w, idx // w] * scale * scale0[b]  (no axis swap here)
  const float s0x = scale0 ? cell * scale0[b * 2] : cell, s0y = scale0 ? cell * scale0[b * 2 + 1] : cell;
  const float s1x = scale1 ? cell * scale1[b * 2] : cell, s1y = scale1 ? cell * scale1[b * 2 + 1] : cell;
  mk0[pos * 2 + 0] = (float)(i % w0) * s0x;
  mk0[pos * 2 + 1] = (float)(i / w0) * s0y;
  mk1[pos * 2 + 0] = (float)(j % w1) * s1x;
  mk1[pos * 2 + 1] = (float)(j / w1) * s1y;
}

// W x W windows of both fine maps (LoFTR loftr_module/fine_preprocess.py:41-49), sequence-major:
// row (seq * M + m) * WW + ww;  seq 0 = image 0's window centred on cell i, seq 1 = image 1's on j.
__global__ void __launch_bounds__(128) fine_gather_2d_kernel(
    const __half* __restrict__ f0, const __half* __restrict__ f1, const long long* __restrict__ b_ids,
    const long long* __restrict__ b1_ids, const long long* __restrict__ i_ids, const long long* __restrict__ j_ids,
    __half* __restrict__ x16, int M, int hf0, int wf0, int wc0, int hf1, int wf1, int wc1, int stride, int W,
    int lo_off) {
  pdl_sync();
  const int m = blockIdx.x, seq = blockIdx.y, c = threadIdx.x;
  const long long b = seq ? b1_ids[m] : b_ids[m];   // map index of this side's image
  const long long cell = seq ? j_ids[m] : i_ids[m];
  const int wc = seq ? wc1 : wc0, hf = seq ? hf1 : hf0, wf = seq ? wf1 : wf0;
  const int cy = (int)(cell / wc), cx = (int)(cell - (long long)cy * wc);
  const int ld = lo_off ? 256 : 128;
  const __half* fb = (seq ? f1 : f0) + b * hf * wf * ld;
  const int WW = W * W, half = W / 2;
  const long long row0 = ((long long)seq * M + m) * WW;
  for (int ww = 0; ww < WW; ++ww) {
    const int y = cy * stride + ww / W - half, x = cx * stride + ww % W - half;
    float v = 0.f;
    if (y >= 0 && y < hf && x >= 0 && x < wf) v = load_split1(fb + ((long long)y * wf + x) * ld, c, lo_off);
    store_split1(x16 + (row0 + ww) * ld, c, v, lo_off);
  }
}

// Linear attention between two small token groups (linear_attention.py:29-61; 8 heads x 16):
// group g: queries q[g][0..L), source kv[g][0..S) = (K' | V).  One CTA per group, thread (h, v) owns
// column v of head h of the 16 x 16 state; tokens stream through shared memory in slabs of 27.
constexpr int kSaSlab = 27;
__global__ void __launch_bounds__(128) seq_attention_kernel(const __half* __restrict__ q,
                                                            const __half* __restrict__ kv,
                                                            __half* __restrict__ out, int L, int S,
                                                            float eps, int lo_q, int lo_kv) {
  pdl_sync();
  __shared__ __align__(16) float a_s[kSaSlab][128];
  __shared__ __align__(16) float b_s[kSaSlab][128];
  __shared__ __align__(16) float ks2[128];
  const int g = blockIdx.x, c = threadIdx.x, h = c >> 4;
  const int ldq = lo_q ? 256 : 128, ldk = lo_kv ? 512 : 256;
  const __half* kvp = kv + (long long)g * S * ldk;
  float col[16];
#pragma unroll
  for (int dd = 0; dd < 16; ++dd) col[dd] = 0.f;
  float ksum_c = 0.f;
  for (int t0 = 0; t0 < S; t0 += kSaSlab) {
    const int cnt = min(kSaSlab, S - t0);
    __syncthreads();
    for (int i = c; i < cnt * 32; i += 128) {     // 32 groups of 8 values per token: K' (16) | V (16)
      const int t = i >> 5, sg = i & 31;
      float f[8];
      load_split8(kvp + (long long)(t0 + t) * ldk, sg * 8, f, lo_kv);
      float* dst = sg < 16 ? &a_s[t][sg * 8] : &b_s[t][(sg - 16) * 8];
      reinterpret_cast<float4*>(dst)[0] = make_float4(f[0], f[1], f[2], f[3]);
      reinterpret_cast<float4*>(dst)[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
    for (int t = 0; t < cnt; ++t) {
      const float vv = b_s[t][c];
      const float4* kr = reinterpret_cast<const float4*>(&a_s[t][h * 16]);
#pragma unroll
      for (int gq = 0; gq < 4; ++gq) {
        const float4 k4 = kr[gq];
        col[4 * gq + 0] = fmaf(k4.x, vv, col[4 * gq + 0]);
        col[4 * gq + 1] = fmaf(k4.y, vv, col[4 * gq + 1]);
        col[4 * gq + 2] = fmaf(k4.z, vv, col[4 * gq + 2]);
        col[4 * gq + 3] = fmaf(k4.w, vv, col[4 * gq + 3]);
      }
      ksum_c += a_s[t][c];
    }
  }
  __syncthreads();
  ks2[c] = ksum_c;
  __syncthreads();
  float ksw[16];
  {
    const float4* a = reinterpret_cast<const float4*>(&ks2[h * 16]);
#pragma unroll
    for (int gq = 0; gq < 4; ++gq) {
      const float4 x = a[gq];
      ksw[4 * gq] = x.x; ksw[4 * gq + 1] = x.y; ksw[4 * gq + 2] = x.z; ksw[4 * gq + 3] = x.w;
    }
  }
  const __half* qp = q + (long long)g * L * ldq;
  __half* op = out + (long long)g * L * ldq;
  for (int t0 = 0; t0 < L; t0 += kSaSlab) {
    const int cnt = min(kSaSlab, L - t0);
    __syncthreads();
    for (int i = c; i < cnt * 16; i += 128) {
      const int t = i >> 4, sg = i & 15;
      float f[8];
      load_split8(qp + (long long)(t0 + t) * ldq, sg * 8, f, lo_q);
      reinterpret_cast<float4*>(&a_s[t][sg * 8])[0] = make_float4(f[0], f[1], f[2], f[3]);
      reinterpret_cast<float4*>(&a_s[t][sg * 8])[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
    for (int t = 0; t < cnt; ++t) {
      const float4* qr = reinterpret_cast<const float4*>(&a_s[t][h * 16]);
      float num = 0.f, den = 0.f;
#pragma unroll
      for (int gq = 0; gq < 4; ++gq) {
        const float4 q4 = qr[gq];
        num = fmaf(q4.x, col[4 * gq + 0], num);
        den = fmaf(q4.x, ksw[4 * gq + 0], den);
        num = fmaf(q4.y, col[4 * gq + 1], num);
        den = fmaf(q4.y, ksw[4 * gq + 1], den);
        num = fmaf(q4.z, col[4 * gq + 2], num);
        den = fmaf(q4.z, ksw[4 * gq + 2], den);
        num = fmaf(q4.w, col[4 * gq + 3], num);
        den = fmaf(q4.w, ksw[4 * gq + 3], den);
      }
      b_s[t][c] = num / (den + eps);
    }
    __syncthreads();
    for (int i = c; i < cnt * 16; i += 128) {
      const int t = i >> 4, sg = i & 15;
      float f[8];
      const float4 a = reinterpret_cast<const float4*>(&b_s[t][sg * 8])[0];
      const float4 b = reinterpret_cast<const float4*>(&b_s[t][sg * 8])[1];
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
      f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
      store_split8(op + (long long)(t0 + t) * ldq, sg * 8, f, lo_q);
    }
  }
}

// LoFTR FineMatching (utils/fine_matching.py:46-70): centre token (WW // 2) of image 0's window
// against the WW tokens of image 1's window; softmax / sqrt(C), expectation + std on the W x W grid
// linspace(-1, 1, W) (x fastest); mkpts1_f = mkpts1_c + coords * (W // 2) * scale * scale1[b].
// x32 fp32 [2][M][WW][128] (sequence-major).  One warp per match.
__global__ void __launch_bounds__(128) fine_match_2d_kernel(
    const float* __restrict__ x32, const float* __restrict__ mk1c, const long long* __restrict__ b_ids,
    const float* __restrict__ scale1, float* __restrict__ expec_f, float* __restrict__ mk1f, int M, int W,
    float fine_scale) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  if (m >= M) return;
  const int WW = W * W;
  const float4 a = reinterpret_cast<const float4*>(x32 + ((long long)m * WW + WW / 2) * 128)[lane];
  const float* f1 = x32 + ((long long)M + m) * WW * 128;
  float sim[3] = {-INFINITY, -INFINITY, -INFINITY};   // this lane owns tokens lane, lane + 32, lane + 64
  for (int r = 0; r < WW; ++r) {
    const float4 w = reinterpret_cast<const float4*>(f1 + (long long)r * 128)[lane];
    float d = a.x * w.x + a.y * w.y + a.z * w.z + a.w * w.w;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if ((r & 31) == lane) sim[r >> 5] = d * 0.08838834764831845f;  // 1/sqrt(128)
  }
  float mx = fmaxf(sim[0], fmaxf(sim[1], sim[2]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float e[3], sum = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    e[k] = (lane + 32 * k < WW) ? expf(sim[k] - mx) : 0.f;
    sum += e[k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  float ex = 0.f, ey = 0.f, exx = 0.f, eyy = 0.f;
  const float step = 2.f / (float)(W - 1);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int r = lane + 32 * k;
    if (r < WW) {
      const float p = e[k] / sum;
      const float gx = -1.f + step * (float)(r % W), gy = -1.f + step * (float)(r / W);
      ex += gx * p;
      ey += gy * p;
      exx += gx * gx * p;
      eyy += gy * gy * p;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ex += __shfl_xor_sync(0xffffffffu, ex, o);
    ey += __shfl_xor_sync(0xffffffffu, ey, o);
    exx += __shfl_xor_sync(0xffffffffu, exx, o);
    eyy += __shfl_xor_sync(0xffffffffu, eyy, o);
  }
  if (lane == 0) {
    const float vx = exx - ex * ex, vy = eyy - ey * ey;
    expec_f[m * 3 + 0] = ex;
    expec_f[m * 3 + 1] = ey;
    expec_f[m * 3 + 2] = sqrtf(fmaxf(vx, 1e-10f)) + sqrtf(fmaxf(vy, 1e-10f));
    float sx = fine_scale, sy = fine_scale;
    if (scale1) {
      const long long b = b_ids[m];
      sx = fine_scale * scale1[b * 2];
      sy = fine_scale * scale1[b * 2 + 1];
    }
    mk1f[m * 2 + 0] = mk1c[m * 2 + 0] + ex * (float)(W / 2) * sx;
    mk1f[m * 2 + 1] = mk1c[m * 2 + 1] + ey * (float)(W / 2) * sy;
  }
}

}  // namespace opp

using namespace opp;

static inline int grid_for(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = (long long)opp::num_sms() * 16;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

extern "C" {

int opp_version(void) { return 100; }
int opp_num_sms(void) { return opp::num_sms(); }

int opp_conv1_im2col(const void* image, int image_u8, void* a_out, int batch, int h, int w, int split,
                     opp_stream_t stream) {
  OPP_REQUIRE(image && a_out, "null pointer");
  OPP_REQUIRE(h % 2 == 0 && w % 2 == 0 && batch > 0, "bad conv1 shape");
  dim3 grid((w / 2 + kC1Tile - 1) / kC1Tile, (h / 2 + kC1Tile - 1) / kC1Tile, batch);
  if (image_u8)
    OPP_CHECK_CUDA(opp::launch_pdl(conv1_im2col_kernel<true>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, image, (__half*)a_out, h, w, split ? 64 : 0));
  else
    OPP_CHECK_CUDA(opp::launch_pdl(conv1_im2col_kernel<false>, dim3(grid), dim3(256), 0, (cudaStream_t)stream, image, (__half*)a_out, h, w, split ? 64 : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_kpt_stats(const float* kpts, float* stats, int batch, int n, opp_stream_t stream) {
  OPP_REQUIRE(kpts && stats && batch > 0 && n > 0, "bad kpt_stats arguments");
  OPP_CHECK_CUDA(opp::launch_pdl(kpt_stats_kernel, dim3(batch), dim3(256), 0, (cudaStream_t)stream, kpts, stats, n));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_kpt_encode(const float* kpts, const float* stats, const float* desc, const float* w1_t,
                   const float* b1, const float* w2_t, const float* b2, const float* w3_t,
                   const float* b3, const float* w4_t, const float* b4, void* tok, int batch, int n,
                   int split, opp_stream_t stream) {
  OPP_REQUIRE(kpts && stats && desc && tok, "null pointer");
  dim3 grid((n + kKeP - 1) / kKeP, batch);
  OPP_CHECK_CUDA(opp::launch_pdl(kpt_encode_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, kpts, stats, desc, w1_t, b1, w2_t, b2,
                                                            w3_t, b3, w4_t, b4, (__half*)tok, n,
                                                            split ? 256 : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

// tokens per CTA of kv_partial: 256 (least partial-state traffic for kv_finalize) unless that leaves
// fewer than 64 CTAs in the grid (batch 1-2), then 128: half the serial loop per CTA
static int kv_chunk_tokens(int s, int batch) {
  const long long ctas = (long long)batch * ((s + kKvChunk - 1) / kKvChunk);
  return ctas < 64 ? kKvChunk / 2 : kKvChunk;
}
int opp_kv_chunks(int s) { return (s + kKvChunk - 1) / kKvChunk; }
int opp_kv_chunks_b(int s, int batch) {
  const int c = kv_chunk_tokens(s, batch);
  return (s + c - 1) / c;
}

int opp_kv_partial(const void* kv16, float* part, int batch, int s, int d, opp_stream_t stream) {
  OPP_REQUIRE(kv16 && part, "null pointer");
  OPP_REQUIRE(d == 256, "kv_partial is built for d = 256 (8 heads x 32), got %d", d);
  const int kv_chunk = kv_chunk_tokens(s, batch);
  dim3 grid((s + kv_chunk - 1) / kv_chunk, batch);
  static unsigned long long attr_done = 0;   // per device
  int dev = 0;
  OPP_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !((attr_done >> dev) & 1ull)) {
    OPP_CHECK_CUDA(cudaFuncSetAttribute(kv_partial_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kKvmSmem));
    attr_done |= 1ull << dev;
  }
  OPP_CHECK_CUDA(opp::launch_pdl(kv_partial_mma_kernel, dim3(grid), dim3(256), kKvmSmem, (cudaStream_t)stream,
                                 (const __half*)kv16, part, s, kv_chunk));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_kv_finalize(const float* part, const float* merge_w, void* mt, float* ksum, int batch,
                    int chunks, int d, float v_len, int split, opp_stream_t stream) {
  OPP_REQUIRE(part && merge_w && mt && ksum, "null pointer");
  OPP_REQUIRE(d % 32 == 0 && d <= 256, "d=%d must be a multiple of the head size 32, <= 256", d);
  dim3 grid(d / 32, batch);
  OPP_CHECK_CUDA(opp::launch_pdl(kv_finalize_kernel, dim3(grid), dim3(1024), 0, (cudaStream_t)stream, part, merge_w, (__half*)mt, ksum,
                                                             chunks, d, 1.f / v_len,
                                                             split ? d : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_lse_finalize(const float* part_m, const float* part_s, float* lse, long long rows,
                     int tiles, opp_stream_t stream) {
  OPP_REQUIRE(part_m && part_s && lse, "null pointer");
  OPP_CHECK_CUDA(opp::launch_pdl(lse_finalize_kernel, dim3((unsigned)((rows + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, 
      part_m, part_s, lse, rows, tiles));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_lse_col_finalize(const float* col_m, const float* col_s, float* lse, int batches, int groups,
                         int cols, const unsigned char* col_mask, opp_stream_t stream) {
  OPP_REQUIRE(col_m && col_s && lse && batches > 0 && groups > 0 && cols > 0, "bad lse_col_finalize arguments");
  OPP_CHECK_CUDA(opp::launch_pdl(lse_col_finalize_kernel, dim3(dim3((cols + 31) / 32, batches)), dim3(32 * kLseColSlices), 0, (cudaStream_t)stream, 
      col_m, col_s, lse, batches, groups, cols, col_mask));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_best_finalize(const float* part_val, const int* part_idx, float* best_val, int* best_idx,
                      long long rows, int tiles, opp_stream_t stream) {
  OPP_REQUIRE(part_val && part_idx && best_val && best_idx, "null pointer");
  OPP_CHECK_CUDA(opp::launch_pdl(best_finalize_kernel, dim3((unsigned)((rows + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, 
      part_val, part_idx, best_val, best_idx, rows, tiles));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_match_select_colmax_set(const float* pt_val, const int* pt_idx, const unsigned* colmax,
                                const float* kpts, const float* img_scale, int batch, int l, int hc,
                                int wc, float thr, int border, float cell, int* scratch,
                                long long* b_ids, long long* i_ids, long long* j_ids, float* mconf,
                                float* mkpts3d, float* mkpts_c, int* count_out, int bank_shared,
                                const int* bank_of_batch, const int* row_count, opp_stream_t stream) {
  OPP_REQUIRE(pt_val && pt_idx && colmax && kpts && scratch && count_out, "null pointer");
  OPP_REQUIRE((bank_of_batch == nullptr) == (row_count == nullptr),
              "bank_of_batch and row_count come together (bank sets)");
  const long long rows = (long long)batch * l;
  const int nblocks = (int)((rows + 1023) / 1024);
  const int s = hc * wc;
  cudaStream_t st = (cudaStream_t)stream;
  if (bank_of_batch) {
    OPP_CHECK_CUDA(opp::launch_pdl(match_count_colmax_kernel<true>, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx,
                                   colmax, rows, l, s, wc, thr, border, scratch, row_count));
  } else {
    OPP_CHECK_CUDA(opp::launch_pdl(match_count_colmax_kernel<false>, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx,
                                   colmax, rows, l, s, wc, thr, border, scratch, row_count));
  }
  OPP_CHECK_CUDA(opp::launch_pdl(match_scan_kernel, dim3(1), dim3(1024), 0, st, scratch, nblocks, count_out));
  if (bank_of_batch) {
    OPP_CHECK_CUDA(opp::launch_pdl(match_scatter_colmax_kernel<true>, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx,
                                   colmax, kpts, img_scale, rows, l, s, wc, thr, border, cell, scratch, b_ids,
                                   i_ids, j_ids, mconf, mkpts3d, mkpts_c, bank_shared, bank_of_batch, row_count));
  } else {
    OPP_CHECK_CUDA(opp::launch_pdl(match_scatter_colmax_kernel<false>, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx,
                                   colmax, kpts, img_scale, rows, l, s, wc, thr, border, cell, scratch, b_ids,
                                   i_ids, j_ids, mconf, mkpts3d, mkpts_c, bank_shared, bank_of_batch, row_count));
  }
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_match_select_colmax(const float* pt_val, const int* pt_idx, const unsigned* colmax,
                            const float* kpts, const float* img_scale, int batch, int l, int hc,
                            int wc, float thr, int border, float cell, int* scratch,
                            long long* b_ids, long long* i_ids, long long* j_ids, float* mconf,
                            float* mkpts3d, float* mkpts_c, int* count_out, int bank_shared,
                            opp_stream_t stream) {
  return opp_match_select_colmax_set(pt_val, pt_idx, colmax, kpts, img_scale, batch, l, hc, wc, thr, border, cell,
                                     scratch, b_ids, i_ids, j_ids, mconf, mkpts3d, mkpts_c, count_out, bank_shared,
                                     nullptr, nullptr, stream);
}

int opp_fine_gather_set(const void* fine, const float* desc3d, const long long* b_ids,
                        const long long* i_ids, const long long* j_ids, float* x32, void* x16, int m,
                        int hf, int wf, int wc, int stride, int n, int split, int bank_shared,
                        int windows, const int* count_dev, const int* bank_of_batch, opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(fine && desc3d && b_ids && i_ids && j_ids && x16, "null pointer");
  if (bank_of_batch)
    OPP_CHECK_CUDA(opp::launch_pdl(fine_gather_kernel<true>, dim3(m), dim3(128), 0, (cudaStream_t)stream,
                                   (const __half*)fine, desc3d, b_ids, i_ids, j_ids, x32, (__half*)x16, hf, wf,
                                   wc, stride, n, split ? 128 : 0, bank_shared, windows, count_dev, bank_of_batch));
  else
    OPP_CHECK_CUDA(opp::launch_pdl(fine_gather_kernel<false>, dim3(m), dim3(128), 0, (cudaStream_t)stream,
                                   (const __half*)fine, desc3d, b_ids, i_ids, j_ids, x32, (__half*)x16, hf, wf,
                                   wc, stride, n, split ? 128 : 0, bank_shared, windows, count_dev, bank_of_batch));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_gather(const void* fine, const float* desc3d, const long long* b_ids,
                    const long long* i_ids, const long long* j_ids, float* x32, void* x16, int m,
                    int hf, int wf, int wc, int stride, int n, int split, int bank_shared,
                    int windows, const int* count_dev, opp_stream_t stream) {
  return opp_fine_gather_set(fine, desc3d, b_ids, i_ids, j_ids, x32, x16, m, hf, wf, wc, stride, n, split,
                             bank_shared, windows, count_dev, nullptr, stream);
}

int opp_fine_attention(const void* qkv, void* msg, int m, int cross, float eps, int split,
                       const int* count_dev, opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(qkv && msg, "null pointer");
  OPP_CHECK_CUDA(opp::launch_pdl(fine_attention_kernel, dim3(m), dim3(128), 0, (cudaStream_t)stream, (const __half*)qkv, (__half*)msg, cross, eps,
                                                             split ? 384 : 0, split ? 128 : 0, count_dev));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_full_attention(const void* q, const void* kv, void* out, int batch, int l, int s, int heads,
                       int head_dim, int split, opp_stream_t stream) {
  OPP_REQUIRE(q && kv && out, "null pointer");
  OPP_REQUIRE(batch > 0 && l > 0 && s > 0 && heads > 0, "empty attention");
  OPP_REQUIRE(head_dim == 32 || head_dim == 16, "full attention is built for head_dim 32 / 16, got %d", head_dim);
  dim3 grid((l + 127) / 128, heads, batch);
  const int dm = heads * head_dim;
  if (head_dim == 32)
    OPP_CHECK_CUDA(opp::launch_pdl(full_attention_kernel<32>, dim3(grid), dim3(128), 0, (cudaStream_t)stream, (const __half*)q, (const __half*)kv,
                                                                     (__half*)out, l, s, heads, split ? dm : 0,
                                                                     split ? 2 * dm : 0));
  else
    OPP_CHECK_CUDA(opp::launch_pdl(full_attention_kernel<16>, dim3(grid), dim3(128), 0, (cudaStream_t)stream, (const __half*)q, (const __half*)kv,
                                                                     (__half*)out, l, s, heads, split ? dm : 0,
                                                                     split ? 2 * dm : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_match(const float* x32, const float* mkpts_c, const long long* b_ids,
                   const float* img_scale, float* expec_f, float* mkpts_f, int m, float fine_scale,
                   const int* count_dev, opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(x32 && mkpts_c && b_ids && expec_f && mkpts_f, "null pointer");
  OPP_CHECK_CUDA(opp::launch_pdl(fine_match_kernel, dim3((m + 3) / 4), dim3(128), 0, (cudaStream_t)stream, x32, mkpts_c, b_ids, img_scale,
                                                                   expec_f, mkpts_f, m, fine_scale, count_dev));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_match_select_2d(const float* pt_val, const int* pt_idx, const unsigned* colmax, const float* scale0,
                        const float* scale1, int batch, int h0, int w0, int h1, int w1, float thr,
                        int border, float cell, int* scratch, long long* b_ids, long long* i_ids,
                        long long* j_ids, float* mconf, float* mkpts0_c, float* mkpts1_c, int* count_out,
                        opp_stream_t stream) {
  OPP_REQUIRE(pt_val && pt_idx && colmax && scratch && count_out, "null pointer");
  const int l = h0 * w0, s = h1 * w1;
  const long long rows = (long long)batch * l;
  const int nblocks = (int)((rows + 1023) / 1024);
  cudaStream_t st = (cudaStream_t)stream;
  OPP_CHECK_CUDA(opp::launch_pdl(match_count_2d_kernel, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx, colmax, rows, l, s, h0, w0, h1, w1, thr,
                                                  border, scratch));
  OPP_CHECK_CUDA(opp::launch_pdl(match_scan_kernel, dim3(1), dim3(1024), 0, st, scratch, nblocks, count_out));
  OPP_CHECK_CUDA(opp::launch_pdl(match_scatter_2d_kernel, dim3(nblocks), dim3(1024), 0, st, pt_val, pt_idx, colmax, scale0, scale1, rows, l, s, h0, w0,
                                                    h1, w1, thr, border, cell, scratch, b_ids, i_ids, j_ids,
                                                    mconf, mkpts0_c, mkpts1_c));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_gather_2d(const void* fine0, const void* fine1, const long long* b_ids, const long long* i_ids,
                       const long long* j_ids, void* x16, int m, int hf0, int wf0, int wc0, int hf1, int wf1,
                       int wc1, int stride, int window, int split, opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(fine0 && fine1 && b_ids && i_ids && j_ids && x16, "null pointer");
  OPP_REQUIRE(window % 2 == 1 && window >= 1 && window <= 9, "window %d unsupported (odd, <= 9)", window);
  OPP_CHECK_CUDA(opp::launch_pdl(fine_gather_2d_kernel, dim3(dim3(m, 2)), dim3(128), 0, (cudaStream_t)stream, 
      (const __half*)fine0, (const __half*)fine1, b_ids, b_ids, i_ids, j_ids, (__half*)x16, m, hf0, wf0, wc0, hf1,
      wf1, wc1, stride, window, split ? 128 : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_gather_2d_images(const void* fine, const long long* img0, const long long* img1, const long long* i_ids,
                              const long long* j_ids, void* x16, int m, int hf, int wf, int wc, int stride,
                              int window, int split, opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(fine && img0 && img1 && i_ids && j_ids && x16, "null pointer");
  OPP_REQUIRE(window % 2 == 1 && window >= 1 && window <= 9, "window %d unsupported (odd, <= 9)", window);
  OPP_CHECK_CUDA(opp::launch_pdl(fine_gather_2d_kernel, dim3(dim3(m, 2)), dim3(128), 0, (cudaStream_t)stream,
      (const __half*)fine, (const __half*)fine, img0, img1, i_ids, j_ids, (__half*)x16, m, hf, wf, wc, hf, wf, wc,
      stride, window, split ? 128 : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_seq_attention(const void* q, const void* kv, void* out, int groups, int l, int s, float eps, int split,
                      opp_stream_t stream) {
  if (groups == 0) return OPP_OK;
  OPP_REQUIRE(q && kv && out && l > 0 && s > 0, "bad seq_attention arguments");
  OPP_CHECK_CUDA(opp::launch_pdl(seq_attention_kernel, dim3(groups), dim3(128), 0, (cudaStream_t)stream, (const __half*)q, (const __half*)kv,
                                                                 (__half*)out, l, s, eps, split ? 128 : 0,
                                                                 split ? 256 : 0));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

int opp_fine_match_2d(const float* x32, const float* mkpts1_c, const long long* b_ids, const float* scale1,
                      float* expec_f, float* mkpts1_f, int m, int window, float fine_scale,
                      opp_stream_t stream) {
  if (m == 0) return OPP_OK;
  OPP_REQUIRE(x32 && mkpts1_c && b_ids && expec_f && mkpts1_f, "null pointer");
  OPP_REQUIRE(window % 2 == 1 && window >= 3 && window <= 9, "window %d unsupported (odd, 3..9)", window);
  OPP_CHECK_CUDA(opp::launch_pdl(fine_match_2d_kernel, dim3((m + 3) / 4), dim3(128), 0, (cudaStream_t)stream, x32, mkpts1_c, b_ids, scale1, expec_f,
                                                                      mkpts1_f, m, window, fine_scale));
  OPP_CHECK_CUDA(cudaGetLastError());
  return OPP_OK;
}

}  // extern "C"
