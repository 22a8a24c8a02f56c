// opp_gemm.cuh — the one tensor-core engine of the hot path.
//
// D[M,N] = A[M,K] * W[N,K]^T on wgmma (fp16 operands, fp32 accumulators), operands staged by TMA
// into 128B- (or, for 32-wide slots, 64B-) swizzled shared memory through an mbarrier ring, persistent over output tiles.  The
// producer warp keeps loading the next tile's operands while the epilogue of the current one runs.
//
// Precision: the reference computes in fp32 and the parity bar is 1e-3 on outputs whose logits
// reach ~1e2, so single fp16 operands (2^-11) are not enough.  In `split` mode every operand is a
// pair of fp16 planes  x = hi + lo  (see opp_common.cuh) and each K-step issues three MMAs into
// the same accumulator:  hi*hi + hi*lo + lo*hi  (the dropped lo*lo term is ~2^-22), i.e. an
// fp32-grade GEMM at 3 tensor-core passes and 2x operand bytes.  split = 0 is plain fp16.
//
// The A operand is either
//   A_ROWS : token rows  [batch][rows][planes*K]  (up to two arrays concatenated along K), or
//   A_CONV : an NHWC feature map read as an implicit-GEMM im2col: for every filter tap the TMA
//            box is the output tile shifted by the tap offset; out-of-bounds coordinates are
//            zero-filled by the TMA unit, which implements the convolution padding for free.
//            Stride-2 convolutions use four parity views (y%2, x%2) of the same tensor.
// Everything after the accumulator (bias / BN / activation / residual / LayerNorm / elu+1 /
// linear-attention normaliser / dual-softmax statistics) is a fused epilogue functor.
//
// Warp roles (384 threads): two MMA warpgroups, then the producer warpgroup, whose first warp issues
// the TMA loads (the other three only wait for the end of the CTA).  The producer warpgroup gives
// its registers up (setmaxnreg 40) so that the MMA warpgroups can hold 232 each.  Warpgroup g
// issues one full-width wgmma per K step (m64nNk16, N = the tile's mma_n) for tile rows
// 64g .. 64g+63 into its registers and then runs the epilogue as epilogue group g, in one of two ways:
//   * the conv epilogues (EpiConv, EpiWin: per-element math) and the token-row epilogues (row /
//     column reductions: LayerNorm, linear-attention normaliser, dual-softmax statistics) read the
//     accumulator registers directly (EpiFromRegs): warp q holds tile rows 64g+16q .. +15 over all N
//     columns.  There is no accumulator tile in shared memory, so the ring takes its space and the
//     producer never waits for an epilogue; the two warpgroups run their epilogues independently.
//   * the fused-upsample conv (EpiConvUp) writes the fp32 accumulator tile to shared memory: warp w
//     owns accumulator rows 32*(w%4) .. +31, one row per thread, and the two groups take alternate
//     32-column chunks.
//
// Reference semantics implemented by the epilogues are cited at each functor
// (paths relative to the reference repo zju3dv/OnePose_Plus_Plus).
#pragma once

#include <type_traits>

#include "opp_common.cuh"

#ifndef OPP_CONV_GROUPS
#define OPP_CONV_GROUPS 2
#endif

namespace opp {

constexpr int kBlockM = 128;
// A ring stage holds one K chunk of kBlockK = 64 fp16.  Its slot width (GemmShape.bk, the kernels'
// BK) is the whole chunk, 128 B = one 128B-swizzle row, or half of it, 32 fp16 = one 64B-swizzle row:
// the stage is then filled and released half by half, so the wide conv tiles (N = 208 / 256, two
// stages) keep loads in flight while the MMAs still hold the other stage.
constexpr int kBlockK = 64;
__host__ __device__ constexpr int gemm_a_bytes(int bk) { return kBlockM * bk * 2; }   // one plane of the A tile
constexpr int kMaxStages = 8;
constexpr int kEpiParamBytes = 4096;   // bias / gamma,beta / lse vectors: 2 KB per epilogue group
constexpr int kMaxEpiWarps = 8;
// two MMA / epilogue warpgroups (Epi::kGroups must be 2) + the producer warpgroup
constexpr int gemm_threads(int groups) { return 128 + 128 * groups; }
constexpr int kProducerRegs = 40;         // setmaxnreg of the producer warpgroup
constexpr int kMmaRegs = 232;             // ... and of the MMA / epilogue warpgroups
static_assert(128 * kProducerRegs + 256 * kMmaRegs <= 65536, "register file of one SM");
// Accumulator widths the mainloop is compiled for (the N of its m64nNk16): a tile of block_n
// columns runs at the smallest one >= block_n.  208 = the 196-channel layers padded to 16.
constexpr int kMmaWidths[] = {64, 128, 208, 256};
constexpr int mma_width_for(int block_n) {
  for (int w : kMmaWidths)
    if (w >= block_n) return w;
  return 0;
}

enum AMode : int { A_ROWS = 0, A_CONV = 1, A_WIN = 2 };

struct TensorMaps {
  CUtensorMap a[4];
  CUtensorMap b;
};

struct GemmShape {
  int batches;      // tiles never straddle a batch
  int rows;         // A_ROWS: valid rows per batch; A_CONV: out_h*out_w
  int m_tiles;      // M tiles per batch
  int n_tiles;
  int n_total;      // valid output columns
  int block_n;      // output columns per tile (multiple of 16, <= 256)
  int mma_n;        // mma_width_for(block_n): W rows staged per tile and accumulator width
  int k_chunks;     // number of 64-wide K chunks per tile (per plane)
  int bk;           // K columns per ring slot: 64, or 32 (two slots per stage; conv_chunk_k and
                    // rows_chunk_k pick it per layer; a compile-time parameter of the kernel)
  int stages;       // ring stages of one K chunk each
  int b_batched;    // W operand has a leading batch dim
  int cluster;      // CTAs per cluster (1, 2, 4): they work on adjacent M tiles of the same
                    // (batch, n_tile) in lockstep and share the W tile through TMA multicast
  int msup;         // ceil(m_tiles / cluster)
  int pair;         // 2: "N-split cluster" (latency shapes of the LayerNorm GEMMs): the two CTAs of the
                    // cluster work on the SAME 128-row M tile, CTA r on columns [r*block_n, +block_n),
                    // independent pipelines, row statistics exchanged through DSMEM (EpiLN); else 0
  int acc_alias;    // the accumulator tile overlays the operand ring (it does not fit beside it):
                    // the producer starts a tile's loads only after the previous epilogue is done
  int debug_skip;   // TIMING EXPERIMENTS ONLY ($OPP_DEBUG_SKIP): 1 = skip W loads, 2 = skip A loads
  int split;        // operands are (hi|lo) plane pairs; 3 MMAs per K-step
  int b_lo;         // element offset of W's lo plane inside a row (= K total)
  // A_ROWS
  int k_chunks_a0;  // chunks read through maps.a[0]; the rest through maps.a[1]
  int a0_lo, a1_lo; // element offsets of the lo planes of the two A arrays (= their K)
  int a0_shared;    // the first A array is [1][rows][..]: one object shared by every batch element
  // A_CONV
  int conv_cchunks; // K chunks per filter tap
  int conv_c;       // padded input channels (multiple of 16); also the lo-plane offset
  int conv_kw;      // filter width/height (1 or 3)
  int conv_pad;
  int conv_stride;  // 1 or 2
  int tile_w, tile_h;    // output tile, tile_w*tile_h == 128
  int tiles_x, tiles_y;  // tiles per image
  int out_w, out_h;
  // A_WIN (sparse 3x3 convolution on per-match windows) reuses the conv fields: tile_w = 8 (window
  // row pitch), tile_h = window rows (7 or 5), tiles_x = windows per M tile (2 or 3; they occupy
  // tiles_x * tile_w * tile_h <= 128 accumulator rows), rows = matches * tile_w * tile_h,
  // m_tiles = ceil(matches / tiles_x), batches = 1.
};

struct EpiCtx {
  uint32_t acc;    // shared-memory word address (byte address / 4) of column 0 of this thread's
                   // accumulator row
  int b, m_tile, n_tile;
  int q;           // warp within the epilogue group
  int a_mode;
  int n0;          // first global column of the tile
  int ncols;       // valid columns in this tile (multiple of 8)
  int etid;        // 0..127 within the epilogue group
  float* smem;     // 2 KB of scratch shared by this epilogue group
  uint8_t* wstage; // kWarpStageBytes private to this warp (transpose buffer for coalesced I/O)
  uint32_t smem_s, wstage_s;   // the same two regions as 32-bit shared-space addresses
  int group;       // epilogue warp group (0/1); groups take alternate 32-column chunks
  int col_first, col_step;
  // rows (lane>>2) + 8*i, i = 0..3 of this warp's quarter of the accumulator tile (EpiFromRegs:
  // i = 0..1, the two rows of this thread's accumulator fragment): element offset grow*ld is NOT
  // stored, only grow (row index in the output) and validity, computed once per tile
  long long sgrow[4];
  unsigned svalid;
  int next_b, next_m_tile;   // the (batch, M tile) this CTA processes next, or next_b = -1
  uint8_t* extra;            // EpiExtraSmem<Epi>::value bytes (EpiLN: DSMEM exchange slots + 2 mbarriers)
  int it;                    // how many tiles this CTA has processed before this one
};

__device__ __forceinline__ void epi_sync(const EpiCtx& c) { named_bar_sync(1 + c.group, 128); }

// bytes of private staging per epilogue warp: kWarpStageBytes unless the epilogue declares
// `static constexpr int kWarpStage` (EpiConvUp stages both planes of a chunk at once)
template <class E, class = void>
struct EpiWarpStage {
  static constexpr int value = 32 * 80;
};
template <class E>
struct EpiWarpStage<E, std::void_t<decltype(E::kWarpStage)>> {
  static constexpr int value = E::kWarpStage;
};
// bytes of extra shared memory behind the warp stages: epilogues declare `static constexpr int kExtraSmem`
template <class E, class = void>
struct EpiExtraSmem {
  static constexpr int value = 0;
};
template <class E>
struct EpiExtraSmem<E, std::void_t<decltype(E::kExtraSmem)>> {
  static constexpr int value = E::kExtraSmem;
};
template <class E>
constexpr int epi_smem_bytes() {
  return 4096 + 8 * EpiWarpStage<E>::value + EpiExtraSmem<E>::value;   // kEpiParamBytes + kMaxEpiWarps * stage
}

// the narrowest mainloop an epilogue is compiled with: epilogues declare `static constexpr int
// kMinMmaN` (fit_tile then widens narrower tiles to it; the columns past ncols are never used)
template <class E, class = void>
struct EpiMinMmaN {
  static constexpr int value = 64;
};
template <class E>
struct EpiMinMmaN<E, std::void_t<decltype(E::kMinMmaN)>> {
  static constexpr int value = E::kMinMmaN;
};

// epilogues that look one tile ahead declare `static constexpr bool kNeedsNext`
template <class E, class = void>
struct EpiNeedsNext : std::false_type {};
template <class E>
struct EpiNeedsNext<E, std::void_t<decltype(E::kNeedsNext)>> : std::true_type {};

// epilogues that run on the accumulator registers declare `static constexpr bool kFromRegs` and
// `template <int N> static void run_frag(const Params&, const GemmShape&, const EpiCtx&, float (&d)[N / 2])`;
// their kernels have no accumulator tile in shared memory
template <class E, class = void>
struct EpiFromRegs : std::false_type {};
template <class E>
struct EpiFromRegs<E, std::void_t<decltype(E::kFromRegs)>> : std::true_type {};

// (global row, validity) of tile row `rit` (0..127)
__device__ __forceinline__ bool epi_row_at(const GemmShape& s, const EpiCtx& c, int rit,
                                           long long& grow, int& row) {
  bool ok;
  if (c.a_mode == A_ROWS) {
    row = c.m_tile * kBlockM + rit;
    ok = row < s.rows;
  } else if (c.a_mode == A_WIN) {
    const int wrows = s.tiles_x * s.tile_w * s.tile_h;   // accumulator rows in use
    row = c.m_tile * wrows + rit;
    ok = rit < wrows && row < s.rows;
  } else {
    const int ty = c.m_tile / s.tiles_x;
    const int tx = c.m_tile - ty * s.tiles_x;
    const int ly = rit / s.tile_w;
    const int oy = ty * s.tile_h + ly;
    const int ox = tx * s.tile_w + (rit - ly * s.tile_w);
    ok = oy < s.out_h && ox < s.out_w;
    row = oy * s.out_w + ox;
  }
  grow = (long long)c.b * s.rows + row;
  return ok;
}

// ---------------------------------------------------------------------------------------------
// Accumulator tile in shared memory (EpiConvUp only): row r, column j at word  r * (mma_n + kAccPad) + j.
// The pad of kAccPad = 4 words puts the 16-byte reads of 8 consecutive rows into distinct banks.
// ---------------------------------------------------------------------------------------------
constexpr int kAccPad = 4;
__host__ __device__ constexpr int gemm_acc_bytes(int mma_n) { return 128 * (mma_n + kAccPad) * 4; }

// 32 consecutive fp32 columns of this thread's accumulator row, starting at word address `waddr`
__device__ __forceinline__ void acc_ld32(uint32_t waddr, float (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 u = lds128(waddr * 4 + 16 * i);
    v[4 * i + 0] = __uint_as_float(u.x);
    v[4 * i + 1] = __uint_as_float(u.y);
    v[4 * i + 2] = __uint_as_float(u.z);
    v[4 * i + 3] = __uint_as_float(u.w);
  }
}

// ---------------------------------------------------------------------------------------------
// Warp-staged, coalesced store of one-row-per-thread values (EpiConvUp): global memory wants whole
// 64/128-byte segments, so every 32x32 chunk goes through a per-warp shared-memory transpose buffer
// (row stride padded by 16 B so both access directions are conflict-light).
// ---------------------------------------------------------------------------------------------
constexpr int kStageRowH = 80;    // 32 fp16 (64 B) + 16 B pad
constexpr int kWarpStageBytes = 32 * kStageRowH;   // 2560 B

// fp16 planes: v = this lane's 32 values for global columns [gcol, gcol+32); nvalid = valid
// columns of the chunk (multiple of 8).  Writes hi (and lo when lo_off != 0).
__device__ __forceinline__ void staged_store_h32(const GemmShape& s, const EpiCtx& c, __half* out,
                                                 long long ld, int lo_off, int gcol,
                                                 const float* v, int nvalid) {
  if (s.debug_skip & 8) return;   // bit 3: timing experiment, epilogue math without the stores
  const int lane = threadIdx.x & 31;
  const uint32_t st = c.wstage_s;
#pragma unroll
  for (int plane = 0; plane < 2; ++plane) {
    if (plane == 1 && lo_off == 0) break;
    const uint32_t mine = st + lane * kStageRowH;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      uint4 u;
      if (plane == 0) {
        u.x = pack_half2(v[8 * g + 0], v[8 * g + 1]);
        u.y = pack_half2(v[8 * g + 2], v[8 * g + 3]);
        u.z = pack_half2(v[8 * g + 4], v[8 * g + 5]);
        u.w = pack_half2(v[8 * g + 6], v[8 * g + 7]);
      } else {
        float l[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          l[j] = v[8 * g + j] - __half2float(__float2half_rn(v[8 * g + j]));
        u.x = pack_half2(l[0], l[1]);
        u.y = pack_half2(l[2], l[3]);
        u.z = pack_half2(l[4], l[5]);
        u.w = pack_half2(l[6], l[7]);
      }
      sts128(mine + g * 16, u);
    }
    __syncwarp();
    const int seg = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = (lane >> 2) + 8 * i;
      if (((c.svalid >> i) & 1u) && seg * 8 < nvalid)
        *reinterpret_cast<uint4*>(out + c.sgrow[i] * ld + plane * lo_off + gcol + seg * 8) =
            lds128(st + rr * kStageRowH + seg * 16);
    }
    __syncwarp();
  }
}

// =============================================================================================
// Epilogues.  Outputs that feed later GEMMs are written as (hi|lo) plane pairs when
// `out_lo` != 0: row layout [hi(n_total) | lo(n_total)], out_lo = n_total.
// =============================================================================================

// ---------------------------------------------------------------------------------------------
// Register-fragment epilogue I/O (EpiFromRegs).  Warp q of MMA warpgroup g holds tile rows
// 64g + 16q .. +15 over all mma_n columns; this lane holds rows (lane>>2) + 8h, h = 0, 1 of them
// (c.sgrow[h], bit h of c.svalid) at columns 8i + 2(lane&3) + {0, 1}: d[4i + 2h + {0, 1}].  Those
// 16 rows are 16 consecutive output rows (one 16-pixel image row of a conv tile, or 16 consecutive
// window rows), so the global I/O of a 32-column slice (fragment columns i = 4j .. 4j+3) goes through
// the warp's stage: lane moves the 16-byte segment (lane&3) of its two rows, 8 rows x 64 B per
// instruction, and the fragment side reads / writes 4 (fp16 pair) or 8 (fp32 pair) bytes, without
// bank conflicts at these row pitches.  A slice's values are v[4 ii + 2h + e] for i = 4j + ii.
// ---------------------------------------------------------------------------------------------
constexpr int kFragRowH = 80;                  // fp16 slice row: 64 B + 16 B pad
constexpr int kFragPlaneH = 16 * kFragRowH;    // one plane of a 16 x 32 fp16 slice (1280 B)
constexpr int kFragRowF = 160;                 // fp32 slice row: 128 B + 32 B pad (16 rows = the whole stage)

__device__ __forceinline__ void sts32u(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t lds32u(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds64f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

__device__ __forceinline__ void sts64f(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// the (tile-row) fragment values of slice j: v[4 ii + 2h + e] = d[4 (4j + ii) + 2h + e]; columns
// past the accumulator width (the second half of the last slice at N = 208) read as `fill`
template <int N>
__device__ __forceinline__ void frag_slice(const float (&d)[N / 2], int j, float (&v)[16], float fill = 0.f) {
#pragma unroll
  for (int k = 0; k < 16; ++k) v[k] = 16 * j + k < N / 2 ? d[16 * j + k] : fill;
}

// + the fp32 vector at smem word address `base` (the epilogue group's bias) per fragment column
__device__ __forceinline__ void frag_add_cols(uint32_t base_s, int col, float (&v)[16]) {
  const int c0 = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const float2 b = lds64f(base_s + 4 * ((col + 8 * ii + c0) & 255));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      v[4 * ii + 2 * h] += b.x;
      v[4 * ii + 2 * h + 1] += b.y;
    }
  }
}

// fp16 planes of slice columns [gcol, gcol + 32) of this warp's 16 rows (hi, and lo when lo_off != 0);
// nvalid = valid columns of the slice (multiple of 8)
__device__ __forceinline__ void frag_store_h(const GemmShape& s, const EpiCtx& c, __half* out, long long ld,
                                             int lo_off, int gcol, const float (&v)[16], int nvalid) {
  if (s.debug_skip & 8) return;   // bit 3: timing experiment, epilogue math without the stores
  const int lane = threadIdx.x & 31, t = lane & 3, rq = lane >> 2;
  const uint32_t st = c.wstage_s;
#pragma unroll
  for (int ii = 0; ii < 4; ++ii)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float a = v[4 * ii + 2 * h], b = v[4 * ii + 2 * h + 1];
      const uint32_t addr = st + (rq + 8 * h) * kFragRowH + 16 * ii + 4 * t;
      sts32u(addr, pack_half2(a, b));
      if (lo_off)
        sts32u(addr + kFragPlaneH, pack_half2(a - __half2float(__float2half_rn(a)),
                                              b - __half2float(__float2half_rn(b))));
    }
  __syncwarp();
#pragma unroll
  for (int plane = 0; plane < 2; ++plane) {
    if (plane == 1 && lo_off == 0) break;
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (((c.svalid >> h) & 1u) && t * 8 < nvalid)
        *reinterpret_cast<uint4*>(out + c.sgrow[h] * ld + plane * lo_off + gcol + t * 8) =
            lds128(st + plane * kFragPlaneH + (rq + 8 * h) * kFragRowH + 16 * t);
  }
  __syncwarp();
}

// fp32 slice columns [gcol, gcol + 32) of this warp's 16 rows (row stride ld floats, 16-byte aligned
// rows): the slice goes through the stage (row pitch kFragRowF) and leaves it in two 16-column halves,
// lane moving the 16-byte segment (lane&3) of its two rows: 8 rows x 64 B per instruction.
// nvalid = valid columns of the slice (multiple of 4).
__device__ __forceinline__ void frag_store_f32(const EpiCtx& c, float* out, long long ld, int gcol,
                                               const float (&v)[16], int nvalid) {
  const int lane = threadIdx.x & 31, t = lane & 3, rq = lane >> 2;
  const uint32_t st = c.wstage_s;
#pragma unroll
  for (int ii = 0; ii < 4; ++ii)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      sts64f(st + (rq + 8 * h) * kFragRowF + 4 * (8 * ii + 2 * t), v[4 * ii + 2 * h], v[4 * ii + 2 * h + 1]);
  __syncwarp();
#pragma unroll
  for (int half = 0; half < 2; ++half)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (((c.svalid >> h) & 1u) && 16 * half + 4 * t < nvalid)
        *reinterpret_cast<uint4*>(out + c.sgrow[h] * ld + gcol + 16 * half + 4 * t) =
            lds128(st + (rq + 8 * h) * kFragRowF + 64 * half + 16 * t);
  __syncwarp();
}

// Residual rows (same layout as the output) of one slice: copied into the warp's stage without
// passing through registers (rows / columns outside the tensor read as 0); frag_load_add then adds
// hi, then lo to the fragment values.
__device__ __forceinline__ void frag_load_issue(const EpiCtx& c, const __half* src, long long ld, int lo_off,
                                                int gcol, int nvalid) {
  const int lane = threadIdx.x & 31, t = lane & 3, rq = lane >> 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool in = ((c.svalid >> h) & 1u) && t * 8 < nvalid;
    const __half* row = in ? src + c.sgrow[h] * ld + gcol + t * 8 : src;
    const uint32_t dst = c.wstage_s + (rq + 8 * h) * kFragRowH + 16 * t;
    cp_async16_zfill(dst, row, in ? 16 : 0);
    if (lo_off) cp_async16_zfill(dst + kFragPlaneH, in ? row + lo_off : src, in ? 16 : 0);
  }
  cp_async_commit();
}
__device__ __forceinline__ void frag_load_add(const EpiCtx& c, int lo_off, float (&v)[16]) {
  const int lane = threadIdx.x & 31, t = lane & 3, rq = lane >> 2;
  const uint32_t st = c.wstage_s;
  cp_async_wait<0>();
  __syncwarp();
#pragma unroll
  for (int plane = 0; plane < 2; ++plane) {
    if (plane == 1 && lo_off == 0) break;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t u = lds32u(st + plane * kFragPlaneH + (rq + 8 * h) * kFragRowH + 16 * ii + 4 * t);
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
        v[4 * ii + 2 * h] += f.x;
        v[4 * ii + 2 * h + 1] += f.y;
      }
  }
  __syncwarp();
}

// + an fp32 row-major matrix (row stride ld floats) at rows row[h], slice columns [gcol, gcol + 32),
// for the rows of c.svalid (the others are left unchanged)
__device__ __forceinline__ void frag_add_f32(const EpiCtx& c, const float* src, long long ld, const int (&row)[2],
                                             int gcol, int nvalid, float (&v)[16]) {
  const int lane = threadIdx.x & 31, t = lane & 3, rq = lane >> 2;
  const uint32_t st = c.wstage_s;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int k = 0; k < 2; ++k) {   // 16-byte segments t and t + 4 of the 128-byte row slice
      const int seg = t + 4 * k;
      if (((c.svalid >> h) & 1u) && seg * 4 < nvalid)
        sts128(st + (rq + 8 * h) * kFragRowF + 16 * seg,
               *reinterpret_cast<const uint4*>(src + (long long)row[h] * ld + gcol + seg * 4));
    }
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!((c.svalid >> h) & 1u)) continue;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
      if (8 * ii < nvalid) {
        const float2 f = lds64f(st + (rq + 8 * h) * kFragRowF + 4 * (8 * ii + 2 * t));
        v[4 * ii + 2 * h] += f.x;
        v[4 * ii + 2 * h + 1] += f.y;
      }
  }
  __syncwarp();
}

__device__ __forceinline__ void frag_act(int act, float slope, float (&v)[16]) {
  if (act == 1) {
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = fmaxf(v[k], 0.f);
  } else if (act == 2) {
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = v[k] > 0.f ? v[k] : v[k] * slope;
  }
}

// the tile's columns of a per-column fp32 vector into this epilogue group's parameter smem: once per
// CTA when the launch has one N tile (every tile has the same columns), else per tile
__device__ __forceinline__ void epi_stage_cols(const GemmShape& s, const EpiCtx& c, const float* src) {
  if (c.it > 0 && s.n_tiles == 1) return;
  epi_sync(c);
  for (int i = c.etid; i < c.ncols; i += 128) sts32f(c.smem_s + 4 * i, src[c.n0 + i]);
  epi_sync(c);
}

// Convolution epilogue: folded-BN bias, residual add, ReLU / LeakyReLU (resnet.py:36-45,112-124,
// 141-147).  Optionally also emits the coarse tokens  x3_out + pe  in token-major order
// (position_encoding.py:37-42 + OnePosePlusModel.py:137-142: NHWC *is* 'n (h w) c').
struct EpiConvParams {
  __half* out;          // NHWC, pixel stride ld (or null)
  long long ld;
  int out_lo;
  const float* bias;    // [n_total]
  const __half* resid;  // same layout as out, or null
  int act;              // 0 none, 1 relu, 2 leaky relu
  float slope;
  __half* tok;          // [B*H*W] rows with the same (ld, out_lo) layout, or null
  const float* pe;      // [H*W][n_total]
  // FPN top-down path (resnet.py:149-157): out = conv(x) + bilinear_x2(up), align_corners=True.
  // up is the coarser map [B][up_h][up_w] with the same (ld, out_lo) channel layout, or null.
  const __half* up;
  int up_h, up_w;
  float up_sy, up_sx;   // (in - 1) / (out - 1)
};
struct EpiConv {
  static constexpr int kGroups = OPP_CONV_GROUPS;
  static constexpr const char* kName = "conv";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  using Params = EpiConvParams;
  // Called before the MMAs of the tile: pull this lane's share of the residual rows towards L2
  // while they run (the conv2 of a BasicBlock was epilogue-bound on this read).
  __device__ static void prefetch(const Params& p, const GemmShape& s, const EpiCtx& c) {
    if (!p.resid) return;
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!((c.svalid >> h) & 1u)) continue;
      const char* row = reinterpret_cast<const char*>(p.resid + c.sgrow[h] * p.ld + c.n0);
      for (int o = 128 * t; o < c.ncols * 2; o += 512) {
        asm volatile("prefetch.global.L2 [%0];" ::"l"(row + o));
        if (p.out_lo) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + 2 * p.out_lo + o));
      }
    }
  }
  // Per element, in this order: acc + bias, + residual hi, + residual lo, activation, the (hi, lo)
  // store, then + pe and the token store.
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    const bool has_res = p.resid != nullptr;
    // the residual of a slice is copied into the stage when the stage is free: before the bias of
    // the tile is staged, and after the stores of the previous slice
    if (has_res) frag_load_issue(c, p.resid, p.ld, p.out_lo, c.n0, c.ncols);
    epi_stage_cols(s, c, p.bias);
    int prow[2] = {0, 0};   // pixel index inside the image of the two fragment rows (tokens)
#pragma unroll
    for (int h = 0; h < 2; ++h) prow[h] = (int)(c.sgrow[h] - (long long)c.b * s.rows);
#pragma unroll
    for (int j = 0; j < (N + 31) / 32; ++j) {
      const int col = 32 * j;
      if (col < c.ncols) {
        const int g0 = c.n0 + col;
        const int nvalid = c.ncols - col;   // >= 8, multiple of 8; columns past it are padding
        float v[16];
        frag_slice<N>(d, j, v);
        frag_add_cols(c.smem_s, col, v);
        if (has_res) frag_load_add(c, p.out_lo, v);
        frag_act(p.act, p.slope, v);
        if (p.out) frag_store_h(s, c, p.out, p.ld, p.out_lo, g0, v, nvalid);
        if (p.tok) {
          frag_add_f32(c, p.pe, s.n_total, prow, g0, nvalid, v);
          frag_store_h(s, c, p.tok, p.ld, p.out_lo, g0, v, nvalid);
        }
        if (has_res && col + 32 < c.ncols) frag_load_issue(c, p.resid, p.ld, p.out_lo, g0 + 32, nvalid - 32);
      }
    }
  }
};

// Sparse 3x3 convolution on per-match windows (A_WIN): the fine branch of the FPN
// (resnet.py:155-157, layer1_outconv2) is only ever read inside the W x W window of each coarse
// match (fine_preprocess.py:40-47 unfolds the map and keeps the matched cells), so the two
// half-resolution 3x3 convolutions are evaluated on those windows alone: conv A on the 7x7
// neighbourhood of a match (what conv B's 5x5 outputs need), conv B on the 5x5 window.
// Output rows are compact: window m, position (ly, lx) -> row (m * tile_h + ly) * 8 + lx.
// j_ids != null: the input is the dense NHWC map and the window origin comes from the match's
// coarse cell: x = stride * cx + org + lx, y likewise; rows whose position lies outside the image
// are written as ZERO (they are the zero padding conv B must see).  j_ids == null: the input is a
// compact window tensor [matches][tile_h + 2][8][C] of a previous A_WIN launch.
struct EpiWin {
  static constexpr int kGroups = OPP_CONV_GROUPS;
  static constexpr const char* kName = "conv_win";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  struct Params {
    __half* out;
    long long ld;
    int out_lo;
    const float* bias;
    int act;
    float slope;
    const long long* b_ids;   // [matches] image of the match (dense input only)
    const long long* j_ids;   // [matches] coarse cell of the match, or null: compact input
    int wc;                   // coarse cells per row
    int stride;               // input pixels per coarse cell (4)
    int org;                  // first output position relative to stride * cell (-3 / -2)
    int in_h, in_w;           // dense map size
  };
  __device__ static void prefetch(const Params&, const GemmShape&, const EpiCtx&) {}
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    epi_stage_cols(s, c, p.bias);
    bool inside[2] = {true, true};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (p.j_ids && ((c.svalid >> h) & 1u)) {
        const int rpm = s.tile_w * s.tile_h;
        const int m = (int)(c.sgrow[h] / rpm);
        const int local = (int)(c.sgrow[h] - (long long)m * rpm);
        const int ly = local / s.tile_w, lx = local - ly * s.tile_w;
        const int jj = (int)p.j_ids[m];
        const int cy = jj / p.wc;
        const int y = p.stride * cy + p.org + ly, x = p.stride * (jj - cy * p.wc) + p.org + lx;
        inside[h] = y >= 0 && y < p.in_h && x >= 0 && x < p.in_w;
      }
    }
#pragma unroll
    for (int j = 0; j < (N + 31) / 32; ++j) {
      const int col = 32 * j;
      if (col < c.ncols) {
        float v[16];
        frag_slice<N>(d, j, v);
        frag_add_cols(c.smem_s, col, v);
        frag_act(p.act, p.slope, v);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (!inside[h]) {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) v[4 * ii + 2 * h] = v[4 * ii + 2 * h + 1] = 0.f;
          }
        frag_store_h(s, c, p.out, p.ld, p.out_lo, c.n0 + col, v, c.ncols - col);
      }
    }
  }
};

// Lateral 1x1 convolution of the FPN top-down path with the bilinear x2 upsample-add fused in
// (resnet.py:149-157: layerN_outconv(x) + F.interpolate(coarser, scale_factor=2, mode="bilinear",
// align_corners=True)); torch semantics: src = dst * (in-1)/(out-1), i0 = floor(src),
// i1 = min(i0+1, in-1).  No residual / activation / tokens on these layers.
//
// A warp owns 2 output rows x 16 columns of the 8x16 tile; their neighbours lie in a 3 x 10 window
// of the coarse map (15 * 0.5 < 8 columns, 1 * 0.5 < 1 row).  Per 32-channel chunk and plane the
// warp fetches those <= 30 pixels' 64-byte segments coalesced into its transpose buffer
// (slot = wy * 10 + wx) and every lane reads its own four neighbours from shared memory.
// Loading on demand would cost one dependent DRAM round trip per chunk and plane (the coarse map
// does not fit in L2), so (i) the NEXT tile's window is pulled into L2 while this tile is processed, (ii) both planes
// of a chunk are loaded together and (iii) the loads of chunk i+1 are issued before the plane-1
// math and the stores of chunk i.
struct EpiConvUp {
  static constexpr int kGroups = OPP_CONV_GROUPS;
  static constexpr const char* kName = "conv_up";   // $OPP_LOG_TILES
  static constexpr bool kNeedsNext = true;   // EpiCtx::next_b / next_m_tile are filled in
  static constexpr int kWarpStage = 2 * 32 * 80;   // hi and lo windows of a chunk side by side
  using Params = EpiConvParams;

  struct Geo {
    int ymin, xmin;
  };
  // (ymin, xmin) of the 3 x 10 source window of warp quarter q of tile (m_tile): floor of the source
  // coordinate of the warp's first output pixel (its minimum in both axes)
  __device__ static Geo window(const Params& p, const GemmShape& s, int m_tile, int q) {
    const int ty = m_tile / s.tiles_x;
    const int oy = min(ty * s.tile_h + (q * 32) / s.tile_w, s.out_h - 1);
    const int ox = min((m_tile - ty * s.tiles_x) * s.tile_w, s.out_w - 1);
    return Geo{(int)(p.up_sy * (float)oy), (int)(p.up_sx * (float)ox)};
  }
  // pixel index (not yet multiplied by the pixel stride) of window slot `slot` (0..29)
  __device__ static long long slot_pixel(const Params& p, int b, const Geo& g, int slot) {
    const int sy_ = slot / 10, sx_ = slot - sy_ * 10;
    return ((long long)b * p.up_h + min(g.ymin + sy_, p.up_h - 1)) * p.up_w + min(g.xmin + sx_, p.up_w - 1);
  }
  __device__ static void prefetch(const Params& p, const GemmShape& s, const EpiCtx& c) {
    // L2 prefetch of the NEXT tile's window for this warp: 30 pixels x (planes * C * 2 B), lane = slot
    if (c.next_b < 0) return;
    const int lane = threadIdx.x & 31;
    if (lane >= 30) return;
    const Geo g = window(p, s, c.next_m_tile, c.q);
    const char* px = reinterpret_cast<const char*>(p.up + slot_pixel(p, c.next_b, g, lane) * p.ld);
    const int bytes = (p.out_lo ? 2 : 1) * s.n_total * 2;
    // the two epilogue groups split the lines of a pixel between them
    for (int o = c.group * 128; o < bytes; o += 128 * kGroups) asm volatile("prefetch.global.L2 [%0];" ::"l"(px + o));
  }
  __device__ static void run(const Params& p, const GemmShape& s, const EpiCtx& c) {
    // the bias of this tile's columns: a persistent CTA may visit both N tiles of a narrowed conv
    epi_sync(c);
    for (int i = c.etid; i < c.ncols; i += 128) sts32f(c.smem_s + 4 * i, p.bias[c.n0 + i]);
    epi_sync(c);
    const int lane = threadIdx.x & 31;
    const int seg = lane & 3;
    // this lane's output pixel and its interpolation weights / neighbour slots
    const Geo g = window(p, s, c.m_tile, c.q);
    float w00, w01, w10, w11;
    uint32_t a00, a01, a10, a11;
    {
      const int rit = c.q * 32 + lane;
      const int ty = c.m_tile / s.tiles_x;
      const int ly = rit / s.tile_w;
      const int oy = min(ty * s.tile_h + ly, s.out_h - 1);
      const int ox = min((c.m_tile - ty * s.tiles_x) * s.tile_w + (rit - ly * s.tile_w), s.out_w - 1);
      const float fy = p.up_sy * (float)oy, fx = p.up_sx * (float)ox;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < p.up_h - 1 ? 1 : 0), x1 = x0 + (x0 < p.up_w - 1 ? 1 : 0);
      const float wy = fy - (float)y0, wx = fx - (float)x0;
      w00 = (1.f - wy) * (1.f - wx);
      w01 = (1.f - wy) * wx;
      w10 = wy * (1.f - wx);
      w11 = wy * wx;
      a00 = c.wstage_s + ((y0 - g.ymin) * 10 + (x0 - g.xmin)) * kStageRowH;
      a01 = c.wstage_s + ((y0 - g.ymin) * 10 + (x1 - g.xmin)) * kStageRowH;
      a10 = c.wstage_s + ((y1 - g.ymin) * 10 + (x0 - g.xmin)) * kStageRowH;
      a11 = c.wstage_s + ((y1 - g.ymin) * 10 + (x1 - g.xmin)) * kStageRowH;
    }
    // the four window pixels this lane stages (slot = lane / 4 + 8 i, 16-byte segment lane % 4)
    int spix[4];   // 32-bit pixel indices (64-bit pointers here spilled and serialised the loads on LDL)
#pragma unroll
    for (int i = 0; i < 4; ++i) spix[i] = (int)slot_pixel(p, c.b, g, min((lane >> 2) + 8 * i, 29));
    const __half* upb = p.up + seg * 8 + c.n0;
    const bool two = p.out_lo != 0;
    uint4 nb[8];   // [plane][slot]: the window segments of the chunk about to be processed
    auto issue = [&](int col) {
      const bool ok = seg * 8 < c.ncols - col;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __half* px = upb + (long long)spix[i] * p.ld + col;
        nb[i] = ok ? *reinterpret_cast<const uint4*>(px) : make_uint4(0, 0, 0, 0);
        nb[4 + i] = (ok && two) ? *reinterpret_cast<const uint4*>(px + p.out_lo) : make_uint4(0, 0, 0, 0);
      }
    };
    // both planes of the window are staged side by side (lo at +kLo) and blended in one sweep: two
    // independent FMA chains per element instead of two dependent stage/sync/blend rounds
    constexpr uint32_t kLo = 32 * kStageRowH;
    auto stage = [&]() {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t a = c.wstage_s + ((lane >> 2) + 8 * i) * kStageRowH + seg * 16;
        sts128(a, nb[i]);
        if (two) sts128(a + kLo, nb[4 + i]);
      }
      __syncwarp();
    };
    auto blend = [&](float* v) {
#pragma unroll
      for (int q4 = 0; q4 < 4; ++q4) {
#pragma unroll
        for (int plane = 0; plane < 2; ++plane) {
          if (plane == 1 && !two) break;
          const uint32_t o = plane * kLo + q4 * 16;
          const uint4 q00 = lds128(a00 + o), q01 = lds128(a01 + o);
          const uint4 q10 = lds128(a10 + o), q11 = lds128(a11 + o);
          const __half2* h00 = reinterpret_cast<const __half2*>(&q00);
          const __half2* h01 = reinterpret_cast<const __half2*>(&q01);
          const __half2* h10 = reinterpret_cast<const __half2*>(&q10);
          const __half2* h11 = reinterpret_cast<const __half2*>(&q11);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 fa = __half22float2(h00[j]), fb = __half22float2(h01[j]);
            const float2 fc = __half22float2(h10[j]), fd = __half22float2(h11[j]);
            v[8 * q4 + 2 * j] += (w00 * fa.x + w01 * fb.x) + (w10 * fc.x + w11 * fd.x);
            v[8 * q4 + 2 * j + 1] += (w00 * fa.y + w01 * fb.y) + (w10 * fc.y + w11 * fd.y);
          }
        }
      }
      __syncwarp();
    };
    if (c.col_first < c.ncols) issue(c.col_first);
    for (int col = c.col_first; col < c.ncols; col += c.col_step) {
      float v[32];
      acc_ld32(c.acc + col, v);
#pragma unroll
      for (int q4 = 0; q4 < 8; ++q4) {
        const uint4 bq = lds128(c.smem_s + 4 * ((col + 4 * q4) & 255));
        v[4 * q4 + 0] += __uint_as_float(bq.x);
        v[4 * q4 + 1] += __uint_as_float(bq.y);
        v[4 * q4 + 2] += __uint_as_float(bq.z);
        v[4 * q4 + 3] += __uint_as_float(bq.w);
      }
      stage();
      // nb is free again: fetch the next chunk's window while this chunk is blended and stored
      const int ncol = col + c.col_step;
      if (ncol < c.ncols) issue(ncol);
      blend(v);
      if (p.act == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
      } else if (p.act == 2) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * p.slope;
      }
      staged_store_h32(s, c, p.out, p.ld, p.out_lo, c.n0 + col, v, c.ncols - col);
    }
  }
};

// =============================================================================================
// Token-row epilogues (A_ROWS), on the accumulator registers like the conv epilogues.  Warp q of
// warpgroup g holds the 16 consecutive token rows 64g + 16q .. +15 of the tile over all N columns, so
// a row never spans the two warpgroups: this lane holds rows (lane>>2) + 8h (c.sgrow[h], bit h of
// c.svalid) at columns 8i + 2(lane&3) + {0, 1}.  A row is spread over the 4 lanes of a quad (row
// reductions: two xor shuffles, every lane ends with the same bits), a column over the two rows of
// a lane and the 8 quads of the warp (column reductions: in the lane, then three xor levels).
// =============================================================================================
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
// (value, column) maximum over the quad; the lowest column wins a tie, whatever the lane order
__device__ __forceinline__ void quad_argmax(float& v, int& idx) {
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) {
      v = ov;
      idx = oi;
    }
  }
}

// Column reductions of a 32-column slice: x[k], k = 2 ii + e, is this lane's value of slice column
// 8 ii + 2 (lane&3) + e.  col_allreduce8: every lane ends with the reduction of its 8 columns over
// the warp's 16 rows (xor butterfly over lane bits 2..4).  col_reduce8: at each level a lane keeps
// one half of its values and trades the other half with lane ^ (4 << lvl) (7 shuffles); lane ends
// with the reduction of slice column frag_lane_col() only.
template <class Op>
__device__ __forceinline__ void col_allreduce8(float (&x)[8], Op op) {
#pragma unroll
  for (int o = 4; o <= 16; o <<= 1)
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = op(x[k], __shfl_xor_sync(0xffffffffu, x[k], o));
}
template <class Op>
__device__ __forceinline__ float col_reduce8(float (&x)[8], Op op) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int lvl = 2; lvl >= 0; --lvl) {
    const int half = 1 << lvl;
    const bool up = (lane >> (2 + lvl)) & 1;
#pragma unroll
    for (int k = 0; k < half; ++k) {
      const float keep = up ? x[half + k] : x[k];
      const float send = up ? x[k] : x[half + k];
      x[k] = op(keep, __shfl_xor_sync(0xffffffffu, send, 4 << lvl));
    }
  }
  return x[0];   // value k = lane >> 2
}
__device__ __forceinline__ int frag_lane_col() {
  const int lane = threadIdx.x & 31, rq = lane >> 2;
  return 8 * (rq >> 1) + 2 * (lane & 3) + (rq & 1);
}
// element k of x (k warp-uniform at run time, x indexed by compile-time constants only)
__device__ __forceinline__ float pick8(const float (&x)[8], int k) {
  float r = x[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) r = k == i ? x[i] : r;
  return r;
}
// the two warps of a 32-row group (q = 2k, 2k+1 of the epilogue group) meet here
__device__ __forceinline__ void pair_sync(const EpiCtx& c) { named_bar_sync(5 + 2 * c.group + (c.q >> 1), 64); }

// fp32 per-column vector of this tile (lse of the other side), staged per tile: it changes with the
// batch and the N tile
__device__ __forceinline__ void epi_stage_cols_b(const GemmShape& s, const EpiCtx& c, const float* src) {
  epi_sync(c);
  for (int i = c.etid; i < c.ncols; i += 128) sts32f(c.smem_s + 4 * i, src[(long long)c.b * s.n_total + c.n0 + i]);
  epi_sync(c);
}

// Plain store with an optional activation on the leading `act_cols` columns.
//   act 1 = ReLU  (transformer.py:41-45 mlp ReLU), act 2 = elu(x)+1 (linear_attention.py:10-11)
// Per element exactly the operations of the shared-memory form: the outputs are bit-identical.
struct EpiStoreF16 {
  static constexpr int kGroups = 2;
  static constexpr const char* kName = "store_f16";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  struct Params {
    __half* out;
    long long ld;   // row stride in elements
    int out_lo;     // 0 or n_total
    int act;
    int act_cols;   // multiple of 32
    // padded positions (query_image_mask, linear_attention.py:49-53): rows with row_mask[grow] == 0
    // are written as zeros (K' and V of a masked source token), or null
    const unsigned char* row_mask;
  };
  __device__ static void prefetch(const Params&, const GemmShape&, const EpiCtx&) {}
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    bool masked[2] = {false, false};
#pragma unroll
    for (int h = 0; h < 2; ++h) masked[h] = p.row_mask && ((c.svalid >> h) & 1u) && p.row_mask[c.sgrow[h]] == 0;
#pragma unroll
    for (int j = 0; j < (N + 31) / 32; ++j) {
      const int col = 32 * j;
      if (col < c.ncols) {
        const int g0 = c.n0 + col;
        const int act = g0 < p.act_cols ? p.act : 0;
        float v[16];
        frag_slice<N>(d, j, v);
        if (act == 1) {
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = fmaxf(v[k], 0.f);
        } else if (act == 2) {
#pragma unroll
          for (int k = 0; k < 16; ++k) v[k] = elu_plus_one_fast(v[k]);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (masked[h]) {
#pragma unroll
            for (int ii = 0; ii < 4; ++ii) v[4 * ii + 2 * h] = v[4 * ii + 2 * h + 1] = 0.f;
          }
        frag_store_h(s, c, p.out, p.ld, p.out_lo, g0, v, c.ncols - col);
      }
    }
  }
};

// Query side of linear attention (linear_attention.py:45,58-59): Q = elu(q)+1,
// Z = 1/(Q . Ksum + eps), output Q * Z * v_length per head of 32 channels.  The matching KV
// state is pre-divided by v_length (linear_attention.py:55-56), so (Q*Z*v_length) @ (KV/v_length)
// reproduces the reference product.  A head is one 32-column slice: its dot is 8 products per lane
// and a quad sum.
struct EpiQ {
  static constexpr int kGroups = 2;
  static constexpr const char* kName = "q";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  struct Params {
    __half* out;
    long long ld;
    int out_lo;
    const float* ksum;  // [batches][n_total]
    float v_len;
    float eps;
    const unsigned char* row_mask;   // Q = 0 on padded query positions (linear_attention.py:49-50), or null
  };
  __device__ static void prefetch(const Params&, const GemmShape&, const EpiCtx&) {}
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    epi_stage_cols_b(s, c, p.ksum);
    const int c0 = 2 * (threadIdx.x & 3);
    bool qmasked[2] = {false, false};
#pragma unroll
    for (int h = 0; h < 2; ++h) qmasked[h] = p.row_mask && ((c.svalid >> h) & 1u) && p.row_mask[c.sgrow[h]] == 0;
#pragma unroll
    for (int j = 0; j < (N + 31) / 32; ++j) {
      const int col = 32 * j;
      if (col < c.ncols) {
        float v[16];
        frag_slice<N>(d, j, v);
        float dot[2] = {0.f, 0.f};
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          const float2 kk = lds64f(c.smem_s + 4 * (col + 8 * ii + c0));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            v[4 * ii + 2 * h] = elu_plus_one_fast(v[4 * ii + 2 * h]);
            v[4 * ii + 2 * h + 1] = elu_plus_one_fast(v[4 * ii + 2 * h + 1]);
            dot[h] = fmaf(v[4 * ii + 2 * h], kk.x, dot[h]);
            dot[h] = fmaf(v[4 * ii + 2 * h + 1], kk.y, dot[h]);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float qd = quad_sum(dot[h]);   // every lane shuffles, masked rows included
          const float z = qmasked[h] ? 0.f : p.v_len / (qd + p.eps);
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            v[4 * ii + 2 * h] *= z;
            v[4 * ii + 2 * h + 1] *= z;
          }
        }
        frag_store_h(s, c, p.out, p.ld, p.out_lo, c.n0 + col, v, 32);
      }
    }
  }
};

// LayerNorm over the full output row (the tile spans all N columns), optional residual add
// (transformer.py:86-94: norm1 after merge; norm2 then x + msg).  A row lives in one quad: mean and
// M2 are two passes over the registers with a quad sum each.  The tile is the whole row (the
// launchers check block_n == mma_n == n, or the 128-column halves of the N-split cluster).
struct EpiLN {
  static constexpr int kGroups = 2;
  static constexpr const char* kName = "ln";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  // N-split cluster (GemmShape.pair == 2): 2 x 128 (mean, M2) slots the peer CTA writes into + 2 mbarriers
  static constexpr int kExtraSmem = 2 * 128 * 8 + 64;
  static constexpr int kExchangeArrivals = 64;   // one writer lane per quad of the 8 MMA warps
  struct Params {
    const float* gamma;
    const float* beta;
    float eps;
    const __half* resid;  // same layout as out16 (ld, out_lo) or null
    int resid_shared;     // resid is [1][rows][..], shared by every batch element
    __half* out16;        // or null
    long long ld;
    int out_lo;
    float* out32;         // fp32 [rows][n_total] or null
  };
  __device__ static void prefetch(const Params& p, const GemmShape& s, const EpiCtx& c) {
    if (!p.resid) return;
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!((c.svalid >> h) & 1u)) continue;
      const long long r = p.resid_shared ? c.sgrow[h] - (long long)c.b * s.rows : c.sgrow[h];
      const char* row = reinterpret_cast<const char*>(p.resid + r * p.ld + c.n0);
      for (int o = 128 * t; o < c.ncols * 2; o += 512) {
        asm volatile("prefetch.global.L2 [%0];" ::"l"(row + o));
        if (p.out_lo) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + 2 * p.out_lo + o));
      }
    }
  }
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    const int lane = threadIdx.x & 31, c0 = 2 * (lane & 3);
    // a shared residual is indexed by the row inside the batch: rebase the pointer once per tile
    const __half* resid = p.resid;
    if (resid && p.resid_shared) resid -= (long long)c.b * s.rows * p.ld;
    // the first slice's residual is copied into the stage while the statistics are computed
    if (resid) frag_load_issue(c, resid, p.ld, p.out_lo, c.n0, c.ncols);
    // gamma / beta of this CTA's columns, staged once per CTA: a LayerNorm GEMM has one N tile, or
    // (N-split cluster) one fixed N half per CTA; the launchers check it
    if (c.it == 0) {
      for (int i = c.etid; i < c.ncols; i += 128) {
        sts32f(c.smem_s + 4 * i, p.gamma[c.n0 + i]);
        sts32f(c.smem_s + 4 * (256 + i), p.beta[c.n0 + i]);
      }
      epi_sync(c);
    }
    float mean[2], m2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float s1 = 0.f;
#pragma unroll
      for (int i = 0; i < N / 8; ++i) s1 += d[4 * i + 2 * h] + d[4 * i + 2 * h + 1];
      mean[h] = quad_sum(s1) / (float)c.ncols;
      float s2 = 0.f;
#pragma unroll
      for (int i = 0; i < N / 8; ++i) {
        const float a = d[4 * i + 2 * h] - mean[h], b = d[4 * i + 2 * h + 1] - mean[h];
        s2 = fmaf(a, a, s2);
        s2 = fmaf(b, b, s2);
      }
      m2[h] = quad_sum(s2);
    }
    if (s.pair == 2) {
      // N-split cluster: the other half of every row is in the peer CTA of the cluster (same M tile,
      // same iteration).  Lane 0 of each quad writes (mean, M2) of its two rows into the PEER's slots
      // of this tile parity and arrives (release.cluster) on the peer's mbarrier; it waits on the
      // local one (acquire.cluster), reads the peer's values for its rows and hands them to its quad.
      // Both CTAs merge "columns 0..127 first", so they get bit-identical statistics.  Two slots /
      // barriers alternate by tile parity: the peer can be one publish ahead, never two (its next
      // publish needs ours, and a lane publishes only after it has read this tile's slots).
      const int par = c.it & 1;
      const int r0 = 64 * c.group + 16 * c.q + (lane >> 2);
      float2* slot = reinterpret_cast<float2*>(c.extra) + par * 128 + r0;
      uint64_t* xbar = reinterpret_cast<uint64_t*>(c.extra + 2 * 128 * 8) + par;
      const uint32_t peer = (uint32_t)(c.n_tile ^ 1);
      float2 o[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
      if ((lane & 3) == 0) {
        st_cluster_f32x2(slot, peer, mean[0], m2[0]);
        st_cluster_f32x2(slot + 8, peer, mean[1], m2[1]);
        mbar_arrive_cluster_release(xbar, peer);
        mbar_wait_cluster(xbar, (uint32_t)((c.it >> 1) & 1));
        o[0] = slot[0];
        o[1] = slot[8];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        o[h].x = __shfl_sync(0xffffffffu, o[h].x, lane & ~3);
        o[h].y = __shfl_sync(0xffffffffu, o[h].y, lane & ~3);
        const float mean_a = c.n_tile == 0 ? mean[h] : o[h].x, m2a = c.n_tile == 0 ? m2[h] : o[h].y;
        const float mean_b = c.n_tile == 0 ? o[h].x : mean[h], m2b = c.n_tile == 0 ? o[h].y : m2[h];
        const float delta = mean_b - mean_a;
        mean[h] = mean_a + delta * 0.5f;                       // both halves have c.ncols columns
        m2[h] = m2a + m2b + delta * delta * (0.5f * (float)c.ncols);
      }
    }
    float rstd[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) rstd[h] = 1.f / sqrtf(m2[h] / (float)s.n_total + p.eps);
#pragma unroll
    for (int j = 0; j < (N + 31) / 32; ++j) {
      const int col = 32 * j;
      if (col < c.ncols) {
        const int nvalid = c.ncols - col;
        float v[16];
        frag_slice<N>(d, j, v);
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          const float2 gq = lds64f(c.smem_s + 4 * (col + 8 * ii + c0));
          const float2 bq = lds64f(c.smem_s + 4 * (256 + col + 8 * ii + c0));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            v[4 * ii + 2 * h] = (v[4 * ii + 2 * h] - mean[h]) * rstd[h] * gq.x + bq.x;
            v[4 * ii + 2 * h + 1] = (v[4 * ii + 2 * h + 1] - mean[h]) * rstd[h] * gq.y + bq.y;
          }
        }
        if (resid) frag_load_add(c, p.out_lo, v);
        if (p.out32) frag_store_f32(c, p.out32, s.n_total, c.n0 + col, v, nvalid);
        if (p.out16) frag_store_h(s, c, p.out16, p.ld, p.out_lo, c.n0 + col, v, nvalid);
        if (resid && col + 32 < c.ncols) frag_load_issue(c, resid, p.ld, p.out_lo, c.n0 + col + 32, nvalid - 32);
      }
    }
  }
};

// fp32 conf_matrix store of one slice (row stride n_total): staged when rows are 16-byte aligned,
// else element by element
__device__ __forceinline__ void conf_store(const GemmShape& s, const EpiCtx& c, float* conf, int col,
                                           const float (&v)[16]) {
  if ((s.n_total & 3) == 0) {
    frag_store_f32(c, conf, (long long)s.n_total, c.n0 + col, v, c.ncols - col);
    return;
  }
  const int c0 = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!((c.svalid >> h) & 1u)) continue;
    float* dst = conf + c.sgrow[h] * (long long)s.n_total + c.n0 + col;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (col + 8 * ii + c0 + e < c.ncols) dst[8 * ii + c0 + e] = v[4 * ii + 2 * h + e];
  }
}

// conf = softmax_dim1(sim) * softmax_dim2(sim) = exp((2*sim - lse_pt) - lse_px) of one slice
// (coarse_matching.py:115), and the running per-row (max, first argmax) over the tile's columns
// (coarse_matching.py:157-165): a lane visits its columns in increasing order.  Rows are 3D points
// (lown = their lse_pt), columns query cells (lse_px staged in smem_s).
__device__ __forceinline__ void conf_slice(const EpiCtx& c, int col, float scale, const float (&lown)[2],
                                           float (&v)[16], float (&best)[2], int (&bidx)[2]) {
  const int c0 = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int ii = 0; ii < 4; ++ii)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int cl = col + 8 * ii + c0 + e;
      const float lo = lds32f(c.smem_s + 4 * (cl & 255));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x2 = 2.f * (v[4 * ii + 2 * h + e] * scale);
        const float x = fast_exp((x2 - lown[h]) - lo);
        v[4 * ii + 2 * h + e] = x;
        if (cl < c.ncols && x > best[h]) {
          best[h] = x;
          bidx[h] = c.n0 + cl;
        }
      }
    }
}
// the per-row (max, argmax) of the tile into partial slot [grow][n_tile]
__device__ __forceinline__ void conf_best_store(const GemmShape& s, const EpiCtx& c, float* part_val, int* part_idx,
                                                float (&best)[2], int (&bidx)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    quad_argmax(best[h], bidx[h]);
    if ((threadIdx.x & 3) == 0 && ((c.svalid >> h) & 1u)) {
      part_val[c.sgrow[h] * s.n_tiles + c.n_tile] = best[h];
      part_idx[c.sgrow[h] * s.n_tiles + c.n_tile] = bidx[h];
    }
  }
}

// Dual-softmax statistics (coarse_matching.py:102-115) of sim = acc*scale in one pass: rows are 3D
// points.  Per row, over this tile's columns, (max, sum exp) into part_m / part_s [grow][n_tile]
// (merged by opp_lse_finalize); in addition every warp reduces each column of a 32-column slice over
// its 16 rows (the column max with an xor butterfly, then the sum of exp(x - that max) with a halving
// one, after which lane holds column frag_lane_col()), the two warps of a 32-row group merge their
// (max, sum) through the odd warp's stage (even warp first), and the even warp writes the pair to
// col_m / col_s [batch][row group][n_total] (row group = 32 rows).  opp_lse_col_finalize merges the
// row groups.
struct EpiLseColParams {
  float* part_m;
  float* part_s;
  float scale;
  float* col_m;   // [batches][row_groups][n_total]
  float* col_s;
  int row_groups; // ceil(rows / 32)
  // query_image_mask: columns with col_mask[b][col] == 0 get sim + (-1e9) (coarse_matching.py:108-114), or null
  const unsigned char* col_mask;
};
// + per-batch row counts: rows l >= row_count[b] (the padding of a bank set) are not rows of the matrix
struct EpiLseColRowsParams : EpiLseColParams {
  const int* row_count;   // [batches]
};

// bits h = 0, 1 of c.svalid restricted to the first row_count[c.b] rows of the batch element
__device__ __forceinline__ unsigned rows_below_count(const GemmShape& s, const EpiCtx& c, const int* row_count) {
  const long long end = (long long)c.b * s.rows + row_count[c.b];
  return c.svalid & ((c.sgrow[0] < end ? 1u : 0u) | (c.sgrow[1] < end ? 2u : 0u));
}

template <bool kMask, bool kRows = false>
struct EpiLseColT {
  static_assert(!(kMask && kRows), "query_image_mask and per-batch row counts are not combined");
  static constexpr int kGroups = 2;
  static constexpr const char* kName = kRows ? "lse_col_rows" : "lse_col";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  // With an n64 mainloop in the same kernel, ptxas serialises every wgmma of it (C7514) next to
  // this epilogue's column butterflies; its GEMMs have >= 4096 columns, so tiles of <= 64 columns
  // (tiny inputs only) run at 128
  static constexpr int kMinMmaN = 128;
  using Params = std::conditional_t<kRows, EpiLseColRowsParams, EpiLseColParams>;
  __device__ static void prefetch(const Params&, const GemmShape&, const EpiCtx&) {}
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    const int lane = threadIdx.x & 31, c0 = 2 * (lane & 3);
    // padded rows are treated like rows outside the tensor: -inf, so they leave the column
    // statistics alone (a wholly padded 32-row group writes (-inf, 0), which the finaliser skips)
    // and their row partials are not written (nothing reads them)
    unsigned valid = c.svalid;
    if constexpr (kRows) valid = rows_below_count(s, c, p.row_count);
    if constexpr (kMask) {   // additive column bias (0 / -1e9) of this tile, shared by the epilogue group
      epi_sync(c);
      for (int i = c.etid; i < c.ncols; i += 128)
        sts32f(c.smem_s + 4 * i, p.col_mask[(long long)c.b * s.n_total + c.n0 + i] ? 0.f : -1e9f);
      epi_sync(c);
    }
    // sim (+ column bias) in place; -inf for rows outside the tensor and columns past the tile
#pragma unroll
    for (int i = 0; i < N / 8; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int cl = 8 * i + c0 + e;
        float cb_ = 0.f;
        if constexpr (kMask) cb_ = lds32f(c.smem_s + 4 * (cl & 255));
#pragma unroll
        for (int h = 0; h < 2; ++h)
          d[4 * i + 2 * h + e] = (((valid >> h) & 1u) && cl < c.ncols) ? d[4 * i + 2 * h + e] * p.scale + cb_
                                                                        : -INFINITY;
      }
    // row partials
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m = -INFINITY;
#pragma unroll
      for (int i = 0; i < N / 8; ++i) m = fmaxf(m, fmaxf(d[4 * i + 2 * h], d[4 * i + 2 * h + 1]));
      m = quad_max(m);
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < N / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * i + c0 + e < c.ncols) sum += fast_exp(d[4 * i + 2 * h + e] - m);
      sum = quad_sum(sum);
      if ((lane & 3) == 0 && ((valid >> h) & 1u)) {
        p.part_m[c.sgrow[h] * s.n_tiles + c.n_tile] = m;
        p.part_s[c.sgrow[h] * s.n_tiles + c.n_tile] = sum;
      }
    }
    // column partials of this warp's 16 rows, one slice at a time
    constexpr int kSlices = (N + 31) / 32;
    float cmax[kSlices], csum[kSlices];
    const int rq = lane >> 2;
#pragma unroll
    for (int j = 0; j < kSlices; ++j) {
      cmax[j] = -INFINITY;
      csum[j] = 0.f;
      if (32 * j < c.ncols) {
        float v[16];
        frag_slice<N>(d, j, v, -INFINITY);
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = fmaxf(v[4 * (k >> 1) + (k & 1)], v[4 * (k >> 1) + 2 + (k & 1)]);
        col_allreduce8(x, [](float a, float b) { return fmaxf(a, b); });
        cmax[j] = pick8(x, rq);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float a = v[4 * (k >> 1) + (k & 1)], b = v[4 * (k >> 1) + 2 + (k & 1)];
          x[k] = (a == -INFINITY ? 0.f : fast_exp(a - x[k])) + (b == -INFINITY ? 0.f : fast_exp(b - x[k]));
        }
        csum[j] = col_reduce8(x, [](float a, float b) { return a + b; });
      }
    }
    // merge the warp pair of the 32-row group: the odd warp hands its partials over in its stage
    const bool odd = (c.q & 1) != 0;
    const uint32_t xs = c.wstage_s + (odd ? 0 : kWarpStageBytes);
    if (odd) {
#pragma unroll
      for (int j = 0; j < kSlices; ++j) sts64f(xs + 8 * (32 * j + lane), cmax[j], csum[j]);
    }
    pair_sync(c);
    if (!odd) {
      const int rg = c.m_tile * 4 + 2 * c.group + (c.q >> 1);   // 32-row group inside the batch
      if (rg < p.row_groups) {
        const long long cbase = ((long long)c.b * p.row_groups + rg) * s.n_total + c.n0;
        const int lc = frag_lane_col();
#pragma unroll
        for (int j = 0; j < kSlices; ++j) {
          const int cl = 32 * j + lc;
          if (cl < c.ncols) {
            const float2 o = lds64f(xs + 8 * (32 * j + lane));
            const float m = fmaxf(cmax[j], o.x);
            const float sa = cmax[j] == -INFINITY ? 0.f : csum[j] * fast_exp(cmax[j] - m);
            const float sb = o.x == -INFINITY ? 0.f : o.y * fast_exp(o.x - m);
            p.col_m[cbase + cl] = m;
            p.col_s[cbase + cl] = sa + sb;
          }
        }
      }
    }
    pair_sync(c);   // the odd warp's stage is free again
  }
};

using EpiLseCol = EpiLseColT<false>;
using EpiLseColMasked = EpiLseColT<true>;   // + query_image_mask (-1e9 on the padded query cells)
using EpiLseColRows = EpiLseColT<false, true>;   // + per-batch row counts (bank sets)

// conf pass with the column maxima folded in: rows are 3D points; conf per element (conf_slice),
// optional fp32 store of conf_matrix, and the per-row (max, first argmax) over this tile's columns
// into part_val / part_idx (merged by opp_best_finalize).  Every warp reduces each
// column of a slice over its 16 rows with a halving butterfly (lane ends with column
// frag_lane_col()), the two warps of a 32-row group merge through the odd warp's stage, and the even
// warp does one atomicMax per column on colmax[b][column] (conf >= 0, so its float bits order like
// unsigned ints; an integer max, so the result does not depend on the order).  The mutual-nearest
// test (coarse_matching.py:157-165) is then  rowmax(i) == colmax(argmax_j(i)), an exact comparison
// of two copies of the same register value.
struct EpiConfColParams {
  const float* lse_own;    // [batches*rows]   (3D points)
  const float* lse_other;  // [batches][n_total] (query cells)
  float scale;
  float* conf;             // [batches*rows][n_total] or null
  float* part_val;         // [batches*rows][n_tiles]
  int* part_idx;
  unsigned* colmax;        // [batches][n_total], zero-initialised
};
// + per-batch row counts: rows l >= row_count[b] never enter colmax and are stored as conf 0; their
// row (max, argmax) partials are written but meaningless (the match selection skips those rows)
struct EpiConfColRowsParams : EpiConfColParams {
  const int* row_count;    // [batches]
};
template <bool kRows>
struct EpiConfColT {
  static constexpr int kGroups = 2;
  static constexpr const char* kName = kRows ? "conf_col_rows" : "conf_col";   // $OPP_LOG_TILES
  static constexpr bool kFromRegs = true;
  // With an n64 mainloop in the same kernel, ptxas serialises every wgmma of it (C7514) next to
  // this epilogue's column butterfly; its GEMMs have >= 4096 columns, so tiles of <= 64 columns
  // (tiny inputs only) run at 128
  static constexpr int kMinMmaN = 128;
  using Params = std::conditional_t<kRows, EpiConfColRowsParams, EpiConfColParams>;
  __device__ static void prefetch(const Params&, const GemmShape&, const EpiCtx&) {}
  template <int N>
  __device__ __forceinline__ static void run_frag(const Params& p, const GemmShape& s, const EpiCtx& c, float (&d)[N / 2]) {
    const int lane = threadIdx.x & 31;
    epi_stage_cols_b(s, c, p.lse_other);
    unsigned valid = c.svalid;
    if constexpr (kRows) valid = rows_below_count(s, c, p.row_count);
    float lown[2], best[2] = {-1.f, -1.f};
    int bidx[2] = {c.n0, c.n0};
#pragma unroll
    for (int h = 0; h < 2; ++h) lown[h] = ((valid >> h) & 1u) ? p.lse_own[c.sgrow[h]] : 0.f;
    constexpr int kSlices = (N + 31) / 32;
    float cmax[kSlices];
#pragma unroll
    for (int j = 0; j < kSlices; ++j) {
      const int col = 32 * j;
      cmax[j] = 0.f;
      if (col < c.ncols) {
        float v[16];
        frag_slice<N>(d, j, v);
        conf_slice(c, col, p.scale, lown, v, best, bidx);
        if constexpr (kRows) {
#pragma unroll
          for (int k = 0; k < 16; ++k)
            if (!((valid >> ((k >> 1) & 1)) & 1u)) v[k] = 0.f;
        }
        if (p.conf) conf_store(s, c, p.conf, col, v);
        // column maxima over this warp's 16 rows (rows outside the tensor contribute 0)
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float a = (valid & 1u) ? v[4 * (k >> 1) + (k & 1)] : 0.f;
          const float b = (valid & 2u) ? v[4 * (k >> 1) + 2 + (k & 1)] : 0.f;
          x[k] = fmaxf(a, b);
        }
        cmax[j] = col_reduce8(x, [](float a, float b) { return fmaxf(a, b); });
      }
    }
    conf_best_store(s, c, p.part_val, p.part_idx, best, bidx);
    // merge the warp pair of the 32-row group: the odd warp hands its maxima over in its stage
    const bool odd = (c.q & 1) != 0;
    const uint32_t xs = c.wstage_s + (odd ? 0 : kWarpStageBytes);
    if (odd) {
#pragma unroll
      for (int j = 0; j < kSlices; ++j) sts32f(xs + 4 * (32 * j + lane), cmax[j]);
    }
    pair_sync(c);
    if (!odd) {
      unsigned* cm = p.colmax + (long long)c.b * s.n_total + c.n0;
      const int lc = frag_lane_col();
#pragma unroll
      for (int j = 0; j < kSlices; ++j) {
        const int cl = 32 * j + lc;
        const float m = fmaxf(cmax[j], lds32f(xs + 4 * (32 * j + lane)));
        if (cl < c.ncols && m > 0.f) atomicMax(cm + cl, __float_as_uint(m));
      }
    }
    pair_sync(c);   // the odd warp's stage is free again
  }
};

using EpiConfCol = EpiConfColT<false>;
using EpiConfColRows = EpiConfColT<true>;   // + per-batch row counts (bank sets)

// =============================================================================================
// The kernel
// =============================================================================================
// keeps the compiler from moving accesses of in-flight wgmma accumulators across the fences
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// KS K steps of one chunk into the accumulator, per element in the order hi*hi, hi*lo, lo*hi.
// Every step count has its own fully unrolled body: a wgmma under a runtime-bounded loop makes
// ptxas serialise all of them.
template <int N, int KS>
__device__ __forceinline__ void mma_k_steps(float (&d)[N / 2], bool split, uint64_t a_hi, uint64_t a_lo,
                                            uint64_t b_hi, uint64_t b_lo) {
#pragma unroll
  for (int k = 0; k < KS; ++k) wgmma_m64nNk16<N>(d, a_hi + 2 * k, b_hi + 2 * k);
  if (split) {
#pragma unroll
    for (int k = 0; k < KS; ++k) wgmma_m64nNk16<N>(d, a_hi + 2 * k, b_lo + 2 * k);
#pragma unroll
    for (int k = 0; k < KS; ++k) wgmma_m64nNk16<N>(d, a_lo + 2 * k, b_hi + 2 * k);
  }
}

template <int A_MODE, class Epi, int BK>
__device__ __forceinline__ void gemm_body(const TensorMaps& maps, const GemmShape& s,
                                          const typename Epi::Params& ep) {
  static_assert(Epi::kGroups == 2, "each of the two MMA warpgroups is one epilogue group");
  static_assert(BK == 64 || BK == 32, "K chunk of one 128B- or 64B-swizzle row");
  constexpr int kABytes = gemm_a_bytes(BK);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int planes = s.split ? 2 : 1;
  const bool nsc = s.pair == 2;   // N-split cluster: two independent CTAs, same M tile, N half = cluster rank
  // the ring: s.stages stages of one 64-wide K chunk each, a stage being kParts slots of BK columns
  // with barriers of their own, so that it is filled and released a slot at a time
  constexpr int kParts = kBlockK / BK;
  const int slots = s.stages * kParts;
  const int b_bytes = s.mma_n * BK * 2;   // one plane of the W tile of a slot
  const int a_stage = kABytes * planes;    // bytes of a slot
  const int b_stage = b_bytes * planes;
  const int ring = slots * (a_stage + b_stage);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + slots * a_stage;
  // register-fragment epilogues have no accumulator tile (and acc_alias = 0); only EpiConvUp has one
  constexpr bool kAccTile = !EpiFromRegs<Epi>::value;
  uint8_t* smem_acc = s.acc_alias ? smem : smem + ring;
  float* epi_smem = reinterpret_cast<float*>(smem + ring + (kAccTile && !s.acc_alias ? gemm_acc_bytes(s.mma_n) : 0));
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi_smem) +
                                               epi_smem_bytes<Epi>());
  uint64_t* full = bars;
  uint64_t* empty = bars + kMaxStages;
  uint64_t* accfree = bars + 2 * kMaxStages;

  constexpr int kProducerWarp = 4 * Epi::kGroups;   // first warp of the producer warpgroup
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // tile schedule: "super tiles" of `cluster` adjacent M tiles; every CTA of a cluster walks the
  // same sequence, so the multicast W loads and the cross-CTA stage releases stay in lockstep.
  // N-split cluster: logically two single-CTA GEMMs (csize 1: no multicast, no shared barriers) that
  // walk the same tile sequence; `nrank` selects the N half.
  const int csize = nsc ? 1 : s.cluster;
  const int prank = s.cluster > 1 ? (int)cluster_ctarank() : 0;   // physical rank in the cluster
  const int crank = nsc ? 0 : prank;
  const int nrank = nsc ? prank : 0;
  const uint16_t cmask = (uint16_t)((1u << csize) - 1u);
  const int cluster_id = blockIdx.x / s.cluster;
  const int n_clusters = gridDim.x / s.cluster;
  const int tiles_per_batch = s.msup * s.n_tiles;
  const int total_tiles = s.batches * tiles_per_batch;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&maps.a[0]);
    tma_prefetch_desc(&maps.b);
  }
  if (warp == 0 && lane == 0) {
    for (int i = 0; i < slots; ++i) {
      mbar_init(&full[i], 1);
      // one arrival per MMA warpgroup of every CTA that reads the (multicast) stage
      mbar_init(&empty[i], 2 * csize);
    }
    // acc_alias: one arrival per epilogue warp of every CTA whose ring the producer writes into
    mbar_init(accfree, 4 * Epi::kGroups * csize);
    if constexpr (EpiExtraSmem<Epi>::value > 0) {
      // EpiLN's DSMEM exchange: the writer lanes of the peer CTA arrive once per tile
      uint64_t* xbar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi_smem) + epi_smem_bytes<Epi>() -
                                                   EpiExtraSmem<Epi>::value + 2 * 128 * 8);
      mbar_init(&xbar[0], Epi::kExchangeArrivals);
      mbar_init(&xbar[1], Epi::kExchangeArrivals);
    }
    fence_mbar_init();
  }
  if (s.cluster > 1) cluster_sync_all(); else __syncthreads();
  // programmatic dependent launch: everything above overlapped with the previous kernel's tail;
  // from here on we read what it wrote.
  pdl_sync();

  if (warp >= kProducerWarp) {
    // ------------------------------------------------------------------ producer warpgroup
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kProducerWarp) {
      // TMA producer.  The loop runs warp-uniformly; only the asynchronous-issue instructions sit
      // under elect_one().
      int stage = 0;
      uint32_t phase = 0;
      const bool skip_b = (s.debug_skip & 1) != 0, skip_a = (s.debug_skip & 2) != 0;
      const int a_tx = A_MODE == A_WIN ? s.tiles_x * s.tile_w * s.tile_h * (BK * 2) * planes : a_stage;
      const uint32_t tx_bytes = (skip_a ? 0 : a_tx) + (skip_b ? 0 : b_stage);
      int it = 0;
      for (int t = cluster_id; t < total_tiles; t += n_clusters, ++it) {
        // the accumulator overlays the ring: wait until every epilogue of the cluster is done with it
        if (s.acc_alias && it > 0) mbar_wait(accfree, (uint32_t)((it - 1) & 1));
        const int b = t / tiles_per_batch;
        const int r = t - b * tiles_per_batch;
        const int msi = r / s.n_tiles;
        const int n_tile = nsc ? nrank : r - msi * s.n_tiles;
        const int m_tile = msi * csize + crank;
        int ox0 = 0, oy0 = 0;
        if (A_MODE == A_CONV) {
          const int ty = m_tile / s.tiles_x;
          oy0 = ty * s.tile_h;
          ox0 = (m_tile - ty * s.tiles_x) * s.tile_w;
        }
        const int bb = s.b_batched ? b : 0;
        const int nrow0 = n_tile * s.block_n;
        // A_WIN: input coordinates of the (up to five) windows of this tile, once per tile
        int win_x[5] = {0, 0, 0, 0, 0}, win_y[5] = {0, 0, 0, 0, 0}, win_z[5] = {0, 0, 0, 0, 0};
        if constexpr (A_MODE == A_WIN) {
          const int cnt = s.rows / (s.tile_w * s.tile_h);
#pragma unroll
          for (int wi = 0; wi < 5; ++wi) {
            int m = m_tile * s.tiles_x + wi;
            m = m < cnt ? m : cnt - 1;
            win_z[wi] = m;
            if (ep.j_ids) {
              const int j = (int)ep.j_ids[m];
              const int cy = j / ep.wc;
              win_z[wi] = (int)ep.b_ids[m];
              win_x[wi] = ep.stride * (j - cy * ep.wc) + ep.org - s.conv_pad;
              win_y[wi] = ep.stride * cy + ep.org - s.conv_pad;
            }
          }
        }
        // incremental (tap, channel-chunk) counters instead of per-chunk divisions
        int cc = 0, ky = 0, kx = 0, kb_tap = 0;
        for (int chunk = 0; chunk < s.k_chunks; ++chunk) {
          // K offset of this 64-wide chunk in A (A_ROWS) or its channel offset (conv modes), and in W
          const bool first = A_MODE == A_ROWS && chunk < s.k_chunks_a0;
          const int ka = A_MODE == A_ROWS ? (first ? chunk : chunk - s.k_chunks_a0) * kBlockK : cc * kBlockK;
          const int kb = A_MODE == A_ROWS ? chunk * kBlockK : kb_tap + ka;
#pragma unroll
          for (int part = 0; part < kParts; ++part) {
            const int kp = part * BK;   // K offset of this slot inside the chunk
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem_a + stage * a_stage;
            uint8_t* sb = smem_b + stage * b_stage;
            {
              // (the second slot of a 16-channel tail chunk, 208 = 3 x 64 + 16, reads zeros past conv_c
              // and the next tap's W columns: the MMA warpgroups issue no MMAs on it)
              if constexpr (A_MODE == A_ROWS) {
                const CUtensorMap* am = first ? &maps.a[0] : &maps.a[1];
                const int lo = first ? s.a0_lo : s.a1_lo;
                const int ba = (first && s.a0_shared) ? 0 : b;
                if (elect_one()) {
                  mbar_expect_tx(&full[stage], tx_bytes);
                  if (!skip_a) {
                    tma_load_3d(am, &full[stage], sa, ka + kp, m_tile * kBlockM, ba);
                    if (s.split) tma_load_3d(am, &full[stage], sa + kABytes, ka + kp + lo, m_tile * kBlockM, ba);
                  }
                }
              } else if constexpr (A_MODE == A_WIN) {
                // one TMA box (BK channels x tile_w x tile_h) per window and plane; windows past the
                // match count re-read the last one (their rows are never stored)
                const int wbytes = s.tile_w * s.tile_h * (BK * 2);
#pragma unroll
                for (int wi = 0; wi < 5; ++wi) {
                  if (wi >= s.tiles_x) break;
                  const int bx = win_x[wi] + kx, by = win_y[wi] + ky, bz = win_z[wi];
                  if (elect_one()) {
                    if (wi == 0) mbar_expect_tx(&full[stage], tx_bytes);
                    if (!skip_a) {
                      tma_load_5d(&maps.a[0], &full[stage], sa + wi * wbytes, ka + kp, 0, bx, by, bz);
                      if (s.split)
                        tma_load_5d(&maps.a[0], &full[stage], sa + kABytes + wi * wbytes, ka + kp, 1, bx, by, bz);
                    }
                  }
                }
              } else {
                int dy = ky - s.conv_pad, dx = kx - s.conv_pad, mi = 0;
                if (s.conv_stride == 2) {
                  const int py = dy & 1, px = dx & 1;
                  dy = (dy - py) >> 1;
                  dx = (dx - px) >> 1;
                  mi = py * 2 + px;
                }
                const CUtensorMap* am = &maps.a[mi];
                if (elect_one()) {
                  mbar_expect_tx(&full[stage], tx_bytes);
                  if (!skip_a) {
                    tma_load_5d(am, &full[stage], sa, ka + kp, 0, ox0 + dx, oy0 + dy, b);
                    if (s.split) tma_load_5d(am, &full[stage], sa + kABytes, ka + kp, 1, ox0 + dx, oy0 + dy, b);
                  }
                }
              }
              if (!skip_b && elect_one()) {
                if (csize == 1) {
                  tma_load_3d(&maps.b, &full[stage], sb, kb + kp, nrow0, bb);
                  if (s.split) tma_load_3d(&maps.b, &full[stage], sb + b_bytes, s.b_lo + kb + kp, nrow0, bb);
                } else {
                  // this CTA fetches rows [crank*slice, +slice) of the W tile and multicasts them into
                  // every CTA of the cluster (each CTA's full barrier expects the whole tile)
                  const int slice = s.mma_n / csize;
                  const int soff = crank * slice * (BK * 2);
                  const int nrow = nrow0 + crank * slice;
                  tma_load_3d_mc(&maps.b, &full[stage], sb + soff, kb + kp, nrow, bb, cmask);
                  if (s.split)
                    tma_load_3d_mc(&maps.b, &full[stage], sb + b_bytes + soff, s.b_lo + kb + kp, nrow, bb, cmask);
                }
              }
            }
            __syncwarp();
            if (++stage == slots) {
              stage = 0;
              phase ^= 1;
            }
          }
          if (A_MODE != A_ROWS && ++cc == s.conv_cchunks) {
            cc = 0;
            kb_tap += s.conv_c;
            if (++kx == s.conv_kw) {
              kx = 0;
              ++ky;
            }
          }
        }
      }
    }
    // warps 1-3 of the producer warpgroup go straight to the final CTA / cluster sync
  } else {
    // ------------------------------------------------------------------ MMA warpgroup g = epilogue group g
    setmaxnreg_inc<kMmaRegs>();
    const int g = warp >> 2;
    const int q = warp & 3;
    EpiCtx c;
    c.etid = q * 32 + lane;
    c.q = q;
    c.a_mode = A_MODE;
    c.group = g;
    c.col_first = 32 * g;
    c.col_step = 32 * Epi::kGroups;
    c.smem = epi_smem + g * (kEpiParamBytes / 8);   // 2 KB (512 floats) per group
    c.wstage = reinterpret_cast<uint8_t*>(epi_smem) + kEpiParamBytes + warp * EpiWarpStage<Epi>::value;
    c.extra = reinterpret_cast<uint8_t*>(epi_smem) + epi_smem_bytes<Epi>() - EpiExtraSmem<Epi>::value;
    c.smem_s = smem_u32(c.smem);
    c.wstage_s = smem_u32(c.wstage);
    // descriptors in 16-byte units: this warpgroup's 64 A rows start 64 * (2 BK) B into the A tile;
    // K advances 16 fp16 = 32 B (+2) inside the 2 BK-byte swizzle row; one wgmma reads all mma_n W rows
    const uint64_t desc_tmpl = BK == 64 ? make_kmajor_sw128_desc(0) : make_kmajor_sw64_desc(0);
    const uint32_t sa0 = ((smem_u32(smem_a) >> 4) & 0x3FFF) + g * ((64 * BK * 2) >> 4);
    const uint32_t sb0 = (smem_u32(smem_b) >> 4) & 0x3FFF;
    const uint32_t a_step = (uint32_t)a_stage >> 4, b_step = (uint32_t)b_stage >> 4;
    const uint32_t a_lo_off = kABytes >> 4, b_lo_off = (uint32_t)b_bytes >> 4;
    const bool split = s.split != 0;
    const bool is_signal = q == 0 && lane == 0;
    const uint32_t pitch = (uint32_t)(s.mma_n + kAccPad);
    const uint32_t acc_w = smem_u32(smem_acc) >> 2;
    // this thread's accumulator fragment: rows r0 and r0 + 8, columns 8 i + c0 + {0, 1}
    const uint32_t r0 = 64 * g + 16 * q + (lane >> 2), c0 = 2 * (lane & 3);
    auto release = [&](int st) {
      if (is_signal) {
        if (csize == 1) mbar_arrive(&empty[st]);
        else
          for (int r = 0; r < csize; ++r) mbar_arrive_cluster(&empty[st], (uint32_t)r);
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    uint32_t sa = sa0, sb = sb0;
    // K steps of a chunk: 4, but in the conv modes the last channel chunk of every filter tap holds
    // only conv_c % 64 channels when conv_c is not a multiple of 64 (196 -> 208 = 3 x 64 + 16); the
    // TMA box reads zeros past conv_c, and the steps that would multiply only those are not issued
    // (for a 16-channel tail; see the dispatch below)
    const int tail_steps = (A_MODE != A_ROWS && (s.conv_c & 63)) ? (s.conv_c & 63) / 16 : 4;
    int it = 0;
    for (int t = cluster_id; t < total_tiles; t += n_clusters, ++it) {
      c.b = t / tiles_per_batch;
      const int r = t - c.b * tiles_per_batch;
      const int msi = r / s.n_tiles;
      c.n_tile = nsc ? nrank : r - msi * s.n_tiles;
      c.m_tile = msi * csize + crank;   // may lie past the last M tile: rows are then invalid
      c.n0 = c.n_tile * s.block_n;
      const int rem = s.n_total - c.n0;
      c.ncols = rem < s.block_n ? rem : s.block_n;
      if constexpr (EpiNeedsNext<Epi>::value) {
        const int tn = t + n_clusters;
        c.next_b = -1;
        c.next_m_tile = 0;
        if (tn < total_tiles) {
          c.next_b = tn / tiles_per_batch;
          c.next_m_tile = ((tn - c.next_b * tiles_per_batch) / s.n_tiles) * csize + crank;
        }
      }
      c.it = it;
      c.svalid = 0;
      if constexpr (kAccTile) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          int rdummy;
          if (epi_row_at(s, c, q * 32 + (lane >> 2) + 8 * i, c.sgrow[i], rdummy)) c.svalid |= 1u << i;
        }
      } else {
        // the two accumulator-fragment rows of this thread
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int rdummy;
          if (epi_row_at(s, c, (int)r0 + 8 * h, c.sgrow[h], rdummy)) c.svalid |= 1u << h;
        }
      }
      c.acc = acc_w + (uint32_t)(q * 32 + lane) * pitch;
      Epi::prefetch(ep, s, c);

      // the tile's MMAs and the accumulator dump, with registers for exactly N accumulator columns
      auto mma_tile = [&](auto n_c, auto tail_c) {
        constexpr int N = decltype(n_c)::value;
        // K steps of each filter tap's last chunk (0: every chunk is 4 steps).  A compile-time
        // count keeps the branch between full and tail chunks out of the mainloop: ptxas
        // serialises wgmmas that sit behind a branch it cannot prove uniform.
        constexpr int TAIL = decltype(tail_c)::value;
        float d[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
        wgmma_fence_acc(d);
        int prev = -1;
        static_assert(TAIL * 16 <= BK, "a tail chunk's channels lie in its first slot");
        // one slot: wait for it, KS K steps (0: the empty second slot of a tail chunk), then release
        // the previous slot
        auto chunk_step = [&](auto ks_c, auto& acc) {
          const uint64_t a_hi = desc_tmpl | sa, b_hi = desc_tmpl | sb;
          const uint64_t a_lo = desc_tmpl | (sa + a_lo_off), b_lo = desc_tmpl | (sb + b_lo_off);
          mbar_wait_hot(&full[stage], phase);
          wgmma_fence();
          mma_k_steps<N, decltype(ks_c)::value>(acc, split, a_hi, a_lo, b_hi, b_lo);
          wgmma_commit();
          wgmma_fence_acc(acc);
          if (prev >= 0) {
            wgmma_wait<1>();
            release(prev);
          }
          prev = stage;
          sa += a_step;
          sb += b_step;
          if (++stage == slots) {
            stage = 0;
            phase ^= 1;
            sa = sa0;
            sb = sb0;
          }
        };
        // one 64-wide chunk: its kParts slots; a tail chunk's steps all lie in the first slot
        auto full_chunk = [&]() {
#pragma unroll
          for (int part = 0; part < kParts; ++part) chunk_step(std::integral_constant<int, BK / 16>{}, d);
        };
        auto tail_chunk = [&]() {
          chunk_step(std::integral_constant<int, TAIL>{}, d);
          if constexpr (kParts == 2) chunk_step(std::integral_constant<int, 0>{}, d);
        };
        if constexpr (TAIL == 0) {
          for (int chunk = 0; chunk < s.k_chunks; ++chunk) full_chunk();
        } else {
          const int taps = s.k_chunks / s.conv_cchunks;
          for (int tap = 0; tap < taps; ++tap) {
            for (int cc = 1; cc < s.conv_cchunks; ++cc) full_chunk();
            tail_chunk();
          }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(d);
        if (prev >= 0) release(prev);

        if constexpr (!kAccTile) {
          if (!(s.debug_skip & 4)) Epi::template run_frag<N>(ep, s, c, d);   // bit 2: timing experiment, no epilogue
        } else {
          // both groups are done reading the previous tile's accumulator
          named_bar_sync(4, 256);
#pragma unroll
          for (int i = 0; i < N / 8; ++i) {
            const uint32_t col = 8 * i + c0;
            sts64f((acc_w + r0 * pitch + col) * 4, d[4 * i], d[4 * i + 1]);
            sts64f((acc_w + (r0 + 8) * pitch + col) * 4, d[4 * i + 2], d[4 * i + 3]);
          }
          named_bar_sync(4, 256);
        }
      };
      // one case per entry of kMmaWidths (fit_tile only produces those)
      auto mma_width = [&](auto tail_c) {
        switch (s.mma_n) {
          case 64:
            if constexpr (EpiMinMmaN<Epi>::value <= 64) mma_tile(std::integral_constant<int, 64>{}, tail_c);
            break;
          case 128: mma_tile(std::integral_constant<int, 128>{}, tail_c); break;
          case 208: mma_tile(std::integral_constant<int, 208>{}, tail_c); break;
          default: mma_tile(std::integral_constant<int, 256>{}, tail_c); break;
        }
      };
      if constexpr (A_MODE == A_ROWS) {
        mma_width(std::integral_constant<int, 0>{});
      } else {
        // a one-step tail is what the 196 -> 208 channel layers need; a 32- or 48-channel tail runs
        // as a full chunk (its extra steps multiply zeros): each further tail variant is one more
        // copy of every mainloop, and the copies together made ptxas spill
        switch (tail_steps) {
          case 1: mma_width(std::integral_constant<int, 1>{}); break;
          default: mma_width(std::integral_constant<int, 0>{}); break;
        }
      }

      if constexpr (kAccTile) {
        if (!(s.debug_skip & 4)) Epi::run(ep, s, c);   // bit 2: timing experiment, no epilogue at all
        if (s.acc_alias) {
          // the producer's next TMA writes land where this warp just read the accumulator
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            if (csize == 1) mbar_arrive(accfree);
            else
              for (int r2 = 0; r2 < csize; ++r2) mbar_arrive_cluster(accfree, (uint32_t)r2);
          }
        }
      }
    }
  }

  pdl_done();
  // a CTA must outlive every multicast write / remote barrier arrival aimed at it
  if (s.cluster > 1) cluster_sync_all(); else __syncthreads();
}

// BK (= GemmShape.bk) is a template parameter, not a runtime branch: a second copy of every mainloop
// in one kernel made ptxas spill
template <int A_MODE, class Epi, int BK = kBlockK>
__global__ void __launch_bounds__(gemm_threads(Epi::kGroups), 1)
gemm_kernel(const __grid_constant__ TensorMaps maps, const GemmShape s, const typename Epi::Params ep) {
  gemm_body<A_MODE, Epi, BK>(maps, s, ep);
}

// Same kernel with the number of valid rows in device memory (the match count of the coarse
// stage): rows = *rows_dev * rows_mult, so a whole forward can be enqueued — or captured in a CUDA
// graph — without a host round trip.  The host-side rows / m_tiles describe the CAPACITY.
template <int A_MODE, class Epi, int BK = kBlockK>
__global__ void __launch_bounds__(gemm_threads(Epi::kGroups), 1)
gemm_kernel_dyn(const __grid_constant__ TensorMaps maps, const GemmShape s_in,
                const typename Epi::Params ep, const int* rows_dev, int rows_mult) {
  GemmShape s = s_in;
  pdl_wait();   // rows_dev is written by the previous kernels of the stream
  const int r = *rows_dev * rows_mult;
  s.rows = r < s_in.rows ? r : s_in.rows;
  const int tile_rows = A_MODE == A_WIN ? s_in.tiles_x * s_in.tile_w * s_in.tile_h : kBlockM;
  s.m_tiles = (s.rows + tile_rows - 1) / tile_rows;
  s.msup = (s.m_tiles + s_in.cluster - 1) / s_in.cluster;
  gemm_body<A_MODE, Epi, BK>(maps, s, ep);
}

// Shared memory of a launch with epilogue Epi: operand ring, the accumulator tile (EpiConvUp only:
// beside the ring, or over it when acc_alias), epilogue scratch, barriers and alignment slack.
inline int gemm_stage_bytes(int mma_n, int split) {
  return (gemm_a_bytes(kBlockK) + mma_n * kBlockK * 2) * (split ? 2 : 1);
}
template <class Epi>
inline int gemm_smem_bytes(const GemmShape& s) {
  const bool acc_tile = !EpiFromRegs<Epi>::value && !s.acc_alias;
  return s.stages * gemm_stage_bytes(s.mma_n, s.split) + (acc_tile ? gemm_acc_bytes(s.mma_n) : 0) +
         epi_smem_bytes<Epi>() + (2 * kMaxStages + 2) * 8 + 16 + 1024;
}
constexpr int kSmemLimit = 227 * 1024;
// Ring depth (stages of one 64-wide K chunk, at most kMaxStages slots) and accumulator placement for s.mma_n: the accumulator tile (if Epi has one) gets its
// own space when that leaves at least two stages, else it overlays the ring (which then holds at
// least the tile).  `cap` (> 1) bounds the ring depth.  Returns false when even that does not fit.
template <class Epi>
inline bool gemm_pick_stages(GemmShape& s, int cap = 0) {
  const int avail = kSmemLimit - epi_smem_bytes<Epi>() - 2048;
  const int sb = gemm_stage_bytes(s.mma_n, s.split);
  const int max_st = kMaxStages * s.bk / kBlockK;   // a barrier pair per slot
  const int ab = EpiFromRegs<Epi>::value ? 0 : gemm_acc_bytes(s.mma_n);
  int st = (avail - ab) / sb;
  s.acc_alias = ab > 0 && st < 2;
  if (s.acc_alias) st = avail / sb;
  if (st > max_st) st = max_st;
  if (st > s.k_chunks * 2 && s.k_chunks * 2 >= 2) st = s.k_chunks * 2;
  if (cap > 1 && st > cap) st = cap;
  if (st < 2) st = 2;
  if (s.acc_alias && st * sb < ab) st = (ab + sb - 1) / sb;
  s.stages = st;
  return st <= max_st && gemm_smem_bytes<Epi>(s) <= kSmemLimit;
}

}  // namespace opp
