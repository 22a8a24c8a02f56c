// opp_gemm.cu — host launchers (C-ABI) for the wgmma GEMM / implicit-GEMM conv engine.
//
// Every entry point takes raw device pointers + sizes + a cudaStream_t, builds the TMA tensor
// maps for the call, and launches one persistent kernel.  No allocation, no synchronisation.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/opp_b200.h"
#include "opp_gemm.cuh"

namespace opp {

static thread_local char g_last_error[512] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_last_error; }

// ---------------------------------------------------------------------------------------------
// driver entry point for cuTensorMapEncodeTiled (no link-time dependency on libcuda)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 132;
  }
  return n;
}

// fp16 tensor map, zero OOB fill, swizzled by the inner box row: 64 fp16 (a K chunk of 64) = 128B
// swizzle, 32 fp16 = 64B swizzle. dims/strides fastest-first; strides in elements for dims 1..rank-1.
static int make_map(CUtensorMap* map, const void* ptr, int rank, const uint64_t* dims,
                    const uint64_t* strides_elems, const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return OPP_ERR_CUDA;
  }
  OPP_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "TMA base pointer not 16B aligned");
  OPP_REQUIRE(box[0] == 64 || box[0] == 32, "TMA inner box %u is not one swizzle row", box[0]);
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    OPP_REQUIRE(box[i] >= 1 && box[i] <= 256, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_elems[i] * 2;
    OPP_REQUIRE((gstr[i] & 15) == 0, "TMA stride %d (%llu B) not a multiple of 16", i,
                (unsigned long long)gstr[i]);
  }
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(ptr), gdim, gstr,
                  bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  box[0] == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu %llu %llu)",
                   (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                   (unsigned long long)(rank > 2 ? dims[2] : 0));
    return OPP_ERR_CUDA;
  }
  return OPP_OK;
}

// A / W operand as [batch][rows][K] with row stride ld (elements), boxes of bk K columns
static int map_rows(CUtensorMap* map, const void* ptr, long long k, long long rows,
                    long long batches, long long ld, long long batch_stride, int box_rows, int bk = kBlockK) {
  uint64_t dims[3] = {(uint64_t)k, (uint64_t)rows, (uint64_t)batches};
  uint64_t str[2] = {(uint64_t)ld, (uint64_t)batch_stride};
  uint32_t box[3] = {(uint32_t)bk, (uint32_t)box_rows, 1};
  return make_map(map, ptr, 3, dims, str, box);
}

// $OPP_LOG_TILES=1: print every distinct GEMM tile configuration to stderr once, when it is first
// launched (which wgmma widths, ring depths and clusters a workload actually uses); every field of
// the line is an integer.  $OPP_LOG_TILES=2: print the configuration of every launch, followed by
// "epi <name>" (the epilogue), so that each launch of a test is attributed a line of its own even
// where launches of the same (n, k) differ only in the epilogue.
static void log_tile_once(int a_mode, const GemmShape& s, const char* epi) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("OPP_LOG_TILES");
    on = e ? atoi(e) : 0;
  }
  if (!on) return;
  static std::mutex mu;
  static char seen[256][128];
  static int n_seen = 0;
  char key[128];
  snprintf(key, sizeof(key), "mode %d n %d block_n %d mma_n %d k %d conv_c %d stages %d alias %d cluster %d pair %d bk %d",
           a_mode, s.n_total, s.block_n, s.mma_n, s.k_chunks * kBlockK, s.conv_c, s.stages, s.acc_alias,
           s.cluster, s.pair, s.bk);
  std::lock_guard<std::mutex> lock(mu);
  if (on == 2) {
    fprintf(stderr, "opp gemm tile: %s epi %s\n", key, epi);
    return;
  }
  for (int i = 0; i < n_seen; ++i)
    if (!strcmp(seen[i], key)) return;
  if (n_seen < 256) strcpy(seen[n_seen++], key);
  fprintf(stderr, "opp gemm tile: %s\n", key);
}

// rows_dev != nullptr: the DYN kernel (device-side row count, rows = *rows_dev * rows_mult)
template <int A_MODE, class Epi, bool DYN = false>
static int launch(const TensorMaps& maps, GemmShape s, const typename Epi::Params& ep,
                  cudaStream_t stream, const int* rows_dev = nullptr, int rows_mult = 1) {
  {
    static int dbg = -1;
    if (dbg < 0) {
      const char* e = getenv("OPP_DEBUG_SKIP");
      dbg = e ? atoi(e) : 0;
    }
    s.debug_skip = dbg;
    static int cap = -1;
    if (cap < 0) {
      const char* e = getenv("OPP_STAGES");
      cap = e ? atoi(e) : 0;
    }
    OPP_REQUIRE(s.mma_n >= EpiMinMmaN<Epi>::value, "GEMM tile width %d below the epilogue's minimum %d",
                s.mma_n, EpiMinMmaN<Epi>::value);
    OPP_REQUIRE(s.mma_n > 0 && gemm_pick_stages<Epi>(s, cap),
                "GEMM tile N=%d (split %d) does not fit in shared memory", s.block_n, s.split);
  }
  const int smem = gemm_smem_bytes<Epi>(s);
  log_tile_once(A_MODE, s, Epi::kName);
  OPP_REQUIRE(s.bk == kBlockK || s.bk == 32, "ring slot width %d not compiled", s.bk);
  const void* kern;
  if constexpr (DYN)
    kern = s.bk == 32 ? (const void*)gemm_kernel_dyn<A_MODE, Epi, 32> : (const void*)gemm_kernel_dyn<A_MODE, Epi>;
  else
    kern = s.bk == 32 ? (const void*)gemm_kernel<A_MODE, Epi, 32> : (const void*)gemm_kernel<A_MODE, Epi>;
  // function attributes are per device: set once per (kernel, device)
  static unsigned long long attr_done[2] = {0, 0};
  unsigned long long& done = attr_done[s.bk == 32];
  int dev = 0;
  OPP_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !((done >> dev) & 1ull)) {
    OPP_CHECK_CUDA(
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    done |= 1ull << dev;
  }
  const long long total = (long long)s.batches * s.msup * s.n_tiles;   // super tiles
  if (total == 0) return OPP_OK;
  const int max_clusters = num_sms() / s.cluster;
  const int n_clusters = (int)(total < max_clusters ? total : max_clusters);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_clusters * s.cluster);
  cfg.blockDim = dim3(gemm_threads(Epi::kGroups));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = s.cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // see pdl_wait() in opp_common.cuh
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  void* kargs[5] = {(void*)&maps, (void*)&s, (void*)&ep, (void*)&rows_dev, (void*)&rows_mult};
  cudaError_t le = cudaLaunchKernelExC(&cfg, kern, kargs);
  if (le != cudaSuccess) {
    set_last_error("cudaLaunchKernelEx failed: %s (grid %d cluster %d pair %d smem %d stages %d "
                   "acc_alias %d block_n %d m_tiles %d n_tiles %d batches %d)",
                   cudaGetErrorString(le), n_clusters * s.cluster, s.cluster, s.pair, smem, s.stages,
                   s.acc_alias, s.block_n, s.m_tiles, s.n_tiles, s.batches);
    return OPP_ERR_CUDA;
  }
  return OPP_OK;
}

static int pick_cluster(int block_n, int m_tiles);

// decide the CTA grouping of a GEMM: a multicast cluster sharing the W tile, or single CTAs
static void pick_grouping(GemmShape& s) {
  s.pair = 0;
  s.cluster = pick_cluster(s.block_n, s.m_tiles);
  s.msup = (s.m_tiles + s.cluster - 1) / s.cluster;
}

// cluster size for a GEMM: the W-tile slices (mma_n / cluster rows) must be whole 8-row swizzle
// groups; $OPP_CLUSTER overrides
static int pick_cluster(int block_n, int m_tiles) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("OPP_CLUSTER");
    forced = e ? atoi(e) : 0;
  }
  int c = forced > 1 ? forced : 2;
  while (c > 1 && (mma_width_for(block_n) % (8 * c) != 0 || m_tiles < c)) c >>= 1;
  return c;
}

// Ring slot width of a convolution layer (A_CONV, A_WIN): 32 channels for the 3x3 layers whose
// padded output width is above 128, else 64.  At N = 208 / 256 a 64-wide stage is 84 / 96 KB and
// only two fit, and the MMA warpgroups keep the previous slot until the next slot's MMAs are issued:
// with one slot per stage they hold both stages and no load is in flight.  Two 32-wide slots per
// stage (the same shared memory) leave a stage's first half free to load while its second half and
// the other stage are read (3x3 layers at batch 64: 15-39 % less time).  The 1x1 layers (2-4 chunks
// per tile) and the N <= 128 layers (three stages) measured 1-15 % slower with 32-wide slots, all but
// one 1x1 lateral (7 % faster).  The slot width sets the order of the fp32 accumulation (the three
// split products per slot), so it depends on the layer only - never on the batch, tile, ring, cluster
// or N split - and the dense and window forms of a layer, and its launches at every batch, give the
// same bits.  $OPP_CONV_BK=32|64 forces one width for every conv layer.
static int conv_chunk_k(int ksize, int c_out_pad) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("OPP_CONV_BK");
    forced = e ? atoi(e) : 0;
  }
  if (forced == 32 || forced == 64) return forced;
  return ksize == 3 && c_out_pad > 128 ? 32 : 64;
}

static int pick_block_n(int n) {
  if (n <= 256) return (n + 15) & ~15;  // single tile
  if (n % 256 == 0) return 256;
  if (n % 128 == 0) return 128;
  return 256;
}

// Ring slot width of a token-row GEMM (A_ROWS): 32 columns when the layer's full-width tile is above
// 128 columns (the coarse transformer's N = 256 / 512 projections and the dual-softmax passes over
// S >= 256 columns), else 64.  A 64-wide fp16x3 stage at N = 256 is 96 KB and only two fit beside the
// epilogue scratch, so, as in conv_chunk_k, one slot per stage leaves no load in flight while the MMAs
// hold both stages.  The rule reads the layer (N, K) only - never the batch, rows, tile width,
// cluster or N split - so that the batch-1 launches (N split, LayerNorm pair cluster, the dynamic-row
// kernels) sum the split products in the same order as the batch-64 ones and give the same bits.
// $OPP_ROWS_BK=32|64 forces one width for every token-row GEMM.
static int rows_chunk_k(int n, int k) {
  static int forced = -1;
  if (forced < 0) {
    const char* e = getenv("OPP_ROWS_BK");
    forced = e ? atoi(e) : 0;
  }
  if (forced == 32 || forced == 64) return forced;
  (void)k;
  return pick_block_n(n) > 128 ? 32 : 64;
}

// Latency shapes (batch 1-2: a GEMM has fewer super tiles than half the SMs, e.g. 16 clusters
// for 4096 tokens): halve the N tile, down to 64 columns, so that 2-4x as many SMs share the MMAs
// and the epilogue of the same output.  A is re-read once per N tile — a few hundred KB from L2.
// Call after pick_grouping() and before the W map is built.  $OPP_NSPLIT=0 disables it.
static void split_n_for_latency(GemmShape& s) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("OPP_NSPLIT");
    on = e ? atoi(e) : 1;
  }
  if (!on) return;
  const int max_clusters = num_sms() / s.cluster;
  while (s.block_n >= 128 && s.block_n % 64 == 0 && s.n_total % (s.block_n / 2) == 0 &&
         (long long)s.batches * s.msup * s.n_tiles * 2 <= max_clusters) {
    s.block_n /= 2;
    s.n_tiles = s.n_total / s.block_n;
  }
}

// Latency shapes of the LayerNorm GEMMs (N = 256 must stay in one row for the statistics): when
// every 128-row M tile can have a 2-CTA cluster of its own, the two CTAs take one 128-column half
// each (GemmShape.pair = 2) and exchange the row statistics through distributed shared memory —
// half the MMA and epilogue time per CTA; A is read twice (L2).  $OPP_LN_NSPLIT=0 disables it.
static void ln_nsplit_cluster(GemmShape& s) {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("OPP_LN_NSPLIT");
    on = e ? atoi(e) : 1;
  }
  if (!on || s.n_total != 256 || s.block_n != 256) return;
  if ((long long)s.batches * s.m_tiles > num_sms() / 2) return;
  s.pair = 2;
  s.cluster = 2;
  s.msup = s.m_tiles;
  s.block_n = 128;
  s.n_tiles = 1;
}

// Narrow the N tile until the operand ring, the accumulator tile (EpiConvUp: beside the ring or over
// it) and the epilogue scratch of Epi fit.  Sets mma_n (the smallest compiled wgmma width
// >= block_n, and >= min_mma_n); call before the W map is built (its box is mma_n / cluster rows).
template <class Epi>
static int fit_tile(GemmShape& s, int min_mma_n = 64) {
  for (;;) {
    s.mma_n = mma_width_for(s.block_n);
    if (s.mma_n < min_mma_n) s.mma_n = min_mma_n;
    GemmShape t = s;
    if (gemm_pick_stages<Epi>(t)) return OPP_OK;
    OPP_REQUIRE(s.pair == 0 && s.block_n > 16, "GEMM tile N=%d (split %d) does not fit in shared memory",
                s.block_n, s.split);
    s.block_n = (s.block_n / 2 + 15) & ~15;
    s.n_tiles = (s.n_total + s.block_n - 1) / s.block_n;
  }
}

// common shape / map setup for token-row GEMMs.  With split, every operand row holds two planes:
// A_i rows are [hi(k_i) | lo(k_i)], W rows are [hi(k0+k1) | lo(k0+k1)].
static int setup_rows(TensorMaps& maps, GemmShape& s, const void* a0, int k0, const void* a1,
                      int k1, const void* w, int w_batched, int batches, long long rows, int n,
                      int split, int n_align = 16, int a0_shared = 0, int nsplit_ok = 0,
                      int min_mma_n = 64) {
  OPP_REQUIRE(a0 && w, "null operand");
  OPP_REQUIRE(k0 > 0 && k0 % 64 == 0 && k1 % 64 == 0, "K (%d,%d) must be multiples of 64", k0,
              k1);
  OPP_REQUIRE(n > 0 && n % n_align == 0, "N=%d must be a multiple of %d", n, n_align);
  OPP_REQUIRE(batches > 0 && rows > 0, "empty GEMM");
  const int planes = split ? 2 : 1;
  memset(&s, 0, sizeof(s));
  s.batches = batches;
  s.rows = (int)rows;
  s.m_tiles = (int)((rows + kBlockM - 1) / kBlockM);
  s.block_n = pick_block_n(n);
  OPP_REQUIRE(s.block_n % 16 == 0 && s.block_n <= 256, "bad block_n %d", s.block_n);
  s.n_tiles = (n + s.block_n - 1) / s.block_n;
  s.n_total = n;
  s.bk = rows_chunk_k(n, k0 + k1);
  s.k_chunks_a0 = k0 / 64;
  s.k_chunks = (k0 + k1) / 64;
  s.b_batched = w_batched;
  s.split = split ? 1 : 0;
  s.a0_lo = k0;
  s.a1_lo = k1;
  s.b_lo = k0 + k1;
  s.a0_shared = a0_shared ? 1 : 0;
  const long long ld0 = (long long)planes * k0, ld1 = (long long)planes * k1;
  int rc = map_rows(&maps.a[0], a0, ld0, rows, a0_shared ? 1 : batches, ld0, rows * ld0, kBlockM, s.bk);
  if (rc) return rc;
  if (k1 > 0) {
    OPP_REQUIRE(a1, "null second A operand");
    rc = map_rows(&maps.a[1], a1, ld1, rows, batches, ld1, rows * ld1, kBlockM, s.bk);
    if (rc) return rc;
  } else {
    maps.a[1] = maps.a[0];
  }
  maps.a[2] = maps.a[0];
  maps.a[3] = maps.a[0];
  pick_grouping(s);
  if (nsplit_ok == 1) split_n_for_latency(s);
  if (nsplit_ok == 2) ln_nsplit_cluster(s);
  rc = fit_tile<EpiLN>(s, min_mma_n);   // the largest scratch of the token-row epilogues
  if (rc) return rc;
  const long long kt = (long long)planes * (k0 + k1);
  return map_rows(&maps.b, w, kt, n, w_batched ? batches : 1, kt, (long long)n * kt,
                  s.pair == 2 ? s.mma_n : s.mma_n / s.cluster, s.bk);
}

}  // namespace opp

using namespace opp;

extern "C" {

const char* opp_last_error(void) { return opp::last_error(); }

int opp_linear_act_f16(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                       long long rows, int n, int act, int act_cols, int split,
                       opp_stream_t stream) {
  return opp_linear_act_f16_b(a0, k0, 0, a1, k1, w, out, 1, rows, n, act, act_cols, split, nullptr, stream);
}

int opp_linear_act_f16_b(const void* a0, int k0, int a0_shared, const void* a1, int k1, const void* w,
                         void* out, int batches, long long rows, int n, int act, int act_cols,
                         int split, const unsigned char* row_mask, opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  int rc = setup_rows(maps, s, a0, k0, a1, k1, w, 0, batches, rows, n, split, 16, a0_shared, 1);
  if (rc) return rc;
  OPP_REQUIRE(out, "null output");
  OPP_REQUIRE(act_cols % 32 == 0, "act_cols=%d must be a multiple of 32", act_cols);
  EpiStoreF16::Params ep{(__half*)out, (long long)n * (split ? 2 : 1), split ? n : 0, act,
                         act_cols, row_mask};
  return launch<A_ROWS, EpiStoreF16>(maps, s, ep, (cudaStream_t)stream);
}

// split operands (hi|lo, three MMAs per K-step) with a SINGLE-plane fp16 output: for tensors whose
// consumer averages over thousands of rows (the K'/V rows of the linear-attention state), so that
// the 2^-12 output rounding is harmless while the row is half as long in HBM.  Same kernel as
// opp_linear_act_f16 (EpiStoreF16 with out_lo = 0).
int opp_linear_act_f16_out1(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                            long long rows, int n, int act, int act_cols, const unsigned char* row_mask,
                            opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  int rc = setup_rows(maps, s, a0, k0, a1, k1, w, 0, 1, rows, n, 1, 16, 0, 1);
  if (rc) return rc;
  OPP_REQUIRE(out, "null output");
  OPP_REQUIRE(act_cols % 32 == 0, "act_cols=%d must be a multiple of 32", act_cols);
  EpiStoreF16::Params ep{(__half*)out, (long long)n, 0, act, act_cols, row_mask};
  return launch<A_ROWS, EpiStoreF16>(maps, s, ep, (cudaStream_t)stream);
}

// Same GEMMs with a device-side row count: rows = *count * rows_per_count (<= cap_rows, the size
// the buffers were allocated for).  Used by the fine stage, whose row count is the number of coarse
// matches found on the device.
int opp_linear_act_f16_dyn(const void* a0, int k0, const void* a1, int k1, const void* w, void* out,
                           long long cap_rows, const int* count, int rows_per_count, int n, int act,
                           int act_cols, int split, opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  int rc = setup_rows(maps, s, a0, k0, a1, k1, w, 0, 1, cap_rows, n, split);
  if (rc) return rc;
  OPP_REQUIRE(out && count && rows_per_count > 0, "bad dynamic-row arguments");
  OPP_REQUIRE(act_cols % 32 == 0, "act_cols=%d must be a multiple of 32", act_cols);
  EpiStoreF16::Params ep{(__half*)out, (long long)n * (split ? 2 : 1), split ? n : 0, act, act_cols, nullptr};
  return launch<A_ROWS, EpiStoreF16, true>(maps, s, ep, (cudaStream_t)stream, count, rows_per_count);
}

int opp_linear_ln_dyn(const void* a0, int k0, const void* a1, int k1, const void* w, const float* gamma,
                      const float* beta, float eps, const void* resid, void* out16, float* out32,
                      long long cap_rows, const int* count, int rows_per_count, int n, int split,
                      opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  OPP_REQUIRE(n == 128 || n == 256, "LayerNorm epilogue needs N in {128,256}, got %d", n);
  int rc = setup_rows(maps, s, a0, k0, a1, k1, w, 0, 1, cap_rows, n, split);
  if (rc) return rc;
  OPP_REQUIRE(s.n_tiles == 1 && s.block_n == n, "LayerNorm row of N=%d split across tiles", n);
  OPP_REQUIRE(gamma && beta && count && rows_per_count > 0, "bad dynamic-row arguments");
  OPP_REQUIRE(out16 || out32, "no output requested");
  EpiLN::Params ep{gamma, beta, eps, (const __half*)resid, 0, (__half*)out16,
                   (long long)n * (split ? 2 : 1), split ? n : 0, out32};
  return launch<A_ROWS, EpiLN, true>(maps, s, ep, (cudaStream_t)stream, count, rows_per_count);
}

int opp_linear_q_f16(const void* x, const void* wq, const float* ksum, void* out, int batches,
                     int rows, int d_model, float v_len, float eps, int split, int x_shared,
                     const unsigned char* row_mask, opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  OPP_REQUIRE(d_model == 256, "opp_linear_q_f16 supports d_model 256 (8 heads x 32), got %d",
              d_model);
  int rc = setup_rows(maps, s, x, d_model, nullptr, 0, wq, 0, batches, rows, d_model, split, 16, x_shared, 1);
  if (rc) return rc;
  OPP_REQUIRE(ksum && out, "null pointer");
  EpiQ::Params ep{(__half*)out, (long long)d_model * (split ? 2 : 1), split ? d_model : 0, ksum,
                  v_len, eps, row_mask};
  return launch<A_ROWS, EpiQ>(maps, s, ep, (cudaStream_t)stream);
}

int opp_linear_ln(const void* a0, int k0, const void* a1, int k1, const void* w, int w_batched,
                  const float* gamma, const float* beta, float eps, const void* resid,
                  int resid_shared, void* out16, float* out32, int batches, long long rows, int n,
                  int split, opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  OPP_REQUIRE(n == 128 || n == 256, "LayerNorm epilogue needs N in {128,256}, got %d", n);
  int rc = setup_rows(maps, s, a0, k0, a1, k1, w, w_batched, batches, rows, n, split, 16, 0, 2);
  if (rc) return rc;
  // EpiLN needs whole rows in one CTA, or the two halves of the N-split cluster
  OPP_REQUIRE(s.n_tiles == 1 && s.block_n * (s.pair == 2 ? 2 : 1) == n,
              "LayerNorm row of N=%d split across tiles", n);
  OPP_REQUIRE(gamma && beta, "null LayerNorm parameters");
  OPP_REQUIRE(out16 || out32, "no output requested");
  EpiLN::Params ep{gamma, beta, eps, (const __half*)resid, resid_shared, (__half*)out16,
                   (long long)n * (split ? 2 : 1), split ? n : 0, out32};
  return launch<A_ROWS, EpiLN>(maps, s, ep, (cudaStream_t)stream);
}

int opp_conv2d_nhwc(const void* in, const void* w, const float* bias, const void* resid,
                    void* out, int batch, int in_h, int in_w, int c_in_pad, int c_out_pad,
                    int ksize, int stride, int act, float slope, void* tok, const float* pe,
                    const void* up, int split, opp_stream_t stream) {
  OPP_REQUIRE(in && w && bias, "null operand");
  OPP_REQUIRE(ksize == 1 || ksize == 3, "kernel size %d unsupported (1 or 3)", ksize);
  OPP_REQUIRE(stride == 1 || stride == 2, "stride %d unsupported", stride);
  OPP_REQUIRE(c_in_pad % 16 == 0 && c_out_pad % 16 == 0 && c_out_pad <= 256,
              "channel counts must be padded to multiples of 16 (got %d -> %d)", c_in_pad,
              c_out_pad);
  OPP_REQUIRE(stride == 1 || (in_h % 2 == 0 && in_w % 2 == 0), "stride 2 needs even H, W");
  OPP_REQUIRE(out || tok, "no output requested");
  const int planes = split ? 2 : 1;
  const int pad = ksize / 2;
  const int out_h = (in_h + 2 * pad - ksize) / stride + 1;
  const int out_w = (in_w + 2 * pad - ksize) / stride + 1;
  TensorMaps maps;
  GemmShape s;
  memset(&s, 0, sizeof(s));
  s.batches = batch;
  s.rows = out_h * out_w;
  s.tile_w = 16;
  s.tile_h = 8;
  s.tiles_x = (out_w + s.tile_w - 1) / s.tile_w;
  s.tiles_y = (out_h + s.tile_h - 1) / s.tile_h;
  s.m_tiles = s.tiles_x * s.tiles_y;
  s.block_n = c_out_pad;
  s.n_tiles = 1;
  s.n_total = c_out_pad;
  s.conv_c = c_in_pad;
  s.bk = conv_chunk_k(ksize, c_out_pad);
  s.conv_cchunks = (c_in_pad + 63) / 64;
  s.k_chunks = ksize * ksize * s.conv_cchunks;
  s.conv_kw = ksize;
  s.conv_pad = pad;
  s.conv_stride = stride;
  s.out_w = out_w;
  s.out_h = out_h;
  s.split = split ? 1 : 0;
  // A maps are 5-D (channel, plane, x, y, image) with channel extent c_in_pad: the last bk-channel
  // box of a row reads zeros past c_in_pad (the mainloop skips the MMA steps of a 16-channel tail)
  const long long C = (long long)planes * c_in_pad;  // pixel stride in elements
  const __half* base = (const __half*)in;
  int rc;
  if (stride == 1) {
    uint64_t dims[5] = {(uint64_t)c_in_pad, (uint64_t)planes, (uint64_t)in_w, (uint64_t)in_h, (uint64_t)batch};
    uint64_t str[4] = {(uint64_t)c_in_pad, (uint64_t)C, (uint64_t)(in_w * C), (uint64_t)((long long)in_h * in_w * C)};
    uint32_t box[5] = {(uint32_t)s.bk, 1, (uint32_t)s.tile_w, (uint32_t)s.tile_h, 1};
    rc = make_map(&maps.a[0], base, 5, dims, str, box);
    if (rc) return rc;
    maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  } else {
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        uint64_t dims[5] = {(uint64_t)c_in_pad, (uint64_t)planes, (uint64_t)(in_w / 2),
                            (uint64_t)(in_h / 2), (uint64_t)batch};
        uint64_t str[4] = {(uint64_t)c_in_pad, (uint64_t)(2 * C), (uint64_t)(2LL * in_w * C),
                           (uint64_t)((long long)in_h * in_w * C)};
        uint32_t box[5] = {(uint32_t)s.bk, 1, (uint32_t)s.tile_w, (uint32_t)s.tile_h, 1};
        rc = make_map(&maps.a[py * 2 + px], base + ((long long)py * in_w + px) * C, 5, dims, str,
                      box);
        if (rc) return rc;
      }
  }
  const long long kplane = (long long)ksize * ksize * c_in_pad;
  s.b_lo = (int)kplane;
  const long long kt = kplane * planes;
  pick_grouping(s);
  split_n_for_latency(s);   // the 1/8-resolution layers at batch 1: 16 clusters -> 64
  rc = up ? fit_tile<EpiConvUp>(s) : fit_tile<EpiConv>(s);
  if (rc) return rc;
  rc = map_rows(&maps.b, w, kt, c_out_pad, 1, kt, (long long)c_out_pad * kt, s.mma_n / s.cluster, s.bk);
  if (rc) return rc;
  OPP_REQUIRE(!up || (out_h % 2 == 0 && out_w % 2 == 0 && out_h >= 4 && out_w >= 4),
              "fused upsample-add needs even output dims >= 4 (got %d x %d)", out_h, out_w);
  EpiConvParams ep{(__half*)out, (long long)c_out_pad * planes, split ? c_out_pad : 0, bias,
                     (const __half*)resid, act, slope, (__half*)tok, pe, (const __half*)up,
                     out_h / 2, out_w / 2,
                     up ? (float)(out_h / 2 - 1) / (float)(out_h - 1) : 0.f,
                     up ? (float)(out_w / 2 - 1) / (float)(out_w - 1) : 0.f};
  if (up) return launch<A_CONV, EpiConvUp>(maps, s, ep, (cudaStream_t)stream);
  return launch<A_CONV, EpiConv>(maps, s, ep, (cudaStream_t)stream);
}

// Row pitch of the compact output windows of opp_conv_win: 8 for both window sides, so that a
// window's box is a whole number of swizzle atoms in the A stage (7x8: two windows = 112 accumulator
// rows; 5x8: three windows = 120 rows, 75 of them valid).
int opp_conv_win_pitch(int) { return 8; }

int opp_conv_win(const void* in, const void* w, const float* bias, void* out, const long long* b_ids,
                 const long long* j_ids, int matches, const int* count, int batch, int in_h, int in_w,
                 int c_in_pad, int c_out_pad, int win, int wc, int stride, int org, int act,
                 float slope, int split, opp_stream_t stream) {
  OPP_REQUIRE(in && w && bias && out, "null operand");
  OPP_REQUIRE(win == 5 || win == 7, "window side %d unsupported (5 or 7)", win);
  OPP_REQUIRE(c_in_pad % 16 == 0 && c_out_pad % 16 == 0 && c_out_pad <= 256,
              "channel counts must be padded to multiples of 16 (got %d -> %d)", c_in_pad, c_out_pad);
  OPP_REQUIRE(matches >= 0 && (j_ids == nullptr) == (b_ids == nullptr), "bad match list");
  OPP_REQUIRE(!j_ids || (wc > 0 && stride > 0 && batch > 0 && in_h > 0 && in_w > 0),
              "dense-input window convolution needs the map size, wc and stride");
  if (matches == 0) return OPP_OK;
  const int planes = split ? 2 : 1;
  TensorMaps maps;
  GemmShape s;
  memset(&s, 0, sizeof(s));
  s.batches = 1;
  const int pitch = opp_conv_win_pitch(win);
  s.tile_w = pitch;
  s.tile_h = win;
  s.tiles_x = 128 / (pitch * win);   // windows per M tile: 2 (7x8) or 3 (5x8)
  s.tiles_y = 1;
  s.rows = matches * pitch * win;
  s.m_tiles = (matches + s.tiles_x - 1) / s.tiles_x;
  s.block_n = c_out_pad;
  s.n_tiles = 1;
  s.n_total = c_out_pad;
  s.conv_c = c_in_pad;
  s.bk = conv_chunk_k(3, c_out_pad);
  s.conv_cchunks = (c_in_pad + 63) / 64;
  s.k_chunks = 9 * s.conv_cchunks;
  s.conv_kw = 3;
  s.conv_pad = 1;
  s.conv_stride = 1;
  s.out_w = pitch;
  s.out_h = win;
  s.split = split ? 1 : 0;
  const long long C = (long long)planes * c_in_pad;
  int rc;
  {
    const uint64_t iw = j_ids ? in_w : 8, ih = j_ids ? in_h : win + 2, ib = j_ids ? batch : matches;
    uint64_t dims[5] = {(uint64_t)c_in_pad, (uint64_t)planes, iw, ih, ib};   // 5-D: see opp_conv2d_nhwc
    uint64_t str[4] = {(uint64_t)c_in_pad, (uint64_t)C, (uint64_t)(iw * C), (uint64_t)(ih * iw * C)};
    uint32_t box[5] = {(uint32_t)s.bk, 1, (uint32_t)pitch, (uint32_t)win, 1};
    rc = make_map(&maps.a[0], in, 5, dims, str, box);
    if (rc) return rc;
    maps.a[1] = maps.a[2] = maps.a[3] = maps.a[0];
  }
  const long long kplane = 9LL * c_in_pad;
  s.b_lo = (int)kplane;
  const long long kt = kplane * planes;
  pick_grouping(s);
  rc = fit_tile<EpiWin>(s);
  if (rc) return rc;
  rc = map_rows(&maps.b, w, kt, c_out_pad, 1, kt, (long long)c_out_pad * kt, s.mma_n / s.cluster, s.bk);
  if (rc) return rc;
  EpiWin::Params ep{(__half*)out, (long long)c_out_pad * planes, split ? c_out_pad : 0, bias, act, slope,
                    b_ids, j_ids, wc, stride, org, in_h, in_w};
  if (count) return launch<A_WIN, EpiWin, true>(maps, s, ep, (cudaStream_t)stream, count, pitch * win);
  return launch<A_WIN, EpiWin>(maps, s, ep, (cudaStream_t)stream);
}

int opp_sim_lse_cols_rows(const void* a, const void* b, float* part_m, float* part_s, float* col_m,
                          float* col_s, int batches, int rows, int cols, int k, float scale, int split,
                          const unsigned char* col_mask, const int* row_count, opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  int rc = setup_rows(maps, s, a, k, nullptr, 0, b, 1, batches, rows, cols, split, 1, 0, 0,
                      EpiLseCol::kMinMmaN);
  if (rc) return rc;
  OPP_REQUIRE(part_m && part_s && col_m && col_s, "null pointer");
  OPP_REQUIRE(!(col_mask && row_count), "col_mask and row_count are not combined");
  EpiLseColParams ep{part_m, part_s, scale, col_m, col_s, (rows + 31) / 32, col_mask};
  if (row_count) {
    EpiLseColRowsParams epr{ep, row_count};
    return launch<A_ROWS, EpiLseColRows>(maps, s, epr, (cudaStream_t)stream);
  }
  if (col_mask) return launch<A_ROWS, EpiLseColMasked>(maps, s, ep, (cudaStream_t)stream);
  return launch<A_ROWS, EpiLseCol>(maps, s, ep, (cudaStream_t)stream);
}

int opp_sim_lse_cols(const void* a, const void* b, float* part_m, float* part_s, float* col_m,
                     float* col_s, int batches, int rows, int cols, int k, float scale, int split,
                     const unsigned char* col_mask, opp_stream_t stream) {
  return opp_sim_lse_cols_rows(a, b, part_m, part_s, col_m, col_s, batches, rows, cols, k, scale, split,
                               col_mask, nullptr, stream);
}

int opp_sim_conf_colmax_rows(const void* a, const void* b, const float* lse_own, const float* lse_other,
                             float* conf, float* part_val, int* part_idx, unsigned* colmax, int batches,
                             int rows, int cols, int k, float scale, int split, const int* row_count,
                             opp_stream_t stream) {
  TensorMaps maps;
  GemmShape s;
  int rc = setup_rows(maps, s, a, k, nullptr, 0, b, 1, batches, rows, cols, split, 1, 0, 0,
                      EpiConfCol::kMinMmaN);
  if (rc) return rc;
  OPP_REQUIRE(lse_own && lse_other && part_val && part_idx && colmax, "null pointer");
  OPP_CHECK_CUDA(cudaMemsetAsync(colmax, 0, (size_t)batches * cols * sizeof(unsigned),
                                 (cudaStream_t)stream));
  EpiConfColParams ep{lse_own, lse_other, scale, conf, part_val, part_idx, colmax};
  if (row_count) {
    EpiConfColRowsParams epr{ep, row_count};
    return launch<A_ROWS, EpiConfColRows>(maps, s, epr, (cudaStream_t)stream);
  }
  return launch<A_ROWS, EpiConfCol>(maps, s, ep, (cudaStream_t)stream);
}

int opp_sim_conf_colmax(const void* a, const void* b, const float* lse_own, const float* lse_other,
                        float* conf, float* part_val, int* part_idx, unsigned* colmax, int batches,
                        int rows, int cols, int k, float scale, int split, opp_stream_t stream) {
  return opp_sim_conf_colmax_rows(a, b, lse_own, lse_other, conf, part_val, part_idx, colmax, batches, rows,
                                  cols, k, scale, split, nullptr, stream);
}

// partial slots per row written by the dual-softmax passes: one per column tile (a row lives in one
// quad of one warp, so a tile leaves one (max, sum) / (max, argmax) per row)
int opp_sim_tiles(int cols) {
  return (cols + pick_block_n(cols) - 1) / pick_block_n(cols);
}

}  // extern "C"
