// surya_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[M, Nout] = epilogue(A[M, K] @ W[N, K]^T)      (torch nn.Linear layout: both operands K-major)
//
// Replaces every cuBLAS call the reference makes through nn.Linear / 1x1 Conv2d on the hot path
// (SURVEY.md §2.2 K1, K3, K5-K7, K9-K11).  Design:
//   * one CTA per SM, persistent over a grouped tile raster (A/W tiles stay L2 resident);
//   * warp 0 = TMA producer (cp.async.bulk.tensor, 128B swizzle, BK = 64 elements per stage), running ahead into the next
//     tile while the consumers finish the current one;
//   * warps 4-11 = two consumer warpgroups: wgmma m64 x BN x 16 on rows [0, 64) and [64, 128) of the tile, fp32
//     accumulators in registers, then staged through shared memory (gemm_epilogue.cuh) for the bias/act/residual/SwiGLU
//     epilogue, which all 8 warps run (tiles wider than 128 columns in two passes).
// Rounding to the storage type happens exactly where eager PyTorch has an op boundary (after the
// Linear, after the activation, after the residual add) so results track the reference path.
//
// DECODE = true is the recognition decode step's variant (GemmArgs::decode, M <= 256 rows against a large weight matrix):
// only the single-pass 16-bit staged epilogue, no grouped mode and no fallback epilogue (epilogue_chunk, a __noinline__
// call).  Without them ptxas gives it no stack frame and, at BN = 128, no spills, and the decode GEMMs run faster
// (DESIGN.md §5).  Both variants give the same bits.
//
// STAGED = true is the plain variant for launches the 16-bit staged epilogue takes (epilogue_v2_ok) outside grouped mode: the
// same code with the fallback epilogue and the grouped A offset compiled out, as in the decode variant.  At BN = 128 that
// removes the plain variant's stack frame and spills.  Same bits: it runs the staged epilogue the plain variant would.
#include "gemm.cuh"

#include <string>
#include <unordered_map>
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

#include <cstdarg>
#include <cstdio>
#include <atomic>
#include <mutex>

namespace sb {

__device__ __forceinline__ void tile_coords(int tile, int m_blocks, int n_blocks, int gm, int& mb, int& nb) {
  int per_group = gm * n_blocks;
  int g = tile / per_group;
  int first = g * gm;
  int gsz = min(m_blocks - first, gm);
  int r = tile - g * per_group;
  mb = first + r % gsz;
  nb = r / gsz;
}

template <typename T, int BN, int STAGES, bool DECODE, bool STAGED = false>
__global__ void __launch_bounds__(384, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const GemmKParams p) {
  constexpr int BM = 128, BK = 64;
  constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int AC = acc_cols<BN>();
  static_assert(!DECODE || BN <= ACC_MAX_COLS, "the decode variant takes single-pass epilogue tiles only");
  static_assert(!STAGED || (!DECODE && BN <= ACC_MAX_COLS), "the staged plain variant takes single-pass epilogue tiles only");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_s = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);             // [128][AC] accumulator tile
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(acc_s) + acc_smem_bytes<BN>();        // 8 x EPI_STAGE_BYTES staging + bias + row scales

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();
  const int m_blocks = (p.M + BM - 1) / BM;
  const int n_blocks = (p.N + BN - 1) / BN;
  const int k_blocks = (p.K + BK - 1) / BK;
  const int num_tiles = m_blocks * n_blocks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], EPI_WARPS);   // a stage is free once every consumer warp's MMAs (and RMS pass) are done with it
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      // Weight tiles of the first pipeline fill do not depend on the previous kernel: request them before the
      // programmatic-dependency wait so that the DRAM latency overlaps the predecessor's tail.
      int early = 0;
      if (p.w_constant && static_cast<int>(blockIdx.x) < num_tiles) {
        int mb, nb;
        if constexpr (DECODE) { mb = static_cast<int>(blockIdx.x) % m_blocks; nb = static_cast<int>(blockIdx.x) / m_blocks; }
        else tile_coords(blockIdx.x, m_blocks, n_blocks, p.group_m, mb, nb);
        early = k_blocks < STAGES ? k_blocks : STAGES;
        for (int kb = 0; kb < early; ++kb) {
          uint8_t* sa = smem + kb * STAGE_BYTES;
          mbar_expect_tx(&full_bar[kb], STAGE_BYTES);
          tma_load_2d(sa + A_BYTES, &tma_b, &full_bar[kb], kb * BK, nb * BN);
        }
      }
      pdl_wait();
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        // The decode variant runs both m-blocks of a weight tile back to back.  At M <= 256 (at most two m-blocks) that is
        // the order tile_coords gives with group_m = 8, so both variants give the same bits.
        int mb, nb;
        if constexpr (DECODE) { mb = tile % m_blocks; nb = tile / m_blocks; }
        else tile_coords(tile, m_blocks, n_blocks, p.group_m, mb, nb);
        for (int kb = 0; kb < k_blocks; ++kb) {
          uint8_t* sa = smem + s * STAGE_BYTES;
          uint8_t* sbp = sa + A_BYTES;
          // B of the first tile's first stages was requested before pdl_wait.  The plain variant requests a stage's A tile
          // before its B tile, the decode variant after it: one order for both was slower on H100 for prefill or for the
          // decode step, whichever it did not come from (DESIGN.md §5).  Grouped mode: A columns of this n-block's group.
          const bool b_in_flight = tile == static_cast<int>(blockIdx.x) && kb < early;
          if (!DECODE && b_in_flight) tma_load_2d(sa, &tma_a, &full_bar[s], kb * BK + (STAGED ? 0 : nb * p.group_k), mb * BM);
          if (!b_in_flight) {
            mbar_wait(&empty_bar[s], ph ^ 1);
            mbar_expect_tx(&full_bar[s], STAGE_BYTES);
            if (!DECODE) tma_load_2d(sa, &tma_a, &full_bar[s], kb * BK + (STAGED ? 0 : nb * p.group_k), mb * BM);
            tma_load_2d(sbp, &tma_b, &full_bar[s], kb * BK, nb * BN);
          }
          if (DECODE) tma_load_2d(sa, &tma_a, &full_bar[s], kb * BK, mb * BM);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumer warpgroups: MMA + epilogue
    pdl_wait();
    const int wg = (warp - 4) >> 2;     // MMA rows [64 wg, 64 wg + 64) of the tile
    const int q = warp & 3;             // epilogue: rows [32 q, 32 q + 32) of the tile
    const int half = wg;                // two warps share a row quarter and alternate column groups
    const int epi_tid = threadIdx.x - 128;
    uint8_t* stage = epi_smem + (warp - 4) * EPI_STAGE_BYTES;
    float* sbias = reinterpret_cast<float*>(epi_smem + EPI_WARPS * EPI_STAGE_BYTES);
    float* srs = sbias + BN;                              // 128 per-row scales of the current tile (folded RMSNorm)
    int s = 0;
    uint32_t ph = 0;
    const bool vec_ok = (p.ldc % 8 == 0) && (!p.residual || p.ldr % 8 == 0);
    const bool v2 = DECODE || STAGED || epilogue_v2_ok(p);   // the host launches these variants only where it applies
    const AccRow acc(acc_s, q * 32 + lane, AC);
    float d[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mb, nb;
      if constexpr (DECODE) { mb = tile % m_blocks; nb = tile / m_blocks; }
      else tile_coords(tile, m_blocks, n_blocks, p.group_m, mb, nb);
      if (v2) {
        asm volatile("bar.sync 1, 256;" ::: "memory");   // all epilogue warps are done with the previous tile's bias
        epilogue_stage_bias<BN>(p, sbias, epi_tid, nb * BN);
        if (p.rowscale && epi_tid < BM) srs[epi_tid] = mb * BM + epi_tid < p.M ? __ldg(p.rowscale + mb * BM + epi_tid) : 0.f;
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      // sum of squares of the tile's 128 A rows (folded RMSNorm), taken from each stage while its MMAs run
      float ssq = 0.f;
      wg_mainloop<T, BN, BK>(d, smem, STAGE_BYTES, A_BYTES, STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane,
                             [&](const uint8_t* slot) {
                               if (p.ssq_inline) ssq = ssq_stage<T>(slot, epi_tid, ssq);
                             });
      if (p.ssq_inline) {
        const float tot = ssq + __shfl_xor_sync(0xffffffffu, ssq, 1);
        if ((epi_tid & 1) == 0) srs[epi_tid >> 1] = rsqrtf(tot * p.ssq_inv_k + p.ssq_eps);
      }
      const int row0 = mb * BM + q * 32;
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += AC) {
        asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free (previous pass / tile read it)
        wg_acc_store<AC / 8>(d, c0 / 8, acc_s + wg * 64 * AC, AC, warp & 3, lane);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (v2) {
          const float rs = (p.ssq_inline || p.rowscale) ? srs[q * 32 + lane] : 1.0f;
          if (!p.am_val || p.store_c)
            epilogue_tile_rt<T>(acc, p, stage, sbias + c0, lane, half,
                                [&](int r) { return row0 + r < p.M ? row0 + r : -1; }, nb * BN + c0, rs, AC / 32);
          if constexpr (BN == AC) {
            if (p.am_val)
              epilogue_tile_argmax<T, BN>(acc, p, epi_smem, sbias, lane, half, q, row0 + lane < p.M ? row0 + lane : -1,
                                          nb * BN, nb, rs);
          }
        } else if (half == 0) {
          const int row = row0 + lane;
          const bool row_ok = row < p.M;
#pragma unroll 1
          for (int c = 0; c < AC / 32; ++c) {
            uint32_t v[32];
            acc.load32(c * 32, v);
            const int col0 = nb * BN + c0 + c * 32;
            if (col0 >= p.N) continue;
            epilogue_chunk<T>(v, p, row, row_ok, col0, vec_ok);
          }
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------- host side
static thread_local char g_err[512] = {0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

static std::atomic<long long> g_launches{0};
long long launch_count() { return g_launches.load(); }
void count_launches(long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int launch_ok() {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("kernel launch failed: %s", cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
  });
  return fn;
}

// cuTensorMapEncodeTiled costs 1-2 us of host time per operand; engines issue the same few hundred (pointer, shape, box)
// combinations every forward / step, so encoded maps are memoised (key = every argument of the encode call).
static CUresult encode_tiled_cached(CUtensorMap* map, CUtensorMapDataType dt, int rank, const void* base, const cuuint64_t* dims,
                                    const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr,
                                    CUtensorMapSwizzle swz) {
  struct Key { uint64_t v[18]; };
  Key k{};
  k.v[0] = reinterpret_cast<uint64_t>(base);
  k.v[1] = (static_cast<uint64_t>(dt) << 40) | (static_cast<uint64_t>(rank) << 32) | static_cast<uint64_t>(swz);
  for (int i = 0; i < rank; ++i) { k.v[2 + i] = dims[i]; k.v[10 + i] = (static_cast<uint64_t>(box[i]) << 32) | estr[i]; }
  for (int i = 0; i + 1 < rank; ++i) k.v[6 + i] = strides[i];
  const std::string key(reinterpret_cast<const char*>(&k), sizeof(k));
  static std::mutex mu;
  static std::unordered_map<std::string, CUtensorMap> cache;
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *map = it->second; return CUDA_SUCCESS; }
  }
  CUresult r = get_encode_fn()(map, dt, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) {
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 16384) cache.clear();
    cache.emplace(key, *map);
  }
  return r;
}

int make_tma_2d_sw(CUtensorMap* map, int dtype, const void* base, int rows, int K, int ld, int box_k, int box_rows,
                   int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)"); return -1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (static_cast<size_t>(ld) * 2) % 16 != 0) {
    set_error("TMA operand must be 16B aligned with a 16B-multiple row pitch (ptr=%p ld=%d)", base, ld);
    return -2;
  }
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_k), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_tiled_cached(map, dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base,
                                   dims, strides, box, estr,
                                   swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                                        : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE));
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(2d) failed: %d (rows=%d K=%d ld=%d box=%dx%d)", (int)r, rows, K, ld, box_k, box_rows);
    return -3;
  }
  return 0;
}

int make_tma_nhwc(CUtensorMap* map, int dtype, const void* base, int N, int H, int W, int C, int box_c, int box_w,
                  int box_h, int stride, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)"); return -1; }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (static_cast<size_t>(C) * 2) % 16 != 0) {
    set_error("NHWC TMA operand must be 16B aligned with C %% 8 == 0 (ptr=%p C=%d)", base, C);
    return -2;
  }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)(box_w * stride), (cuuint32_t)(box_h * stride), 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = encode_tiled_cached(map, dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base,
                                   dims, strides, box, estr,
                                   swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                                        : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE));
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(nhwc) failed: %d (N=%d H=%d W=%d C=%d box=%d,%d,%d stride=%d)", (int)r, N, H, W, C,
              box_c, box_w, box_h, stride);
    return -3;
  }
  return 0;
}

// Shared memory per CTA: STAGES ring slots + barriers + the fp32 accumulator tile + epilogue staging, within the 227 KB an
// sm_90 block may use.  Stage counts are the most that fit for each tile width.
constexpr size_t SMEM_LIMIT = 227 * 1024;
template <int BN, int STAGES> constexpr size_t gemm_smem_bytes() {
  return STAGES * (128 * 64 * 2 + BN * 64 * 2) + 1024 /*align slack*/ + 256 /*barriers*/ + acc_smem_bytes<BN>() + epi_smem_bytes<BN>();
}

template <typename T, int BN, int STAGES, bool DECODE, bool STAGED = false>
static int launch_cfg(const GemmArgs& a, cudaStream_t stream) {
  constexpr size_t SMEM = gemm_smem_bytes<BN, STAGES>();
  static_assert(SMEM <= SMEM_LIMIT, "GEMM tile does not fit in shared memory");
  static bool attr_set = false;
  auto kern = gemm_tn_kernel<T, BN, STAGES, DECODE, STAGED>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%zu) failed: %s", SMEM, cudaGetErrorString(e));
      return -10;
    }
    attr_set = true;
  }
  CUtensorMap ma, mb;
  int rc = make_tma_2d(&ma, a.dtype, a.A, a.M, a.group_k ? a.a_cols : a.K, a.lda, 128);
  if (rc) return rc;
  rc = make_tma_2d(&mb, a.dtype, a.W, a.N, a.K, a.ldw, BN);  // grouped: W is [N, K] with K = padded per-group depth
  if (rc) return rc;
  const GemmKParams p = gemm_kparams(a);
  int m_blocks = (a.M + 127) / 128, n_blocks = (a.N + BN - 1) / BN;
  int tiles = m_blocks * n_blocks;
  int grid = tiles < num_sms() ? tiles : num_sms();
  if (launch_pdl(kern, dim3(grid), dim3(384), SMEM, stream, ma, mb, p) != cudaSuccess) { /* reported by launch_ok */ }
  return launch_ok();
}

// Ring stages per tile width: the most that fit beside the accumulator tile and the epilogue staging.  The decode variant
// takes the single-pass widths only.
template <typename T, bool DECODE>
static int launch_bn(const GemmArgs& a, int bn, cudaStream_t stream) {
  switch (bn) {
    case 128:
      // plain launches the staged epilogue takes run without the fallback epilogue (BN 128 only: the width where it costs
      // the plain variant spills)
      if (!DECODE && !a.group_k && epilogue_v2_ok(gemm_kparams(a))) return launch_cfg<T, 128, 4, false, true>(a, stream);
      return launch_cfg<T, 128, 4, DECODE>(a, stream);
    case 64: return launch_cfg<T, 64, 6, DECODE>(a, stream);
    case 32: return launch_cfg<T, 32, 8, DECODE>(a, stream);
  }
  if constexpr (!DECODE) {
    if (bn == 256) return launch_cfg<T, 256, 2, false>(a, stream);
    if (bn == 96) return launch_cfg<T, 96, 5, false>(a, stream);
  }
  set_error("unsupported BN %d", bn);
  return -12;
}

template <typename T>
static int launch_typed(const GemmArgs& a, cudaStream_t stream) {
  if (a.decode) {
    // Tile width per decode shape, measured on H100 (DESIGN.md §5): 32 for the 1280- / 1920-wide qkv and o projections, 128
    // for gate/up; the argmax epilogue keeps gemm_argmax_tile's width, which sized the caller's partial buffers.
    const int bn = a.force_bn ? a.force_bn : a.am_val ? gemm_argmax_tile(a.M, a.N) : a.N >= 4096 ? 128 : 32;
    return launch_bn<T, true>(a, bn, stream);
  }
  int bn = a.force_bn;
  if (bn >= 1000) return gemm_splitk_launch(a, bn / 1000, bn % 1000, stream);   // forced split-K: 1000 * pk + BN
  if (bn == 0 && a.allow_splitk && !a.rowscale && !a.ssq_inline && !a.am_val) {
    int sbn = 0;
    const int pk = splitk_plan(a, &sbn);
    if (pk >= 2) return gemm_splitk_launch(a, pk, sbn, stream);
  }
  if (bn == 0) {
    // Big problems: 128x128 tiles (a 256-wide tile keeps only two ring stages beside its accumulator tile, and its epilogue
    // runs in two passes).  Otherwise the main loop is bound by DRAM latency x bytes in flight per SM, so prefer a single
    // wave of many small tiles: cost = waves * bytes per k-block, with a penalty when fewer than ~60 % of the SMs would be
    // streaming the weight matrix.
    const int sms = num_sms();
    const int m_blocks = (a.M + 127) / 128;
    if (a.N <= 128 && m_blocks >= sms) {
      // narrow outputs over many rows (1x1 "project" convs): the launch streams A; a tile wider than N only adds zero-filled W
      // loads and MMA / epilogue work
      bn = a.N <= 32 ? 32 : a.N <= 64 ? 64 : a.N <= 96 ? 96 : 128;
    } else if (m_blocks * ((a.N + 127) / 128) >= (sms * 3) / 4) {
      bn = 128;
    } else {
      const int cands[4] = {128, 96, 64, 32};
      double best = 1e30;
      for (int i = 0; i < 4; ++i) {
        const int c = cands[i];
        if (a.swiglu && (c % 32)) continue;
        const int tiles = m_blocks * ((a.N + c - 1) / c);
        const int waves = (tiles + sms - 1) / sms;
        double cost = static_cast<double>(waves) * (128 + c);
        const double occ = 0.6 * sms / tiles;
        if (occ > 1.0) cost *= occ;
        if (cost < best) { best = cost; bn = c; }
      }
    }
  }
  if (a.am_val && a.force_bn == 0) bn = gemm_argmax_tile(a.M, a.N);   // the caller sized its partial buffers with this
  if (a.group_k) bn = a.group_n;  // one n-block per channel group
  return launch_bn<T, false>(a, bn, stream);
}

int gemm_argmax_tile(int M, int N) {
  (void)M;
  return N >= 1024 ? 128 : 64;   // the argmax epilogue runs on single-pass tiles (<= ACC_MAX_COLS columns)
}

int gemm_launch(const GemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return 0;
  // Every epilogue may store C and load the residual in 16-byte vectors, and none of them combines these options; the
  // arguments are rejected here rather than faulting the device or being dropped silently on one path.
  if ((reinterpret_cast<uintptr_t>(a.C) & 15) != 0) {
    set_error("gemm: C must be 16B aligned (ptr=%p)", a.C);
    return -19;
  }
  if ((reinterpret_cast<uintptr_t>(a.residual) & 15) != 0) {
    set_error("gemm: the residual must be 16B aligned (ptr=%p)", a.residual);
    return -19;
  }
  if (a.swiglu && a.residual) { set_error("gemm: the swiglu epilogue takes no residual"); return -20; }
  if (a.out_f32 && (a.residual || a.swiglu)) { set_error("gemm: out_f32 takes no residual and no swiglu"); return -20; }
  const bool staged = epilogue_v2_ok(gemm_kparams(a));   // the kernels' own rule for the 16-bit staged epilogue
  if (a.rowscale || a.ssq_inline || a.am_val) {
    // these ride on the staged 16-bit epilogue only (and on the plain kernel: split-K would change who owns a row's columns)
    if (!staged || a.group_k || a.force_bn >= 1000) {
      set_error("gemm: rowscale / ssq_inline / argmax epilogues need the 16-bit staged epilogue (N %% 8 == 0, 16-byte pitches), "
                "no grouped or split-K mode");
      return -15;
    }
    if (a.rowscale && a.ssq_inline) { set_error("gemm: rowscale and ssq_inline are exclusive"); return -15; }
    if (a.am_val && (!a.am_idx || !a.am_sum || a.am_ld <= 0)) { set_error("gemm: incomplete argmax partial buffers"); return -15; }
    if (a.am_val && a.force_bn > ACC_MAX_COLS) { set_error("gemm: the argmax epilogue needs a tile width <= %d", ACC_MAX_COLS); return -15; }
  }
  if (a.swiglu && (a.N % 2 != 0)) {
    set_error("swiglu epilogue needs an even N");
    return -13;
  }
  if (a.dtype != DT_BF16 && a.dtype != DT_F16) { set_error("unsupported dtype %d", a.dtype); return -14; }
  if (a.decode) {
    if (a.decode != 1) {
      set_error("gemm: decode must be 0 or 1 (got %d)", a.decode);
      return -21;
    }
    if (a.M > 256 || a.out_f32 || a.group_k || a.force_bn >= 1000) {
      set_error("gemm: the decode kernel takes M <= 256 (got %d), 16-bit output, no grouped or forced split-K mode", a.M);
      return -21;
    }
    if (a.force_bn != 0 && a.force_bn != 32 && a.force_bn != 64 && a.force_bn != 128) {
      set_error("gemm: the decode kernel's tile width is 32, 64 or 128 (got %d)", a.force_bn);
      return -21;
    }
    if (!staged) {
      set_error("gemm: the decode kernel needs the 16-bit staged epilogue (N %% 8 == 0, N %% 16 == 0 with swiglu, 16-byte pitches)");
      return -21;
    }
  }
  if (gemm_skinny_ok(a)) return gemm_skinny_launch(a, stream);
  if (a.dtype == DT_BF16) return launch_typed<__nv_bfloat16>(a, stream);
  return launch_typed<__half>(a, stream);
}

}  // namespace sb
