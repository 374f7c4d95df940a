// surya_b200 — wgmma GEMM for the recognition decode step (M <= 256 rows against a large weight matrix).
//
//   C[M, Nout] = epilogue(A[M, K] @ W[N, K]^T), same contract and same bits as gemm_tn_kernel (gemm_wgmma.cu).
//
// Same roles, main loop (wg_mainloop) and epilogue helpers as gemm_tn_kernel: warp 0 = TMA producer, warps 4-11 = two
// consumer warpgroups on rows [0, 64) / [64, 128) of a 128 x BN tile, then the 8-warp staged 16-bit epilogue.  What it leaves
// out is what the decode step never uses: the grouped 1x1-conv mode, the fp32 / unaligned fallback epilogue (epilogue_chunk,
// a __noinline__ call) and the two-pass epilogue of 256-wide tiles.  Without them ptxas gives the kernel no stack frame and,
// at BN = 128, no spills (gemm_tn_kernel: 264-312 bytes of stack, 56 / 96 bytes of spill stores / loads at BN = 128), and
// the decode GEMMs run 2-23 % faster (DESIGN.md §5).  The tile order is gemm_tn_kernel's at M <= 256: tile t is
// (m-block t % m_blocks, n-block t / m_blocks), so both m-blocks of a weight tile run back to back.
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

namespace sb {

int make_tma_2d(CUtensorMap* map, int dtype, const void* base, int rows, int K, int ld, int box_rows);

namespace {

constexpr int BM = 128, BK = 64;
constexpr uint32_t A_BYTES = BM * BK * 2;

template <int BN> constexpr int dec_stages() { return BN == 32 ? 8 : BN == 64 ? 6 : 4; }
template <int BN> constexpr size_t dec_smem_bytes() {
  return dec_stages<BN>() * (A_BYTES + BN * BK * 2) + 1024 /*align slack*/ + 256 /*barriers*/ + acc_smem_bytes<BN>() +
         epi_smem_bytes<BN>();
}

}  // namespace

template <typename T, int BN>
__global__ void __launch_bounds__(384, 1)
gemm_decode_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmKParams p) {
  constexpr int STAGES = dec_stages<BN>();
  constexpr uint32_t B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  static_assert(BN <= ACC_MAX_COLS, "single-pass epilogue tiles only");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_s = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(acc_s) + acc_smem_bytes<BN>();

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
      mbar_init(&empty_bar[i], EPI_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      // weight tiles of the first ring fill do not depend on the previous kernel: request them before the wait
      int early = 0;
      if (p.w_constant && static_cast<int>(blockIdx.x) < num_tiles) {
        const int nb = static_cast<int>(blockIdx.x) / m_blocks;
        early = k_blocks < STAGES ? k_blocks : STAGES;
        for (int kb = 0; kb < early; ++kb) {
          mbar_expect_tx(&full_bar[kb], STAGE_BYTES);
          tma_load_2d(smem + kb * STAGE_BYTES + A_BYTES, &tma_b, &full_bar[kb], kb * BK, nb * BN);
        }
      }
      pdl_wait();
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mb = tile % m_blocks, nb = tile / m_blocks;
        for (int kb = 0; kb < k_blocks; ++kb) {
          uint8_t* sa = smem + s * STAGE_BYTES;
          if (!(tile == static_cast<int>(blockIdx.x) && kb < early)) {
            mbar_wait(&empty_bar[s], ph ^ 1);
            mbar_expect_tx(&full_bar[s], STAGE_BYTES);
            tma_load_2d(sa + A_BYTES, &tma_b, &full_bar[s], kb * BK, nb * BN);
          }
          tma_load_2d(sa, &tma_a, &full_bar[s], kb * BK, mb * BM);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumer warpgroups: MMA + epilogue
    pdl_wait();
    const int wg = (warp - 4) >> 2;
    const int q = warp & 3;
    const int half = wg;
    const int epi_tid = threadIdx.x - 128;
    uint8_t* stage = epi_smem + (warp - 4) * EPI_STAGE_BYTES;
    float* sbias = reinterpret_cast<float*>(epi_smem + EPI_WARPS * EPI_STAGE_BYTES);
    float* srs = sbias + BN;
    int s = 0;
    uint32_t ph = 0;
    const AccRow acc(acc_s, q * 32 + lane, BN);
    float d[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mb = tile % m_blocks, nb = tile / m_blocks;
      asm volatile("bar.sync 1, 256;" ::: "memory");   // all epilogue warps are done with the previous tile's bias
      epilogue_stage_bias<BN>(p, sbias, epi_tid, nb * BN);
      if (p.rowscale && epi_tid < BM) srs[epi_tid] = mb * BM + epi_tid < p.M ? __ldg(p.rowscale + mb * BM + epi_tid) : 0.f;
      asm volatile("bar.sync 1, 256;" ::: "memory");
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
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free (previous tile read it)
      wg_acc_store<BN / 8>(d, 0, acc_s + wg * 64 * BN, BN, warp & 3, lane);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const float rs = (p.ssq_inline || p.rowscale) ? srs[q * 32 + lane] : 1.0f;
      if (!p.am_val || p.store_c)
        epilogue_tile_rt<T>(acc, p, stage, sbias, lane, half, [&](int r) { return row0 + r < p.M ? row0 + r : -1; }, nb * BN,
                            rs, BN / 32);
      if (p.am_val)
        epilogue_tile_argmax<T, BN>(acc, p, epi_smem, sbias, lane, half, q, row0 + lane < p.M ? row0 + lane : -1, nb * BN, nb,
                                    rs);
    }
  }
}

// ----------------------------------------------------------------------------------- host side
namespace {

template <typename T, int BN>
int launch_decode(const GemmArgs& a, cudaStream_t stream) {
  constexpr size_t SMEM = dec_smem_bytes<BN>();
  static_assert(SMEM <= 227 * 1024, "GEMM tile does not fit in shared memory");
  auto kern = gemm_decode_kernel<T, BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(smem=%zu) failed: %s", SMEM, cudaGetErrorString(e));
      return -10;
    }
    attr_set = true;
  }
  CUtensorMap ma, mb;
  int rc = make_tma_2d(&ma, a.dtype, a.A, a.M, a.K, a.lda, BM);
  if (rc) return rc;
  rc = make_tma_2d(&mb, a.dtype, a.W, a.N, a.K, a.ldw, BN);
  if (rc) return rc;
  GemmKParams p{};
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.C = a.C; p.ldc = a.ldc;
  p.bias = a.bias;
  p.residual = a.residual; p.ldr = a.ldr;
  p.act = a.act; p.swiglu = a.swiglu; p.out_f32 = 0;
  p.group_m = 1; p.group_k = 0;
  p.w_constant = a.w_constant;
  p.rowscale = a.rowscale;
  p.ssq_inline = a.ssq_inline;
  p.ssq_eps = a.ssq_eps;
  p.ssq_inv_k = 1.0f / static_cast<float>(a.ssq_k > 0 ? a.ssq_k : a.K);
  p.am_val = a.am_val; p.am_idx = a.am_idx; p.am_sum = a.am_sum; p.am_ld = a.am_ld; p.store_c = a.store_c;
  const int tiles = ((a.M + BM - 1) / BM) * ((a.N + BN - 1) / BN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  if (launch_pdl(kern, dim3(grid), dim3(384), SMEM, stream, ma, mb, p) != cudaSuccess) { /* reported by launch_ok */ }
  return launch_ok();
}

// Tile width per decode shape, measured on H100 (DESIGN.md §5): 32 for the 1280- / 1920-wide qkv and o projections, 128 for
// gate/up; the argmax epilogue keeps gemm_argmax_tile's width, which sized the caller's partial buffers.
int decode_bn(const GemmArgs& a) {
  if (a.force_bn) return a.force_bn;
  if (a.am_val) return gemm_argmax_tile(a.M, a.N);
  return a.N >= 4096 ? 128 : 32;
}

}  // namespace

int gemm_decode_check(const GemmArgs& a) {
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
  const bool v2 = a.ldc % 8 == 0 && (!a.residual || a.ldr % 8 == 0) &&
                  (a.swiglu ? ((a.act == ACT_SILU || a.act == ACT_GELU_TANH) && a.N % 16 == 0) : a.N % 8 == 0);
  if (!v2) {
    set_error("gemm: the decode kernel needs the 16-bit staged epilogue (N %% 8 == 0, N %% 16 == 0 with swiglu, 16-byte pitches)");
    return -21;
  }
  return 0;
}

int gemm_decode_launch(const GemmArgs& a, cudaStream_t stream) {
  const int bn = decode_bn(a);
  if (a.dtype == DT_BF16) {
    if (bn == 32) return launch_decode<__nv_bfloat16, 32>(a, stream);
    if (bn == 64) return launch_decode<__nv_bfloat16, 64>(a, stream);
    return launch_decode<__nv_bfloat16, 128>(a, stream);
  }
  if (bn == 32) return launch_decode<__half, 32>(a, stream);
  if (bn == 64) return launch_decode<__half, 64>(a, stream);
  return launch_decode<__half, 128>(a, stream);
}

}  // namespace sb
