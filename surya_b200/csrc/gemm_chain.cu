// surya_b200 — a CHAIN of dependent skinny GEMMs in ONE persistent launch (recognition decode steps, M <= 256).
//
//   for phase in phases:   C_p[M, Nout_p] = epilogue_p(A_p[M, K_p] @ W_p[N_p, K_p]^T)        A_{p+1} may be C_p
//
// Why: inside the decode graph a 256-row GEMM spends a large share of its time on things other than data movement — launch,
// block scheduling behind the previous kernel's 200 KB CTAs, barrier / descriptor set-up, pipeline ramp, drain and the
// completion -> dependent-launch hand-over.  A decoder layer is a chain  o_proj -> gate_up -> down ->
// next layer's qkv  where each GEMM needs the complete rows of its predecessor, so the kernels cannot be fused tile-wise; they
// CAN share one launch: one CTA per SM stays resident, set up once, and cross a grid-wide barrier (one global counter, release /
// acquire) between phases.  Numerics are those of gemm_tn_kernel with the same tile width (same k order, same epilogue).
//
// Layout of a CTA (384 threads) is gemm_tn_kernel's: warp 0 = TMA producer, warps 4-11 = two consumer warpgroups (wgmma, the
// in-kernel sum of squares of the folded RMSNorm, epilogue).  Differences:
//   * the tile width BN is a per-phase RUNTIME value (32 / 64 / 96 / 128, dispatched to a compile-time main loop): one 4-stage
//     ring of 32 KB slots (16 KB of A + up to 16 KB of W) serves every phase, the accumulator tile has 128-column rows;
//   * the ring's barriers keep their phase across phases of the chain, so no barrier is re-initialised;
//   * grid barrier: bar[0] counts arrivals (monotonic inside a launch), bar[1] counts exits; the last CTA to leave resets both.
//     Every CTA is resident by construction (grid <= SM count, 1 CTA / SM); a spin that exceeds 2 s raises bar[2] and moves on
//     so that a scheduling surprise produces a loud error instead of a hung GPU.
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

namespace sb {

int make_tma_2d(CUtensorMap* map, int dtype, const void* base, int rows, int K, int ld, int box_rows);

constexpr int CH_MAX_PHASES = 4;
constexpr int CH_STAGES = 4;
constexpr int CH_BN_MAX = 128;
constexpr uint32_t CH_A_BYTES = 128 * 64 * 2;
constexpr uint32_t CH_SLOT_BYTES = CH_A_BYTES + CH_BN_MAX * 64 * 2;          // 32 KB

struct ChainPhase {
  int M, N, K, bn;
  void* C; int ldc;
  const float* bias;
  const void* residual; int ldr;
  int act, swiglu;
  int ssq_inline; float ssq_eps, ssq_inv_k;
};
struct ChainParams {
  int n_phases;
  ChainPhase ph[CH_MAX_PHASES];
  unsigned int* bar;       // [0] arrivals, [1] exits, [2] timeout flag
  int group_m;
  unsigned long long* dbg; // optional timeline of CTA 0 (globaltimer ns): [8*phase + {0 start, 1 first tile data landed,
                           // 3 accumulator ready, 4 epilogue done, 5 barrier passed}]
};
struct ChainMaps { CUtensorMap a[CH_MAX_PHASES]; CUtensorMap b[CH_MAX_PHASES]; };

__device__ __forceinline__ void ch_tile_coords(int tile, int m_blocks, int n_blocks, int gm, int& mb, int& nb) {
  int per_group = gm * n_blocks;
  int g = tile / per_group;
  int first = g * gm;
  int gsz = min(m_blocks - first, gm);
  int r = tile - g * per_group;
  mb = first + r % gsz;
  nb = r / gsz;
}

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// All threads of the CTA call it.  Orders: this CTA's global writes (generic proxy) -> every other CTA's reads after the
// barrier, including TMA (async proxy) reads issued by thread 0 / warp 0.
__device__ __forceinline__ void chain_grid_sync(unsigned int* bar, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    asm volatile("fence.proxy.async;" ::: "memory");
    red_release_add(bar, 1u);
    const unsigned long long t0 = globaltimer_ns();
    while (ld_acquire_u32(bar) < target) {
      if (globaltimer_ns() - t0 > 2000000000ull) {      // 2 s: something is badly wrong; fail loudly instead of hanging
        bar[2] = 1u;
        break;
      }
    }
    asm volatile("fence.proxy.async;" ::: "memory");
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(384, 1) gemm_chain_kernel(const __grid_constant__ ChainMaps maps, const ChainParams p) {
  constexpr int BM = 128, BK = 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + CH_STAGES * CH_SLOT_BYTES);
  uint64_t* empty_bar = full_bar + CH_STAGES;
  float* acc_s = reinterpret_cast<float*>(smem + CH_STAGES * CH_SLOT_BYTES + 256);      // [128][CH_BN_MAX] accumulator tile
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(acc_s) + acc_smem_bytes<CH_BN_MAX>();

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_trigger();

  if (warp == 0 && lane == 0) {
    for (int i = 0; i < p.n_phases; ++i) {
      tma_prefetch_desc(&maps.a[i]);
      tma_prefetch_desc(&maps.b[i]);
    }
    for (int i = 0; i < CH_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], EPI_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  // pipeline state, carried across phases by each role
  int s = 0;            // ring slot
  uint32_t ph = 0;      // and its phase bit
  float d[CH_BN_MAX / 2];

  auto stamp = [&](int slot) {
    if (p.dbg && blockIdx.x == 0) p.dbg[slot] = globaltimer_ns();
  };
  for (int pi = 0; pi < p.n_phases; ++pi) {
    const ChainPhase& P = p.ph[pi];
    if (threadIdx.x == 0) stamp(8 * pi + 0);
    const int bn = P.bn;
    const int m_blocks = (P.M + BM - 1) / BM;
    const int n_blocks = (P.N + bn - 1) / bn;
    const int k_blocks = (P.K + BK - 1) / BK;
    const int num_tiles = m_blocks * n_blocks;
    const uint32_t stage_bytes = CH_A_BYTES + static_cast<uint32_t>(bn) * BK * 2;

    if (warp == 0) {
      // ---------------------------------------------------------------- TMA producer
      if (lane == 0) {
        int early = 0;
        if (pi == 0) {
          // weights do not depend on the previous kernel: request the first tile's W k-blocks before the dependency wait
          if (static_cast<int>(blockIdx.x) < num_tiles) {
            int mb, nb;
            ch_tile_coords(blockIdx.x, m_blocks, n_blocks, p.group_m, mb, nb);
            early = k_blocks < CH_STAGES ? k_blocks : CH_STAGES;
            for (int kb = 0; kb < early; ++kb) {
              mbar_expect_tx(&full_bar[kb], stage_bytes);
              tma_load_2d(smem + kb * CH_SLOT_BYTES + CH_A_BYTES, &maps.b[0], &full_bar[kb], kb * BK, nb * bn);
            }
          }
          pdl_wait();
        }
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          int mb, nb;
          ch_tile_coords(tile, m_blocks, n_blocks, p.group_m, mb, nb);
          for (int kb = 0; kb < k_blocks; ++kb) {
            uint8_t* sa = smem + s * CH_SLOT_BYTES;
            if (pi == 0 && tile == static_cast<int>(blockIdx.x) && kb < early) {
              tma_load_2d(sa, &maps.a[0], &full_bar[s], kb * BK, mb * BM);
            } else {
              mbar_wait(&empty_bar[s], ph ^ 1);
              mbar_expect_tx(&full_bar[s], stage_bytes);
              tma_load_2d(sa, &maps.a[pi], &full_bar[s], kb * BK, mb * BM);
              tma_load_2d(sa + CH_A_BYTES, &maps.b[pi], &full_bar[s], kb * BK, nb * bn);
            }
            if (++s == CH_STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    } else if (warp >= 4) {
      // ---------------------------------------------------------------- consumer warpgroups: MMA + epilogue
      if (pi == 0) pdl_wait();
      const int wg = (warp - 4) >> 2;
      const int q = warp & 3;
      const int half = wg;
      const int epi_tid = threadIdx.x - 128;
      uint8_t* stage = epi_smem + (warp - 4) * EPI_STAGE_BYTES;
      float* sbias = reinterpret_cast<float*>(epi_smem + EPI_WARPS * EPI_STAGE_BYTES);
      float* srs = sbias + CH_BN_MAX;
      const AccRow acc(acc_s, q * 32 + lane, CH_BN_MAX);
      GemmKParams g{};
      g.M = P.M; g.N = P.N; g.K = P.K; g.C = P.C; g.ldc = P.ldc; g.bias = P.bias; g.residual = P.residual; g.ldr = P.ldr;
      g.act = P.act; g.swiglu = P.swiglu;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mb, nb;
        ch_tile_coords(tile, m_blocks, n_blocks, p.group_m, mb, nb);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        epilogue_stage_bias_rt(g, sbias, epi_tid, nb * bn, bn);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        // main loop; when the phase folds an RMSNorm, the rows' sum of squares is taken from the A tiles on the way
        float ssq = 0.f;
        const bool first = tile == static_cast<int>(blockIdx.x);
        bool landed = false;
        auto on_stage = [&](const uint8_t* slot) {
          if (first && !landed && epi_tid == 0) stamp(8 * pi + 1);
          landed = true;
          if (P.ssq_inline) ssq = ssq_stage<T>(slot, epi_tid, ssq);
        };
        switch (bn) {
          case 32: wg_mainloop<T, 32, BK>(d, smem, CH_SLOT_BYTES, CH_A_BYTES, CH_STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane, on_stage); break;
          case 64: wg_mainloop<T, 64, BK>(d, smem, CH_SLOT_BYTES, CH_A_BYTES, CH_STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane, on_stage); break;
          case 96: wg_mainloop<T, 96, BK>(d, smem, CH_SLOT_BYTES, CH_A_BYTES, CH_STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane, on_stage); break;
          default: wg_mainloop<T, 128, BK>(d, smem, CH_SLOT_BYTES, CH_A_BYTES, CH_STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane, on_stage); break;
        }
        if (P.ssq_inline) {
          const float tot = ssq + __shfl_xor_sync(0xffffffffu, ssq, 1);
          if ((epi_tid & 1) == 0) srs[epi_tid >> 1] = rsqrtf(tot * P.ssq_inv_k + P.ssq_eps);
        }
        if (epi_tid == 0 && first) stamp(8 * pi + 3);
        asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free
        float* dst = acc_s + wg * 64 * CH_BN_MAX;
        switch (bn) {
          case 32: wg_acc_store<4>(d, 0, dst, CH_BN_MAX, warp & 3, lane); break;
          case 64: wg_acc_store<8>(d, 0, dst, CH_BN_MAX, warp & 3, lane); break;
          case 96: wg_acc_store<12>(d, 0, dst, CH_BN_MAX, warp & 3, lane); break;
          default: wg_acc_store<16>(d, 0, dst, CH_BN_MAX, warp & 3, lane); break;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const int row0 = mb * BM + q * 32;
        const float rs = P.ssq_inline ? srs[q * 32 + lane] : 1.0f;
        epilogue_tile_rt<T>(acc, g, stage, sbias, lane, half, [&](int r) { return row0 + r < P.M ? row0 + r : -1; }, nb * bn, rs,
                            bn / 32);
        if (epi_tid == 0 && first) stamp(8 * pi + 4);
      }
    }
    if (pi + 1 < p.n_phases) chain_grid_sync(p.bar, static_cast<unsigned int>(pi + 1) * gridDim.x);
    if (threadIdx.x == 0) stamp(8 * pi + 5);
  }

  if (threadIdx.x == 0 && p.n_phases > 1) {
    __threadfence();
    const unsigned int old = atomicAdd(&p.bar[1], 1u);
    if (old == gridDim.x - 1) {       // every CTA is past its last barrier: re-arm the counters for the next launch
      p.bar[0] = 0u;
      p.bar[1] = 0u;
      __threadfence();
    }
  }
}

// ----------------------------------------------------------------------------------- host side
int gemm_chain_bn(int M, int N, int swiglu) {
  // widest single wave: the smallest tile width whose tile count still fits the SM count (more CTAs stream the weights);
  // past that, the widest tile
  const int sms = num_sms();
  const int m_blocks = (M + 127) / 128;
  const int cands[4] = {32, 64, 96, 128};
  for (int c : cands) {
    (void)swiglu;                       // every candidate is a multiple of 32, which the SwiGLU epilogue needs
    if (m_blocks * ((N + c - 1) / c) <= sms) return c;
  }
  return 128;
}

template <typename T>
static int chain_launch_typed(const GemmArgs* ph, int n, unsigned int* bar, cudaStream_t stream) {
  constexpr size_t SMEM = CH_STAGES * CH_SLOT_BYTES + 1024 + 256 + acc_smem_bytes<CH_BN_MAX>() + epi_smem_bytes<CH_BN_MAX>();
  static_assert(SMEM <= 227 * 1024, "gemm_chain does not fit in shared memory");
  auto kern = gemm_chain_kernel<T>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    if (e != cudaSuccess) { set_error("gemm_chain: cudaFuncSetAttribute(smem=%zu) failed: %s", SMEM, cudaGetErrorString(e)); return -10; }
    attr_set = true;
  }
  ChainMaps maps;
  ChainParams p{};
  p.n_phases = n;
  p.bar = bar;
  p.group_m = 8;
  p.dbg = ph[0].dbg;
  for (int i = 0; i < n; ++i) {
    const GemmArgs& a = ph[i];
    const int bn = a.force_bn > 0 ? a.force_bn : gemm_chain_bn(a.M, a.N, a.swiglu);
    if (bn != 32 && bn != 64 && bn != 96 && bn != 128) { set_error("gemm_chain: tile width %d not in {32, 64, 96, 128}", bn); return -12; }
    int rc = make_tma_2d(&maps.a[i], a.dtype, a.A, a.M, a.K, a.lda, 128);
    if (rc) return rc;
    rc = make_tma_2d(&maps.b[i], a.dtype, a.W, a.N, a.K, a.ldw, bn);
    if (rc) return rc;
    ChainPhase& q = p.ph[i];
    q.M = a.M; q.N = a.N; q.K = a.K; q.bn = bn;
    q.C = a.C; q.ldc = a.ldc; q.bias = a.bias; q.residual = a.residual; q.ldr = a.ldr;
    q.act = a.act; q.swiglu = a.swiglu;
    q.ssq_inline = a.ssq_inline; q.ssq_eps = a.ssq_eps;
    q.ssq_inv_k = 1.0f / static_cast<float>(a.ssq_k > 0 ? a.ssq_k : a.K);
  }
  if (launch_pdl(kern, dim3(num_sms()), dim3(384), SMEM, stream, maps, p) != cudaSuccess) { /* reported by launch_ok */ }
  return launch_ok();
}

// Launch phases[0..n) as one persistent kernel.  Every phase must satisfy the staged 16-bit epilogue's alignment rules; rowscale /
// argmax epilogues / grouped / fp32 outputs are not available here.  bar: 3 zero-initialised uint32 owned by the caller.
int gemm_chain_launch(const GemmArgs* phases, int n, unsigned int* bar, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n > CH_MAX_PHASES) { set_error("gemm_chain: at most %d phases", CH_MAX_PHASES); return -11; }
  if (!bar) { set_error("gemm_chain: null barrier counters"); return -11; }
  for (int i = 0; i < n; ++i) {
    const GemmArgs& a = phases[i];
    if (a.dtype != phases[0].dtype) { set_error("gemm_chain: mixed dtypes"); return -13; }
    if (a.M <= 0 || a.N <= 0 || a.K <= 0) { set_error("gemm_chain: empty phase %d", i); return -13; }
    const bool v2 = !a.out_f32 && a.ldc % 8 == 0 && (!a.residual || a.ldr % 8 == 0) &&
                    (a.swiglu ? ((a.act == ACT_SILU || a.act == ACT_GELU_TANH) && a.N % 16 == 0) : a.N % 8 == 0);
    if (!v2 || a.group_k || a.rowscale || a.am_val) {
      set_error("gemm_chain: phase %d needs the plain staged 16-bit epilogue (no fp32 out / grouped / rowscale / argmax)", i);
      return -14;
    }
  }
  return phases[0].dtype == DT_BF16 ? chain_launch_typed<__nv_bfloat16>(phases, n, bar, stream)
                                    : chain_launch_typed<__half>(phases, n, bar, stream);
}

}  // namespace sb
