// surya_b200 — split-K wgmma GEMM for skinny problems (decode steps: M <= 256 rows against a large weight matrix).
//
//   C[M, Nout] = epilogue(A[M, K] @ W[N, K]^T), same contract as gemm_tn_kernel (gemm_wgmma.cu).
//
// Why: with M = 256 the plain kernel needs many small N tiles to occupy the SMs, and every CTA re-reads a whole 128-row slab
// of A (80 % of its bytes at BN = 32) from L2 — the launch is bound by L2 throughput on activation re-reads
// (DESIGN.md §4).  Here a thread-block CLUSTER of PK CTAs shares one 128 x BN output tile and splits K, so each CTA reads
// only K/PK of A and W.  The PK fp32 partial tiles are combined with a reduce-scatter through distributed shared memory:
// rank j owns a slice of the tile's columns, every rank pushes its partials for that slice into j's receive buffer
// (st.shared::cluster), one cluster barrier, then j sums the PK partials in rank order (deterministic) and runs the usual
// epilogue (bias -> round -> act -> round -> (+residual | SwiGLU product) -> round) on its slice.
//
// Roles per CTA (384 threads): warp 0 = TMA producer (weight tiles requested before griddepcontrol.wait), warps 4-11 = two
// consumer warpgroups (wgmma on rows [0, 64) / [64, 128), then the scatter of their fragments); warps 4-7 run the final epilogue
// (one per 32-row quarter).
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

namespace sb {

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f2(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

constexpr int SK_THREADS = 384;
constexpr int SK_MAX_PK = 8;

// first 8-column unit owned by rank j when n_units units are dealt to pk ranks
__device__ __host__ __forceinline__ int sk_first_unit(int j, int n_units, int pk) { return (j * n_units) / pk; }

template <typename T, int BN>
__global__ void __launch_bounds__(SK_THREADS, 1)
gemm_splitk_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmKParams p,
                   int pk, int rstride, int STAGES) {
  constexpr int BM = 128, BK = 64;
  constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int N_UNITS = BN / 8;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  // STAGES (<= 8) is a launch parameter: as many pipeline stages as fit beside the receive buffer
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + 8;
  float* recv = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);   // [pk][128][rstride]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = static_cast<int>(cluster_ctarank());        // == blockIdx.x (grid.x == cluster.x == pk)
  const int nb = blockIdx.y, mb = blockIdx.z;
  pdl_trigger();
  const int k_blocks = (p.K + BK - 1) / BK;
  const int kb0 = (rank * k_blocks) / pk, kb1 = ((rank + 1) * k_blocks) / pk;
  const int my_kb = kb1 - kb0;

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
  // Phase 1 of the cluster barrier = "every CTA of the cluster is running" (required before touching a peer's shared
  // memory); arrive now, wait only right before the first remote store so the wait hides behind the main loop.
  cluster_arrive_relaxed();

  if (warp == 0) {
    if (lane == 0) {
      int early = 0;
      if (p.w_constant) {
        early = my_kb < STAGES ? my_kb : STAGES;
        for (int i = 0; i < early; ++i) {
          mbar_expect_tx(&full_bar[i], STAGE_BYTES);
          tma_load_2d(smem + i * STAGE_BYTES + A_BYTES, &tma_b, &full_bar[i], (kb0 + i) * BK, nb * BN);
        }
      }
      pdl_wait();
      int s = 0;
      uint32_t ph = 0;
      for (int i = 0; i < my_kb; ++i) {
        uint8_t* sa = smem + s * STAGE_BYTES;
        if (i < early) {
          tma_load_2d(sa, &tma_a, &full_bar[s], (kb0 + i) * BK, mb * BM);
        } else {
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], STAGE_BYTES);
          tma_load_2d(sa, &tma_a, &full_bar[s], (kb0 + i) * BK, mb * BM);
          tma_load_2d(sa + A_BYTES, &tma_b, &full_bar[s], (kb0 + i) * BK, nb * BN);
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ---------------------------------------------------------------- consumers: partial tile, then scatter it
    pdl_wait();
    const int wg = (warp - 4) >> 2;
    float d[BN / 2];
    if (my_kb > 0) {
      int s = 0;
      uint32_t ph = 0;
      wg_mainloop<T, BN, BK>(d, smem, STAGE_BYTES, A_BYTES, STAGES, full_bar, empty_bar, s, ph, my_kb, wg, lane,
                             [](const uint8_t*) {});
    } else {
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) d[j] = 0.f;
    }
    const uint32_t recv_local = smem_u32(recv);
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);       // fragment rows r0 and r0 + 8 of the tile
    const int c = (lane & 3) * 2;
    cluster_wait();
#pragma unroll
    for (int unit = 0; unit < N_UNITS; ++unit) {                  // n8 block == 8-column unit
      int owner = 0;                                              // largest j with first_unit(j) <= unit
      while (owner + 1 < pk && sk_first_unit(owner + 1, N_UNITS, pk) <= unit) ++owner;
      const int local_col = (unit - sk_first_unit(owner, N_UNITS, pk)) * 8 + c;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t off = ((static_cast<uint32_t>(rank) * BM + r0 + 8 * h) * rstride + local_col) * 4u;
        st_cluster_f2(mapa_shared(recv_local + off, static_cast<uint32_t>(owner)), d[4 * unit + 2 * h], d[4 * unit + 2 * h + 1]);
      }
    }
  }

  __syncwarp();
  if (warp < 4) cluster_wait();     // producer and idle warps complete phase 1 here
  // every partial of this cluster's tile is in its owner's receive buffer after this barrier
  cluster_sync_all();

  if (warp >= 4 && warp < 8) {
    const int q = warp & 3;
    const int row_t = q * 32 + lane;
    const int row = mb * BM + row_t;
    const int u0 = sk_first_unit(rank, N_UNITS, pk), u1 = sk_first_unit(rank + 1, N_UNITS, pk);
    if (row < p.M) {
      for (int u = u0; u < u1; ++u) {
        const int col0 = nb * BN + u * 8;
        if (col0 >= p.N) break;
        const int lc = (u - u0) * 8;
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = 0.f;
        for (int r = 0; r < pk; ++r) {             // fixed order: deterministic sum
          const float4 a = *reinterpret_cast<const float4*>(&recv[(static_cast<size_t>(r) * BM + row_t) * rstride + lc]);
          const float4 b = *reinterpret_cast<const float4*>(&recv[(static_cast<size_t>(r) * BM + row_t) * rstride + lc + 4]);
          x[0] += a.x; x[1] += a.y; x[2] += a.z; x[3] += a.w;
          x[4] += b.x; x[5] += b.y; x[6] += b.z; x[7] += b.w;
        }
        if (p.bias) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (col0 + j < p.N) x[j] += __ldg(p.bias + col0 + j);
        }
        if (p.swiglu) {
          T* crow = reinterpret_cast<T*>(p.C) + static_cast<size_t>(row) * p.ldc;
          const int oc0 = col0 >> 1, n_out = p.N >> 1;
          T o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float g = rnd<T>(x[2 * i]);
            const float uu = rnd<T>(x[2 * i + 1]);
            const float sact = rnd<T>(apply_act(g, p.act));
            o[i] = from_f<T>(sact * uu);
          }
          if ((p.ldc & 3) == 0 && oc0 + 4 <= n_out) {
            *reinterpret_cast<uint2*>(crow + oc0) = *reinterpret_cast<const uint2*>(o);
          } else {
            for (int i = 0; i < 4; ++i)
              if (oc0 + i < n_out) crow[oc0 + i] = o[i];
          }
        } else {
          T* crow = reinterpret_cast<T*>(p.C) + static_cast<size_t>(row) * p.ldc;
          const T* rrow = p.residual ? reinterpret_cast<const T*>(p.residual) + static_cast<size_t>(row) * p.ldr : nullptr;
          const bool full = (col0 + 8 <= p.N) && (p.ldc & 7) == 0 && (!rrow || (p.ldr & 7) == 0);
          T rr[8];
          if (rrow) {
            if (full) *reinterpret_cast<uint4*>(rr) = *reinterpret_cast<const uint4*>(rrow + col0);
            else
              for (int j = 0; j < 8; ++j) rr[j] = (col0 + j < p.N) ? rrow[col0 + j] : from_f<T>(0.f);
          }
          T o[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float y = rnd<T>(x[j]);
            if (p.act != ACT_NONE) y = rnd<T>(apply_act(y, p.act));
            if (rrow) y = y + to_f<T>(rr[j]);
            o[j] = from_f<T>(y);
          }
          if (full) *reinterpret_cast<uint4*>(crow + col0) = *reinterpret_cast<const uint4*>(o);
          else
            for (int j = 0; j < 8; ++j)
              if (col0 + j < p.N) crow[col0 + j] = o[j];
        }
      }
    }
  }

}

static int sk_rstride(int bn, int pk) { return ((bn / 8 + pk - 1) / pk) * 8 + 4; }   // +4 floats: rows land in different banks
static size_t sk_recv_bytes(int bn, int pk) { return static_cast<size_t>(pk) * 128 * sk_rstride(bn, pk) * 4; }
static int sk_stages(int bn, int pk, int k_blocks) {
  const size_t stage = 128 * 64 * 2 + static_cast<size_t>(bn) * 64 * 2;
  const size_t room = 227 * 1024 - 1024 - 256 - sk_recv_bytes(bn, pk);
  int st = static_cast<int>(room / stage);
  const int need = (k_blocks + pk - 1) / pk;
  if (st > need) st = need;
  if (st > 8) st = 8;
  return st;
}

template <typename T, int BN>
static int launch_splitk(const GemmArgs& a, int pk, cudaStream_t stream) {
  const int rstride = sk_rstride(BN, pk);
  const int stages = sk_stages(BN, pk, (a.K + 63) / 64);
  if (stages < 2) { set_error("split-K GEMM: no room for the pipeline (BN=%d pk=%d)", BN, pk); return -15; }
  const size_t smem = static_cast<size_t>(stages) * (128 * 64 * 2 + BN * 64 * 2) + 1024 + 256 + sk_recv_bytes(BN, pk);
  auto kern = gemm_splitk_kernel<T, BN>;
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(smem=%zu) failed: %s", smem, cudaGetErrorString(e)); return -10; }
    attr_smem = smem;
  }
  CUtensorMap ma, mb;
  int rc = make_tma_2d(&ma, a.dtype, a.A, a.M, a.K, a.lda, 128);
  if (rc) return rc;
  rc = make_tma_2d(&mb, a.dtype, a.W, a.N, a.K, a.ldw, BN);
  if (rc) return rc;
  const GemmKParams p = gemm_kparams(a);
  const int m_blocks = (a.M + 127) / 128, n_blocks = (a.N + BN - 1) / BN;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pk, n_blocks, m_blocks);
  cfg.blockDim = dim3(SK_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = pk; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  cudaLaunchKernelEx(&cfg, kern, ma, mb, p, pk, rstride, stages);
  return launch_ok();
}

// Chooses a split for skinny GEMMs; returns 0 when the plain kernel should be used.  A cluster launch costs more than a plain
// one and large clusters are placed less freely, so the split is kept to <= 3 CTAs and used only when the per-CTA k-chain is
// long (the decoder's down projections, K = 3424 / 4096).  Everything else stays on the plain kernel.
int splitk_plan(const GemmArgs& a, int* bn_out) {
  if (a.out_f32 || a.group_k || a.M > 256 || a.swiglu) return 0;
  const int k_blocks = (a.K + 63) / 64;
  if (k_blocks < 40 || a.N < 64) return 0;
  const int sms = num_sms();
  const int tiles = ((a.M + 127) / 128) * ((a.N + 63) / 64);
  int pk = 3;
  while (pk >= 2 && tiles * pk > sms) --pk;
  if (pk < 2) return 0;
  *bn_out = 64;
  return pk;
}

int gemm_splitk_launch(const GemmArgs& a, int pk, int bn, cudaStream_t stream) {
  if (pk < 1 || pk > SK_MAX_PK) { set_error("split-K factor %d out of range", pk); return -16; }   // pk = 1: cluster of one (benchmarks)
  if (a.out_f32 || a.group_k) { set_error("split-K GEMM: fp32 output / grouped mode not supported"); return -17; }
  if (a.dtype == DT_BF16) {
    if (bn == 128) return launch_splitk<__nv_bfloat16, 128>(a, pk, stream);
    if (bn == 64) return launch_splitk<__nv_bfloat16, 64>(a, pk, stream);
  } else if (a.dtype == DT_F16) {
    if (bn == 128) return launch_splitk<__half, 128>(a, pk, stream);
    if (bn == 64) return launch_splitk<__half, 64>(a, pk, stream);
  }
  set_error("split-K GEMM: unsupported dtype / BN (%d, %d)", a.dtype, bn);
  return -18;
}

}  // namespace sb
