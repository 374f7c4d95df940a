// surya_b200 — GEMM for M <= 16 rows (ADETR layout / table decode steps at batch 16, tiny recognition batches).
//
//   C[M, Nout] = epilogue(A[M, K] @ W[N, K]^T), same contract and rounding points as gemm_tn_kernel.
//
// Why: at 16 rows the wgmma kernel's fixed costs (mbarrier / tensor-map set-up, a 128-row MMA tile that is 7/8 padding)
// dwarf the work: a decode step of the layout decoder is 48 such GEMMs.  This kernel is the light-weight path: weights stream straight from HBM into
// registers (16 B per lane, fully coalesced), the 16 activation rows come from L2, and the products run on mma.sync
// m16n8k16 — M = 16 is exactly one MMA tile, so no tensor-core lane is padding.
//   * CTA = 8 warps = one group of 8 output columns; the warps split K eight ways and meet in shared memory in warp order
//     (deterministic); N / 8 CTAs stream the weight matrix together (128 CTAs for a 1024-wide layer, 1024 for the 8192-wide MLP).
//   * k is consumed in blocks of 32: a lane's 16 contiguous bytes of W (and of each of its two A rows) feed two MMAs through a
//     fixed permutation of the k index — legal because both operands use the same permutation.
//   * epilogue: bias -> round -> act -> round -> (+residual | GLU product) -> round, identical to gemm_epilogue.cuh.
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

namespace sb {

struct SkinnyParams {
  const void* A; int lda;
  const void* W; int ldw;
  void* C; int ldc;
  int M, N, K;
  const float* bias;
  const void* residual; int ldr;
  int act, swiglu;
  int w_constant;   // W is never written by a preceding kernel: its first loads may precede the dependency wait
};

template <typename T> struct MmaSkinny;
template <> struct MmaSkinny<__nv_bfloat16> {
  static __device__ __forceinline__ void run(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
};
template <> struct MmaSkinny<__half> {
  static __device__ __forceinline__ void run(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
};

constexpr int SK_WARPS = 8;
constexpr int SK_UNROLL = 4;     // 32-wide k blocks whose loads are issued before the first MMA

template <typename T>
__global__ void __launch_bounds__(SK_WARPS * 32) gemm_skinny_kernel(const SkinnyParams p) {
  __shared__ float part[SK_WARPS][16 * 8];
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * 8;
  const int r = lane >> 2, q = lane & 3;          // fragment row / k quad
  const int n = n0 + r;                           // this lane's weight row (B fragment column)
  const bool n_ok = n < p.N;
  // K split: contiguous runs of 32-wide blocks per warp
  const int kblocks = p.K / 32;
  const int kb0 = (warp * kblocks) / SK_WARPS, kb1 = ((warp + 1) * kblocks) / SK_WARPS;
  const T* Wrow = reinterpret_cast<const T*>(p.W) + static_cast<size_t>(n_ok ? n : 0) * p.ldw + q * 8;
  const T* A0 = reinterpret_cast<const T*>(p.A) + static_cast<size_t>(r < p.M ? r : 0) * p.lda + q * 8;
  const T* A1 = reinterpret_cast<const T*>(p.A) + static_cast<size_t>(r + 8 < p.M ? r + 8 : 0) * p.lda + q * 8;
  const bool a0_ok = r < p.M, a1_ok = r + 8 < p.M;
  float c[4] = {0.f, 0.f, 0.f, 0.f};
  // constant weights (w_constant) do not depend on the previous kernel: their first batch of loads goes out before the
  // dependency wait.  Any other W may still be being written by the previous kernel, so it is read after the wait.
  if (!p.w_constant) pdl_wait();
  uint4 w[SK_UNROLL];
  int kb = kb0;
#pragma unroll
  for (int u = 0; u < SK_UNROLL; ++u)
    w[u] = (n_ok && kb + u < kb1) ? *reinterpret_cast<const uint4*>(Wrow + static_cast<size_t>(kb + u) * 32) : make_uint4(0u, 0u, 0u, 0u);
  if (p.w_constant) pdl_wait();
  for (; kb < kb1; kb += SK_UNROLL) {
    uint4 a0[SK_UNROLL], a1[SK_UNROLL];
#pragma unroll
    for (int u = 0; u < SK_UNROLL; ++u) {
      const bool ok = kb + u < kb1;
      a0[u] = (ok && a0_ok) ? *reinterpret_cast<const uint4*>(A0 + static_cast<size_t>(kb + u) * 32) : make_uint4(0u, 0u, 0u, 0u);
      a1[u] = (ok && a1_ok) ? *reinterpret_cast<const uint4*>(A1 + static_cast<size_t>(kb + u) * 32) : make_uint4(0u, 0u, 0u, 0u);
    }
    uint4 wn[SK_UNROLL];
#pragma unroll
    for (int u = 0; u < SK_UNROLL; ++u)       // next batch of weights in flight while this one multiplies
      wn[u] = (n_ok && kb + SK_UNROLL + u < kb1) ? *reinterpret_cast<const uint4*>(Wrow + static_cast<size_t>(kb + SK_UNROLL + u) * 32)
                                                  : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int u = 0; u < SK_UNROLL; ++u) {
      if (kb + u >= kb1) break;
      // 8 consecutive k per lane: (x, y) feed the first MMA's k slots {2q, 2q+1 | 2q+8, 2q+9}, (z, w) the second MMA's
      MmaSkinny<T>::run(c, a0[u].x, a1[u].x, a0[u].y, a1[u].y, w[u].x, w[u].y);
      MmaSkinny<T>::run(c, a0[u].z, a1[u].z, a0[u].w, a1[u].w, w[u].z, w[u].w);
    }
#pragma unroll
    for (int u = 0; u < SK_UNROLL; ++u) w[u] = wn[u];
  }
  // C fragment: c0,c1 -> (row r, cols 2q, 2q+1); c2,c3 -> (row r + 8, same cols)
  part[warp][r * 8 + 2 * q] = c[0];
  part[warp][r * 8 + 2 * q + 1] = c[1];
  part[warp][(r + 8) * 8 + 2 * q] = c[2];
  part[warp][(r + 8) * 8 + 2 * q + 1] = c[3];
  __syncthreads();
  // 128 outputs (16 rows x 8 columns); in GLU mode column pairs (2i, 2i+1) = (gate, up) collapse into one output
  const int t = threadIdx.x;
  if (t < 128) {
    const int row = t >> 3, col = t & 7;
    float x = 0.f;
#pragma unroll
    for (int wv = 0; wv < SK_WARPS; ++wv) x += part[wv][row * 8 + col];
    const int gcol = n0 + col;
    if (p.bias && gcol < p.N) x += __ldg(p.bias + gcol);
    part[0][row * 8 + col] = x;      // each thread wrote back only its own slot of warp 0's tile (already consumed by itself)
  }
  __syncthreads();
  if (t < 128) {
    const int row = t >> 3, col = t & 7;
    if (row < p.M) {
      if (p.swiglu) {
        if ((col & 1) == 0 && n0 + col < p.N) {
          const float g = rnd<T>(part[0][row * 8 + col]);
          const float u = rnd<T>(part[0][row * 8 + col + 1]);
          const float sact = rnd<T>(apply_act(g, p.act));
          reinterpret_cast<T*>(p.C)[static_cast<size_t>(row) * p.ldc + ((n0 + col) >> 1)] = from_f<T>(sact * u);
        }
      } else if (n0 + col < p.N) {
        float y = rnd<T>(part[0][row * 8 + col]);
        if (p.act != ACT_NONE) y = rnd<T>(apply_act(y, p.act));
        if (p.residual) y = y + to_f<T>(reinterpret_cast<const T*>(p.residual)[static_cast<size_t>(row) * p.ldr + n0 + col]);
        reinterpret_cast<T*>(p.C)[static_cast<size_t>(row) * p.ldc + n0 + col] = from_f<T>(y);
      }
    }
  }
}

bool gemm_skinny_ok(const GemmArgs& a) {
  if (a.M > 16 || a.M <= 0 || a.out_f32 || a.group_k || a.rowscale || a.ssq_inline || a.am_val || a.force_bn > 0) return false;
  if (a.K % 32 || a.lda % 8 || a.ldw % 8) return false;
  if ((reinterpret_cast<uintptr_t>(a.A) | reinterpret_cast<uintptr_t>(a.W)) & 15) return false;
  if (a.swiglu && (a.N % 2)) return false;
  return true;
}

int gemm_skinny_launch(const GemmArgs& a, cudaStream_t stream) {
  SkinnyParams p;
  p.A = a.A; p.lda = a.lda; p.W = a.W; p.ldw = a.ldw; p.C = a.C; p.ldc = a.ldc;
  p.M = a.M; p.N = a.N; p.K = a.K; p.bias = a.bias; p.residual = a.residual; p.ldr = a.ldr; p.act = a.act; p.swiglu = a.swiglu;
  p.w_constant = a.w_constant;
  const dim3 grid((a.N + 7) / 8), block(SK_WARPS * 32);
  if (a.dtype == DT_BF16) launch_pdl(gemm_skinny_kernel<__nv_bfloat16>, grid, block, 0, stream, p);
  else launch_pdl(gemm_skinny_kernel<__half>, grid, block, 0, stream, p);
  return launch_ok();
}

}  // namespace sb
