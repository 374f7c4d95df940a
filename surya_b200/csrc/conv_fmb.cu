// surya_b200 — FusedMBConv in one kernel: 3x3 conv (expand, + folded BN, Hardswish) -> 1x1 project (+ folded BN, + identity
// shortcut), the expanded tensor never leaves the SM.
//
// Stands in for FusedMBConv.forward (surya/detection/model/encoderdecoder.py:228-270) of the EfficientViT stages 0 and 1 and
// replaces the op pair conv_igemm -> gemm of det_engine.cu.  At BASELINE config 3 the four blocks write and re-read
// 2.1 + 1.0 + 1.0 + 0.5 GB of expanded activations per 32-page forward.
//
// Back-to-back GEMM per 128-pixel tile (8 rows x 16 px); two consumer warpgroups, each owning 64 of the tile's pixels end to end:
//   for each chunk j of 128 mid channels:
//     GEMM1  acc1 (registers, 128 cols) = sum over 9 taps x Cin/BKC channel chunks of  A1 (tap box, TMA)  x  W1[j] (TMA)
//     epi1   acc1 + shift -> round -> Hardswish -> round -> the warpgroup's 128B-swizzled A2 tile in shared memory (2 k-blocks)
//     GEMM2  acc2 (registers, Cout cols) += A2 x W2[:, chunk j] (TMA)
//   epi2     acc2 + shift (+ block input) -> round -> NHWC store
// Rounding points are those of the two separate kernels (expand output in T after the shift, after Hardswish; project output
// in T after the shift, after the residual add); the fp32 sum over the mid channels runs in the same k order as gemm_tn_kernel.
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "ops.cuh"
#include "sb_ptx.cuh"

#include <cstdlib>

namespace sb {

struct FmbParams {
  int n_img, H, W, Ho, Wo, Cin, Cmid, Cout, stride;
  int tiles_x, tiles_y;
  const float* bias1;     // [Cmid]
  const float* bias2;     // [Cout]
  const void* residual;   // NHWC [n_img, Ho, Wo, Cout] or null
  void* out;              // NHWC [n_img, Ho, Wo, Cout]
};

template <typename T, int BKC, int COUT, int STAGES, int NW2>
__global__ void __launch_bounds__(384, 1)
fmb_fused_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_w1,
                 const __grid_constant__ CUtensorMap tma_w2, const FmbParams fp) {
  constexpr int TW = 16, TH = 8, CH = 128;                           // mid-channel chunk
  constexpr uint32_t A1_BYTES = 128 * BKC * 2;
  constexpr uint32_t W1_BYTES = CH * BKC * 2;
  constexpr uint32_t S1_BYTES = A1_BYTES + W1_BYTES;
  constexpr uint32_t A2_KB_BYTES = 64 * 64 * 2;                      // one 64-channel k-block of a warpgroup's A2 tile (8 KB)
  constexpr uint32_t A2_WG_BYTES = 2 * A2_KB_BYTES;                  // 64 pixels x 128 mid channels
  constexpr uint32_t W2_KB_BYTES = COUT * 64 * 2, W2_BYTES = 2 * W2_KB_BYTES;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint8_t* s_1 = smem;
  uint8_t* s_a2 = s_1 + STAGES * S1_BYTES;
  uint8_t* s_w2 = s_a2 + 2 * A2_WG_BYTES;
  float* s_b1 = reinterpret_cast<float*>(s_w2 + NW2 * W2_BYTES);
  float* s_b2 = s_b1 + fp.Cmid;
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_b2 + COUT);
  uint64_t* s1_full = bars;
  uint64_t* s1_empty = s1_full + STAGES;
  uint64_t* w2_full = s1_empty + STAGES;
  uint64_t* w2_empty = w2_full + NW2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = fp.tiles_x * fp.tiles_y;
  const int num_tiles = fp.n_img * tiles_per_img;
  const int nch = fp.Cmid / CH;
  const int cpb = fp.Cin / BKC;                                      // channel chunks per tap
  const int kb1 = 9 * cpb;                                           // GEMM1 k-blocks per mid chunk

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_a); tma_prefetch_desc(&tma_w1); tma_prefetch_desc(&tma_w2);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&s1_full[i], 1); mbar_init(&s1_empty[i], EPI_WARPS); }
    for (int i = 0; i < NW2; ++i) { mbar_init(&w2_full[i], 1); mbar_init(&w2_empty[i], EPI_WARPS); }
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < fp.Cmid; i += blockDim.x) s_b1[i] = fp.bias1 ? fp.bias1[i] : 0.f;
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) s_b2[i] = fp.bias2 ? fp.bias2[i] : 0.f;
  __syncthreads();

  auto coords = [&](int tile, int& img, int& oy0, int& ox0) {
    img = tile / tiles_per_img;
    const int t = tile - img * tiles_per_img;
    oy0 = (t / fp.tiles_x) * TH;
    ox0 = (t % fp.tiles_x) * TW;
  };

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int s = 0; uint32_t ph = 0; int wb = 0; uint32_t wph = 0;
      auto load_w2 = [&](int j) {
        mbar_wait(&w2_empty[wb], wph ^ 1);
        mbar_expect_tx(&w2_full[wb], W2_BYTES);
        tma_load_2d(s_w2 + wb * W2_BYTES, &tma_w2, &w2_full[wb], j * CH, 0);
        tma_load_2d(s_w2 + wb * W2_BYTES + W2_KB_BYTES, &tma_w2, &w2_full[wb], j * CH + 64, 0);
        if (++wb == NW2) { wb = 0; wph ^= 1; }
      };
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int img, oy0, ox0;
        coords(tile, img, oy0, ox0);
        const int x0 = ox0 * fp.stride - 1, y0 = oy0 * fp.stride - 1;
        for (int j = 0; j < nch; ++j) {
          int kcol = 0;
          for (int r = 0; r < 3; ++r)
            for (int sx = 0; sx < 3; ++sx)
              for (int cc = 0; cc < cpb; ++cc, kcol += BKC) {
                mbar_wait(&s1_empty[s], ph ^ 1);
                uint8_t* sa = s_1 + s * S1_BYTES;
                mbar_expect_tx(&s1_full[s], S1_BYTES);
                tma_load_4d(sa, &tma_a, &s1_full[s], cc * BKC, x0 + sx, y0 + r, img);
                tma_load_2d(sa + A1_BYTES, &tma_w1, &s1_full[s], kcol, j * CH);
                if (++s == STAGES) { s = 0; ph ^= 1; }
              }
          load_w2(j);
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumer warpgroups: pixels [64 wg, 64 wg + 64) of the tile
    const int wg = (warp - 4) >> 2, ww = warp & 3;
    const int r0 = ww * 16 + (lane >> 2), c = (lane & 3) * 2;        // fragment rows r0, r0 + 8 (of the warpgroup), columns 8j + c
    uint8_t* a2 = s_a2 + wg * A2_WG_BYTES;
    int s = 0; uint32_t ph = 0; int wb = 0; uint32_t wph = 0;
    constexpr int NCH = 64;                                          // partial-sum width (register budget: d1 + d2 + part)
    float d1[CH / 2], d2[COUT / 2], part[NCH / 2];
    T* out = reinterpret_cast<T*>(fp.out);
    const T* res = reinterpret_cast<const T*>(fp.residual);
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int img, oy0, ox0;
      coords(tile, img, oy0, ox0);
      for (int j = 0; j < nch; ++j) {
        // GEMM1: expanded chunk j (per-k-block partial sums added in fp32, gemm_epilogue.cuh)
        wg_mainloop<T, CH, BKC, NCH>(d1, s_1, S1_BYTES, A1_BYTES, STAGES, s1_full, s1_empty, s, ph, kb1, wg, lane,
                                     [](const uint8_t*) {});
        // epi1: + shift -> round -> Hardswish -> round -> A2 (row r, mid channel cc: k-block cc / 64, 16-byte chunk (cc % 64) / 8)
        const float* bs = s_b1 + j * CH;
#pragma unroll
        for (int jb = 0; jb < CH / 8; ++jb) {
          const int cc = jb * 8 + c;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const uint32_t t = Pk<T>::pack(d1[4 * jb + 2 * h] + bs[cc], d1[4 * jb + 2 * h + 1] + bs[cc + 1]);
            const uint32_t o = Pk<T>::pack(act_ct<ACT_HARDSWISH>(Pk<T>::lo(t)), act_ct<ACT_HARDSWISH>(Pk<T>::hi(t)));
            *reinterpret_cast<uint32_t*>(a2 + (cc >> 6) * A2_KB_BYTES + r * 128 + ((((cc & 63) >> 3) ^ (r & 7)) << 4) + (cc & 7) * 2) = o;
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> wgmma operand reads
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        // GEMM2: acc2 += A2 x W2[:, chunk j], one 64-channel k-block at a time (the k-blocks of the unfused project GEMM)
        mbar_wait(&w2_full[wb], wph);
        if (j == 0) {
#pragma unroll
          for (int i = 0; i < COUT / 2; ++i) d2[i] = 0.f;
        }
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint64_t da = wgmma_desc_k128(smem_u32(a2 + kk * A2_KB_BYTES));
          const uint64_t db = wgmma_desc_k128(smem_u32(s_w2 + wb * W2_BYTES + kk * W2_KB_BYTES));
#pragma unroll
          for (int cn = 0; cn < COUT / NCH; ++cn) {
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64k16<T, NCH>(part, da + 2 * k, db + ((cn * NCH * 128) >> 4) + 2 * k, k != 0 ? 1u : 0u);
            wgmma_commit();
            wg_promote<NCH>(d2 + cn * (NCH / 2), part);
          }
        }
        release(&w2_empty[wb]);                                      // A2 and the W2 buffer are free again
        if (++wb == NW2) { wb = 0; wph ^= 1; }
      }
      // epi2: + shift (+ block input) -> round -> NHWC store
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = wg * 64 + r0 + 8 * h;                          // tile pixel (m / 16, m % 16)
        const int oy = oy0 + (m >> 4), ox = ox0 + (m & 15);
        if (oy >= fp.Ho || ox >= fp.Wo) continue;
        const size_t pix = (static_cast<size_t>(img) * fp.Ho + oy) * fp.Wo + ox;
#pragma unroll
        for (int jb = 0; jb < COUT / 8; ++jb) {
          const int cc = jb * 8 + c;
          uint32_t o = Pk<T>::pack(d2[4 * jb + 2 * h] + s_b2[cc], d2[4 * jb + 2 * h + 1] + s_b2[cc + 1]);
          if (res) {
            const uint32_t rr = __ldg(reinterpret_cast<const unsigned int*>(res + pix * COUT + cc));
            o = Pk<T>::pack(Pk<T>::lo(o) + Pk<T>::lo(rr), Pk<T>::hi(o) + Pk<T>::hi(rr));
          }
          *reinterpret_cast<uint32_t*>(out + pix * COUT + cc) = o;
        }
      }
    }
  }
}

bool fmb_fused_ok(int Cin, int Cmid, int Cout, int ksize, int stride, int pad, int act1, int act2) {
  static int en = -1;
  if (en < 0) { const char* e = getenv("SB_FMB_FUSED"); en = (e && e[0] == '0') ? 0 : 1; }
  if (!en) return false;
  if (ksize != 3 || pad != 1 || (stride != 1 && stride != 2) || act1 != ACT_HARDSWISH || act2 != ACT_NONE) return false;
  if (Cin != 64 && Cin != 128) return false;
  if (Cmid % 128 || Cmid < 128 || Cmid > 1024) return false;
  return Cout == 64 || Cout == 128;
}

template <typename T, int BKC, int COUT, int STAGES, int NW2>
static int launch_fmb(int dtype, const void* in, const void* w1, const void* w2, const FmbParams& fp, cudaStream_t st) {
  constexpr size_t S1 = static_cast<size_t>(128 * BKC * 2) * 2;
  const size_t SMEM = STAGES * S1 + 32768 + NW2 * (COUT * 256) + (fp.Cmid + COUT) * 4 + 512 + 1024;
  auto kern = fmb_fused_kernel<T, BKC, COUT, STAGES, NW2>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess) {
    cudaGetLastError();
    set_error("fmb_fused: cudaFuncSetAttribute(smem=%zu) failed", SMEM);
    return -10;
  }
  CUtensorMap ma, m1, m2;
  int rc = make_tma_nhwc(&ma, dtype, in, fp.n_img, fp.H, fp.W, fp.Cin, BKC, 16, 8, fp.stride, BKC * 2);
  if (rc) return rc;
  rc = make_tma_2d_sw(&m1, dtype, w1, fp.Cmid, 9 * fp.Cin, 9 * fp.Cin, BKC, 128, BKC * 2);
  if (rc) return rc;
  rc = make_tma_2d(&m2, dtype, w2, COUT, fp.Cmid, fp.Cmid, COUT);
  if (rc) return rc;
  const int tiles = fp.n_img * fp.tiles_x * fp.tiles_y;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, 384, SMEM, st>>>(ma, m1, m2, fp);
  return launch_ok();
}

// in NHWC [n_img, H, W, Cin]; w1 T [Cmid][9*Cin] (tap-major, BN folded), bias1 fp32 [Cmid]; w2 T [Cout][Cmid], bias2 fp32 [Cout];
// residual NHWC [n_img, Ho, Wo, Cout] or null; out NHWC [n_img, Ho, Wo, Cout].
int fmb_fused(int dtype, const void* in, const void* w1, const float* bias1, const void* w2, const float* bias2,
              const void* residual, void* out, int n_img, int H, int W, int Cin, int Cmid, int Cout, int stride, cudaStream_t st) {
  if (n_img <= 0) return 0;
  if (!fmb_fused_ok(Cin, Cmid, Cout, 3, stride, 1, ACT_HARDSWISH, ACT_NONE)) { set_error("fmb_fused: unsupported shape"); return -1; }
  FmbParams fp{};
  fp.n_img = n_img; fp.H = H; fp.W = W; fp.Ho = (H + 2 - 3) / stride + 1; fp.Wo = (W + 2 - 3) / stride + 1;
  fp.Cin = Cin; fp.Cmid = Cmid; fp.Cout = Cout; fp.stride = stride;
  fp.tiles_x = (fp.Wo + 15) / 16; fp.tiles_y = (fp.Ho + 7) / 8;
  fp.bias1 = bias1; fp.bias2 = bias2; fp.residual = residual; fp.out = out;
#define FMB(T_) \
  do { \
    if (Cout == 64) return launch_fmb<T_, 64, 64, 3, 2>(dtype, in, w1, w2, fp, st); \
    return launch_fmb<T_, 64, 128, 3, 1>(dtype, in, w1, w2, fp, st); \
  } while (0)
  if (dtype == DT_BF16) FMB(__nv_bfloat16); else FMB(__half);
#undef FMB
}

}  // namespace sb
