// surya_b200 — 3x3 (k x k) dense convolution as an implicit GEMM on wgmma, NHWC activations.
//
//   out[n, oy, ox, :] = epilogue( sum_{r,s,c} in[n, oy*stride + r - pad, ox*stride + s - pad, c] * W[:, r, s, c] )
//
// Replaces the cuDNN implicit-GEMM convolutions of the detection backbone's ConvBlock / FusedMBConv
// (surya/detection/model/encoderdecoder.py:130-171, 228-270; SURVEY.md §2.2 K1).  Same warp-specialised
// pipeline as gemm_wgmma.cu; the only difference is the A operand: for k-block (tap r,s ; channel chunk c0)
// the producer issues ONE 4-D TMA tile load {BKC channels, TW pixels, TH rows, 1 image} at the tap-shifted
// coordinate.  TMA zero-fills out-of-bounds pixels (= the convolution's zero padding) and its elementStrides
// implement stride 2, so no im2col matrix is ever materialised.  BN is folded into W/bias at pack time.
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "ops.cuh"
#include "sb_ptx.cuh"

namespace sb {

struct ConvKParams {
  GemmKParams g;  // M unused; N = Cout
  int n_img, Ho, Wo, Cin, ksize, stride, pad;
  int tiles_x, tiles_y;
  int desc_lbo, desc_sbo;   // halo variant: A-descriptor strides
};

template <typename T, int BN, int BKC, int STAGES>
__global__ void __launch_bounds__(384, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                  const ConvKParams cp) {
  constexpr int BM = 128, TW = 16, TH = 8;
  constexpr uint32_t A_BYTES = BM * BKC * 2, B_BYTES = BN * BKC * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  static_assert(BKC == 64 || BKC == 32, "channel chunk must be 64 (128B swizzle) or 32 (64B swizzle)");
  static_assert(BN <= ACC_MAX_COLS, "one epilogue pass per tile");
  const GemmKParams& p = cp.g;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* acc_s = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + 256);
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(acc_s) + acc_smem_bytes<BN>();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = cp.tiles_x * cp.tiles_y;
  const int m_blocks = cp.n_img * tiles_per_img;
  const int n_blocks = (p.N + BN - 1) / BN;
  const int cpb = cp.Cin / BKC;                       // channel chunks per tap
  const int k_blocks = cp.ksize * cp.ksize * cpb;
  const int num_tiles = m_blocks * n_blocks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_a); tma_prefetch_desc(&tma_b);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], EPI_WARPS); }
    mbar_fence_init();
  }
  __syncthreads();

  auto coords = [&](int tile, int& img, int& oy0, int& ox0, int& nb) {
    // n-block fastest inside a group of 8 m-blocks: the (small) weight matrix and the input halo stay L2-hot
    int mb;
    int per_group = p.group_m * n_blocks;
    int g = tile / per_group;
    int first = g * p.group_m;
    int gsz = min(m_blocks - first, p.group_m);
    int r = tile - g * per_group;
    mb = first + r % gsz;
    nb = r / gsz;
    img = mb / tiles_per_img;
    int t = mb - img * tiles_per_img;
    oy0 = (t / cp.tiles_x) * TH;
    ox0 = (t % cp.tiles_x) * TW;
  };

  if (warp == 0) {
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int img, oy0, ox0, nb;
        coords(tile, img, oy0, ox0, nb);
        // nested (tap row, tap column, channel chunk) loops: this single thread's dependent integer math paces narrow tiles,
        // so no runtime division per k-block
        const int x0 = ox0 * cp.stride - cp.pad, y0 = oy0 * cp.stride - cp.pad, n0 = nb * BN;
        int kcol = 0;
        for (int r = 0; r < cp.ksize; ++r) {
          for (int sx = 0; sx < cp.ksize; ++sx) {
            for (int cc = 0; cc < cpb; ++cc, kcol += BKC) {
              mbar_wait(&empty_bar[s], ph ^ 1);
              uint8_t* sa = smem + s * STAGE_BYTES;
              mbar_expect_tx(&full_bar[s], STAGE_BYTES);
              tma_load_4d(sa, &tma_a, &full_bar[s], cc * BKC, x0 + sx, y0 + r, img);
              tma_load_2d(sa + A_BYTES, &tma_b, &full_bar[s], kcol, n0);
              if (++s == STAGES) { s = 0; ph ^= 1; }
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;
    const int q = warp & 3;
    const int half = wg;
    const int epi_tid = threadIdx.x - 128;
    uint8_t* stage = epi_smem + (warp - 4) * EPI_STAGE_BYTES;
    float* sbias = reinterpret_cast<float*>(epi_smem + EPI_WARPS * EPI_STAGE_BYTES);
    int s = 0; uint32_t ph = 0;
    const bool vec_ok = (p.ldc % 8 == 0) && (!p.residual || p.ldr % 8 == 0);
    const bool v2 = epilogue_v2_ok(p);
    const AccRow acc(acc_s, q * 32 + lane, BN);
    float d[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int img, oy0, ox0, nb;
      coords(tile, img, oy0, ox0, nb);
      if (v2) {
        asm volatile("bar.sync 1, 256;" ::: "memory");
        epilogue_stage_bias<BN>(p, sbias, epi_tid, nb * BN);
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      wg_mainloop<T, BN, BKC>(d, smem, STAGE_BYTES, A_BYTES, STAGES, full_bar, empty_bar, s, ph, k_blocks, wg, lane,
                              [](const uint8_t*) {});
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free
      wg_acc_store<BN / 8>(d, 0, acc_s + wg * 64 * BN, BN, warp & 3, lane);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (v2) {
        epilogue_tile_rt<T>(acc, p, stage, sbias, lane, half,
                            [&](int r) {
                              const int mm = q * 32 + r;
                              const int yy = oy0 + mm / TW, xx = ox0 + mm % TW;
                              return (yy < cp.Ho && xx < cp.Wo) ? (img * cp.Ho + yy) * cp.Wo + xx : -1;
                            }, nb * BN, 1.0f, BN / 32);
      } else if (half == 0) {
        const int m = q * 32 + lane;
        const int oy = oy0 + m / TW, ox = ox0 + m % TW;
        const bool row_ok = oy < cp.Ho && ox < cp.Wo;
        const int row = (img * cp.Ho + oy) * cp.Wo + ox;
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          uint32_t v[32];
          acc.load32(c * 32, v);
          const int col0 = nb * BN + c * 32;
          if (col0 >= p.N) continue;
          epilogue_chunk<T>(v, p, row, row_ok, col0, vec_ok);
        }
      }
    }
  }
}

template <typename T, int BN, int BKC, int STAGES>
static int launch_conv(const ConvArgs& a, cudaStream_t stream) {
  constexpr uint32_t STAGE_BYTES = 128 * BKC * 2 + BN * BKC * 2;
  constexpr size_t SMEM = STAGES * STAGE_BYTES + 1024 + 256 + acc_smem_bytes<BN>() + epi_smem_bytes<BN>();
  static_assert(SMEM <= 227 * 1024, "convolution tile does not fit in shared memory");
  auto kern = conv_igemm_kernel<T, BN, BKC, STAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess) {
      cudaGetLastError();
      set_error("conv: cudaFuncSetAttribute(smem=%zu) failed", SMEM);
      return -10;
    }
    attr_set = true;
  }
  const int Ho = (a.H + 2 * a.pad - a.ksize) / a.stride + 1, Wo = (a.W + 2 * a.pad - a.ksize) / a.stride + 1;
  CUtensorMap ma, mb;
  const int sw = BKC * 2;
  int rc = make_tma_nhwc(&ma, a.dtype, a.in, a.n_img, a.H, a.W, a.Cin, BKC, 16, 8, a.stride, sw);
  if (rc) return rc;
  rc = make_tma_2d_sw(&mb, a.dtype, a.weight, a.Cout, a.ksize * a.ksize * a.Cin, a.ksize * a.ksize * a.Cin, BKC, BN, sw);
  if (rc) return rc;
  ConvKParams cp{};
  cp.g.M = a.n_img * Ho * Wo; cp.g.N = a.Cout; cp.g.K = a.ksize * a.ksize * a.Cin;
  cp.g.C = a.out; cp.g.ldc = a.Cout; cp.g.bias = a.bias; cp.g.residual = a.residual; cp.g.ldr = a.Cout;
  cp.g.act = a.act; cp.g.swiglu = 0; cp.g.out_f32 = 0; cp.g.group_m = 8; cp.g.group_k = 0; cp.g.w_constant = 0;
  cp.n_img = a.n_img; cp.Ho = Ho; cp.Wo = Wo; cp.Cin = a.Cin; cp.ksize = a.ksize; cp.stride = a.stride; cp.pad = a.pad;
  cp.tiles_x = (Wo + 15) / 16; cp.tiles_y = (Ho + 7) / 8;
  const int tiles = a.n_img * cp.tiles_x * cp.tiles_y * ((a.Cout + BN - 1) / BN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, 384, SMEM, stream>>>(ma, mb, cp);
  return launch_ok();
}


// ------------------------------------------------------------------------------------------------ halo-tile variant
// Narrow convolutions (Cin = Cout = 32: the stem's ResidualBlock at 512^2) are far from their DRAM floor with the tap-box kernel
// above: nine {32 ch, 16 px, 8 rows} boxes per tile are 1152 separate 64-byte TMA lines and a 9x re-read of the input through L2.  A first fix (one halo box per tile, builder warps copying it into nine swizzled tap tiles)
// moved the bound to the shared-memory pipe (144 KB of LDS + STS per tile).
// This version never forms tap tiles: the halo is re-laid once per tile into four CHANNEL-CHUNK PLANES (16 bytes = 8 channels per
// pixel and plane, pixels contiguous), which is exactly wgmma's un-swizzled K-major canonical layout when the tile is 8 pixels
// wide: core matrix = 8 pixels x 16 B contiguous, SBO = one halo row (10 px x 16 B), LBO = one plane.  A tap (ty, tx) is then
// nothing but a start-address offset of (ty * 10 + tx) * 16 bytes in the A descriptor (and the second consumer warpgroup's 64
// rows start 8 halo rows further).  Per tile: 1 TMA box (180 lines), 23 KB of LDS + STS, 18 MMAs per warpgroup.  Weights
// (9 x 32 x 32, 64B-swizzled) are loaded once per CTA.  Stride 1, pad 1.
constexpr int HALO_BUFS = 8;       // halo boxes in flight (TMA staging, pixel-major)
constexpr int HALO_PLANES = 3;     // re-laid tiles between the builders and the MMA warp
constexpr int HALO_PLANE_PITCH = 180 * 16 + 32;   // +32: the four planes start in different bank groups (conflict-free STS)

template <typename T>
__global__ void __launch_bounds__(512, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tma_halo, const __grid_constant__ CUtensorMap tma_b, const ConvKParams cp) {
  constexpr int BM = 128, TW = 8, TH = 16, BN = 32, CIN = 32, TAPS = 9;
  constexpr int HW_ = TW + 2, HH_ = TH + 2, HPIX = HW_ * HH_;      // 10 x 18 = 180 halo pixels
  constexpr uint32_t W_BYTES = TAPS * BN * CIN * 2;          // 18 KB
  constexpr uint32_t HALO_BYTES = HPIX * CIN * 2;            // 11 520 B
  constexpr uint32_t PLANES_BYTES = 4 * HALO_PLANE_PITCH;    // 11 648 B per re-laid tile
  const GemmKParams& p = cp.g;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint8_t* s_w = smem;
  uint8_t* s_halo = s_w + W_BYTES;
  uint8_t* s_pl = s_halo + HALO_BUFS * HALO_BYTES;
  uint64_t* pfull_bar = reinterpret_cast<uint64_t*>(s_pl + HALO_PLANES * PLANES_BYTES);
  uint64_t* pempty_bar = pfull_bar + HALO_PLANES;
  uint64_t* hfull_bar = pempty_bar + HALO_PLANES;
  uint64_t* hempty_bar = hfull_bar + HALO_BUFS;
  uint64_t* w_bar = hempty_bar + HALO_BUFS;
  float* acc_s = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(pfull_bar) + 512);    // [128][32] accumulator tile
  uint8_t* epi_smem = reinterpret_cast<uint8_t*>(acc_s) + acc_smem_bytes<BN>();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = cp.tiles_x * cp.tiles_y;
  const int num_tiles = cp.n_img * tiles_per_img;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_halo); tma_prefetch_desc(&tma_b);
    for (int i = 0; i < HALO_PLANES; ++i) { mbar_init(&pfull_bar[i], 4); mbar_init(&pempty_bar[i], EPI_WARPS); }
    for (int i = 0; i < HALO_BUFS; ++i) { mbar_init(&hfull_bar[i], 1); mbar_init(&hempty_bar[i], 4); }
    mbar_init(w_bar, 1);
    mbar_fence_init();
  }
  __syncthreads();

  auto coords = [&](int tile, int& img, int& oy0, int& ox0) {
    img = tile / tiles_per_img;
    const int t = tile - img * tiles_per_img;
    oy0 = (t / cp.tiles_x) * TH;
    ox0 = (t % cp.tiles_x) * TW;
  };

  if (warp == 0) {
    if (lane == 0) {
      mbar_expect_tx(w_bar, W_BYTES);
      for (int t = 0; t < TAPS; ++t) tma_load_2d(s_w + t * BN * CIN * 2, &tma_b, w_bar, t * CIN, 0);
      int hb = 0; uint32_t hph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int img, oy0, ox0;
        coords(tile, img, oy0, ox0);
        mbar_wait(&hempty_bar[hb], hph ^ 1);
        mbar_expect_tx(&hfull_bar[hb], HALO_BYTES);
        tma_load_4d(s_halo + hb * HALO_BYTES, &tma_halo, &hfull_bar[hb], 0, ox0 - 1, oy0 - 1, img);
        if (++hb == HALO_BUFS) { hb = 0; hph ^= 1; }
      }
    }
  } else if (warp >= 12) {
    // builders: 16-byte moves, thread -> (pixel = k * 32 + i / 4, chunk = i % 4): a quarter warp reads 2 pixels = 128 contiguous
    // bytes and writes 2 x 16 B into each of the four planes (plane pitch chosen so the eight stores hit eight bank groups)
    const int i = threadIdx.x - 384;
    const int c = i & 3, p0 = i >> 2;
    int pb = 0; uint32_t pph = 0; int hb = 0; uint32_t hph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      mbar_wait(&hfull_bar[hb], hph);
      const uint8_t* halo = s_halo + hb * HALO_BYTES;
      mbar_wait(&pempty_bar[pb], pph ^ 1);
      uint8_t* pl = s_pl + pb * PLANES_BYTES + c * HALO_PLANE_PITCH;
      uint4 v[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const int px = p0 + k * 32;
        v[k] = px < HPIX ? *reinterpret_cast<const uint4*>(halo + px * (CIN * 2) + c * 16) : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const int px = p0 + k * 32;
        if (px < HPIX) *reinterpret_cast<uint4*>(pl + px * 16) = v[k];
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) { mbar_arrive(&pfull_bar[pb]); mbar_arrive(&hempty_bar[hb]); }
      if (++pb == HALO_PLANES) { pb = 0; pph ^= 1; }
      if (++hb == HALO_BUFS) { hb = 0; hph ^= 1; }
    }
  } else if (warp >= 4) {
    // consumer warpgroups: 9 taps x 2 MMAs on the re-laid planes, then the epilogue
    const int wg = (warp - 4) >> 2;
    const int q = warp & 3;
    const int half = wg;
    const int epi_tid = threadIdx.x - 128;
    uint8_t* stage = epi_smem + (warp - 4) * EPI_STAGE_BYTES;
    float* sbias = reinterpret_cast<float*>(epi_smem + EPI_WARPS * EPI_STAGE_BYTES);
    const uint32_t lbo = static_cast<uint32_t>(cp.desc_lbo), sbo = static_cast<uint32_t>(cp.desc_sbo);
    int pb = 0; uint32_t pph = 0;
    const AccRow acc(acc_s, q * 32 + lane, BN);
    float d[BN / 2];
    epilogue_stage_bias<BN>(p, sbias, epi_tid, 0);
    asm volatile("bar.sync 1, 256;" ::: "memory");
    mbar_wait(w_bar, 0);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int img, oy0, ox0;
      coords(tile, img, oy0, ox0);
      mbar_wait(&pfull_bar[pb], pph);
      const uint32_t a0 = smem_u32(s_pl + pb * PLANES_BYTES) + wg * (TH / 2) * HW_ * 16;   // this warpgroup's 8 pixel rows
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
#pragma unroll
      for (int t = 0; t < TAPS; ++t) {
        // one tap = one 32-channel k-block of the tap-box kernel (BKC = 32): same partial sums, same fp32 additions
        const int ty = t / 3, tx = t % 3;
        const uint64_t db = wgmma_desc_k64(smem_u32(s_w + t * BN * CIN * 2));
        float part[BN / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < CIN / 16; ++k) {
          // k-th pair of channel-chunk planes, start shifted by the tap
          const uint64_t da = wgmma_desc_plain(a0 + (ty * HW_ + tx) * 16 + k * 2 * HALO_PLANE_PITCH, lbo, sbo);
          wgmma_m64k16<T, BN>(part, da, db + 2 * k, k != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wg_promote<BN>(d, part);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&pempty_bar[pb]);
      if (++pb == HALO_PLANES) { pb = 0; pph ^= 1; }
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the accumulator tile is free
      wg_acc_store<BN / 8>(d, 0, acc_s + wg * 64 * BN, BN, warp & 3, lane);
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // Cout = ldc = ldr = 32 and 16-bit output: the staged epilogue's requirements (epilogue_v2_ok) always hold here
      epilogue_tile_rt<T>(acc, p, stage, sbias, lane, half,
                          [&](int r) {
                            const int mm = q * 32 + r;
                            const int yy = oy0 + mm / TW, xx = ox0 + mm % TW;
                            return (yy < cp.Ho && xx < cp.Wo) ? (img * cp.Ho + yy) * cp.Wo + xx : -1;
                          }, 0, 1.0f, BN / 32);
    }
  }
}

static bool conv_halo_ok(const ConvArgs& a) {
  return a.ksize == 3 && a.stride == 1 && a.pad == 1 && a.Cin == 32 && a.Cout == 32;
}

template <typename T>
static int launch_conv_halo(const ConvArgs& a, cudaStream_t stream) {
  constexpr size_t SMEM = 9 * 2048 + HALO_BUFS * 11520 + HALO_PLANES * 4 * HALO_PLANE_PITCH + 512 + acc_smem_bytes<32>() + epi_smem_bytes<32>() + 1024;
  static_assert(SMEM <= 227 * 1024, "conv_halo does not fit in shared memory");
  auto kern = conv_halo_kernel<T>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess) {
      cudaGetLastError();
      set_error("conv_halo: cudaFuncSetAttribute(smem=%zu) failed", SMEM);
      return -10;
    }
    attr_set = true;
  }
  CUtensorMap mh, mb;
  int rc = make_tma_nhwc(&mh, a.dtype, a.in, a.n_img, a.H, a.W, a.Cin, 32, 10, 18, 1, 0);
  if (rc) return rc;
  rc = make_tma_2d_sw(&mb, a.dtype, a.weight, a.Cout, 9 * a.Cin, 9 * a.Cin, 32, 32, 64);
  if (rc) return rc;
  ConvKParams cp{};
  cp.g.M = a.n_img * a.H * a.W; cp.g.N = a.Cout; cp.g.K = 9 * a.Cin;
  cp.g.C = a.out; cp.g.ldc = a.Cout; cp.g.bias = a.bias; cp.g.residual = a.residual; cp.g.ldr = a.Cout;
  cp.g.act = a.act; cp.g.swiglu = 0; cp.g.out_f32 = 0; cp.g.group_m = 8; cp.g.group_k = 0; cp.g.w_constant = 0;
  cp.n_img = a.n_img; cp.Ho = a.H; cp.Wo = a.W; cp.Cin = a.Cin; cp.ksize = 3; cp.stride = 1; cp.pad = 1;
  cp.tiles_x = (a.W + 7) / 8; cp.tiles_y = (a.H + 15) / 16;
  cp.desc_lbo = HALO_PLANE_PITCH; cp.desc_sbo = 10 * 16;   // LBO: next 16-byte k chunk (plane); SBO: next 8-row group (halo row)
  const int tiles = a.n_img * cp.tiles_x * cp.tiles_y;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, 512, SMEM, stream>>>(mh, mb, cp);
  return launch_ok();
}

template <typename T>
static int conv_typed(const ConvArgs& a, cudaStream_t st) {
  // tiles up to 128 output channels: a single epilogue pass, and the ring keeps >= 4 stages beside the accumulator tile
  const int bn = a.Cout >= 128 ? 128 : (a.Cout >= 64 ? 64 : 32);
  if (a.Cin % 64 == 0) {
    switch (bn) {
      case 128: return launch_conv<T, 128, 64, 4>(a, st);
      case 64: return launch_conv<T, 64, 64, 6>(a, st);
      default: return launch_conv<T, 32, 64, 8>(a, st);
    }
  }
  if (a.Cin % 32 == 0) {
    switch (bn) {
      case 128: return launch_conv<T, 128, 32, 8>(a, st);
      case 64: return launch_conv<T, 64, 32, 8>(a, st);
      default: return launch_conv<T, 32, 32, 12>(a, st);
    }
  }
  set_error("conv_igemm: Cin must be a multiple of 32 (got %d)", a.Cin);
  return -20;
}

int conv_igemm(const ConvArgs& a, cudaStream_t st) {
  if (a.n_img <= 0) return 0;
  if (a.stride != 1 && a.stride != 2) { set_error("conv_igemm: stride must be 1 or 2"); return -21; }
  if (a.Cout % 8) { set_error("conv_igemm: Cout must be a multiple of 8"); return -22; }
  if (conv_halo_ok(a)) return a.dtype == DT_BF16 ? launch_conv_halo<__nv_bfloat16>(a, st) : launch_conv_halo<__half>(a, st);
  return a.dtype == DT_BF16 ? conv_typed<__nv_bfloat16>(a, st) : conv_typed<__half>(a, st);
}

}  // namespace sb
