// surya_b200 — detection decode head in one kernel: bilinear up-sampling + channel concat + 1x1 "fuse" conv (+ folded BN, ReLU)
// + classifier + sigmoid.  Stands in for DecodeHead.forward after the per-stage linear_c projections
// (surya/detection/model/encoderdecoder.py:699-722) and replaces the op sequence upsample_cat -> gemm -> classifier of det_ops.cu.
//
// Why: at BASELINE config 3 (32 pages, 1024^2) the 512-channel map at 256^2 is 2.1 GB; the unfused path writes it twice and reads
// it twice (8.6 GB of the ~24 GB a forward moves).  Here it never exists:
//   * the A operand of the fuse GEMM (128 pixels x 512 channels per tile) is PRODUCED in shared memory: the three low-resolution
//     branches by four builder warps (bilinear blend of the branch maps, which are L2 resident: 0.26 / 1 / 4 MB per page, with the
//     same pinned arithmetic and the same rounding to the storage type as upsample_cat_kernel), the full-resolution branch by TMA;
//     everything lands in the 128B-swizzled K-major layout wgmma reads;
//   * two consumer warpgroups (64 pixels each) run the GEMM as eight passes of N = 64 over the same A tile, accumulators in
//     registers (per-k-block partial sums added in fp32, like the unfused GEMM), weights streamed by TMA (8 KB per k-block and pass);
//   * after each pass the epilogue adds the folded-BN shift, rounds to the storage type, applies ReLU and multiplies straight
//     into the two classifier rows (fp32 accumulation of the rounded 16-bit values), so the fused map is never written either;
//     the four lanes sharing a pixel meet through shuffles in a fixed order; sigmoid and the NCHW store finish the pixel.
// Rounding points are those of the unfused kernels (branch value -> T, fuse output -> T, classifier logit -> T, sigmoid -> T);
// only the fp32 summation order inside the 512-long classifier dot differs from classifier_kernel (lane-strided there, strided by
// the fragment layout here).
#include "gemm.cuh"
#include "gemm_epilogue.cuh"
#include "ops.cuh"
#include "sb_ptx.cuh"

#include <cstdlib>

namespace sb {

constexpr int HEAD_KB = 8;          // k-blocks of 64 channels (K = 512)
constexpr int HEAD_N = 512;

struct HeadParams {
  const void* src[HEAD_KB];         // per k-block: source map (NHWC [B, hs, ws, CS]) or null when the block comes by TMA
  int hs[HEAD_KB], ws[HEAD_KB], c0[HEAD_KB];   // source size and first channel of the block inside the source
  int tma_c0[HEAD_KB];              // TMA blocks: first channel inside the identity source
  int CS;                           // channels per source map
  int B, HO, WO, tiles_x, tiles_y;
  const float* fuse_bias;           // [512] fp32 (folded BN shift)
  const void* cls_w;                // T [2][512]
  const void* cls_b;                // T [2]
  void* out;                        // T NCHW [B, 2, HO*WO]
};


template <typename T>
__global__ void __launch_bounds__(512, 1)
head_fused_kernel(const __grid_constant__ CUtensorMap tma_id, const __grid_constant__ CUtensorMap tma_w, const HeadParams hp) {
  constexpr int TW = 16, TH = 8, BK = 64, BNP = 64, PASSES = HEAD_N / BNP;
  constexpr uint32_t A_BYTES = 128 * BK * 2;           // 16 KB per k-block
  constexpr uint32_t W_BYTES = BNP * BK * 2;           // 8 KB per k-block and pass
  constexpr int W_STAGES = 8;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // array + offset keeps the shared address space (STS / LDS, not generic ST / LD)
  uint8_t* s_a = smem;                                  // 8 x 16 KB
  uint8_t* s_w = s_a + HEAD_KB * A_BYTES;               // 8 x 8 KB
  float* s_bias = reinterpret_cast<float*>(s_w + W_STAGES * W_BYTES);      // [512]
  T* s_cls = reinterpret_cast<T*>(s_bias + HEAD_N);                          // [2][512]
  uint64_t* afull_bar = reinterpret_cast<uint64_t*>(s_cls + 2 * HEAD_N);
  uint64_t* aempty_bar = afull_bar + HEAD_KB;
  uint64_t* wfull_bar = aempty_bar + HEAD_KB;
  uint64_t* wempty_bar = wfull_bar + W_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_img = hp.tiles_x * hp.tiles_y;
  const int num_tiles = hp.B * tiles_per_img;
  const int HW = hp.HO * hp.WO;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tma_id); tma_prefetch_desc(&tma_w);
    for (int i = 0; i < HEAD_KB; ++i) { mbar_init(&afull_bar[i], hp.src[i] ? 4 : 1); mbar_init(&aempty_bar[i], EPI_WARPS); }
    for (int i = 0; i < W_STAGES; ++i) { mbar_init(&wfull_bar[i], 1); mbar_init(&wempty_bar[i], EPI_WARPS); }
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < HEAD_N; i += blockDim.x) {
    s_bias[i] = hp.fuse_bias[i];
    s_cls[i] = reinterpret_cast<const T*>(hp.cls_w)[i];
    s_cls[HEAD_N + i] = reinterpret_cast<const T*>(hp.cls_w)[HEAD_N + i];
  }
  __syncthreads();

  auto coords = [&](int tile, int& img, int& oy0, int& ox0) {
    img = tile / tiles_per_img;
    const int t = tile - img * tiles_per_img;
    oy0 = (t / hp.tiles_x) * TH;
    ox0 = (t % hp.tiles_x) * TW;
  };

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer: weights (every pass) + identity-branch A blocks
    if (lane == 0) {
      int ws_ = 0; uint32_t wph = 0; uint32_t aph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int img, oy0, ox0;
        coords(tile, img, oy0, ox0);
        for (int kb = 0; kb < HEAD_KB; ++kb) {
          if (hp.src[kb]) continue;
          mbar_wait(&aempty_bar[kb], aph ^ 1);
          mbar_expect_tx(&afull_bar[kb], A_BYTES);
          tma_load_4d(s_a + kb * A_BYTES, &tma_id, &afull_bar[kb], hp.tma_c0[kb], ox0, oy0, img);
        }
        aph ^= 1;
        for (int h = 0; h < PASSES; ++h) {
          for (int kb = 0; kb < HEAD_KB; ++kb) {
            mbar_wait(&wempty_bar[ws_], wph ^ 1);
            mbar_expect_tx(&wfull_bar[ws_], W_BYTES);
            tma_load_2d(s_w + ws_ * W_BYTES, &tma_w, &wfull_bar[ws_], kb * BK, h * BNP);
            if (++ws_ == W_STAGES) { ws_ = 0; wph ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 12) {
    // ------------------------------------------------------------------ A builders (low-resolution branches)
    // thread -> 16-byte chunk c of pixel rows it*16 + i/8: eight lanes read one source pixel's 128 contiguous bytes per corner
    const int i = threadIdx.x - 384;
    const int c = i & 7, rsub = i >> 3;
    uint32_t aph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int img, oy0, ox0;
      coords(tile, img, oy0, ox0);
      for (int kb = 0; kb < HEAD_KB; ++kb) {
        if (!hp.src[kb]) continue;
        const int hs = hp.hs[kb], ws = hp.ws[kb];
        const T* base = reinterpret_cast<const T*>(hp.src[kb]) + static_cast<size_t>(img) * hs * ws * hp.CS + hp.c0[kb] + c * 8;
        const float ry = static_cast<float>(hs) / hp.HO, rx = static_cast<float>(ws) / hp.WO;
        mbar_wait(&aempty_bar[kb], aph ^ 1);
        uint8_t* dst = s_a + kb * A_BYTES;
        // two batches of four pixel rows: 16 independent 16-byte loads in flight per thread before the first blend.  The x / y
        // weights of an integer up-sampling ratio (2, 4, 8) are multiples of 1/16, exact in the 16-bit storage type, so the blend
        // runs on fma16 (exact 16-bit products) of the loaded values: p = lx*b + hx*a, q = lx*d + hx*c (both exact products + one
        // rounding each, identical to the fp32 expression), then hy*p + ly*q in fp32.
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
          uint4 v00[4], v01[4], v10[4], v11[4];
          float lyv[4], lxv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int r = (half * 4 + u) * 16 + rsub;           // tile row = pixel (r / 16, r % 16)
            const int oy = min(oy0 + (r >> 4), hp.HO - 1), ox = min(ox0 + (r & 15), hp.WO - 1);
            // torch upsample_bilinear2d, align_corners=False: src = (dst + 0.5) * (in/out) - 0.5, clamped at 0
            const float sy = fmaxf((oy + 0.5f) * ry - 0.5f, 0.f), sx = fmaxf((ox + 0.5f) * rx - 0.5f, 0.f);
            const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
            const int y1 = y0 + (y0 < hs - 1 ? 1 : 0), x1 = x0 + (x0 < ws - 1 ? 1 : 0);
            lyv[u] = sy - y0; lxv[u] = sx - x0;
            v00[u] = __ldg(reinterpret_cast<const uint4*>(base + (y0 * ws + x0) * hp.CS));
            v01[u] = __ldg(reinterpret_cast<const uint4*>(base + (y0 * ws + x1) * hp.CS));
            v10[u] = __ldg(reinterpret_cast<const uint4*>(base + (y1 * ws + x0) * hp.CS));
            v11[u] = __ldg(reinterpret_cast<const uint4*>(base + (y1 * ws + x1) * hp.CS));
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int r = (half * 4 + u) * 16 + rsub;
            const float ly = lyv[u], lx = lxv[u], hy = 1.f - ly, hx = 1.f - lx;
            const unsigned short lxh = bits_of<T>(from_f<T>(lx)), hxh = bits_of<T>(from_f<T>(hx));
            const unsigned short *e00 = reinterpret_cast<const unsigned short*>(&v00[u]), *e01 = reinterpret_cast<const unsigned short*>(&v01[u]);
            const unsigned short *e10 = reinterpret_cast<const unsigned short*>(&v10[u]), *e11 = reinterpret_cast<const unsigned short*>(&v11[u]);
            uint32_t pk[4];
#pragma unroll
            for (int j = 0; j < 8; j += 2) {
              float o2[2];
#pragma unroll
              for (int jj = 0; jj < 2; ++jj) {
                const float p_ = fma16<T>(lxh, e01[j + jj], fma16<T>(hxh, e00[j + jj], 0.f));
                const float q_ = fma16<T>(lxh, e11[j + jj], fma16<T>(hxh, e10[j + jj], 0.f));
                o2[jj] = __fmaf_rn(ly, q_, __fmul_rn(hy, p_));
              }
              pk[j >> 1] = Pk<T>::pack(o2[0], o2[1]);
            }
            *reinterpret_cast<uint4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(&afull_bar[kb]);
      }
      aph ^= 1;
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers: MMA passes, + shift, round, ReLU, classifier dot, sigmoid
    const int wg = (warp - 4) >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c = (lane & 3) * 2;   // fragment rows r0, r0 + 8; columns 8j + c
    int ws_ = 0; uint32_t wph = 0; uint32_t aph = 0;
    const unsigned short* wc0 = reinterpret_cast<const unsigned short*>(s_cls);
    const unsigned short* wc1 = wc0 + HEAD_N;
    float d[BNP / 2], part[BNP / 2];
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int img, oy0, ox0;
      coords(tile, img, oy0, ox0);
      float dot[2][2] = {{0.f, 0.f}, {0.f, 0.f}};     // [row r0 / r0 + 8][classifier output]
      for (int h = 0; h < PASSES; ++h) {
#pragma unroll
        for (int i = 0; i < BNP / 2; ++i) d[i] = 0.f;
        for (int kb = 0; kb < HEAD_KB; ++kb) {
          if (h == 0) mbar_wait(&afull_bar[kb], aph);
          mbar_wait(&wfull_bar[ws_], wph);
          const uint64_t da = wgmma_desc_k128(smem_u32(s_a + kb * A_BYTES) + wg * 64 * 128);
          const uint64_t db = wgmma_desc_k128(smem_u32(s_w + ws_ * W_BYTES));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) wgmma_m64k16<T, BNP>(part, da + 2 * k, db + 2 * k, k != 0 ? 1u : 0u);
          wgmma_commit();
          wg_promote<BNP>(d, part);
          release(&wempty_bar[ws_]);
          if (h == PASSES - 1) release(&aempty_bar[kb]);
          if (++ws_ == W_STAGES) { ws_ = 0; wph ^= 1; }
        }
#pragma unroll
        for (int jb = 0; jb < BNP / 8; ++jb) {
          const int cb = h * BNP + jb * 8 + c;
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const float x0 = fmaxf(d[4 * jb + 2 * hh] + s_bias[cb], 0.f);
            const float x1 = fmaxf(d[4 * jb + 2 * hh + 1] + s_bias[cb + 1], 0.f);
            const uint32_t pk = Pk<T>::pack(x0, x1);        // rounded to T: what the unfused path stores
            const unsigned short lo = static_cast<unsigned short>(pk & 0xffffu), hi = static_cast<unsigned short>(pk >> 16);
            dot[hh][0] = fma16<T>(lo, wc0[cb], dot[hh][0]);
            dot[hh][1] = fma16<T>(lo, wc1[cb], dot[hh][1]);
            dot[hh][0] = fma16<T>(hi, wc0[cb + 1], dot[hh][0]);
            dot[hh][1] = fma16<T>(hi, wc1[cb + 1], dot[hh][1]);
          }
        }
      }
      aph ^= 1;
      // the four lanes holding a pixel's columns meet in a fixed order
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int o = 0; o < 2; ++o) {
          dot[hh][o] += __shfl_xor_sync(0xffffffffu, dot[hh][o], 1);
          dot[hh][o] += __shfl_xor_sync(0xffffffffu, dot[hh][o], 2);
        }
      if ((lane & 3) == 0) {
        const T* cb_ = reinterpret_cast<const T*>(hp.cls_b);
        T* out = reinterpret_cast<T*>(hp.out);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = r0 + 8 * hh;
          const int oy = oy0 + (row >> 4), ox = ox0 + (row & 15);
          if (oy >= hp.HO || ox >= hp.WO) continue;
          const size_t pix = static_cast<size_t>(oy) * hp.WO + ox;
#pragma unroll
          for (int o = 0; o < 2; ++o) {
            const float v = rnd<T>(dot[hh][o] + to_f<T>(cb_[o]));
            out[(static_cast<size_t>(img) * 2 + o) * HW + pix] = from_f<T>(1.f / (1.f + expf(-v)));
          }
        }
      }
    }
  }
}

bool det_head_fused_ok(int n_src, int CS, int n_out, int cin, int cout, const int* hs, const int* ws, int HO, int WO) {
  static int en = -1;
  if (en < 0) { const char* e = getenv("SB_DET_FUSED_HEAD"); en = (e && e[0] == '0') ? 0 : 1; }
  if (!en || n_src != 4 || CS != 128 || n_out != 2 || cin != 512 || cout != 512) return false;
  int ident = 0;
  for (int i = 0; i < n_src; ++i) {
    if (hs[i] == HO && ws[i] == WO) { ++ident; continue; }
    // integer up-sampling ratios up to 8: the bilinear weights are then multiples of 1/16 (exact in fp16 / bf16, see the builders)
    if (hs[i] <= 0 || ws[i] <= 0 || HO % hs[i] || WO % ws[i]) return false;
    const int fy = HO / hs[i], fx = WO / ws[i];
    if ((fy != 2 && fy != 4 && fy != 8) || (fx != 2 && fx != 4 && fx != 8)) return false;
  }
  return ident == 1;
}

template <typename T>
static int launch_head(const HeadParams& hp, const CUtensorMap& mid, const CUtensorMap& mw, cudaStream_t st) {
  constexpr size_t SMEM = 8 * 16384 + 8 * 8192 + 512 * 4 + 2 * 512 * 2 + 512 + 1024;
  auto kern = head_fused_kernel<T>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess) {
      cudaGetLastError();
      set_error("det_head_fused: cudaFuncSetAttribute(smem=%zu) failed", SMEM);
      return -10;
    }
    attr_set = true;
  }
  const int tiles = hp.B * hp.tiles_x * hp.tiles_y;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  kern<<<grid, 512, SMEM, st>>>(mid, mw, hp);
  return launch_ok();
}

// srcs / hs / ws / ch_off: the four branch maps of the UPCAT op (NHWC, CS channels each, channel offset in the concat order);
// fuse_w: T [512][512] K-major (BN folded), fuse_bias fp32 [512]; cls_w T [2][512], cls_b T [2]; logits T NCHW [B, 2, HO*WO].
int det_head_fused(int dtype, const void* const* srcs, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                   const void* fuse_w, const float* fuse_bias, const void* cls_w, const void* cls_b, void* logits, int B, int HO,
                   int WO, cudaStream_t st) {
  if (B <= 0) return 0;
  if (!det_head_fused_ok(n_src, CS, 2, 512, 512, hs, ws, HO, WO)) { set_error("det_head_fused: unsupported head shape"); return -1; }
  if (!fuse_w || !fuse_bias || !cls_w || !cls_b || !logits) { set_error("det_head_fused: null argument"); return -1; }
  HeadParams hp{};
  const void* ident = nullptr;
  for (int j = 0; j < n_src; ++j) {
    if (ch_off[j] % 64 || ch_off[j] < 0 || ch_off[j] + CS > 512) { set_error("det_head_fused: bad channel offset %d", ch_off[j]); return -1; }
    const bool is_id = hs[j] == HO && ws[j] == WO;
    if (is_id) ident = srcs[j];
    for (int k = 0; k < CS / 64; ++k) {
      const int kb = ch_off[j] / 64 + k;
      hp.src[kb] = is_id ? nullptr : srcs[j];
      hp.hs[kb] = hs[j]; hp.ws[kb] = ws[j]; hp.c0[kb] = k * 64; hp.tma_c0[kb] = k * 64;
    }
  }
  hp.CS = CS; hp.B = B; hp.HO = HO; hp.WO = WO; hp.tiles_x = (WO + 15) / 16; hp.tiles_y = (HO + 7) / 8;
  hp.fuse_bias = fuse_bias; hp.cls_w = cls_w; hp.cls_b = cls_b; hp.out = logits;
  CUtensorMap mid, mw;
  int rc = make_tma_nhwc(&mid, dtype, ident, B, HO, WO, CS, 64, 16, 8, 1, 128);
  if (rc) return rc;
  rc = make_tma_2d(&mw, dtype, fuse_w, 512, 512, 512, 64);
  if (rc) return rc;
  return dtype == DT_BF16 ? launch_head<__nv_bfloat16>(hp, mid, mw, st) : launch_head<__half>(hp, mid, mw, st);
}

}  // namespace sb
