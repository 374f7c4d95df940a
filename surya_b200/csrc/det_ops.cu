// surya_b200 — CUDA-core kernels of the detection path (NHWC fp16/bf16 activations; all HBM-bound).
//
//   stem_conv      Stem.in_conv: 3x3 s2 conv 3->32 + folded BN + Hardswish from the NCHW input
//                  (surya/detection/model/encoderdecoder.py:484-495)
//   dwconv         depthwise k x k conv (+bias, +Hardswish): MBConv.depth_conv (:202-211) and LiteMLA.aggreg[0] (:313-320)
//   lite_mla       ReLU linear attention core, fp32: kv = relu(k)^T [v,1]; out = relu(q) kv; out[:-1]/(out[-1]+eps)
//                  (:332-338, 352-359)
//   upsample_cat   DecodeHead: bilinear(align_corners=False) upsample of the 4 projected maps to the stage-0 size and
//                  channel concat in reversed order (:703-716)
//   classifier     1x1 conv 512->2 + bias + sigmoid, NCHW output (:720, :747)
//   upsample_nchw  DetectionPredictor's x4 bilinear upsample to fp32 (surya/detection/__init__.py:120-132)
#include "gemm_epilogue.cuh"
#include "ops.cuh"
#include "sb_ptx.cuh"

#include <cstdlib>

namespace sb {

// x * min(max(x + 3, 0), 6) * (1/6) in fp32: the expression of ATen's CUDA kernel (ActivationHardswishKernel.cu) and of the GEMM
// epilogue (act_ct<ACT_HARDSWISH>).  Round 1 divided by 6 here (ATen's CPU form): a true fp32 division is ~8 instructions plus a
// slow-path call per value, which made the epilogue of the depthwise kernel twice as long as its convolution.
__device__ __forceinline__ float hardswish_f(float x) { return x * fminf(fmaxf(x + 3.0f, 0.0f), 6.0f) * (1.0f / 6.0f); }

// ------------------------------------------------------------------------------------------------ stem conv
// in: NCHW [B,3,H,W] (T or float); w: fp32 [32][r][s][c] (27 per output channel, BN folded); out NHWC [B,H/2,W/2,CO].
template <typename T, typename InT, int CO>
__global__ void __launch_bounds__(128) stem_conv_kernel(const InT* __restrict__ in, const float* __restrict__ w,
                                                        const float* __restrict__ bias, T* __restrict__ out, int H, int W) {
  // weights transposed to [27 taps][CO] so one LDS.128 feeds four output channels of a tap (broadcast across the warp)
  __shared__ __align__(16) float sw[27][CO];
  __shared__ __align__(16) float sb_[CO];
  for (int i = threadIdx.x; i < CO * 27; i += blockDim.x) sw[i % 27][i / 27] = w[i];
  for (int i = threadIdx.x; i < CO; i += blockDim.x) sb_[i] = bias[i];
  __syncthreads();
  const int Ho = H >> 1, Wo = W >> 1;
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y, b = blockIdx.z;
  if (ox >= Wo) return;
  float x[27];
  const InT* img = in + static_cast<size_t>(b) * 3 * H * W;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = oy * 2 + r - 1;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ix = ox * 2 + s - 1;
      const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = 0.f;
        if (ok) {
          const InT* p = img + (static_cast<size_t>(c) * H + iy) * W + ix;
          if constexpr (sizeof(InT) == 4) v = rnd<T>(static_cast<float>(*p));  // .to(model dtype) of the pixel batch
          else v = to_f<InT>(*p);
        }
        x[(r * 3 + s) * 3 + c] = v;
      }
    }
  }
  float acc[CO];
#pragma unroll
  for (int j = 0; j < CO; ++j) acc[j] = sb_[j];
#pragma unroll
  for (int k = 0; k < 27; ++k) {
#pragma unroll
    for (int j4 = 0; j4 < CO / 4; ++j4) {
      const float4 w4 = *reinterpret_cast<const float4*>(&sw[k][j4 * 4]);
      acc[j4 * 4 + 0] += x[k] * w4.x; acc[j4 * 4 + 1] += x[k] * w4.y; acc[j4 * 4 + 2] += x[k] * w4.z; acc[j4 * 4 + 3] += x[k] * w4.w;
    }
    if ((k & 3) == 3) asm volatile("" ::: "memory");   // bound the number of hoisted weight loads
  }
  T* o = out + ((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * CO;
#pragma unroll
  for (int co8 = 0; co8 < CO; co8 += 8) {
    uint4 pack;
    T* pe = reinterpret_cast<T*>(&pack);
#pragma unroll
    for (int j = 0; j < 8; ++j) pe[j] = from_f<T>(hardswish_f(rnd<T>(acc[co8 + j])));
    *reinterpret_cast<uint4*>(o + co8) = pack;
  }
}

int det_stem_conv(int dtype, const void* in, int in_f32, const float* w, const float* bias, void* out, int B, int H,
                  int W, int cout, cudaStream_t st) {
  if (cout != 32) { set_error("det_stem_conv: only 32 output channels are instantiated (got %d)", cout); return -1; }
  if ((H | W) & 1) { set_error("det_stem_conv: H and W must be even"); return -1; }
  if (B > 65535 || H / 2 > 65535) { set_error("det_stem_conv: batch / height too large for the grid"); return -1; }
  dim3 grid((W / 2 + 127) / 128, H / 2, B);
  if (dtype == DT_F16) {
    if (in_f32) stem_conv_kernel<__half, float, 32><<<grid, 128, 0, st>>>((const float*)in, w, bias, (__half*)out, H, W);
    else stem_conv_kernel<__half, __half, 32><<<grid, 128, 0, st>>>((const __half*)in, w, bias, (__half*)out, H, W);
  } else {
    if (in_f32) stem_conv_kernel<__nv_bfloat16, float, 32><<<grid, 128, 0, st>>>((const float*)in, w, bias, (__nv_bfloat16*)out, H, W);
    else stem_conv_kernel<__nv_bfloat16, __nv_bfloat16, 32><<<grid, 128, 0, st>>>((const __nv_bfloat16*)in, w, bias, (__nv_bfloat16*)out, H, W);
  }
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ depthwise conv
// in NHWC [B,H,W,C]; w: T [k*k][C] (tap-major); bias fp32 [C] or null.
// CTA = 32 output columns x 8 channel vectors (64 channels = one 128 B line per pixel); every thread owns 8 channels of one
// output column and walks TY output rows with the k x k weights in registers, so each input row it touches is loaded once per
// column instead of once per tap row (L1 absorbs the overlap between neighbouring columns).  fp32 accumulation in tap order
// (r, s) — the same order as a direct per-pixel loop; the multiply-adds take the 16-bit operands as loaded (sb_ptx.cuh fma16).
// A shared-memory-tiled, double-buffered persistent variant (cp.async halo tiles, 2 CTAs/SM) was slower and dropped (git
// history: "shared-memory tiled ... depthwise 3x3"): the kernel is not bound by the L1 re-fetch of neighbouring columns.
template <typename T, int KS, int STRIDE, int TY>
__global__ void __launch_bounds__(256, 2) dwconv_kernel(const T* __restrict__ in, const T* __restrict__ w,
                                                        const float* __restrict__ bias, T* __restrict__ out, int H, int W, int C,
                                                        int Ho, int Wo, int pad, int act, int c_blocks, int groups_per_cta) {
  constexpr int ROWS = (TY - 1) * STRIDE + KS;
  const int cvec = threadIdx.x & 7, xl = threadIdx.x >> 3;
  const int cb = blockIdx.x % c_blocks, xb = blockIdx.x / c_blocks;
  const int c8 = (cb * 8 + cvec) * 8;
  const int ox = xb * 32 + xl;
  const int b = blockIdx.z;
  __shared__ uint4 wsm[KS * KS][8];
  for (int i = threadIdx.x; i < KS * KS * 8; i += 256) {
    const int t = i >> 3, cv = i & 7, cc = (cb * 8 + cv) * 8;
    wsm[t][cv] = cc < C ? *reinterpret_cast<const uint4*>(w + static_cast<size_t>(t) * C + cc) : make_uint4(0u, 0u, 0u, 0u);
  }
  const bool active = c8 < C && ox < Wo;
  const T* img = in + static_cast<size_t>(b) * H * W * C + (active ? c8 : 0);
  const int ix0 = ox * STRIDE - pad;
  // each CTA walks `groups_per_cta` consecutive groups of TY output rows: the weight staging and CTA launch are paid once and
  // the second CTA resident on the SM computes while this one waits for its loads
  for (int gi = 0; gi < groups_per_cta; ++gi) {
    const int oy0 = (blockIdx.y * groups_per_cta + gi) * TY;
    if (oy0 >= Ho) break;
    const int iy0 = oy0 * STRIDE - pad;
    constexpr bool PRELOAD = KS == 3;    // 3x3: issue every load of the group up front; 5x5: stream rows (register budget)
    constexpr int PR = PRELOAD ? ROWS : 1;
    uint4 xv[PR][KS];
    auto load_row = [&](int rr, uint4 (&dst)[KS]) {
      const int iy = iy0 + rr;
      const bool row_ok = active && iy >= 0 && iy < H;
#pragma unroll
      for (int s_ = 0; s_ < KS; ++s_) {
        const int ix = ix0 + s_;
        dst[s_] = make_uint4(0u, 0u, 0u, 0u);
        if (row_ok && ix >= 0 && ix < W) dst[s_] = *reinterpret_cast<const uint4*>(img + (static_cast<size_t>(iy) * W + ix) * C);
      }
    };
    if constexpr (PRELOAD) {
#pragma unroll
      for (int rr = 0; rr < ROWS; ++rr) load_row(rr, xv[rr]);
    }
    if (gi == 0) __syncthreads();        // weights staged (the first group's loads are already in flight)
    float acc[TY][8];
#pragma unroll
    for (int y = 0; y < TY; ++y)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[y][j] = 0.f;
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {
      if constexpr (!PRELOAD) load_row(rr, xv[0]);
#pragma unroll
      for (int y = 0; y < TY; ++y) {
        const int r = rr - y * STRIDE;          // tap row of output row y that reads input row rr (compile-time after unrolling)
        if (r < 0 || r >= KS) continue;
#pragma unroll
        for (int s_ = 0; s_ < KS; ++s_) {
          const unsigned short* xe = reinterpret_cast<const unsigned short*>(&xv[PRELOAD ? rr : 0][s_]);
          const uint4 wq = wsm[r * KS + s_][cvec];
          const unsigned short* we = reinterpret_cast<const unsigned short*>(&wq);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[y][j] = fma16<T>(xe[j], we[j], acc[y][j]);    // FHFMA: no conversions
        }
      }
    }
    if (active) {
      float bv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) bv[j] = bias ? __ldg(bias + c8 + j) : 0.f;
#pragma unroll
      for (int y = 0; y < TY; ++y) {
        const int oy = oy0 + y;
        if (oy >= Ho) break;
        uint32_t pk[4];                              // pairwise conversions: one F2FP per two values and rounding point
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          uint32_t t = Pk<T>::pack(acc[y][j] + bv[j], acc[y][j + 1] + bv[j + 1]);
          if (act == ACT_HARDSWISH) t = Pk<T>::pack(hardswish_f(Pk<T>::lo(t)), hardswish_f(Pk<T>::hi(t)));
          pk[j >> 1] = t;
        }
        *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * C + c8) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      }
    }
  }
}

template <typename T, int KS, int STRIDE, int TY>
static void launch_dw(const void* in, const void* w, const float* bias, void* out, int B, int H, int W, int C, int Ho, int Wo,
                      int pad, int act, cudaStream_t st) {
  const int c_blocks = (C + 63) / 64;
  const int gx = c_blocks * ((Wo + 31) / 32);
  const int groups = (Ho + TY - 1) / TY;
  // keep >= ~8 CTAs per SM in the grid, otherwise walk up to 4 row groups per CTA
  int per = 4;
  while (per > 1 && static_cast<long long>(gx) * ((groups + per - 1) / per) * B < 8LL * num_sms()) per >>= 1;
  dim3 grid(gx, (groups + per - 1) / per, B);
  dwconv_kernel<T, KS, STRIDE, TY><<<grid, 256, 0, st>>>((const T*)in, (const T*)w, bias, (T*)out, H, W, C, Ho, Wo, pad, act, c_blocks,
                                                         per);
}

int det_dwconv(int dtype, const void* in, const void* w, const float* bias, void* out, int B, int H, int W, int C, int ks,
               int stride, int pad, int act, cudaStream_t st) {
  if (C % 8) { set_error("det_dwconv: C must be a multiple of 8"); return -1; }
  if (B > 65535) { set_error("det_dwconv: batch too large for the grid"); return -1; }
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  if (Ho <= 0 || Wo <= 0) return 0;
#define DW(T_) \
  do { \
    if (ks == 3 && stride == 1) launch_dw<T_, 3, 1, 4>(in, w, bias, out, B, H, W, C, Ho, Wo, pad, act, st); \
    else if (ks == 3 && stride == 2) launch_dw<T_, 3, 2, 2>(in, w, bias, out, B, H, W, C, Ho, Wo, pad, act, st); \
    else if (ks == 5 && stride == 1) launch_dw<T_, 5, 1, 2>(in, w, bias, out, B, H, W, C, Ho, Wo, pad, act, st); \
    else if (ks == 5 && stride == 2) launch_dw<T_, 5, 2, 1>(in, w, bias, out, B, H, W, C, Ho, Wo, pad, act, st); \
    else { set_error("det_dwconv: kernel size 3 or 5, stride 1 or 2"); return -1; } \
  } while (0)
  if (dtype == DT_F16) DW(__half); else DW(__nv_bfloat16);
#undef DW
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ LiteMLA core
// qkv_a / qkv_b: token-major [B*HW, 3*heads*DIM] (plain qkv and aggregated qkv); head h of scale s reads channels
// [h*3*DIM, (h+1)*3*DIM) = (q | k | v).  out: [B*HW, 2*heads*DIM], channel = (s*heads + h)*DIM + d.
// One CTA per (image, scale*heads + h).  fp32 throughout; rounded to T once at the end (reference: .float() ... .to(dtype)).
// Tiling (a first version was shared-memory bound: 2.5 FMA per LDS in phase 1 and one broadcast LDS.128 per 4 FMA in phase 2):
//   phase 1  kv[i][j] = sum_t relu(k[t][i]) * [v[t] | 1][j]: thread = (2 rows i, 8 columns j, one quarter of each token tile):
//            3 shared loads per 18 FMA; the four token-quarters meet in shared memory in a fixed order;
//   phase 2  out[t] = relu(q[t]) kv: thread = (4 tokens, 8 columns): 2 LDS.128 + 1 LDS.32 per 36 FMA; every thread also carries
//            the denominator column of its tokens, and multiplies by 1 / (den + eps) (one division per token instead of 32).
template <typename T, int DIM>
__global__ void __launch_bounds__(256, 2) lite_mla_kernel(const T* __restrict__ qkv_a, const T* __restrict__ qkv_b,
                                                       T* __restrict__ out, int HW, int heads, float eps) {
  static_assert(DIM == 32, "thread mapping below assumes 32-wide heads");
  constexpr int DVP = 36;                       // 33 columns (v | ones) padded to a float4 multiple
  constexpr int TT = 64;                        // tokens staged per tile
  __shared__ __align__(16) float kv[DIM * DVP];
  __shared__ __align__(16) float tk[TT][DIM];
  __shared__ __align__(16) float tv[TT][DIM];
  __shared__ __align__(16) float part[4][DIM * DVP];
  const int b = blockIdx.x, hh = blockIdx.y;
  const int scale = hh / heads, h = hh % heads;
  const int ld = 3 * heads * DIM;
  const T* src = (scale == 0 ? qkv_a : qkv_b) + static_cast<size_t>(b) * HW * ld + h * 3 * DIM;
  const int tid = threadIdx.x;
  // ---- phase 1
  const int tq = tid >> 6, ip = (tid & 63) >> 2, jq = tid & 3;
  float acc0[8], acc1[8], ones0 = 0.f, ones1 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
  for (int t0 = 0; t0 < HW; t0 += TT) {
    __syncthreads();
#pragma unroll
    for (int rep = 0; rep < (TT * 8) / 256; ++rep) {
      const int i = tid + rep * 256;
      const int t = i >> 3, pt = i & 7;          // parts 0..3 = k, 4..7 = v (k | v are 128 contiguous bytes per token)
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if (t0 + t < HW) u = *reinterpret_cast<const uint4*>(src + static_cast<size_t>(t0 + t) * ld + DIM + pt * 8);
      const T* e = reinterpret_cast<const T*>(&u);
      float f[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = to_f<T>(e[j]);
      if (pt < 4) {
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
      }
      float* dstp = pt < 4 ? &tk[t][pt * 8] : &tv[t][(pt - 4) * 8];
      *reinterpret_cast<float4*>(dstp) = make_float4(f[0], f[1], f[2], f[3]);
      *reinterpret_cast<float4*>(dstp + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
    __syncthreads();
#pragma unroll 4
    for (int tt = 0; tt < TT / 4; ++tt) {        // rows past HW were staged as zeros
      const int t = tq * (TT / 4) + tt;
      const float2 kx = *reinterpret_cast<const float2*>(&tk[t][2 * ip]);
      const float4 va = *reinterpret_cast<const float4*>(&tv[t][8 * jq]);
      const float4 vb = *reinterpret_cast<const float4*>(&tv[t][8 * jq + 4]);
      const float vv[8] = {va.x, va.y, va.z, va.w, vb.x, vb.y, vb.z, vb.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) { acc0[j] += kx.x * vv[j]; acc1[j] += kx.y * vv[j]; }
      ones0 += kx.x;
      ones1 += kx.y;
    }
  }
  {
    float* p0 = &part[tq][(2 * ip) * DVP + 8 * jq];
    float* p1 = p0 + DVP;
    *reinterpret_cast<float4*>(p0) = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
    *reinterpret_cast<float4*>(p0 + 4) = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
    *reinterpret_cast<float4*>(p1) = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
    *reinterpret_cast<float4*>(p1 + 4) = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
    if (jq == 0) {
      float* o0 = &part[tq][(2 * ip) * DVP + DIM];
      *reinterpret_cast<float4*>(o0) = make_float4(ones0, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(o0 + DVP) = make_float4(ones1, 0.f, 0.f, 0.f);
    }
  }
  __syncthreads();
  for (int e = tid; e < DIM * DVP; e += 256) kv[e] = ((part[0][e] + part[1][e]) + part[2][e]) + part[3][e];
  __syncthreads();
  // ---- phase 2
  T* dst = out + static_cast<size_t>(b) * HW * (2 * heads * DIM) + (scale * heads + h) * DIM;
  const int ldo = 2 * heads * DIM;
  const int js = tid & 3;
  for (int g = tid >> 2; g * 4 < HW; g += 64) {
    const int t0 = g * 4;
    float oa[4][8], den[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      den[k] = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) oa[k][j] = 0.f;
    }
#pragma unroll 1
    for (int c = 0; c < DIM / 8; ++c) {
      uint4 qv[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int t = min(t0 + k, HW - 1);
        qv[k] = *reinterpret_cast<const uint4*>(src + static_cast<size_t>(t) * ld + c * 8);
      }
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        const int i = c * 8 + ii;
        const float4 ka = *reinterpret_cast<const float4*>(&kv[i * DVP + 8 * js]);
        const float4 kb = *reinterpret_cast<const float4*>(&kv[i * DVP + 8 * js + 4]);
        const float kd = kv[i * DVP + DIM];
        const float kk[8] = {ka.x, ka.y, ka.z, ka.w, kb.x, kb.y, kb.z, kb.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float x = fmaxf(to_f<T>(reinterpret_cast<const T*>(&qv[k])[ii]), 0.f);
#pragma unroll
          for (int j = 0; j < 8; ++j) oa[k][j] += x * kk[j];
          den[k] += x * kd;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (t0 + k >= HW) break;
      const float r = 1.0f / (den[k] + eps);
      uint4 pa;
      T* ea = reinterpret_cast<T*>(&pa);
#pragma unroll
      for (int j = 0; j < 8; ++j) ea[j] = from_f<T>(oa[k][j] * r);
      *reinterpret_cast<uint4*>(dst + static_cast<size_t>(t0 + k) * ldo + 8 * js) = pa;
    }
  }
}

int det_lite_mla(int dtype, const void* qkv_a, const void* qkv_b, void* out, int B, int HW, int heads, int dim, float eps,
                 cudaStream_t st) {
  if (dim != 32) { set_error("det_lite_mla: head dim 32 is instantiated (got %d)", dim); return -1; }
  dim3 grid(B, 2 * heads), block(256);
  if (dtype == DT_F16)
    lite_mla_kernel<__half, 32><<<grid, block, 0, st>>>((const __half*)qkv_a, (const __half*)qkv_b, (__half*)out, HW, heads, eps);
  else
    lite_mla_kernel<__nv_bfloat16, 32><<<grid, block, 0, st>>>((const __nv_bfloat16*)qkv_a, (const __nv_bfloat16*)qkv_b,
                                                               (__nv_bfloat16*)out, HW, heads, eps);
  return launch_ok();
}

// bilinear blend with a pinned operation order (no compiler-chosen FMA contraction): the decode-head up-sampler, the fp32
// up-sampler and the post-processing front half must produce the same bits, and so must the fused head's builders
// (det_head.cu), which evaluate this expression for the integer ratios whose weights are exact in the 16-bit type
__device__ __forceinline__ float bilerp(float hy, float ly, float hx, float lx, float a, float b, float c, float d) {
  const float p = __fmaf_rn(lx, b, __fmul_rn(hx, a));
  const float q = __fmaf_rn(lx, d, __fmul_rn(hx, c));
  return __fmaf_rn(ly, q, __fmul_rn(hy, p));
}

// ------------------------------------------------------------------------------------------------ decode-head upsample + concat
// src maps NHWC [B, hs, ws, CS]; dst NHWC [B, HO, WO, n_src*CS], map i written at channel offset ch_off[i].
struct UpcatParams {
  const void* src[4];
  int hs[4], ws[4], ch_off[4];
  int n_src, CS, HO, WO, B;
};

constexpr int UPCAT_ROWS = 4;   // output rows per thread: 16 independent 16-byte loads in flight, one 16-byte store per row

template <typename T>
__global__ void __launch_bounds__(256) upsample_cat_kernel(const UpcatParams p, T* __restrict__ dst) {
  const int cv = p.CS >> 3;
  const int CT = p.n_src * p.CS;
  const int t = blockIdx.x * 256 + threadIdx.x;        // (ox, source, channel vector) within one output row
  if (t >= p.WO * p.n_src * cv) return;
  const int c8 = (t % cv) * 8;
  const int r = t / cv;
  const int si = r % p.n_src, ox = r / p.n_src;
  const int oy0 = blockIdx.y * UPCAT_ROWS, b = blockIdx.z;
  const T* src = reinterpret_cast<const T*>(p.src[si]);
  const int hs = p.hs[si], ws = p.ws[si];
  T* drow = dst + (static_cast<size_t>(b) * p.HO * p.WO + ox) * CT + p.ch_off[si] + c8;
  if (hs == p.HO && ws == p.WO) {
    uint4 v[UPCAT_ROWS];
#pragma unroll
    for (int y = 0; y < UPCAT_ROWS; ++y)
      if (oy0 + y < p.HO) v[y] = *reinterpret_cast<const uint4*>(src + ((static_cast<size_t>(b) * hs + oy0 + y) * ws + ox) * p.CS + c8);
#pragma unroll
    for (int y = 0; y < UPCAT_ROWS; ++y)
      if (oy0 + y < p.HO) *reinterpret_cast<uint4*>(drow + static_cast<size_t>(oy0 + y) * p.WO * CT) = v[y];
    return;
  }
  // torch upsample_bilinear2d, align_corners=False: src = (dst + 0.5) * (in/out) - 0.5, clamped at 0
  const float sx = fmaxf((ox + 0.5f) * (static_cast<float>(ws) / p.WO) - 0.5f, 0.f);
  const int x0 = static_cast<int>(sx);
  const int x1 = x0 + (x0 < ws - 1 ? 1 : 0);
  const float lx = sx - x0, hx = 1.f - lx;
  const T* base = src + static_cast<size_t>(b) * hs * ws * p.CS + c8;
  uint4 v00[UPCAT_ROWS], v01[UPCAT_ROWS], v10[UPCAT_ROWS], v11[UPCAT_ROWS];
  float ly[UPCAT_ROWS];
#pragma unroll
  for (int y = 0; y < UPCAT_ROWS; ++y) {
    const int oy = min(oy0 + y, p.HO - 1);
    const float sy = fmaxf((oy + 0.5f) * (static_cast<float>(hs) / p.HO) - 0.5f, 0.f);
    const int y0 = static_cast<int>(sy);
    const int y1 = y0 + (y0 < hs - 1 ? 1 : 0);
    ly[y] = sy - y0;
    v00[y] = *reinterpret_cast<const uint4*>(base + (y0 * ws + x0) * p.CS);
    v01[y] = *reinterpret_cast<const uint4*>(base + (y0 * ws + x1) * p.CS);
    v10[y] = *reinterpret_cast<const uint4*>(base + (y1 * ws + x0) * p.CS);
    v11[y] = *reinterpret_cast<const uint4*>(base + (y1 * ws + x1) * p.CS);
  }
#pragma unroll
  for (int y = 0; y < UPCAT_ROWS; ++y) {
    if (oy0 + y >= p.HO) break;
    const float hy = 1.f - ly[y];
    const T *e00 = reinterpret_cast<const T*>(&v00[y]), *e01 = reinterpret_cast<const T*>(&v01[y]);
    const T *e10 = reinterpret_cast<const T*>(&v10[y]), *e11 = reinterpret_cast<const T*>(&v11[y]);
    uint4 pack;
    T* pe = reinterpret_cast<T*>(&pack);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      pe[j] = from_f<T>(bilerp(hy, ly[y], hx, lx, to_f<T>(e00[j]), to_f<T>(e01[j]), to_f<T>(e10[j]), to_f<T>(e11[j])));
    }
    *reinterpret_cast<uint4*>(drow + static_cast<size_t>(oy0 + y) * p.WO * CT) = pack;
  }
}

int det_upsample_cat(int dtype, const void* const* src, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                     void* dst, int B, int HO, int WO, cudaStream_t st) {
  if (n_src > 4 || CS % 8) { set_error("det_upsample_cat: at most 4 sources, CS multiple of 8"); return -1; }
  UpcatParams p;
  for (int i = 0; i < n_src; ++i) { p.src[i] = src[i]; p.hs[i] = hs[i]; p.ws[i] = ws[i]; p.ch_off[i] = ch_off[i]; }
  p.n_src = n_src; p.CS = CS; p.HO = HO; p.WO = WO; p.B = B;
  if (B > 65535 || HO > 65535) { set_error("det_upsample_cat: batch / height too large for the grid"); return -1; }
  dim3 grid((WO * n_src * (CS / 8) + 255) / 256, (HO + UPCAT_ROWS - 1) / UPCAT_ROWS, B);
  if (dtype == DT_F16) upsample_cat_kernel<__half><<<grid, 256, 0, st>>>(p, (__half*)dst);
  else upsample_cat_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(p, (__nv_bfloat16*)dst);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ classifier + sigmoid
// x NHWC [P, C]; w T [n_out][C]; b T [n_out]; out NCHW [B, n_out, HW] T: sigmoid(T(x.w + b)); one warp per pixel.
template <typename T, int NOUT>
__global__ void __launch_bounds__(256) classifier_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                         const T* __restrict__ b, T* __restrict__ out, long long P,
                                                         int C, int HW) {
  const long long pix = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (pix >= P) return;
  const T* xr = x + pix * C;
  float acc[NOUT];
#pragma unroll
  for (int o = 0; o < NOUT; ++o) acc[o] = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    const uint4 xv = *reinterpret_cast<const uint4*>(xr + c);
    const unsigned short* xe = reinterpret_cast<const unsigned short*>(&xv);
#pragma unroll
    for (int o = 0; o < NOUT; ++o) {
      const uint4 wv = *reinterpret_cast<const uint4*>(w + static_cast<size_t>(o) * C + c);
      const unsigned short* we = reinterpret_cast<const unsigned short*>(&wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[o] = fma16<T>(xe[j], we[j], acc[o]);
    }
  }
#pragma unroll
  for (int o = 0; o < NOUT; ++o) acc[o] = warp_sum(acc[o]);
  if (lane == 0) {
    const long long bimg = pix / HW, hw = pix % HW;
#pragma unroll
    for (int o = 0; o < NOUT; ++o) {
      float v = rnd<T>(acc[o] + to_f<T>(b[o]));
      out[(bimg * NOUT + o) * HW + hw] = from_f<T>(1.f / (1.f + expf(-v)));
    }
  }
}

int det_classifier(int dtype, const void* x, const void* w, const void* b, void* out, long long P, int C, int HW, int n_out,
                   cudaStream_t st) {
  if (n_out != 2 || C % 8) { set_error("det_classifier: 2 labels and C %% 8 == 0 are instantiated"); return -1; }
  const int grid = static_cast<int>((P + 7) / 8);
  if (dtype == DT_F16)
    classifier_kernel<__half, 2><<<grid, 256, 0, st>>>((const __half*)x, (const __half*)w, (const __half*)b, (__half*)out, P, C, HW);
  else
    classifier_kernel<__nv_bfloat16, 2><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w,
                                                              (const __nv_bfloat16*)b, (__nv_bfloat16*)out, P, C, HW);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ x4 bilinear to fp32 (NCHW)
template <typename T>
__global__ void __launch_bounds__(256) upsample_nchw_kernel(const T* __restrict__ in, float* __restrict__ out, int hs, int ws,
                                                            int HO, int WO) {
  // one thread = 4 consecutive output columns of row blockIdx.y in plane blockIdx.z (float4 store when WO % 4 == 0)
  const int ox0 = (blockIdx.x * 256 + threadIdx.x) * 4;
  if (ox0 >= WO) return;
  const int oy = blockIdx.y, pl = blockIdx.z;
  const float sy = fmaxf((oy + 0.5f) * (static_cast<float>(hs) / HO) - 0.5f, 0.f);
  const int y0 = static_cast<int>(sy);
  const int y1 = y0 + (y0 < hs - 1 ? 1 : 0);
  const float ly = sy - y0, hy = 1.f - ly;
  const T* r0 = in + (static_cast<size_t>(pl) * hs + y0) * ws;
  const T* r1 = in + (static_cast<size_t>(pl) * hs + y1) * ws;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int ox = min(ox0 + j, WO - 1);
    const float sx = fmaxf((ox + 0.5f) * (static_cast<float>(ws) / WO) - 0.5f, 0.f);
    const int x0 = static_cast<int>(sx);
    const int x1 = x0 + (x0 < ws - 1 ? 1 : 0);
    const float lx = sx - x0, hx = 1.f - lx;
    const float t = bilerp(hy, ly, hx, lx, to_f<T>(r0[x0]), to_f<T>(r0[x1]), to_f<T>(r1[x0]), to_f<T>(r1[x1]));
    v[j] = rnd<T>(t);  // F.interpolate runs in the model dtype; .float() afterwards
  }
  float* o = out + (static_cast<size_t>(pl) * HO + oy) * WO + ox0;
  if ((WO & 3) == 0) {
    *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (ox0 + j < WO) o[j] = v[j];
  }
}

int det_upsample_nchw(int dtype, const void* in, float* out, int planes, int hs, int ws, int HO, int WO, cudaStream_t st) {
  if (planes <= 0) return 0;
  if (planes > 65535 || HO > 65535) { set_error("det_upsample_nchw: too many planes / rows for the grid"); return -1; }
  dim3 grid((WO + 1023) / 1024, HO, planes);
  if (dtype == DT_F16) upsample_nchw_kernel<__half><<<grid, 256, 0, st>>>((const __half*)in, out, hs, ws, HO, WO);
  else upsample_nchw_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)in, out, hs, ws, HO, WO);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ uint8 pages -> network input
// SegformerImageProcessor on the device (surya/detection/processor.py:94-95, 126-146): x = (u8 * (1/255) - mean) / std in fp32,
// NHWC uint8 -> NCHW engine dtype.  Pages cross PCIe as 3 bytes per pixel instead of 6 (fp16) or 12 (fp32).
template <typename T>
__global__ void __launch_bounds__(256) det_normalize_u8_kernel(const unsigned char* __restrict__ in, T* __restrict__ out, long long HW) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= HW) return;
  const int b = blockIdx.y;
  const unsigned char* px = in + (static_cast<size_t>(b) * HW + i) * 3;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = __fdiv_rn(__fsub_rn(__fmul_rn(static_cast<float>(px[c]), 1.0f / 255.0f), mean[c]), stdv[c]);
    out[(static_cast<size_t>(b) * 3 + c) * HW + i] = from_f<T>(v);
  }
}

int det_normalize_u8(int dtype, const unsigned char* in, void* out, int B, int H, int W, cudaStream_t st) {
  if (B <= 0) return 0;
  if (B > 65535) { set_error("det_normalize_u8: too many pages for the grid"); return -1; }
  const long long HW = static_cast<long long>(H) * W;
  dim3 grid(static_cast<unsigned int>((HW + 255) / 256), B);
  if (dtype == DT_F16) det_normalize_u8_kernel<__half><<<grid, 256, 0, st>>>(in, (__half*)out, HW);
  else det_normalize_u8_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(in, (__nv_bfloat16*)out, HW);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ post-processing front half
// Device side of DetectionPredictor.batch_detection's tail + get_dynamic_thresholds + the binarisation of detect_boxes
// (surya/detection/__init__.py:120-132, surya/detection/heatmap.py:14-24, 33): for the TEXT channel of every page
//   line  = F.interpolate(logits, (HO, WO), bilinear).float()        (values are the model-dtype roundings, kept as 16-bit)
//   avg   = mean of the n - int(0.9 n) largest pixels               (np.partition in the reference)
//   sf    = clip(avg / 0.7, 0, 1) ** 0.5 ; low = clip(low_text * sf, 0.1, 0.6) ; tt = clip(text_threshold * sf, 0.15, 0.8)
//   mask  = line > low                                              (uint8, what cv2.connectedComponentsWithStats consumes)
// Because the up-sampled values are 16-bit floats in [0, 1], the top-10 % mean is EXACT from a histogram over the bit
// pattern (<= 15 361 bins for fp16, <= 16 257 for bf16): no sort, no selection passes.  The host receives 3 bytes per pixel
// (16-bit map + mask) instead of 8 (two fp32 channels) and no longer runs np.partition over a megapixel per page.
constexpr int FRONT_BINS = 16384;

template <typename T>
__device__ __forceinline__ unsigned short bits16(float v) {
  T t = from_f<T>(v);
  return *reinterpret_cast<unsigned short*>(&t);
}

// chunk_tab (optional, int32 [n_chunks, 4]): chunk c = blockIdx.y belongs to page chunk_tab[c][0] and writes its first
// chunk_tab[c][2] rows at row chunk_tab[c][1] of the packed stitched map; without it chunk c is page c at row c * HO.
template <typename T>
__global__ void __launch_bounds__(256) det_front_map_kernel(const T* __restrict__ logits, int plane_stride, T* __restrict__ map,
                                                            unsigned int* __restrict__ hist, int hs, int ws, int HO, int WO,
                                                            int rows_per_block, const int* __restrict__ chunk_tab) {
  // block = rows_per_block output rows of chunk blockIdx.y; thread = 4 consecutive columns at a time
  extern __shared__ unsigned int sh[];
  for (int i = threadIdx.x; i < FRONT_BINS; i += 256) sh[i] = 0u;
  __syncthreads();
  const int ch = blockIdx.y;
  const int pg = chunk_tab ? chunk_tab[ch * 4 + 0] : ch;
  const int row0 = chunk_tab ? chunk_tab[ch * 4 + 1] : ch * HO;
  const int rows = chunk_tab ? chunk_tab[ch * 4 + 2] : HO;
  const T* in = logits + static_cast<size_t>(ch) * plane_stride;
  const int oy0 = blockIdx.x * rows_per_block;
  for (int r = 0; r < rows_per_block; ++r) {
    const int oy = oy0 + r;
    if (oy >= rows) break;
    const float sy = fmaxf((oy + 0.5f) * (static_cast<float>(hs) / HO) - 0.5f, 0.f);
    const int y0 = static_cast<int>(sy);
    const int y1 = y0 + (y0 < hs - 1 ? 1 : 0);
    const float ly = sy - y0, hy = 1.f - ly;
    const T* r0 = in + static_cast<size_t>(y0) * ws;
    const T* r1 = in + static_cast<size_t>(y1) * ws;
    T* orow = map + (static_cast<size_t>(row0) + oy) * WO;
    for (int ox = threadIdx.x; ox < WO; ox += 256) {
      const float sx = fmaxf((ox + 0.5f) * (static_cast<float>(ws) / WO) - 0.5f, 0.f);
      const int x0 = static_cast<int>(sx);
      const int x1 = x0 + (x0 < ws - 1 ? 1 : 0);
      const float lx = sx - x0, hx = 1.f - lx;
      // same expression as upsample_nchw_kernel: the two paths must agree bit for bit
      const float t = bilerp(hy, ly, hx, lx, to_f<T>(r0[x0]), to_f<T>(r0[x1]), to_f<T>(r1[x0]), to_f<T>(r1[x1]));
      const T o = from_f<T>(t);
      orow[ox] = o;
      unsigned short b = *reinterpret_cast<const unsigned short*>(&o);
      if (b & 0x8000u) b = 0;                        // -0 / negatives cannot come out of a sigmoid; keep the index in range
      atomicAdd(&sh[b < FRONT_BINS ? b : FRONT_BINS - 1], 1u);
    }
  }
  __syncthreads();
  unsigned int* gh = hist + static_cast<size_t>(pg) * FRONT_BINS;
  for (int i = threadIdx.x; i < FRONT_BINS; i += 256)
    if (sh[i]) atomicAdd(&gh[i], sh[i]);
}

// page_tab (optional, int32 [B, 2]): page b spans page_tab[b][1] rows of WO pixels from row page_tab[b][0] of the packed map;
// without it every page has n_pix pixels from pixel b * n_pix.
template <typename T>
__global__ void __launch_bounds__(256) det_front_threshold_kernel(unsigned int* __restrict__ hist, float* __restrict__ thr,
                                                                  long long n_pix, float text_threshold, float low_text,
                                                                  float typical, const int* __restrict__ page_tab, int WO) {
  // one block per page: walk the histogram from the top bin down until n - int(0.9 n) pixels are covered
  __shared__ unsigned int cnt[256];
  __shared__ double sum[256];
  __shared__ long long s_before[257];
  unsigned int* gh = hist + static_cast<size_t>(blockIdx.x) * FRONT_BINS;
  if (page_tab) n_pix = static_cast<long long>(page_tab[blockIdx.x * 2 + 1]) * WO;
  const long long k = n_pix - static_cast<long long>(static_cast<double>(n_pix) * 0.9);   // int(len * 0.9) truncates
  constexpr int PER = FRONT_BINS / 256;
  // thread t owns bins [hi - PER + 1, hi] counted from the top: t = 0 holds the largest values
  const int t = threadIdx.x;
  const int top = FRONT_BINS - 1 - t * PER;
  unsigned int c = 0;
  for (int j = 0; j < PER; ++j) c += gh[top - j];
  cnt[t] = c;
  __syncthreads();
  if (t == 0) {
    long long acc = 0;
    for (int i = 0; i < 256; ++i) { s_before[i] = acc; acc += cnt[i]; }
    s_before[256] = acc;
  }
  __syncthreads();
  // each thread adds what falls inside the top-k set from its own bins
  double sm = 0.0;
  long long before = s_before[t];
  for (int j = 0; j < PER && before < k; ++j) {
    const int b = top - j;
    const unsigned int cb = gh[b];
    if (!cb) continue;
    const long long take = (before + cb <= k) ? cb : (k - before);
    unsigned short bits = static_cast<unsigned short>(b);
    const float v = to_f<T>(*reinterpret_cast<const T*>(&bits));
    sm += static_cast<double>(take) * static_cast<double>(v);
    before += cb;
  }
  sum[t] = sm;
  __syncthreads();
  if (t == 0) {
    double tot = 0.0;
    for (int i = 0; i < 256; ++i) tot += sum[i];
    const float avg = k > 0 ? static_cast<float>(tot / static_cast<double>(k)) : 0.f;
    float sf = avg / typical;
    sf = fminf(fmaxf(sf, 0.f), 1.f);
    sf = sqrtf(sf);
    const float low = fminf(fmaxf(low_text * sf, 0.1f), 0.6f);
    const float tt = fminf(fmaxf(text_threshold * sf, 0.15f), 0.8f);
    thr[blockIdx.x * 4 + 0] = tt;
    thr[blockIdx.x * 4 + 1] = low;
    thr[blockIdx.x * 4 + 2] = avg;
    thr[blockIdx.x * 4 + 3] = sf;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < FRONT_BINS; i += 256) gh[i] = 0u;      // ready for the next call
}

template <typename T>
__global__ void __launch_bounds__(256) det_front_mask_kernel(const T* __restrict__ map, const float* __restrict__ thr,
                                                             unsigned char* __restrict__ mask, long long n_pix,
                                                             const int* __restrict__ page_tab, int WO) {
  const float low = thr[blockIdx.y * 4 + 1];
  size_t base = static_cast<size_t>(blockIdx.y) * n_pix;
  if (page_tab) {
    base = static_cast<size_t>(page_tab[blockIdx.y * 2]) * WO;
    n_pix = static_cast<long long>(page_tab[blockIdx.y * 2 + 1]) * WO;
  }
  const T* m = map + base;
  unsigned char* o = mask + base;
  const long long i0 = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) * 8;
  if (i0 + 8 <= n_pix) {
    const uint4 u = *reinterpret_cast<const uint4*>(m + i0);
    const T* e = reinterpret_cast<const T*>(&u);
    unsigned long long pk = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) pk |= static_cast<unsigned long long>(to_f<T>(e[j]) > low ? 1u : 0u) << (8 * j);
    *reinterpret_cast<unsigned long long*>(o + i0) = pk;
  } else {
    for (long long i = i0; i < n_pix; ++i) o[i] = to_f<T>(m[i]) > low ? 1 : 0;
  }
}

int det_text_front(int dtype, const void* logits, int n_labels, int B, int hs, int ws, int HO, int WO, void* map16,
                   unsigned char* mask, float* thr, unsigned int* hist, float text_threshold, float low_text, cudaStream_t st,
                   const int* chunk_tab, int n_pages, const int* page_tab, int max_page_rows) {
  if (B <= 0) return 0;
  if (B > 65535) { set_error("det_text_front: too many pages for the grid"); return -1; }
  const long long n_pix = static_cast<long long>(HO) * WO;
  if (n_pix % 8 || (chunk_tab && WO % 8)) { set_error("det_text_front: H*W (stitched: W) must be a multiple of 8"); return -1; }
  if (!chunk_tab) { n_pages = B; max_page_rows = HO; }
  if (n_pages <= 0) return 0;
  if (n_pages > 65535) { set_error("det_text_front: too many pages for the grid"); return -1; }
  const int rows_per_block = 16;
  dim3 g1((HO + rows_per_block - 1) / rows_per_block, B);
  const size_t smem = FRONT_BINS * sizeof(unsigned int);
  const int plane_stride = n_labels * hs * ws;         // channel 0 of chunk b
  dim3 g3(static_cast<unsigned int>((static_cast<long long>(max_page_rows) * WO / 8 + 255) / 256), n_pages);
  if (dtype == DT_F16) {
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(det_front_map_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
    det_front_map_kernel<__half><<<g1, 256, smem, st>>>((const __half*)logits, plane_stride, (__half*)map16, hist, hs, ws, HO, WO, rows_per_block, chunk_tab);
    if (int rc = launch_ok()) return rc;
    det_front_threshold_kernel<__half><<<n_pages, 256, 0, st>>>(hist, thr, n_pix, text_threshold, low_text, 0.7f, page_tab, WO);
    if (int rc = launch_ok()) return rc;
    det_front_mask_kernel<__half><<<g3, 256, 0, st>>>((const __half*)map16, thr, mask, n_pix, page_tab, WO);
  } else {
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(det_front_map_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
    det_front_map_kernel<__nv_bfloat16><<<g1, 256, smem, st>>>((const __nv_bfloat16*)logits, plane_stride, (__nv_bfloat16*)map16, hist, hs, ws, HO, WO, rows_per_block, chunk_tab);
    if (int rc = launch_ok()) return rc;
    det_front_threshold_kernel<__nv_bfloat16><<<n_pages, 256, 0, st>>>(hist, thr, n_pix, text_threshold, low_text, 0.7f, page_tab, WO);
    if (int rc = launch_ok()) return rc;
    det_front_mask_kernel<__nv_bfloat16><<<g3, 256, 0, st>>>((const __nv_bfloat16*)map16, thr, mask, n_pix, page_tab, WO);
  }
  return launch_ok();
}

}  // namespace sb
