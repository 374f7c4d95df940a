// surya_b200 — encoder image preprocessing of the layout and table_rec predictors on the device: uint8 pages (or rectangles of
// them) -> NCHW pixel values in the engine dtype at the encoder size.
//
// Replaces SuryaEncoderImageProcessor.process_inner (surya/common/donut/processor.py:61-116) for RGB input:
//   cv2.resize(img, (W, H), interpolation=self.resample)   resample is Image.Resampling.BILINEAR == 2, which cv2 reads as
//                                                         INTER_CUBIC: a bicubic resize of the uint8 image, aspect ratio not kept
//   pad_image to max_size                                 nothing to do at the encoder size
//   astype(float64) * (1/255) -> float32, normalize(mean 0.5, std 0.5) in float32, then the predictor's cast to the model dtype
//   (surya/layout/__init__.py:78-81; table_rec uses the same processor, surya/table_rec/processor.py:19-21).
// A job reads a source rectangle (x0, y0, w, h) of a resident page, so ImageSlicer's crops (surya/layout/slicer.py:48-66) need no
// copy.  A job that gives the page height is bounded: taps outside the page read 0, as PIL's Image.crop fills a crop box that
// extends past the page with black before the table processor's resize (surya/scripts/table_recognition.py:63-70), so the
// expanded table boxes also need no copy.  The cubic taps (index relative to the rectangle, clamped to it = border replicate,
// and Keys weights with A = -0.75 from a double-precision coordinate) are computed on the host per (source extent, destination
// extent) by surya_b200/layout_pages.py.
// Arithmetic (the model of OpenCV's uint8 cubic resize that oracle/layout_pages_oracle.py restates and pins to cv2): four
// horizontal sums, each float32 tap by tap, then the vertical float32 sum, round half to even, clamp to 0..255.
#include "ops.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace sb {

namespace {

constexpr int LP_TX = 32, LP_TY = 8;
enum { LJ_SRC_OFF = 0, LJ_PITCH, LJ_X0, LJ_Y0, LJ_XTAB, LJ_YTAB, LJ_OUT, LJ_PAGE_H, LJ_STRIDE = 8 };

template <typename T> __device__ __forceinline__ T to_dt(float v);
template <> __device__ __forceinline__ __half to_dt<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 to_dt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(LP_TX * LP_TY) layout_preprocess_kernel(const unsigned char* __restrict__ pages,
                                                                          const long long* __restrict__ jobs,
                                                                          const int* __restrict__ tap_idx, const float* __restrict__ tap_w,
                                                                          int H, int W, T* __restrict__ out) {
  const long long* j = jobs + static_cast<size_t>(blockIdx.z) * LJ_STRIDE;
  const int x0 = blockIdx.x * LP_TX, y0 = blockIdx.y * LP_TY;
  __shared__ int sxi[LP_TX][4], syi[LP_TY][4];
  __shared__ float sxw[LP_TX][4], syw[LP_TY][4];
  const int tid = threadIdx.y * LP_TX + threadIdx.x;
  if (tid < LP_TX * 4) {
    const int d = tid >> 2, k = tid & 3;
    if (x0 + d < W) {
      const size_t e = (static_cast<size_t>(j[LJ_XTAB]) + x0 + d) * 4 + k;
      sxi[d][k] = tap_idx[e] + static_cast<int>(j[LJ_X0]);
      sxw[d][k] = tap_w[e];
    }
  } else if (tid < (LP_TX + LP_TY) * 4) {
    const int d = (tid - LP_TX * 4) >> 2, k = tid & 3;
    if (y0 + d < H) {
      const size_t e = (static_cast<size_t>(j[LJ_YTAB]) + y0 + d) * 4 + k;
      syi[d][k] = tap_idx[e] + static_cast<int>(j[LJ_Y0]);
      syw[d][k] = tap_w[e];
    }
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= W || y >= H) return;
  const unsigned char* src = pages + j[LJ_SRC_OFF];
  const int page_w = static_cast<int>(j[LJ_PITCH]), page_h = static_cast<int>(j[LJ_PAGE_H]);
  const size_t pitch = static_cast<size_t>(page_w) * 3;
  float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int sy = syi[threadIdx.y][r];
    const bool row_in = page_h == 0 || (sy >= 0 && sy < page_h);
    const unsigned char* row = src + static_cast<ptrdiff_t>(sy) * static_cast<ptrdiff_t>(pitch);
    float hs[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int sx = sxi[threadIdx.x][t];
      const bool in = row_in && (page_h == 0 || (sx >= 0 && sx < page_w));   // outside a bounded job's page: PIL's 0 fill
      const unsigned char* px = row + sx * 3;
      const float w = sxw[threadIdx.x][t];
#pragma unroll
      for (int c = 0; c < 3; ++c) hs[c] = __fadd_rn(hs[c], __fmul_rn(in ? static_cast<float>(px[c]) : 0.f, w));
    }
    const float w = syw[threadIdx.y][r];
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(hs[c], w));
  }
  const size_t plane = static_cast<size_t>(H) * W;
  T* o = out + static_cast<size_t>(j[LJ_OUT]) * 3 * plane + static_cast<size_t>(y) * W + x;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fminf(fmaxf(rintf(acc[c]), 0.f), 255.f);                                 // saturate_cast<uchar>
    const float r = static_cast<float>(static_cast<double>(v) * (1.0 / 255.0));              // astype(float64) * (1/255) -> float32
    o[c * plane] = to_dt<T>(__fdiv_rn(__fsub_rn(r, 0.5f), 0.5f));                             // (x - 0.5) / 0.5 in float32
  }
}

}  // namespace

}  // namespace sb

extern "C" int sb_layout_preprocess(int dtype, const unsigned char* pages, const long long* jobs, int n_jobs, const int* tap_idx,
                                    const float* tap_w, int out_h, int out_w, void* out, void* stream) {
  using namespace sb;
  if (n_jobs == 0) return 0;
  if (!pages || !jobs || !tap_idx || !tap_w || !out) { set_error("sb_layout_preprocess: null argument"); return -1; }
  if (n_jobs < 0 || n_jobs > 65535 || out_h <= 0 || out_w <= 0) {
    set_error("sb_layout_preprocess: %d jobs (1..65535) of %dx%d outputs", n_jobs, out_h, out_w);
    return -2;
  }
  if (dtype != DT_F16 && dtype != DT_BF16) { set_error("sb_layout_preprocess: dtype must be fp16 or bf16"); return -3; }
  const dim3 grid((out_w + LP_TX - 1) / LP_TX, (out_h + LP_TY - 1) / LP_TY, n_jobs), block(LP_TX, LP_TY);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == DT_F16)
    layout_preprocess_kernel<__half><<<grid, block, 0, st>>>(pages, jobs, tap_idx, tap_w, out_h, out_w, static_cast<__half*>(out));
  else
    layout_preprocess_kernel<__nv_bfloat16><<<grid, block, 0, st>>>(pages, jobs, tap_idx, tap_w, out_h, out_w,
                                                                    static_cast<__nv_bfloat16*>(out));
  return launch_ok();
}
