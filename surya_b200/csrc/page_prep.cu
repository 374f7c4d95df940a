// surya_b200 — detection page preparation on the device: ragged uint8 pages -> processor-size uint8 chunks.
//
// Replaces, per chunk of a page, the host PIL chain of DetectionPredictor (surya/detection/util.py:7-36 split_image +
// ImageOps.pad; surya/detection/__init__.py:50-62 prepare_image: thumbnail(LANCZOS, reducing_gap=2.0) then resize(LANCZOS)).
// surya_b200/page_prep.py plans every chunk as a chain of at most five jobs (box-average pre-reduce, horizontal and vertical
// Lanczos passes of the thumbnail, horizontal and vertical passes of the stretch) and computes PIL's fixed-point weights once per
// (source extent, box, destination extent).  This file only does PIL's integer arithmetic on top of them:
//   reduce      ((sum + n / 2) * uint32(2^32f / (256 n)f)) >> 24 over the n pixels of a block (ImagingReduceNxN / Corners)
//   resample    clip8((2^21 + sum_t src[t] * w[t]) >> 22), the uint8 intermediate between the two passes (ImagingResample*_8bpc)
// so the chunks equal PIL's bytes exactly.  Rows past a chunk's source rows read as the padding colour of ImageOps.pad.
#include "ops.cuh"

namespace sb {

namespace {

enum { PR_KIND = 0, PR_SRC_OFF, PR_SRC_W, PR_SRC_H, PR_SRC_VALID, PR_SRC_PAGE, PR_DST_OFF, PR_DST_W, PR_DST_H, PR_DST_OUT, PR_FX,
       PR_FY, PR_KSIZE, PR_COEF, PR_BOUNDS, PR_STRIDE = 16 };
enum { PRK_REDUCE = 0, PRK_HORIZ = 1, PRK_VERT = 2 };

// ImageOps.pad(color=255) on an RGB image fills (255, 0, 0)
__device__ __forceinline__ void fetch(const unsigned char* __restrict__ src, int w, int valid, int x, int y, int v[3]) {
  if (y >= valid) { v[0] = 255; v[1] = 0; v[2] = 0; return; }
  const unsigned char* p = src + (static_cast<size_t>(y) * w + x) * 3;
  v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
}

__device__ __forceinline__ unsigned char clip8(int v) {
  v >>= 22;
  return static_cast<unsigned char>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void __launch_bounds__(256) page_resize_kernel(const unsigned char* __restrict__ pages, unsigned char* scratch,
                                                          unsigned char* out, const long long* __restrict__ desc,
                                                          const int* __restrict__ tables) {
  const long long* d = desc + static_cast<size_t>(blockIdx.y) * PR_STRIDE;
  const int kind = static_cast<int>(d[PR_KIND]);
  const int sw = static_cast<int>(d[PR_SRC_W]), sh = static_cast<int>(d[PR_SRC_H]), valid = static_cast<int>(d[PR_SRC_VALID]);
  const int dw = static_cast<int>(d[PR_DST_W]), dh = static_cast<int>(d[PR_DST_H]);
  const unsigned char* src = (d[PR_SRC_PAGE] ? pages : scratch) + d[PR_SRC_OFF];
  unsigned char* dst = (d[PR_DST_OUT] ? out : scratch) + d[PR_DST_OFF];
  const long long n = static_cast<long long>(dw) * dh;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int y = static_cast<int>(i / dw), x = static_cast<int>(i % dw);
    unsigned char o[3];
    int v[3];
    if (kind == PRK_REDUCE) {
      const int fx = static_cast<int>(d[PR_FX]), fy = static_cast<int>(d[PR_FY]);
      const int x0 = x * fx, y0 = y * fy, x1 = min(x0 + fx, sw), y1 = min(y0 + fy, sh);
      unsigned int s[3] = {0u, 0u, 0u};
      for (int yy = y0; yy < y1; ++yy)
        for (int xx = x0; xx < x1; ++xx) {
          fetch(src, sw, valid, xx, yy, v);
          s[0] += v[0]; s[1] += v[1]; s[2] += v[2];
        }
      const unsigned int cnt = static_cast<unsigned int>((x1 - x0) * (y1 - y0));
      const unsigned int m = __float2uint_rz(__fdiv_rn(4294967296.0f, static_cast<float>(256u * cnt)));
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = static_cast<unsigned char>(((s[c] + cnt / 2) * m) >> 24);
    } else {
      const bool horiz = kind == PRK_HORIZ;
      const int pos = horiz ? x : y;
      const int ksize = static_cast<int>(d[PR_KSIZE]);
      const int* b = tables + d[PR_BOUNDS] + 2 * pos;
      const int* k = tables + d[PR_COEF] + static_cast<size_t>(pos) * ksize;
      const int t0 = b[0], cnt = b[1];
      int ss[3] = {1 << 21, 1 << 21, 1 << 21};
      for (int t = 0; t < cnt; ++t) {
        if (horiz) fetch(src, sw, valid, t0 + t, y, v);
        else fetch(src, sw, valid, x, t0 + t, v);
        const int kt = k[t];
        ss[0] += v[0] * kt; ss[1] += v[1] * kt; ss[2] += v[2] * kt;
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = clip8(ss[c]);
    }
    unsigned char* q = dst + static_cast<size_t>(i) * 3;
    q[0] = o[0]; q[1] = o[1]; q[2] = o[2];
  }
}

}  // namespace

int det_page_resize(const unsigned char* pages, unsigned char* scratch, unsigned char* out, const long long* desc, const int* tables,
                    int n_steps, const int* step_jobs, const long long* step_max_px, cudaStream_t st) {
  long long first = 0;
  for (int s = 0; s < n_steps; ++s) {
    const int jobs = step_jobs[s];
    if (jobs <= 0) continue;
    if (jobs > 65535) { set_error("det_page_resize: at most 65535 jobs per step"); return -1; }
    const long long blocks = (step_max_px[s] + 255) / 256;
    dim3 grid(static_cast<unsigned int>(blocks < 4096 ? (blocks > 0 ? blocks : 1) : 4096), jobs);
    page_resize_kernel<<<grid, 256, 0, st>>>(pages, scratch, out, desc + first * PR_STRIDE, tables);
    if (int rc = launch_ok()) return rc;
    first += jobs;
  }
  return 0;
}

}  // namespace sb
