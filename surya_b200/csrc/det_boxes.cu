// surya_b200 — back half of the detection post-processing on the device (surya/detection/heatmap.py:33-107): text-line tables
// from the binarised mask and the 16-bit text map that det_text_front leaves on the device.
//
//   ccl_local      4-connected union-find inside a 32x32 tile (shared memory), labels = global raster index of the tile root
//   ccl_merge      unions across tile borders in global memory
//   ccl_flatten    every foreground pixel -> its root; roots counted per row
//   row_scan       per-page exclusive scan of the row counts
//   ccl_number     roots numbered in raster order (= cv2.connectedComponentsWithStats(connectivity=4)'s label order)
//   comp_stats     area, bounding box and peak map value per component, warp-aggregated
//   comp_keep      keep filter (area >= 10, peak >= text threshold), dilation kernel size, output index and point offset
//   row_extents    per source row of every kept component: leftmost / rightmost pixel
//   dilated_rows   per dilated row: the leftmost / rightmost pixel of cv2.dilate's output, written as two points
//
// The host is left with cv2.minAreaRect over two points per dilated row, which gives the same rectangle as over every dilated
// pixel (the hull is the same), so the boxes stay bit-identical to detect_boxes.
#include "ops.cuh"
#include "sb_ptx.cuh"

#include <climits>

namespace sb {
namespace {

constexpr int TILE = 32;
constexpr unsigned FULL = 0xffffffffu;
constexpr int MIN_AREA = 10;            // heatmap.py:44 `if size < 10: continue`

// Union-find over raster indices with parent[x] <= x everywhere.  A root is the smallest index of its set, so after the last
// union every component's root is its first pixel in raster order.
__device__ __forceinline__ int find_root(const volatile int* parent, int x) {
  // terminates: each step goes to a strictly smaller index (parent[x] < x unless x is a root), and indices are >= 0
  int p = parent[x];
  while (p != x) { x = p; p = parent[x]; }
  return x;
}

template <typename AtomicMin>
__device__ __forceinline__ void unite(volatile int* parent, int a, int b, AtomicMin amin) {
  // Links the larger root under the smaller one with an atomic min.  When the min finds that the larger index is no longer a
  // root, it continues from the parent it found.  Every pass that does not finish lowers max(a, b) strictly: the new b is the
  // old parent, which is < b, and find_root only moves to lower roots.  Indices are >= 0, so the loop terminates.
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = amin(const_cast<int*>(parent) + b, a);
    if (old == b) return;
    b = old;
  }
}

struct SmemMin { __device__ int operator()(int* p, int v) const { return atomicMin(p, v); } };
struct GmemMin { __device__ int operator()(int* p, int v) const { return atomicMin(p, v); } };

__device__ __forceinline__ int isqrt_exact(int m) {
  // int(np.sqrt(m)): np.sqrt is correctly rounded in fp64, so that is floor(sqrt(m)); sqrtf alone is not guaranteed to be
  int r = static_cast<int>(sqrtf(static_cast<float>(m)));
  while (r > 0 && r * r > m) --r;
  while ((r + 1) * (r + 1) <= m) ++r;
  return r;
}

__device__ __forceinline__ float bits_to_f(unsigned bits, int bf16) {
  const unsigned short u = static_cast<unsigned short>(bits);
  return bf16 ? __bfloat162float(__ushort_as_bfloat16(u)) : __half2float(__ushort_as_half(u));
}

// Component id of a pixel after ccl_number: background -1; a root holds -(id + 2); every other pixel holds its root's index.
__device__ __forceinline__ int comp_id(const int* L, int i) {
  const int v = L[i];
  if (v == -1) return -1;
  return v < -1 ? -v - 2 : -L[v] - 2;
}

// Exclusive scan over a 1024-thread block; `total` gets the block sum.  sh: 32 ints of shared memory.
__device__ __forceinline__ int block_scan_1024(int v, int* sh, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(FULL, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) sh[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = sh[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(FULL, s, d);
      if (lane >= d) s += y;
    }
    sh[lane] = s;
  }
  __syncthreads();
  const int r = (wid ? sh[wid - 1] : 0) + x - v;
  total = sh[31];
  __syncthreads();
  return r;
}

// Per-page scratch, carved out of the caller's buffer (sizes in the header comment of sb_det_text_boxes).
struct Scratch {
  int* label;                     // [B][n]
  int *area, *x0, *x1, *y0, *y1;  // [B][C], C = ceil(n / 2) components at most (4-connectivity)
  unsigned* peak;                 // [B][C] 16-bit pattern of the largest map value
  int* keep;                      // [B][C] output index or -1
  int *row_cnt, *row_off;         // [B][H]
  int *ext_lo, *ext_hi;           // [B][R], R = max_points / 2 dilated rows
  int* ncomp;                     // [B]
  long long n, C, R;
};

// ------------------------------------------------------------------------------------------------ labelling
__global__ void __launch_bounds__(256) ccl_local_kernel(const unsigned char* __restrict__ mask, int* __restrict__ label, int H,
                                                        int W, long long n) {
  __shared__ int s[TILE * TILE];
  const unsigned char* m = mask + blockIdx.z * n;
  int* L = label + blockIdx.z * n;
  const int lx = threadIdx.x, tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
  const int x = tx0 + lx;
  bool fg[TILE / 8];
#pragma unroll
  for (int r = 0; r < TILE / 8; ++r) {
    const int ly = threadIdx.y + 8 * r, y = ty0 + ly;
    fg[r] = x < W && y < H && m[static_cast<long long>(y) * W + x];
    s[ly * TILE + lx] = fg[r] ? ly * TILE + lx : -1;
  }
  __syncthreads();
  volatile int* vs = s;
#pragma unroll
  for (int r = 0; r < TILE / 8; ++r) {
    const int ly = threadIdx.y + 8 * r, l = ly * TILE + lx;
    if (!fg[r]) continue;
    if (lx > 0 && vs[l - 1] >= 0) unite(vs, l, l - 1, SmemMin());
    if (ly > 0 && vs[l - TILE] >= 0) unite(vs, l, l - TILE, SmemMin());
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < TILE / 8; ++r) {
    const int ly = threadIdx.y + 8 * r, y = ty0 + ly;
    if (x >= W || y >= H) continue;
    int g = -1;
    if (fg[r]) {
      // tile-local raster order is global raster order restricted to the tile, so the local minimum is the global one
      const int root = find_root(vs, ly * TILE + lx);
      g = (ty0 + root / TILE) * W + tx0 + root % TILE;
    }
    L[static_cast<long long>(y) * W + x] = g;
  }
}

// Thread t < 32: the pixel on the tile's top edge against the one above; t >= 32: the left edge against the one to the left.
__global__ void __launch_bounds__(64) ccl_merge_kernel(const unsigned char* __restrict__ mask, int* label, int H, int W,
                                                       long long n) {
  const unsigned char* m = mask + blockIdx.z * n;
  volatile int* L = label + blockIdx.z * n;
  const int t = threadIdx.x & 31, tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
  int i = -1, j = -1;
  if (threadIdx.x < 32) {
    const int x = tx0 + t;
    if (ty0 > 0 && x < W) { i = ty0 * W + x; j = i - W; }
  } else {
    const int y = ty0 + t;
    if (tx0 > 0 && y < H) { i = y * W + tx0; j = i - 1; }
  }
  if (i >= 0 && m[i] && m[j]) unite(L, i, j, GmemMin());
}

// One warp per row: every foreground pixel gets its root, and the row's roots are counted.
__global__ void __launch_bounds__(256) ccl_flatten_kernel(int* label, int* __restrict__ row_cnt, int H, int W, long long n) {
  const int y = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (y >= H) return;
  volatile int* L = label + blockIdx.y * n;
  int cnt = 0;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane, i = y * W + x;
    bool root = false;
    if (x < W) {
      const int v = L[i];
      if (v >= 0) {
        const int r = find_root(L, v);
        L[i] = r;
        root = r == i;
      }
    }
    cnt += __popc(__ballot_sync(FULL, root));
  }
  if (lane == 0) row_cnt[static_cast<long long>(blockIdx.y) * H + y] = cnt;
}

__global__ void __launch_bounds__(1024) row_scan_kernel(const int* __restrict__ row_cnt, int* __restrict__ row_off,
                                                        int* __restrict__ ncomp, int H) {
  __shared__ int sh[32];
  const int* c = row_cnt + static_cast<long long>(blockIdx.x) * H;
  int* o = row_off + static_cast<long long>(blockIdx.x) * H;
  int carry = 0;
  for (int y0 = 0; y0 < H; y0 += 1024) {
    const int y = y0 + threadIdx.x;
    int tot;
    const int e = block_scan_1024(y < H ? c[y] : 0, sh, tot);
    if (y < H) o[y] = carry + e;
    carry += tot;
  }
  if (threadIdx.x == 0) ncomp[blockIdx.x] = carry;
}

// One warp per row: roots get consecutive ids in raster order, and their component's stats are reset.
__global__ void __launch_bounds__(256) ccl_number_kernel(Scratch s, int H, int W) {
  const int y = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (y >= H) return;
  const int b = blockIdx.y;
  int* L = s.label + b * s.n;
  const long long cb = b * s.C;
  int next = s.row_off[static_cast<long long>(b) * H + y];
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane, i = y * W + x;
    const bool root = x < W && L[i] == i;
    const unsigned bal = __ballot_sync(FULL, root);
    if (root) {
      const int id = next + __popc(bal & ((1u << lane) - 1u));
      L[i] = -id - 2;
      s.area[cb + id] = 0;
      s.x0[cb + id] = INT_MAX;
      s.x1[cb + id] = -1;
      s.y0[cb + id] = y;          // the root is the component's first pixel in raster order
      s.y1[cb + id] = -1;
      s.peak[cb + id] = 0u;
    }
    next += __popc(bal);
  }
}

// One warp per row segment of 32 pixels: lanes of one component (found with __match_any_sync) are combined before the atomics,
// so a long text line costs one atomic per 32 pixels.  Component pixels are > low_text > 0, so the largest 16-bit pattern is the
// largest value for fp16 and bf16 alike.
__global__ void __launch_bounds__(256) comp_stats_kernel(Scratch s, const unsigned short* __restrict__ map16, int H, int W) {
  const int y = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (y >= H) return;
  const int b = blockIdx.y;
  const int* L = s.label + b * s.n;
  const unsigned short* mp = map16 + b * s.n;
  const long long cb = b * s.C;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane, i = y * W + x;
    const int id = x < W ? comp_id(L, i) : -1;
    const unsigned grp = __match_any_sync(FULL, id);
    if (id < 0) continue;
    const unsigned pk = __reduce_max_sync(grp, static_cast<unsigned>(mp[i]));
    if (lane == __ffs(grp) - 1) {
      atomicAdd(s.area + cb + id, __popc(grp));
      atomicMin(s.x0 + cb + id, x);
      atomicMax(s.x1 + cb + id, x0 + 31 - __clz(grp));
      atomicMax(s.y1 + cb + id, y);
      atomicMax(s.peak + cb + id, pk);
    }
  }
}

// One block per page, components in id (= raster) order: the keep filter of heatmap.py:43-60, the dilation kernel size of :47-58
// and two scans, one giving each kept component its output index, one its first dilated row.
__global__ void __launch_bounds__(1024) comp_keep_kernel(Scratch s, const float* __restrict__ thr, int bf16, int H, int W,
                                                         int max_boxes, int* __restrict__ count, int* __restrict__ overflow,
                                                         int* __restrict__ box, float* __restrict__ peak_out) {
  __shared__ int sh_k[32], sh_r[32];
  const int b = blockIdx.x;
  const int nc = s.ncomp[b];
  const float tt = thr[b * 4 + 0];
  const long long cb = b * s.C;
  int kept_base = 0, row_base = 0;
  for (int c0 = 0; c0 < nc; c0 += 1024) {
    const int id = c0 + threadIdx.x;
    bool kept = false;
    int ks = 0, x0d = 0, y0d = 0, x1d = 0, y1d = 0, rows = 0;
    float pk = 0.f;
    if (id < nc) {
      pk = bits_to_f(s.peak[cb + id], bf16);
      // `if size < 10: continue` and `if line_max < text_threshold: continue`, compared in fp32 like NumPy does
      kept = s.area[cb + id] >= MIN_AREA && !(pk < tt);
      if (kept) {
        const int x0 = s.x0[cb + id], x1 = s.x1[cb + id], y0 = s.y0[cb + id], y1 = s.y1[cb + id];
        ks = isqrt_exact(min(x1 - x0 + 1, y1 - y0 + 1)) + 1;
        // getStructuringElement(MORPH_RECT, (ks, ks)) has its anchor at ks / 2: output pixel p reads p - a .. p - a + ks - 1
        const int a = ks / 2, lead = ks - 1 - a;
        x0d = max(0, x0 - lead); x1d = min(W - 1, x1 + a);
        y0d = max(0, y0 - lead); y1d = min(H - 1, y1 + a);
        rows = y1d - y0d + 1;
      }
    }
    int nk, nr;
    const int k = kept_base + block_scan_1024(kept ? 1 : 0, sh_k, nk);
    const int r0 = row_base + block_scan_1024(rows, sh_r, nr);
    if (id < nc) {
      const bool fits = kept && k < max_boxes && r0 + rows <= s.R;
      s.keep[cb + id] = fits ? k : -1;
      if (fits) {
        int* o = box + (static_cast<long long>(b) * max_boxes + k) * 7;
        o[0] = x0d; o[1] = y0d; o[2] = x1d; o[3] = y1d; o[4] = 2 * r0; o[5] = 2 * rows; o[6] = ks;
        peak_out[static_cast<long long>(b) * max_boxes + k] = pk;
      }
    }
    kept_base += nk;
    row_base += nr;
  }
  if (threadIdx.x == 0) {
    count[b] = kept_base;
    overflow[b] = (kept_base > max_boxes || row_base > s.R) ? 1 : 0;
  }
}

// One warp per row segment: leftmost / rightmost pixel of every kept component on this row, into its dilated-row slot.
__global__ void __launch_bounds__(256) row_extents_kernel(Scratch s, const int* __restrict__ box, int max_boxes, int H, int W) {
  const int y = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (y >= H) return;
  const int b = blockIdx.y;
  const int* L = s.label + b * s.n;
  const long long cb = b * s.C;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane, i = y * W + x;
    const int id = x < W ? comp_id(L, i) : -1;
    const int k = id >= 0 ? s.keep[cb + id] : -1;
    const unsigned grp = __match_any_sync(FULL, k);
    if (k < 0 || lane != __ffs(grp) - 1) continue;
    const int* o = box + (static_cast<long long>(b) * max_boxes + k) * 7;
    const long long slot = b * s.R + o[4] / 2 + (y - o[1]);
    atomicMin(s.ext_lo + slot, x);
    atomicMax(s.ext_hi + slot, x0 + 31 - __clz(grp));
  }
}

// One warp per kept component, one lane per dilated row Y: cv2.dilate's row Y is the union of source rows Y - a .. Y - a + ks - 1
// widened by ks - 1 - a on the left and a on the right.  The window of heatmap.py:49-52 is ks wider than the component on every
// side, so only the image border clips.  Rows of the range that are not source rows still hold the neutral INT_MAX / -1.
__global__ void __launch_bounds__(256) dilated_rows_kernel(Scratch s, const int* __restrict__ count, const int* __restrict__ overflow,
                                                           const int* __restrict__ box, int* __restrict__ points, int max_boxes,
                                                           int max_points, int W) {
  const int b = blockIdx.y;
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (overflow[b] || k >= count[b]) return;
  const int* o = box + (static_cast<long long>(b) * max_boxes + k) * 7;
  const int y0d = o[1], y1d = o[3], p0 = o[4], rows = o[5] / 2, ks = o[6];
  const int a = ks / 2, lead = ks - 1 - a;
  const int* lo = s.ext_lo + b * s.R + p0 / 2;      // indexed by image row - y0d
  const int* hi = s.ext_hi + b * s.R + p0 / 2;
  int* pt = points + static_cast<long long>(b) * max_points * 2 + 2 * p0;
  for (int r = lane; r < rows; r += 32) {
    const int Y = y0d + r;
    int l = INT_MAX, h = -1;
    for (int j = max(y0d, Y - a); j <= min(y1d, Y - a + ks - 1); ++j) {
      l = min(l, lo[j - y0d]);
      h = max(h, hi[j - y0d]);
    }
    pt[4 * r + 0] = max(0, l - lead);
    pt[4 * r + 1] = Y;
    pt[4 * r + 2] = min(W - 1, h + a);
    pt[4 * r + 3] = Y;
  }
}

}  // namespace

size_t det_text_boxes_scratch_bytes(int B, int H, int W, int max_points) {
  const size_t n = static_cast<size_t>(H) * W, C = (n + 1) / 2, R = static_cast<size_t>(max_points / 2);
  return static_cast<size_t>(B) * (4 * n + 28 * C + 8 * static_cast<size_t>(H) + 8 * R + 4);
}

int det_text_boxes(int dtype, const void* map16, const unsigned char* mask, const float* thr, int B, int H, int W,
                   int max_boxes, int max_points, void* scratch, int* count, int* overflow, int* box, float* peak, int* points,
                   cudaStream_t st) {
  const long long n = static_cast<long long>(H) * W;
  if (n >= (1LL << 30)) { set_error("det_text_boxes: %d x %d pixels per page do not fit the int32 labels", H, W); return -1; }
  if (B > 65535) { set_error("det_text_boxes: too many pages for the grid"); return -1; }
  if (dtype != DT_F16 && dtype != DT_BF16) { set_error("det_text_boxes: map must be fp16 or bf16"); return -1; }
  Scratch s;
  s.n = n; s.C = (n + 1) / 2; s.R = max_points / 2;
  char* p = static_cast<char*>(scratch);
  auto take = [&](long long elems) { int* q = reinterpret_cast<int*>(p); p += static_cast<size_t>(B) * elems * 4; return q; };
  s.label = take(n);
  s.area = take(s.C); s.x0 = take(s.C); s.x1 = take(s.C); s.y0 = take(s.C); s.y1 = take(s.C);
  s.peak = reinterpret_cast<unsigned*>(take(s.C));
  s.keep = take(s.C);
  s.row_cnt = take(H); s.row_off = take(H);
  s.ext_lo = take(s.R); s.ext_hi = take(s.R);
  s.ncomp = take(1);
  const size_t ext_bytes = static_cast<size_t>(B) * s.R * 4;
  if (ext_bytes) {
    cudaMemsetAsync(s.ext_lo, 0x7f, ext_bytes, st);      // 0x7f7f7f7f: above any x
    cudaMemsetAsync(s.ext_hi, 0xff, ext_bytes, st);      // -1: below any x
  }
  const unsigned short* m16 = static_cast<const unsigned short*>(map16);
  const dim3 tiles((W + TILE - 1) / TILE, (H + TILE - 1) / TILE, B);
  const dim3 rows((H + 7) / 8, B);
  ccl_local_kernel<<<tiles, dim3(TILE, 8), 0, st>>>(mask, s.label, H, W, n);
  if (int rc = launch_ok()) return rc;
  ccl_merge_kernel<<<tiles, 64, 0, st>>>(mask, s.label, H, W, n);
  if (int rc = launch_ok()) return rc;
  ccl_flatten_kernel<<<rows, 256, 0, st>>>(s.label, s.row_cnt, H, W, n);
  if (int rc = launch_ok()) return rc;
  row_scan_kernel<<<B, 1024, 0, st>>>(s.row_cnt, s.row_off, s.ncomp, H);
  if (int rc = launch_ok()) return rc;
  ccl_number_kernel<<<rows, 256, 0, st>>>(s, H, W);
  if (int rc = launch_ok()) return rc;
  comp_stats_kernel<<<rows, 256, 0, st>>>(s, m16, H, W);
  if (int rc = launch_ok()) return rc;
  comp_keep_kernel<<<B, 1024, 0, st>>>(s, thr, dtype == DT_BF16 ? 1 : 0, H, W, max_boxes, count, overflow, box, peak);
  if (int rc = launch_ok()) return rc;
  row_extents_kernel<<<rows, 256, 0, st>>>(s, box, max_boxes, H, W);
  if (int rc = launch_ok()) return rc;
  dilated_rows_kernel<<<dim3((max_boxes + 7) / 8, B), 256, 0, st>>>(s, count, overflow, box, points, max_boxes, max_points, W);
  return launch_ok();
}

}  // namespace sb
