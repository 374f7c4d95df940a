// surya_b200 — kernels of the layout / table_rec path (Donut-Swin encoder + ADETR decoder) that the recognition and
// detection paths do not already provide.
//
//   layernorm          nn.LayerNorm (surya/common/donut/encoder.py:117,163,544-548; layout/model/decoder.py:73)
//   patch4_gather      im2col of the 4x4 stride-4 patch-embedding conv (encoder.py:228-230) -> GEMM operand
//   add_bcast_rows     + 2-D sin-cos stage table / learned position_embeddings (encoder.py:773-776; layout encoder.py:76-77)
//   swin_window_attn   shifted-window attention with relative-position bias and -100 shift mask
//                      (encoder.py:383-442, 562-590, 598-664): windows, cyclic shift and un-shift are pure index maps,
//                      so tokens stay in natural (b, y, x) order for every GEMM / LayerNorm around it
//   patch_merge_gather 2x2 neighbourhood concat in the reference's channel order (encoder.py:301-312)
//   bbox_embed_sum     BboxEmbedding: 15 table gathers with integer corner arithmetic (layout/model/decoder.py:36-57)
//   attn_single_query  q_len = 1 attention over a fixed K/V set with arbitrary strides (ADETR cross-attention,
//                      surya/common/adetr/decoder.py:150-194)
#include "ops.cuh"
#include "sb_ptx.cuh"

namespace sb {

// ------------------------------------------------------------------------------------------------ LayerNorm
// A row is held in registers by LPR = min(32, C/8) lanes (one global read, two-pass statistics from registers); for narrow rows
// (C = 128, 256) a warp normalises 32/LPR rows at once.  Rows wider than 8 * 32 * LN_MAXV elements take the streaming kernel.
constexpr int LN_MAXV = 4;

template <typename T>
__global__ void __launch_bounds__(128) layernorm_reg_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                            const T* __restrict__ b, T* __restrict__ y, int rows, int C, float eps,
                                                            int lpr) {
  const int lane = threadIdx.x & 31;
  const int rows_per_warp = 32 / lpr;
  const int sub = lane / lpr, sl = lane % lpr;
  const long long warp_id = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long row = warp_id * rows_per_warp + sub;
  const bool ok = row < rows;
  const T* xr = x + (ok ? row : 0) * C;
  uint4 v[LN_MAXV];
  float s = 0.f;
#pragma unroll
  for (int it = 0; it < LN_MAXV; ++it) {
    const int i = (it * lpr + sl) * 8;
    v[it] = make_uint4(0u, 0u, 0u, 0u);
    if (ok && i < C) {
      v[it] = *reinterpret_cast<const uint4*>(xr + i);
      const T* e = reinterpret_cast<const T*>(&v[it]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += to_f<T>(e[j]);
    }
  }
  for (int o = lpr >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int it = 0; it < LN_MAXV; ++it) {
    const int i = (it * lpr + sl) * 8;
    if (ok && i < C) {
      const T* e = reinterpret_cast<const T*>(&v[it]);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = to_f<T>(e[j]) - mean; q += d * d; }
    }
  }
  for (int o = lpr >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
  if (!ok) return;
  T* yr = y + row * C;
#pragma unroll
  for (int it = 0; it < LN_MAXV; ++it) {
    const int i = (it * lpr + sl) * 8;
    if (i < C) {
      const uint4 wu = *reinterpret_cast<const uint4*>(w + i);
      const uint4 bu = *reinterpret_cast<const uint4*>(b + i);
      const T *e = reinterpret_cast<const T*>(&v[it]), *we = reinterpret_cast<const T*>(&wu), *be = reinterpret_cast<const T*>(&bu);
      uint4 o;
      T* oe = reinterpret_cast<T*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) oe[j] = from_f<T>((to_f<T>(e[j]) - mean) * rstd * to_f<T>(we[j]) + to_f<T>(be[j]));
      *reinterpret_cast<uint4*>(yr + i) = o;
    }
  }
}

template <typename T>
__global__ void layernorm_kernel(const T* __restrict__ x, const T* __restrict__ w, const T* __restrict__ b,
                                 T* __restrict__ y, int rows, int C, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const T* xr = x + static_cast<size_t>(row) * C;
  T* yr = y + static_cast<size_t>(row) * C;
  float s = 0.f;
  for (int i = lane * 8; i < C; i += 256) {
    uint4 u = *reinterpret_cast<const uint4*>(xr + i);
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) s += to_f<T>(e[j]);
  }
  const float mean = warp_sum(s) / C;
  float v = 0.f;
  for (int i = lane * 8; i < C; i += 256) {
    uint4 u = *reinterpret_cast<const uint4*>(xr + i);
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) { float d = to_f<T>(e[j]) - mean; v += d * d; }
  }
  const float rstd = rsqrtf(warp_sum(v) / C + eps);
  for (int i = lane * 8; i < C; i += 256) {
    uint4 u = *reinterpret_cast<const uint4*>(xr + i);
    uint4 wu = *reinterpret_cast<const uint4*>(w + i);
    uint4 bu = *reinterpret_cast<const uint4*>(b + i);
    const T *e = reinterpret_cast<const T*>(&u), *we = reinterpret_cast<const T*>(&wu), *be = reinterpret_cast<const T*>(&bu);
    uint4 o;
    T* oe = reinterpret_cast<T*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) oe[j] = from_f<T>((to_f<T>(e[j]) - mean) * rstd * to_f<T>(we[j]) + to_f<T>(be[j]));
    *reinterpret_cast<uint4*>(yr + i) = o;
  }
}

int layernorm(int dtype, const void* x, const void* w, const void* b, void* y, int rows, int C, float eps, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (C % 8) { set_error("layernorm: C must be a multiple of 8"); return -1; }
  const int vecs = C / 8;
  int lpr = 32;
  while (lpr > 1 && (lpr >> 1) >= vecs) lpr >>= 1;       // smallest power of two >= vecs, capped at 32
  if (vecs <= lpr * LN_MAXV && (vecs % lpr == 0 || lpr == 32)) {
    const int rows_per_warp = 32 / lpr;
    const long long warps = (static_cast<long long>(rows) + rows_per_warp - 1) / rows_per_warp;
    dim3 grid(static_cast<unsigned>((warps + 3) / 4)), block(128);
    if (dtype == DT_F16) layernorm_reg_kernel<__half><<<grid, block, 0, st>>>((const __half*)x, (const __half*)w, (const __half*)b, (__half*)y, rows, C, eps, lpr);
    else layernorm_reg_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, rows, C, eps, lpr);
    return launch_ok();
  }
  dim3 grid((rows + 3) / 4), block(128);
  if (dtype == DT_F16) layernorm_kernel<__half><<<grid, block, 0, st>>>((const __half*)x, (const __half*)w, (const __half*)b, (__half*)y, rows, C, eps);
  else layernorm_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, rows, C, eps);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ patch-embed im2col
// in NCHW [B, Cin, H, W]; out [B*gh*gw, Kp]: column = c*P*P + ky*P + kx (Conv2d weight flatten order), zero padded to Kp.
template <typename T, typename InT>
__global__ void __launch_bounds__(256) patch_gather_kernel(const InT* __restrict__ in, T* __restrict__ out, int Cin, int H, int W,
                                                          int P, int Kp) {
  // one thread = 8 consecutive output columns of one patch (16-byte store); (patch row, image) come from the grid
  const int gw = (W + P - 1) / P, gh = (H + P - 1) / P;     // a partial last patch row / column is zero padded (maybe_pad)
  const int groups = Kp >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= gw * groups) return;
  const int g8 = t % groups, gx = t / groups;
  const int gy = blockIdx.y, b = blockIdx.z;
  const int K = Cin * P * P, PP = P * P;
  uint4 pack;
  T* pe = reinterpret_cast<T*>(&pack);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = g8 * 8 + j;
    float v = 0.f;
    if (col < K) {
      const int c = col / PP, r = col - c * PP;
      const int ky = r / P, kx = r - ky * P;
      const int yy = gy * P + ky, xx = gx * P + kx;
      if (yy < H && xx < W) {
        const InT* p = in + ((static_cast<size_t>(b) * Cin + c) * H + yy) * W + xx;
        if constexpr (sizeof(InT) == 4) v = static_cast<float>(*p); else v = to_f<InT>(*p);
      }
    }
    pe[j] = from_f<T>(v);
  }
  *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(b) * gh + gy) * gw + gx) * Kp + g8 * 8) = pack;
}

int patch_gather(int dtype, const void* in, int in_f32, void* out, int B, int Cin, int H, int W, int P, int Kp, cudaStream_t st) {
  if (B <= 0) return 0;
  if (P <= 0 || Kp % 8 || Kp < Cin * P * P) { set_error("patch_gather: Kp >= Cin*P*P and Kp %% 8 == 0"); return -1; }
  const int gh = (H + P - 1) / P, gw = (W + P - 1) / P;
  if (B > 65535 || gh > 65535) { set_error("patch_gather: batch / rows too large for the grid"); return -1; }
  dim3 grid((gw * (Kp / 8) + 255) / 256, gh, B);
#define PG(T_, I_) patch_gather_kernel<T_, I_><<<grid, 256, 0, st>>>((const I_*)in, (T_*)out, Cin, H, W, P, Kp)
  if (dtype == DT_F16) { if (in_f32) PG(__half, float); else PG(__half, __half); }
  else { if (in_f32) PG(__nv_bfloat16, float); else PG(__nv_bfloat16, __nv_bfloat16); }
#undef PG
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ x[b, t, :] += tab[t, :]
template <typename T>
__global__ void add_bcast_rows_kernel(T* __restrict__ x, const T* __restrict__ tab, long long rows, int rows_per_batch, int C) {
  const int cv = C >> 3;
  const long long total = rows * cv;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = (idx % cv) * 8;
    const long long r = idx / cv;
    uint4 xv = *reinterpret_cast<const uint4*>(x + r * C + c8);
    const uint4 tv = *reinterpret_cast<const uint4*>(tab + static_cast<size_t>(r % rows_per_batch) * C + c8);
    T* xe = reinterpret_cast<T*>(&xv);
    const T* te = reinterpret_cast<const T*>(&tv);
#pragma unroll
    for (int j = 0; j < 8; ++j) xe[j] = from_f<T>(to_f<T>(xe[j]) + to_f<T>(te[j]));
    *reinterpret_cast<uint4*>(x + r * C + c8) = xv;
  }
}

int add_bcast_rows(int dtype, void* x, const void* tab, long long rows, int rows_per_batch, int C, cudaStream_t st) {
  if (C % 8) { set_error("add_bcast_rows: C must be a multiple of 8"); return -1; }
  const long long total = rows * (C / 8);
  int grid = static_cast<int>((total + 255) / 256);
  if (grid > num_sms() * 32) grid = num_sms() * 32;
  if (dtype == DT_F16) add_bcast_rows_kernel<__half><<<grid, 256, 0, st>>>((__half*)x, (const __half*)tab, rows, rows_per_batch, C);
  else add_bcast_rows_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((__nv_bfloat16*)x, (const __nv_bfloat16*)tab, rows, rows_per_batch, C);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ 2x2 patch-merging gather
// x [B, H, W, C] -> y [B, ceil(H/2), ceil(W/2), 4C], channel blocks (dy,dx) = (0,0), (1,0), (0,1), (1,1); an odd H / W is zero
// padded by one row / column (DonutSwinPatchMerging.maybe_pad, encoder.py:281-287)
template <typename T>
__global__ void patch_merge_gather_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int H, int W, int C) {
  const int cv = C >> 3, Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = static_cast<long long>(B) * Ho * Wo * 4 * cv;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c8 = (idx % cv) * 8;
    long long r = idx / cv;
    const int blk = r % 4;
    r /= 4;
    const int ox = r % Wo, oy = (r / Wo) % Ho;
    const int b = r / (static_cast<long long>(Wo) * Ho);
    const int dy = blk & 1, dx = blk >> 1;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (2 * oy + dy < H && 2 * ox + dx < W)
      v = *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(b) * H + 2 * oy + dy) * W + 2 * ox + dx) * C + c8);
    *reinterpret_cast<uint4*>(y + (((static_cast<size_t>(b) * Ho + oy) * Wo + ox) * 4 + blk) * C + c8) = v;
  }
}

int patch_merge_gather(int dtype, const void* x, void* y, int B, int H, int W, int C, cudaStream_t st) {
  if (C % 8) { set_error("patch_merge_gather: C must be a multiple of 8"); return -1; }
  const long long total = static_cast<long long>(B) * ((H + 1) / 2) * ((W + 1) / 2) * 4 * (C / 8);
  int grid = static_cast<int>((total + 255) / 256);
  if (grid > num_sms() * 32) grid = num_sms() * 32;
  if (dtype == DT_F16) patch_merge_gather_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (__half*)y, B, H, W, C);
  else patch_merge_gather_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, B, H, W, C);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ Swin window attention
template <typename T> struct MmaS;
template <> struct MmaS<__nv_bfloat16> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) { __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&v); }
};
template <> struct MmaS<__half> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) { __half2 v = __floats2half2_rn(lo, hi); return *reinterpret_cast<uint32_t*>(&v); }
};

// qkv [B*H*W, 3C] natural token order (q | k | v, head h at h*32); bias_table T [225, nh]; out [B*H*W, C].
// One CTA = one 8x8 window x 4 heads (128 contiguous channels per token); warp w owns query rows 16w..16w+15.
// H, W that are not multiples of the window are handled like DonutSwinLayer.maybe_pad (encoder.py:591-596): the token grid is
// padded with ZERO rows (after layernorm_before) to Hp x Wp, so a pad token's q / k / v is the QKV bias; windows, the cyclic shift
// and the shift mask live on the padded grid and pad query rows are dropped (the reference crops them, encoder.py:657-659).
template <typename T>
__global__ void __launch_bounds__(128) swin_window_attn_kernel(const T* __restrict__ qkv, const float* __restrict__ qkv_bias,
                                                               const T* __restrict__ bias_table, T* __restrict__ out, int Hr,
                                                               int Wr, int H, int W, int C, int nh, int shift, float scale) {
  constexpr int WS = 8, NT = 64, HD = 32, HG = 4, LDS = HG * HD + 8;
  extern __shared__ __align__(16) uint8_t smem_sw[];
  T* sQ = reinterpret_cast<T*>(smem_sw);
  T* sK = sQ + NT * LDS;
  T* sV = sK + NT * LDS;
  float* sBias = reinterpret_cast<float*>(sV + NT * LDS);   // [225][HG]
  __shared__ int s_tok[NT];
  __shared__ int s_reg[NT];

  const int nwx = W / WS, nwy = H / WS;
  const int win = blockIdx.x % (nwx * nwy);
  const int b = blockIdx.x / (nwx * nwy);
  const int hg = blockIdx.y;                 // head group
  const int wy = win / nwx, wx = win % nwx;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;

  if (tid < NT) {
    const int py = tid / WS, px = tid % WS;
    const int ys = wy * WS + py, xs = wx * WS + px;                 // coordinates in the shifted image
    const int y = (ys + shift) % H, x = (xs + shift) % W;           // torch.roll(-shift) source (H, W = padded grid)
    s_tok[tid] = (y < Hr && x < Wr) ? (b * Hr + y) * Wr + x : -1;   // -1 = pad token
    int ry = 0, rx = 0;
    if (shift > 0) {
      ry = ys < H - WS ? 0 : (ys < H - shift ? 1 : 2);
      rx = xs < W - WS ? 0 : (xs < W - shift ? 1 : 2);
    }
    s_reg[tid] = ry * 3 + rx;
  }
  for (int i = tid; i < 225 * HG; i += 128) {
    const int e = i / HG, hh = i % HG;
    sBias[i] = to_f<T>(bias_table[static_cast<size_t>(e) * nh + hg * HG + hh]);
  }
  __syncthreads();
  // gather Q, K, V rows of this window for the 4 heads (256 contiguous bytes per token and tensor)
  constexpr int VPR = HG * HD / 8;  // 16
  for (int i = tid; i < NT * VPR; i += 128) {
    const int r = i / VPR, c = i % VPR;
    if (s_tok[r] >= 0) {
      const T* base = qkv + static_cast<size_t>(s_tok[r]) * (3 * C) + hg * HG * HD + c * 8;
      *reinterpret_cast<uint4*>(sQ + r * LDS + c * 8) = *reinterpret_cast<const uint4*>(base);
      *reinterpret_cast<uint4*>(sK + r * LDS + c * 8) = *reinterpret_cast<const uint4*>(base + C);
      *reinterpret_cast<uint4*>(sV + r * LDS + c * 8) = *reinterpret_cast<const uint4*>(base + 2 * C);
    } else {
      // Linear(0) = bias, rounded to T like any other GEMM output row
      const float* bq = qkv_bias + hg * HG * HD + c * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        sQ[r * LDS + c * 8 + j] = from_f<T>(bq[j]);
        sK[r * LDS + c * 8 + j] = from_f<T>(bq[C + j]);
        sV[r * LDS + c * 8 + j] = from_f<T>(bq[2 * C + j]);
      }
    }
  }
  __syncthreads();

  const int rbase = warp * 16;
  const int q0 = rbase + g, q1 = q0 + 8;
  const int q0y = q0 / WS, q0x = q0 % WS, q1y = q1 / WS, q1x = q1 % WS;
  const int reg0 = s_reg[q0], reg1 = s_reg[q1];
  for (int hh = 0; hh < HG; ++hh) {
    const int co = hh * HD;
    uint32_t aQ[2][4];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      aQ[ks][0] = *reinterpret_cast<const uint32_t*>(sQ + q0 * LDS + co + ks * 16 + 2 * t);
      aQ[ks][1] = *reinterpret_cast<const uint32_t*>(sQ + q1 * LDS + co + ks * 16 + 2 * t);
      aQ[ks][2] = *reinterpret_cast<const uint32_t*>(sQ + q0 * LDS + co + ks * 16 + 8 + 2 * t);
      aQ[ks][3] = *reinterpret_cast<const uint32_t*>(sQ + q1 * LDS + co + ks * 16 + 8 + 2 * t);
    }
    float S[8][4];
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      S[nt][0] = S[nt][1] = S[nt][2] = S[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (nt * 8 + g) * LDS + co + ks * 16 + 2 * t);
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (nt * 8 + g) * LDS + co + ks * 16 + 8 + 2 * t);
        MmaS<T>::run(S[nt], aQ[ks], b0, b1);
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = nt * 8 + 2 * t + (e & 1);
        const int ky = key / WS, kx = key % WS;
        const int qy = e < 2 ? q0y : q1y, qx = e < 2 ? q0x : q1x;
        float add = sBias[((qy - ky + WS - 1) * (2 * WS - 1) + (qx - kx + WS - 1)) * HG + hh];
        if (shift > 0 && s_reg[key] != (e < 2 ? reg0 : reg1)) add = rnd<T>(add - 100.0f);   // mask + bias summed in T
        const float sv = S[nt][e] * scale + add;
        S[nt][e] = sv;
        if (e < 2) mx0 = fmaxf(mx0, sv); else mx1 = fmaxf(mx1, sv);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      S[nt][0] = __expf(S[nt][0] - mx0); S[nt][1] = __expf(S[nt][1] - mx0);
      S[nt][2] = __expf(S[nt][2] - mx1); S[nt][3] = __expf(S[nt][3] - mx1);
      l0 += S[nt][0] + S[nt][1];
      l1 += S[nt][2] + S[nt][3];
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    float O[4][4];
#pragma unroll
    for (int dn = 0; dn < 4; ++dn) O[dn][0] = O[dn][1] = O[dn][2] = O[dn][3] = 0.f;
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      uint32_t aP[4];
      aP[0] = MmaS<T>::pack(S[2 * kc][0] * i0, S[2 * kc][1] * i0);
      aP[1] = MmaS<T>::pack(S[2 * kc][2] * i1, S[2 * kc][3] * i1);
      aP[2] = MmaS<T>::pack(S[2 * kc + 1][0] * i0, S[2 * kc + 1][1] * i0);
      aP[3] = MmaS<T>::pack(S[2 * kc + 1][2] * i1, S[2 * kc + 1][3] * i1);
      const int mid = lane >> 3, r = lane & 7;
#pragma unroll
      for (int dn = 0; dn < 4; dn += 2) {
        uint32_t bv[4];
        const T* addr = sV + (kc * 16 + (mid & 1) * 8 + r) * LDS + co + (dn + (mid >> 1)) * 8;
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                     : "=r"(bv[0]), "=r"(bv[1]), "=r"(bv[2]), "=r"(bv[3]) : "r"(smem_u32(addr)));
        MmaS<T>::run(O[dn], aP, bv[0], bv[1]);
        MmaS<T>::run(O[dn + 1], aP, bv[2], bv[3]);
      }
    }
    const int tk0 = s_tok[q0], tk1 = s_tok[q1];
    T* o0 = out + static_cast<size_t>(tk0 < 0 ? 0 : tk0) * C + (hg * HG + hh) * HD;
    T* o1 = out + static_cast<size_t>(tk1 < 0 ? 0 : tk1) * C + (hg * HG + hh) * HD;
#pragma unroll
    for (int dn = 0; dn < 4; ++dn) {
      if (tk0 >= 0) *reinterpret_cast<uint32_t*>(o0 + dn * 8 + 2 * t) = MmaS<T>::pack(O[dn][0], O[dn][1]);
      if (tk1 >= 0) *reinterpret_cast<uint32_t*>(o1 + dn * 8 + 2 * t) = MmaS<T>::pack(O[dn][2], O[dn][3]);
    }
  }
}

int swin_window_attn(int dtype, const void* qkv, const float* qkv_bias, const void* bias_table, void* out, int B, int H, int W, int C,
                     int nh, int shift, cudaStream_t st) {
  if (nh % 4 || C != nh * 32) {
    set_error("swin_window_attn: needs head_dim 32 and heads in groups of 4 (C=%d nh=%d)", C, nh);
    return -1;
  }
  if (H < 8 || W < 8) {
    // the reference shrinks the window to min(H, W) here (encoder.py:550-558) and then fails on its own 8x8 relative-position bias
    set_error("swin_window_attn: token grid %dx%d is smaller than the 8x8 window", H, W);
    return -1;
  }
  const int Hp = (H + 7) / 8 * 8, Wp = (W + 7) / 8 * 8;
  if ((Hp != H || Wp != W) && !qkv_bias) {
    set_error("swin_window_attn: a %dx%d grid needs window padding, which needs the QKV bias (pad tokens are Linear(0))", H, W);
    return -1;
  }
  constexpr size_t SMEM = 3 * 64 * (128 + 8) * 2 + 225 * 4 * 4;
  dim3 grid(B * (Hp / 8) * (Wp / 8), nh / 4), block(128);
  const float scale = 0.17677669529663687f;  // 32^-0.5
  if (dtype == DT_F16) {
    static bool set = false;
    if (!set) { cudaFuncSetAttribute(swin_window_attn_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM); set = true; }
    swin_window_attn_kernel<__half><<<grid, block, SMEM, st>>>((const __half*)qkv, qkv_bias, (const __half*)bias_table, (__half*)out, H, W, Hp, Wp, C, nh, shift, scale);
  } else {
    static bool set = false;
    if (!set) { cudaFuncSetAttribute(swin_window_attn_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM); set = true; }
    swin_window_attn_kernel<__nv_bfloat16><<<grid, block, SMEM, st>>>((const __nv_bfloat16*)qkv, qkv_bias, (const __nv_bfloat16*)bias_table, (__nv_bfloat16*)out, H, W, Hp, Wp, C, nh, shift, scale);
  }
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ BboxEmbedding
// boxes i64 [n, 7] = (cx, cy, w, h, xskew, yskew, label); tables T [15][...]: w,h,cx,cy,xskew,yskew,x1,y1,..,y4 each
// [vocab, Hd], label [label_count, Hd].  Sums follow the reference's association order, one rounding per add.
struct BboxTables { const void* t[15]; };

template <typename T>
__global__ void bbox_embed_sum_kernel(const long long* __restrict__ boxes, BboxTables tabs, T* __restrict__ out, int n, int Hd,
                                      int bbox_size) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const long long* bx = boxes + static_cast<size_t>(r) * 7;
  const long long cx = bx[0], cy = bx[1], w = bx[2], h = bx[3], xs = bx[4], ys = bx[5], label = bx[6];
  auto trunc_div2 = [](long long v) { return static_cast<long long>(static_cast<double>(v) / 2.0); };  // (x / 2).to(long)
  const long long xa = trunc_div2(xs - bbox_size / 2), ya = trunc_div2(ys - bbox_size / 2);
  auto fdiv2 = [](long long v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); };                            // python floor //
  auto cl = [&](long long v) { return v < 0 ? 0LL : (v > bbox_size ? static_cast<long long>(bbox_size) : v); };
  const long long hw = fdiv2(w), hh = fdiv2(h);
  const long long idx[15] = {w, h, cx, cy, xs, ys,
                             cl(cx - hw - xa), cl(cy - hh - ya), cl(cx + hw - xa), cl(cy + hh + ya),
                             cl(cx + hw + xa), cl(cy + hh + ya), cl(cx - hw + xa), cl(cy - hh - ya), label};
  const T* rows[15];
#pragma unroll
  for (int i = 0; i < 15; ++i) rows[i] = reinterpret_cast<const T*>(tabs.t[i]) + static_cast<size_t>(idx[i]) * Hd;
  T* o = out + static_cast<size_t>(r) * Hd;
  for (int c = threadIdx.x; c < Hd; c += blockDim.x) {
    auto f = [&](int i) { return to_f<T>(rows[i][c]); };
    const float size = rnd<T>(rnd<T>(rnd<T>(f(0) + f(1)) + f(2)) + f(3));
    const float skew = rnd<T>(f(4) + f(5));
    float corner = rnd<T>(f(6) + f(7));
#pragma unroll
    for (int i = 8; i < 14; ++i) corner = rnd<T>(corner + f(i));
    const float e = rnd<T>(rnd<T>(rnd<T>(f(14) + size) + skew) + corner);
    o[c] = from_f<T>(e);
  }
}

int bbox_embed_sum(int dtype, const long long* boxes, const void* const* tables, void* out, int n, int Hd, int bbox_size,
                   cudaStream_t st) {
  if (n <= 0) return 0;
  BboxTables tb;
  for (int i = 0; i < 15; ++i) tb.t[i] = tables[i];
  if (dtype == DT_F16) bbox_embed_sum_kernel<__half><<<n, 128, 0, st>>>(boxes, tb, (__half*)out, n, Hd, bbox_size);
  else bbox_embed_sum_kernel<__nv_bfloat16><<<n, 128, 0, st>>>(boxes, tb, (__nv_bfloat16*)out, n, Hd, bbox_size);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ single-query attention
// q [B, nh*HD]; K/V element (set, kvh, j, c) at base + set*bs + kvh*hs + j*ts + c with set = kv_index ? kv_index[b] : b;
// out [B, nh*HD]. One CTA per (b, kv head).
template <typename T, int HD, int G>
__global__ void __launch_bounds__(128) attn_single_query_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ K,
                                                                const T* __restrict__ V, long long bs, long long hs,
                                                                long long ts, T* __restrict__ out, int ldo, int n_keys,
                                                                float scale, const int* __restrict__ kv_index) {
  constexpr int VPR = HD / 8, NKG = 128 / VPR;
  extern __shared__ __align__(16) uint8_t smem_sq[];
  T* q_t = reinterpret_cast<T*>(smem_sq);            // [G][HD] query rows, kept in T (first G*HD floats' worth of space)
  float* red = reinterpret_cast<float*>(smem_sq) + G * HD;   // [NKG][G][HD]
  float* sc = red + NKG * G * HD;                    // [G][n_keys]
  __shared__ float s_red[4][G];
  __shared__ float s_m[G], s_l[G];
  const int b = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const T* qr = q + static_cast<size_t>(b) * ldq + kvh * G * HD;
  for (int i = tid; i < G * HD; i += 128) q_t[i] = qr[i];
  const long long set = kv_index ? kv_index[b] : b;     // K/V set of this query row (many rows may share one set)
  const T* kb = K + set * bs + kvh * hs;
  const T* vb = V + set * bs + kvh * hs;
  __syncthreads();
  float tmax[G];
#pragma unroll
  for (int gq = 0; gq < G; ++gq) tmax[gq] = -INFINITY;
  // The kernel is a latency chain, not a bandwidth problem (64 CTAs x 4 warps, 147 KB of K / V each): every global load of a thread's
  // next key used to wait for the arithmetic of the previous one.  Keys are therefore taken KU at a time with all their row loads
  // issued first; the multiply-add order per accumulator is unchanged, so results are bit-identical to the one-key-at-a-time loop.
  constexpr int KU = 2;
  for (int j0 = tid; j0 < n_keys; j0 += 128 * KU) {
    uint4 kv[KU][VPR];
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const int j = j0 + u * 128;
      if (j < n_keys) {
        const uint4* kr = reinterpret_cast<const uint4*>(kb + j * ts);
#pragma unroll
        for (int c = 0; c < VPR; ++c) kv[u][c] = kr[c];
      }
    }
#pragma unroll
    for (int u = 0; u < KU; ++u) {
      const int j = j0 + u * 128;
      if (j >= n_keys) break;
      float acc[G];
#pragma unroll
      for (int gq = 0; gq < G; ++gq) acc[gq] = 0.f;
#pragma unroll
      for (int c = 0; c < VPR; ++c) {
        const unsigned short* kb16 = reinterpret_cast<const unsigned short*>(&kv[u][c]);
#pragma unroll
        for (int gq = 0; gq < G; ++gq) {      // FHFMA: 16-bit q and k, fp32 accumulate, no conversions (bit-identical to fmaf on floats)
          const uint4 qv = *reinterpret_cast<const uint4*>(q_t + gq * HD + c * 8);
          const unsigned short* qb = reinterpret_cast<const unsigned short*>(&qv);
#pragma unroll
          for (int x = 0; x < 8; ++x) acc[gq] = fma16<T>(qb[x], kb16[x], acc[gq]);
        }
      }
#pragma unroll
      for (int gq = 0; gq < G; ++gq) {
        const float sv = acc[gq] * scale;
        sc[gq * n_keys + j] = sv;
        tmax[gq] = fmaxf(tmax[gq], sv);
      }
    }
  }
#pragma unroll
  for (int gq = 0; gq < G; ++gq) { const float m = warp_max(tmax[gq]); if (lane == 0) s_red[warp][gq] = m; }
  __syncthreads();
  if (tid < G) s_m[tid] = fmaxf(fmaxf(s_red[0][tid], s_red[1][tid]), fmaxf(s_red[2][tid], s_red[3][tid]));
  __syncthreads();
  float tsum[G];
#pragma unroll
  for (int gq = 0; gq < G; ++gq) tsum[gq] = 0.f;
  for (int j = tid; j < n_keys; j += 128) {
#pragma unroll
    for (int gq = 0; gq < G; ++gq) {
      const float pv = __expf(sc[gq * n_keys + j] - s_m[gq]);
      tsum[gq] += pv;
      sc[gq * n_keys + j] = pv;
    }
  }
#pragma unroll
  for (int gq = 0; gq < G; ++gq) { const float s = warp_sum(tsum[gq]); if (lane == 0) s_red[warp][gq] = s; }
  __syncthreads();
  if (tid < G) s_l[tid] = s_red[0][tid] + s_red[1][tid] + s_red[2][tid] + s_red[3][tid];
  __syncthreads();
  const int chunk = tid % VPR, kg = tid / VPR;
  if (kg < NKG) {
    float acc[G][8];
#pragma unroll
    for (int gq = 0; gq < G; ++gq)
#pragma unroll
      for (int x = 0; x < 8; ++x) acc[gq][x] = 0.f;
    constexpr int VU = 6;                       // V rows in flight per thread (576 keys / 16 key groups = 6 rounds of 6)
    for (int j0 = kg; j0 < n_keys; j0 += NKG * VU) {
      uint4 vv[VU];
#pragma unroll
      for (int u = 0; u < VU; ++u) {
        const int j = j0 + u * NKG;
        if (j < n_keys) vv[u] = *reinterpret_cast<const uint4*>(vb + j * ts + chunk * 8);
      }
#pragma unroll
      for (int u = 0; u < VU; ++u) {
        const int j = j0 + u * NKG;
        if (j >= n_keys) break;
        const unsigned short* vb16 = reinterpret_cast<const unsigned short*>(&vv[u]);
#pragma unroll
        for (int gq = 0; gq < G; ++gq) {
          const unsigned short pb = bits_of<T>(from_f<T>(sc[gq * n_keys + j] / s_l[gq]));
#pragma unroll
          for (int x = 0; x < 8; ++x) acc[gq][x] = fma16<T>(pb, vb16[x], acc[gq][x]);
        }
      }
    }
#pragma unroll
    for (int gq = 0; gq < G; ++gq)
#pragma unroll
      for (int x = 0; x < 8; ++x) red[(kg * G + gq) * HD + chunk * 8 + x] = acc[gq][x];
  }
  __syncthreads();
  T* orow = out + static_cast<size_t>(b) * ldo + kvh * G * HD;
  for (int i = tid; i < G * HD; i += 128) {
    float s = 0.f;
#pragma unroll
    for (int k2 = 0; k2 < NKG; ++k2) s += red[k2 * G * HD + i];
    orow[i] = from_f<T>(s);
  }
}

template <typename T, int G>
static int launch_sq(const void* q, int ldq, const void* K, const void* V, long long bs, long long hs, long long ts, void* out,
                     int ldo, int B, int nkv, int n_keys, float scale, const int* kv_index, cudaStream_t st) {
  constexpr int HD = 64, NKG = 128 / (HD / 8);
  const size_t smem = (static_cast<size_t>(G) * HD + static_cast<size_t>(NKG) * G * HD + static_cast<size_t>(G) * n_keys) * sizeof(float);
  auto kern = attn_single_query_kernel<T, HD, G>;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      cudaGetLastError();
      set_error("attn_single_query: %zu bytes of shared memory exceed the device limit", smem);
      return -3;
    }
    attr = smem;
  }
  kern<<<dim3(B, nkv), 128, smem, st>>>((const T*)q, ldq, (const T*)K, (const T*)V, bs, hs, ts, (T*)out, ldo, n_keys, scale,
                                        kv_index);
  return launch_ok();
}

int attn_single_query(int dtype, const void* q, int ldq, const void* K, const void* V, long long bs, long long hs, long long ts,
                      void* out, int ldo, int B, int nh, int nkv, int head_dim, int n_keys, float scale, cudaStream_t st,
                      const int* kv_index) {
  if (head_dim != 64) { set_error("attn_single_query: head_dim 64 is instantiated (got %d)", head_dim); return -1; }
  if (nkv <= 0 || nh % nkv) { set_error("attn_single_query: nh (%d) must be a positive multiple of nkv (%d)", nh, nkv); return -1; }
  if (n_keys <= 0) { set_error("attn_single_query: n_keys must be positive (got %d)", n_keys); return -1; }
  const int G = nh / nkv;
#define SQ(T_) \
  (G == 1 ? launch_sq<T_, 1>(q, ldq, K, V, bs, hs, ts, out, ldo, B, nkv, n_keys, scale, kv_index, st) : \
   G == 2 ? launch_sq<T_, 2>(q, ldq, K, V, bs, hs, ts, out, ldo, B, nkv, n_keys, scale, kv_index, st) : \
   G == 4 ? launch_sq<T_, 4>(q, ldq, K, V, bs, hs, ts, out, ldo, B, nkv, n_keys, scale, kv_index, st) : -9)
  int rc = dtype == DT_F16 ? SQ(__half) : SQ(__nv_bfloat16);
#undef SQ
  if (rc == -9) set_error("attn_single_query: GQA group %d not instantiated (1/2/4)", G);
  return rc;
}

// ------------------------------------------------------------------------------------------------ table_rec LabelEmbedding
// LabelEmbedding.forward (table_rec/model/decoder.py:46-73): out[:, :box_w] = (size + skew) + corner with corner = x1+y1+x3+y3,
// out[:, box_w:] = (category + merges) + colspan; every add rounds to T like the eager graph does.
struct LabelTables { const void* t[13]; };   // w,h,cx,cy,xskew,yskew,x1,y1,x3,y3 (width box_w) | category,merge,colspan (width prop_w)

template <typename T>
__global__ void label_embed_kernel(const long long* __restrict__ boxes, LabelTables tabs, T* __restrict__ out, int n, int box_w,
                                   int prop_w, int bbox_size, int vocab) {
  const int r = blockIdx.x;
  if (r >= n) return;
  const long long* bx = boxes + static_cast<size_t>(r) * 10;
  auto cv = [&](long long v) { return v < 0 ? 0LL : (v > vocab ? static_cast<long long>(vocab) : v); };
  const long long cx = cv(bx[0]), cy = cv(bx[1]), w = cv(bx[2]), h = cv(bx[3]), xs = cv(bx[4]), ys = cv(bx[5]);
  const long long cat = cv(bx[6]), mrg = cv(bx[7]), col = cv(bx[8]);
  auto trunc_div2 = [](long long v) { return static_cast<long long>(static_cast<double>(v) / 2.0); };
  const long long xa = trunc_div2(xs - bbox_size / 2), ya = trunc_div2(ys - bbox_size / 2);
  auto cl = [&](long long v) { return v < 0 ? 0LL : (v > bbox_size ? static_cast<long long>(bbox_size) : v); };
  const long long hw = w / 2, hh = h / 2;
  const long long idx[13] = {w, h, cx, cy, xs, ys, cl(cx - hw - xa), cl(cy - hh - ya), cl(cx + hw + xa), cl(cy + hh + ya),
                             cat, mrg, col};
  T* o = out + static_cast<size_t>(r) * (box_w + prop_w);
  for (int c = threadIdx.x; c < box_w + prop_w; c += blockDim.x) {
    float e;
    if (c < box_w) {
      auto f = [&](int i) { return to_f<T>(reinterpret_cast<const T*>(tabs.t[i])[static_cast<size_t>(idx[i]) * box_w + c]); };
      const float size = rnd<T>(rnd<T>(rnd<T>(f(0) + f(1)) + f(2)) + f(3));
      const float skew = rnd<T>(f(4) + f(5));
      const float corner = rnd<T>(rnd<T>(rnd<T>(f(6) + f(7)) + f(8)) + f(9));
      e = rnd<T>(rnd<T>(size + skew) + corner);
    } else {
      const int pc = c - box_w;
      auto f = [&](int i) { return to_f<T>(reinterpret_cast<const T*>(tabs.t[i])[static_cast<size_t>(idx[i]) * prop_w + pc]); };
      e = rnd<T>(rnd<T>(f(10) + f(11)) + f(12));
    }
    o[c] = from_f<T>(e);
  }
}

int label_embed(int dtype, const long long* boxes, const void* const* tables, void* out, int n, int box_w, int prop_w,
                int bbox_size, int vocab, cudaStream_t st) {
  if (n <= 0) return 0;
  LabelTables tb;
  for (int i = 0; i < 13; ++i) tb.t[i] = tables[i];
  if (dtype == DT_F16) label_embed_kernel<__half><<<n, 128, 0, st>>>(boxes, tb, (__half*)out, n, box_w, prop_w, bbox_size, vocab);
  else label_embed_kernel<__nv_bfloat16><<<n, 128, 0, st>>>(boxes, tb, (__nv_bfloat16*)out, n, box_w, prop_w, bbox_size, vocab);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ next box token
// The predictors' per-step token formation, on the device: columns 0..5 = trunc(clamp(bbox * bbox_size, 0, bbox_size))
// (layout/__init__.py:125-137; table_rec/__init__.py:88-93 + shaper.dict_to_labels), then one column per head:
// mode 0 = argmax (first maximum), mode 1 = round-half-even(max(v, 1)) (table colspan).  done[b] = token of head `done_head`
// is eos or pad (table_rec/__init__.py:84-87).  Optional decode-loop state so that a whole step can live in a CUDA graph:
// cache_pos[b] is advanced (decoder_position_ids + 1) and the step's tokens / raw head outputs are appended to history
// arrays at row (cache_pos[b] - hist_base[0]).
// Optional page rule (rule.page_wh non-null): LayoutPredictor's header/footer relabelling (layout/__init__.py:147-174) on head 0.
struct StepHeads { const float* p[4]; int n[4]; int mode[4]; float* hist[4]; };

// rounding of one torch op on 16-bit CPU tensors: the float result rounded to the model dtype
__device__ __forceinline__ float round_dt(float v, int dtype) {
  return dtype == DT_F16 ? __half2float(__float2half_rn(v)) : __bfloat162float(__float2bfloat16_rn(v));
}

// prediction_to_polygon (layout/util.py:4-40) from the model-dtype row [bbox * bbox_size x6, class] that the predictor builds
// (layout/__init__.py:127, 137), then the position test of the rule in Python float (double): corner 0 below 0.8 and corner 2
// above 0.2 of the page on both axes.
__device__ __forceinline__ bool header_footer_misplaced(const float* bb, float bbox_size, const PageRule& r, int b) {
  float v[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) v[i] = round_dt(__fmul_rn(bb[i], bbox_size), r.dtype);
  const float hw = round_dt(__fdiv_rn(v[2], 2.f), r.dtype), hh = round_dt(__fdiv_rn(v[3], 2.f), r.dtype);
  const float x1 = round_dt(__fsub_rn(v[0], hw), r.dtype), x2 = round_dt(__fadd_rn(v[0], hw), r.dtype);
  const float y1 = round_dt(__fsub_rn(v[1], hh), r.dtype), y2 = round_dt(__fadd_rn(v[1], hh), r.dtype);
  const float sx = floorf(round_dt(__fdiv_rn(round_dt(__fsub_rn(v[4], r.skew_scaler), r.dtype), 2.f), r.dtype));
  const float sy = floorf(round_dt(__fdiv_rn(round_dt(__fsub_rn(v[5], r.skew_scaler), r.dtype), 2.f), r.dtype));
  // |skew| < skew_min -> 0 only ever clears a (signed) zero: the floors are integers
  const double pw = r.page_wh[2 * b], ph = r.page_wh[2 * b + 1];
  const double ws = pw / static_cast<double>(bbox_size), hs = ph / static_cast<double>(bbox_size);
  const double p0x = static_cast<double>(round_dt(__fsub_rn(x1, sx), r.dtype)) * ws;
  const double p0y = static_cast<double>(round_dt(__fsub_rn(y1, sy), r.dtype)) * hs;
  const double p2x = static_cast<double>(round_dt(__fadd_rn(x2, sx), r.dtype)) * ws;
  const double p2y = static_cast<double>(round_dt(__fadd_rn(y2, sy), r.dtype)) * hs;
  return p0y < ph * .8 && p2y > ph * .2 && p0x < pw * .8 && p2x > pw * .2;
}

__global__ void box_next_token_kernel(const float* __restrict__ bbox, StepHeads hd, int n_heads, float bbox_size,
                                      long long* __restrict__ out, unsigned char* __restrict__ done, int done_head, int eos,
                                      int pad, int B, int* __restrict__ cache_pos, const int* __restrict__ hist_base, int hist_T,
                                      long long* __restrict__ hist_tok, float* __restrict__ hist_bbox,
                                      unsigned char* __restrict__ hist_done, PageRule rule) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int ncol = 6 + n_heads;
  long long tok[10];
  for (int i = 0; i < 6; ++i) {
    float v = bbox[b * 6 + i] * bbox_size;
    v = fminf(fmaxf(v, 0.f), bbox_size);
    tok[i] = static_cast<long long>(v);
  }
  unsigned char dn = 0;
  for (int k = 0; k < n_heads; ++k) {
    const float* p = hd.p[k] + static_cast<size_t>(b) * hd.n[k];
    long long t;
    if (hd.mode[k] == 1) {
      t = static_cast<long long>(rintf(fmaxf(p[0], 1.f)));
    } else {
      int best = 0;
      float bv = p[0];
      for (int j = 1; j < hd.n[k]; ++j)
        if (p[j] > bv) { bv = p[j]; best = j; }
      t = best;
    }
    tok[6 + k] = t;
    if (k == done_head) dn = (t == eos || t == pad) ? 1 : 0;
  }
  // header / footer rule: the class logit of a misplaced PageHeader / PageFooter is set to 0 and the first maximum taken again;
  // the new class feeds the next step and the modified logits go to the history (done still comes from the first argmax)
  long long zeroed = -1;
  if (rule.page_wh && !dn && !(rule.sticky && rule.sticky[b]) && (tok[6] == rule.header || tok[6] == rule.footer) &&
      header_footer_misplaced(bbox + static_cast<size_t>(b) * 6, bbox_size, rule, b)) {
    const float* p = hd.p[0] + static_cast<size_t>(b) * hd.n[0];
    zeroed = tok[6];
    int best = 0;
    float bv = zeroed == 0 ? 0.f : p[0];
    for (int j = 1; j < hd.n[0]; ++j) {
      const float v = j == zeroed ? 0.f : p[j];
      if (v > bv) { bv = v; best = j; }
    }
    tok[6] = best;
  }
  int row = -1;
  if (cache_pos) {
    const int pos = cache_pos[b];
    if (hist_base) row = pos - hist_base[0];
    cache_pos[b] = pos + 1;
  }
  if (row >= 0 && row < hist_T) {
    const size_t r = static_cast<size_t>(row) * B + b;
    if (hist_tok)
      for (int i = 0; i < ncol; ++i) hist_tok[r * ncol + i] = tok[i];
    if (hist_bbox)
      for (int i = 0; i < 6; ++i) hist_bbox[r * 6 + i] = bbox[b * 6 + i];
    for (int k = 0; k < n_heads; ++k)
      if (hd.hist[k])
        for (int j = 0; j < hd.n[k]; ++j)
          hd.hist[k][r * hd.n[k] + j] = (k == 0 && j == zeroed) ? 0.f : hd.p[k][static_cast<size_t>(b) * hd.n[k] + j];
    if (hist_done && done_head >= 0) hist_done[r] = dn;
  }
  // the token buffer may alias nothing this step still reads: written last
  for (int i = 0; i < ncol; ++i) out[static_cast<size_t>(b) * ncol + i] = tok[i];
  if (done && done_head >= 0) done[b] = dn;
}

int box_next_token(const float* bbox, const float* const* heads, const int* head_n, const int* head_mode, int n_heads,
                   float bbox_size, long long* out, unsigned char* done, int done_head, int eos, int pad, int B, int* cache_pos,
                   const int* hist_base, int hist_T, long long* hist_tok, float* hist_bbox, float* const* hist_heads,
                   unsigned char* hist_done, cudaStream_t st, const PageRule& rule) {
  if (B <= 0) return 0;
  if (n_heads < 0 || n_heads > 4) { set_error("box_next_token: at most 4 heads"); return -1; }
  if (rule.page_wh && (n_heads < 1 || head_mode[0] != 0)) { set_error("box_next_token: the page rule needs an argmax class head 0"); return -1; }
  StepHeads h{};
  for (int i = 0; i < n_heads; ++i) {
    h.p[i] = heads[i]; h.n[i] = head_n[i]; h.mode[i] = head_mode[i];
    h.hist[i] = hist_heads ? hist_heads[i] : nullptr;
  }
  box_next_token_kernel<<<(B + 63) / 64, 64, 0, st>>>(bbox, h, n_heads, bbox_size, out, done, done_head, eos, pad, B, cache_pos,
                                                      hist_base, hist_T, hist_tok, hist_bbox, hist_done, rule);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------------ sticky done + active count
// The stop rule of TableRecPredictor.inference_loop (table_rec/__init__.py:111-115) on the device: sticky[b] |= done[b], and
// n_active[0] = the number of rows not yet done.  One CTA, so that the count is written by one store after the block reduce.
__global__ void __launch_bounds__(256) rows_done_count_kernel(const unsigned char* __restrict__ done, unsigned char* __restrict__ sticky,
                                                              int* __restrict__ n_active, int B) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  int cnt = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const unsigned char d = sticky[b] | done[b];
    sticky[b] = d;
    cnt += d ? 0 : 1;
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0) n_active[0] = s_cnt;
}

int rows_done_count(const unsigned char* done, unsigned char* sticky, int* n_active, int B, cudaStream_t st) {
  if (B <= 0) return 0;
  rows_done_count_kernel<<<1, 256, 0, st>>>(done, sticky, n_active, B);
  return launch_ok();
}

}  // namespace sb
