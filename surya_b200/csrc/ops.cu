// surya_b200 — row-wise / gather / rotary / head kernels (CUDA-core, HBM-bound; warp-shuffle reductions).
//
// Reference semantics (file:line relative to the reference checkout):
//   rmsnorm            surya/common/surya/decoder/__init__.py:241-258, encoder/__init__.py:90-104
//   rope_vision        surya/common/surya/encoder/__init__.py:188-199, 523-550
//   rope_decoder       surya/common/surya/decoder/__init__.py:53-84, 346-361
//   embed_splice       surya/common/surya/__init__.py:197-272
//   argmax / score     surya/recognition/__init__.py:294-324
//   bbox head          surya/common/surya/__init__.py:329
#include "ops.cuh"
#include "gemm_epilogue.cuh"
#include "sb_ptx.cuh"

namespace sb {

// ------------------------------------------------------------------------------------------ rmsnorm
// One warp per row. y = weight * T(x * rsqrt(mean(x^2) + eps)); optional row gather (src_rows).
template <typename T>
__global__ void rmsnorm_kernel(const T* __restrict__ x, int ldx, const T* __restrict__ w, T* __restrict__ y, int ldy,
                               int rows, int H, float eps, const int* __restrict__ src_rows, int mode) {
  pdl_trigger();
  pdl_wait();
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
  int srow = src_rows ? src_rows[row] : row;
  const T* xr = x + static_cast<size_t>(srow) * ldx;
  T* yr = y + static_cast<size_t>(row) * ldy;
  float ss = 0.f;
  const int nv = H >> 3;
  for (int i = lane; i < nv; i += 32) {
    uint4 u = *reinterpret_cast<const uint4*>(xr + i * 8);
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = to_f<T>(e[j]);
      ss += f * f;
    }
  }
  for (int i = (nv << 3) + lane; i < H; i += 32) {
    float f = to_f<T>(xr[i]);
    ss += f * f;
  }
  ss = warp_sum(ss);
  // mode 0: Qwen2RMSNorm  y = w * T(x * rsqrt(mean + eps))
  // mode 1: SuryaADETRDecoderRMSNorm (adetr/decoder.py:29-47)  y = T(clamp(x * rsqrt(max(mean, eps)) * (1 + w)))
  float inv = mode ? rsqrtf(fmaxf(ss / static_cast<float>(H), eps)) : rsqrtf(ss / static_cast<float>(H) + eps);
  const float tmax = sizeof(T) == 2 && !TypeInfo<T>::is_bf16 ? 65504.f : 3.3895313892515355e38f;
  for (int i = lane; i < nv; i += 32) {
    uint4 u = *reinterpret_cast<const uint4*>(xr + i * 8);
    uint4 wv = *reinterpret_cast<const uint4*>(w + i * 8);
    const T* e = reinterpret_cast<const T*>(&u);
    const T* we = reinterpret_cast<const T*>(&wv);
    uint4 o;
    T* oe = reinterpret_cast<T*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (mode) {
        float v = to_f<T>(e[j]) * inv * (1.0f + to_f<T>(we[j]));
        v = fminf(fmaxf(v, -tmax), tmax);
        oe[j] = from_f<T>(v != v ? 0.f : v);
      } else {
        float n = rnd<T>(to_f<T>(e[j]) * inv);
        oe[j] = from_f<T>(to_f<T>(we[j]) * n);
      }
    }
    *reinterpret_cast<uint4*>(yr + i * 8) = o;
  }
  for (int i = (nv << 3) + lane; i < H; i += 32) {
    if (mode) {
      float v = to_f<T>(xr[i]) * inv * (1.0f + to_f<T>(w[i]));
      v = fminf(fmaxf(v, -tmax), tmax);
      yr[i] = from_f<T>(v != v ? 0.f : v);
    } else {
      float n = rnd<T>(to_f<T>(xr[i]) * inv);
      yr[i] = from_f<T>(to_f<T>(w[i]) * n);
    }
  }
}

int rmsnorm(int dtype, const void* x, int ldx, const void* w, void* y, int ldy, int rows, int H, float eps,
            const int* src_rows, cudaStream_t st, int mode) {
  if (rows <= 0) return 0;
  if (ldx % 8 || ldy % 8) { set_error("rmsnorm: row pitch must be a multiple of 8 elements"); return -1; }
  int wpb = 4;
  dim3 grid((rows + wpb - 1) / wpb), block(32 * wpb);
  if (dtype == DT_BF16)
    launch_pdl(rmsnorm_kernel<__nv_bfloat16>, grid, block, 0, st, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)w,
               (__nv_bfloat16*)y, ldy, rows, H, eps, src_rows, mode);
  else
    launch_pdl(rmsnorm_kernel<__half>, grid, block, 0, st, (const __half*)x, ldx, (const __half*)w, (__half*)y, ldy, rows, H,
               eps, src_rows, mode);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ row 1/rms (folded RMSNorm)
// rs[row] = rsqrt(sum_k x[row,k]^2 / H + eps) for GEMMs that fold the norm weight into W (gemm.cuh: rowscale).  Two threads
// per row add the squares in exactly the order the GEMM's in-kernel pass does (gemm_epilogue.cuh: ssq_stage — per 64-column
// block, thread h takes elements [32h, 32h + 32) in order; the halves meet at the end), so a sequence prefilled through this
// kernel and continued by decode steps sees bit-identical scales.
template <typename T>
__global__ void row_rstd_kernel(const T* __restrict__ x, int ldx, float* __restrict__ rs, int rows, int H, float eps,
                                const int* __restrict__ src_rows) {
  pdl_trigger();
  pdl_wait();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = t >> 1, hf = t & 1;
  float acc = 0.f;
  if (row < rows) {
    const T* xr = x + static_cast<size_t>(src_rows ? src_rows[row] : row) * ldx;
    constexpr int UB = 4;                 // k-blocks whose 16 loads are issued before the (strictly ordered) fma chain
    int k0 = 0;
    for (; k0 + 64 * UB <= H; k0 += 64 * UB) {
      uint4 u[UB][4];
#pragma unroll
      for (int b = 0; b < UB; ++b)
#pragma unroll
        for (int j = 0; j < 4; ++j) u[b][j] = *reinterpret_cast<const uint4*>(xr + k0 + b * 64 + hf * 32 + j * 8);
#pragma unroll
      for (int b = 0; b < UB; ++b)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const T* e = reinterpret_cast<const T*>(&u[b][j]);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float f = to_f<T>(e[i]);
            acc = fmaf(f, f, acc);
          }
        }
    }
    for (; k0 < H; k0 += 64) {
      const int c0 = k0 + hf * 32;
      if (c0 + 32 <= H) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 u = *reinterpret_cast<const uint4*>(xr + c0 + j * 8);
          const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float f = to_f<T>(e[i]);
            acc = fmaf(f, f, acc);
          }
        }
      } else {
        for (int c = c0; c < c0 + 32 && c < H; ++c) {
          const float f = to_f<T>(xr[c]);
          acc = fmaf(f, f, acc);
        }
      }
    }
  }
  const float tot = acc + __shfl_xor_sync(0xffffffffu, acc, 1);
  if (row < rows && hf == 0) rs[row] = rsqrtf(tot * (1.0f / static_cast<float>(H)) + eps);
}

int row_rstd(int dtype, const void* x, int ldx, float* rs, int rows, int H, float eps, const int* src_rows, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (ldx % 8) { set_error("row_rstd: row pitch must be a multiple of 8 elements"); return -1; }
  dim3 grid((rows * 2 + 31) / 32), block(32);      // one warp per 16 rows: small batches spread over many SMs
  if (dtype == DT_BF16)
    launch_pdl(row_rstd_kernel<__nv_bfloat16>, grid, block, 0, st, (const __nv_bfloat16*)x, ldx, rs, rows, H, eps, src_rows);
  else
    launch_pdl(row_rstd_kernel<__half>, grid, block, 0, st, (const __half*)x, ldx, rs, rows, H, eps, src_rows);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ decode tail
// Everything between the lm_head GEMM of one greedy step and the first GEMM of the next (one block per batch row):
//   * reduce the GEMM's per-tile (max, first argmax, sum exp) partials -> token, score = max softmax = 1 / sum exp(l - max),
//     done = tok in {EOS, PAD}, next id = PAD if done (RecognitionPredictor.process_outputs, surya/recognition/__init__.py:294-324);
//   * bbox head on the final hidden state with the final RMSNorm folded in: sig = T(sigmoid(T(rs * (x . Wb') + b))),
//     box = trunc(sig * bbox_size) (surya/common/surya/__init__.py:323-330);
//   * optional device-side bookkeeping of sb_rec_decode_steps: history append at *step, token feedback, position + 1, and the
//     next step's input embedding written over this row of x (embed_tokens lookup of the decoder's next call);
//   * the last block to finish advances *step.
struct TailParams {
  const float* am_val; const int* am_idx; const float* am_sum; int am_ld, n_tiles;
  const void* x; int ldx; int H; float eps;
  const void* bbox_w; const void* bbox_b; int n_box; float bbox_size;
  const void* embed; void* x_next; int ldx_next;
  long long* tok; float* score; long long* bbox; float* bbox_sig; unsigned char* done; long long* next_ids;
  int* step; unsigned int* counter; int B;
  long long* tok_hist; float* score_hist; long long* bbox_hist; unsigned char* done_hist;
  long long* ids_io; int* pos_io;
  int eos, pad;
};

template <typename T>
__global__ void __launch_bounds__(128) decode_tail_kernel(const TailParams p) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ float s_red[4][8];
  __shared__ float s_m[4], s_s[4];
  __shared__ int s_i[4];
  __shared__ long long s_next;
  const int s = p.step ? *p.step : 0;
  // ---- token / score
  AmPartial a{-INFINITY, 0x7fffffff, 0.f};
  for (int t = tid; t < p.n_tiles; t += 128) {
    const size_t o = static_cast<size_t>(b) * p.am_ld + t;
    am_combine(a, AmPartial{p.am_val[o], p.am_idx[o], p.am_sum[o]});
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    AmPartial c{__shfl_xor_sync(0xffffffffu, a.m, o), __shfl_xor_sync(0xffffffffu, a.i, o), __shfl_xor_sync(0xffffffffu, a.s, o)};
    am_combine(a, c);
  }
  if (lane == 0) { s_m[warp] = a.m; s_i[warp] = a.i; s_s[warp] = a.s; }
  // ---- bbox head partial sums: n_box dot products + the row's sum of squares
  const T* xr = reinterpret_cast<const T*>(p.x) + static_cast<size_t>(b) * p.ldx;
  float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const bool want_box = p.bbox || p.bbox_sig;
  if (want_box) {
    for (int k = tid; k < p.H; k += 128) {
      const float xv = to_f<T>(xr[k]);
      acc[6] = fmaf(xv, xv, acc[6]);
      for (int o = 0; o < p.n_box; ++o)
        acc[o] = fmaf(xv, to_f<T>(reinterpret_cast<const T*>(p.bbox_w)[static_cast<size_t>(o) * p.H + k]), acc[o]);
    }
#pragma unroll
    for (int o = 0; o < 7; ++o) {
      const float v = warp_sum(acc[o]);
      if (lane == 0) s_red[warp][o] = v;
    }
  }
  __syncthreads();
  if (tid == 0) {
    AmPartial r{s_m[0], s_i[0], s_s[0]};
    for (int w = 1; w < 4; ++w) am_combine(r, AmPartial{s_m[w], s_i[w], s_s[w]});
    const bool d = (r.i == p.eos) || (r.i == p.pad);
    const float sc = d ? 0.f : 1.f / r.s;
    const long long nxt = d ? p.pad : r.i;
    s_next = nxt;
    if (p.tok) p.tok[b] = r.i;
    if (p.score) p.score[b] = sc;
    if (p.done) p.done[b] = d ? 1 : 0;
    if (p.next_ids) p.next_ids[b] = nxt;
    const size_t ho = static_cast<size_t>(s) * p.B + b;
    if (p.tok_hist) p.tok_hist[ho] = r.i;
    if (p.score_hist) p.score_hist[ho] = sc;
    if (p.done_hist) p.done_hist[ho] = d ? 1 : 0;
    if (p.ids_io) p.ids_io[b] = nxt;
    if (p.pos_io) p.pos_io[b] += 1;
  }
  if (want_box && tid < p.n_box) {
    const float ssq = s_red[0][6] + s_red[1][6] + s_red[2][6] + s_red[3][6];
    const float rs = rsqrtf(ssq * (1.0f / static_cast<float>(p.H)) + p.eps);
    const float dot = s_red[0][tid] + s_red[1][tid] + s_red[2][tid] + s_red[3][tid];
    float v = rnd<T>(fmaf(dot, rs, to_f<T>(reinterpret_cast<const T*>(p.bbox_b)[tid])));
    v = rnd<T>(1.f / (1.f + expf(-v)));
    const long long box = static_cast<long long>(v * p.bbox_size);
    if (p.bbox_sig) p.bbox_sig[static_cast<size_t>(b) * p.n_box + tid] = v;
    if (p.bbox) p.bbox[static_cast<size_t>(b) * p.n_box + tid] = box;
    if (p.bbox_hist) p.bbox_hist[(static_cast<size_t>(s) * p.B + b) * p.n_box + tid] = box;
  }
  __syncthreads();
  // ---- next step's input embedding (after every read of this row of x above)
  if (p.x_next) {
    const uint4* e = reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.embed) + static_cast<size_t>(s_next) * p.H);
    uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.x_next) + static_cast<size_t>(b) * p.ldx_next);
    for (int i = tid; i < (p.H >> 3); i += 128) o[i] = e[i];
  }
  if (p.step) {
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      const unsigned int old = atomicAdd(p.counter, 1u);
      if (old == gridDim.x - 1) {       // every other block has read *step and finished: advance it for the next launch
        *p.counter = 0u;
        *p.step = s + 1;
      }
    }
  }
}

int decode_tail(int dtype, const DecodeTailArgs& a, cudaStream_t st) {
  if (a.rows <= 0) return 0;
  if (a.n_box > 6) { set_error("decode_tail: at most 6 box outputs"); return -1; }
  if (a.x_next && (a.H % 8 || a.ldx_next % 8)) { set_error("decode_tail: H and pitch must be multiples of 8"); return -1; }
  TailParams p;
  p.am_val = a.am_val; p.am_idx = a.am_idx; p.am_sum = a.am_sum; p.am_ld = a.am_ld; p.n_tiles = a.n_tiles;
  p.x = a.x; p.ldx = a.ldx; p.H = a.H; p.eps = a.eps;
  p.bbox_w = a.bbox_w; p.bbox_b = a.bbox_b; p.n_box = a.n_box; p.bbox_size = a.bbox_size;
  p.embed = a.embed; p.x_next = a.x_next; p.ldx_next = a.ldx_next;
  p.tok = a.tok; p.score = a.score; p.bbox = a.bbox; p.bbox_sig = a.bbox_sig; p.done = a.done; p.next_ids = a.next_ids;
  p.step = a.step; p.counter = a.counter; p.B = a.rows;
  p.tok_hist = a.tok_hist; p.score_hist = a.score_hist; p.bbox_hist = a.bbox_hist; p.done_hist = a.done_hist;
  p.ids_io = a.ids_io; p.pos_io = a.pos_io;
  p.eos = a.eos; p.pad = a.pad;
  if (dtype == DT_BF16) launch_pdl(decode_tail_kernel<__nv_bfloat16>, dim3(a.rows), dim3(128), 0, st, p);
  else launch_pdl(decode_tail_kernel<__half>, dim3(a.rows), dim3(128), 0, st, p);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ device-side stop rules
// The per-row scheduler state of the continuous-batching loop on the device (SURVEY §8 f3): after every greedy step the stop
// rules of RecognitionPredictor.prediction_loop (surya/recognition/__init__.py:568-601: EOS / PAD, max_tokens, detect_repeat_token)
// are evaluated here instead of in a per-token Python loop on the host.  One thread per batch row:
//   gen_count[r]   tokens generated for the row's prompt so far (the prefill token counts: the host seeds 1)
//   ring[r][R]     the row's last R = max_repeats tokens (slot = index % R; the host seeds slot 0 with the prefill token)
//   row_done[r]    sticky: a stop rule fired (or the row is idle); such rows keep stepping like every row of the reference's
//                  batch does, their tokens are not counted
//   n_valid[r]     steps of the current host round trip whose outputs belong to the row (1 + index of its stopping step)
//   n_active[0]    rows still running after this step (one int for the host to poll)
// detect_repeat_token (surya/recognition/util.py:59-69): with at least R tokens, u = distinct values among the last R; stop when
// u <= 5 and the last u tokens equal the u tokens before them.
constexpr int STOP_MAX_RING = 64;

__global__ void __launch_bounds__(256) stop_rules_kernel(const long long* __restrict__ tok_hist, const unsigned char* __restrict__ done_hist,
                                                         const int* __restrict__ step_dev, int step_host, int B, int* __restrict__ gen_count,
                                                         long long* __restrict__ ring, unsigned char* __restrict__ row_done,
                                                         int* __restrict__ n_valid, int* __restrict__ n_active, int max_tokens, int R) {
  pdl_trigger();
  pdl_wait();
  __shared__ int s_active;
  if (threadIdx.x == 0) s_active = 0;
  __syncthreads();
  const int s = step_dev ? (*step_dev - 1) : step_host;        // the step decode_tail has just written
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    if (row_done[r]) continue;
    const size_t ho = static_cast<size_t>(s) * B + r;
    const long long tok = tok_hist[ho];
    const int cnt = gen_count[r] + 1;
    gen_count[r] = cnt;
    long long* rg = ring + static_cast<size_t>(r) * R;
    rg[(cnt - 1) % R] = tok;
    bool stop = (done_hist[ho] != 0) || (cnt >= max_tokens);
    if (!stop && cnt >= R) {
      // last_n[j] for j = 0..R-1 (oldest first) lives at ring slot (cnt + j) % R
      int u = 0;
      for (int j = 0; j < R && u <= 5; ++j) {
        const long long v = rg[(cnt + j) % R];
        bool seen = false;
        for (int k = 0; k < j; ++k) seen |= (rg[(cnt + k) % R] == v);
        u += seen ? 0 : 1;
      }
      if (u <= 5 && 2 * u <= R) {          // a window shorter than 2u: Python's last_n[-2u:-u] is shorter than last_n[-u:], never equal
        bool same = true;
        for (int j = 0; j < u; ++j) same &= (rg[(cnt + R - u + j) % R] == rg[(cnt + R - 2 * u + j) % R]);
        stop = same;
      }
    }
    n_valid[r] = s + 1;
    if (stop) row_done[r] = 1;
    else atomicAdd(&s_active, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0 && n_active) *n_active = s_active;
}

int stop_rules(const long long* tok_hist, const unsigned char* done_hist, const int* step_dev, int step_host, int B, int* gen_count,
               long long* ring, unsigned char* row_done, int* n_valid, int* n_active, int max_tokens, int max_repeats,
               cudaStream_t st) {
  if (B <= 0) return 0;
  if (!tok_hist || !done_hist || !gen_count || !ring || !row_done || !n_valid) { set_error("stop_rules: null argument"); return -1; }
  if (max_repeats < 2 || max_repeats > STOP_MAX_RING) { set_error("stop_rules: max_repeats %d outside [2, %d]", max_repeats, STOP_MAX_RING); return -2; }
  launch_pdl(stop_rules_kernel, dim3(1), dim3(256), 0, st, tok_hist, done_hist, step_dev, step_host, B, gen_count, ring, row_done,
             n_valid, n_active, max_tokens, max_repeats);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ gather + pad rows
// dst[i, 0:K] = src[perm[i], 0:K] (converted from SrcT), dst[i, K:Kp] = 0.
template <typename T, typename SrcT>
__global__ void gather_pad_kernel(const SrcT* __restrict__ src, int lds, const int* __restrict__ perm,
                                  T* __restrict__ dst, int ldd, int rows, int K, int Kp) {
  int row = blockIdx.x;
  if (row >= rows) return;
  int s = perm ? perm[row] : row;
  const SrcT* sr = src + static_cast<size_t>(s) * lds;
  T* dr = dst + static_cast<size_t>(row) * ldd;
  for (int i = threadIdx.x; i < Kp; i += blockDim.x) {
    float v = 0.f;
    if (i < K) {
      if constexpr (sizeof(SrcT) == 4) v = static_cast<float>(sr[i]);
      else v = to_f<SrcT>(sr[i]);
    }
    dr[i] = from_f<T>(v);
  }
}

int gather_pad_rows(int dtype, const void* src, int src_is_f32, int lds, const int* perm, void* dst, int ldd, int rows,
                    int K, int Kp, cudaStream_t st) {
  if (rows <= 0) return 0;
  dim3 grid(rows), block(128);
  if (dtype == DT_BF16) {
    if (src_is_f32)
      gather_pad_kernel<__nv_bfloat16, float><<<grid, block, 0, st>>>((const float*)src, lds, perm,
                                                                      (__nv_bfloat16*)dst, ldd, rows, K, Kp);
    else
      gather_pad_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, block, 0, st>>>(
          (const __nv_bfloat16*)src, lds, perm, (__nv_bfloat16*)dst, ldd, rows, K, Kp);
  } else {
    if (src_is_f32)
      gather_pad_kernel<__half, float><<<grid, block, 0, st>>>((const float*)src, lds, perm, (__half*)dst, ldd, rows,
                                                               K, Kp);
    else
      gather_pad_kernel<__half, __half><<<grid, block, 0, st>>>((const __half*)src, lds, perm, (__half*)dst, ldd,
                                                                rows, K, Kp);
  }
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ vision 2-D RoPE
// qkv row = [q(nh*d) | k(nh*d) | v(nh*d)]; rotates q and k in place, fp32 math, one rounding at the end.
// freq index i < d/2: i < d/4 -> row_pos * inv_freq[i], else col_pos * inv_freq[i - d/4].
template <typename T>
__global__ void rope_vision_kernel(T* __restrict__ qkv, int ld, const int2* __restrict__ pos,
                                   const float* __restrict__ inv_freq, int n_tok, int nh, int d) {
  int tok = blockIdx.x;
  if (tok >= n_tok) return;
  const int half = d >> 1, quarter = d >> 2;
  int2 p = pos[tok];
  T* row = qkv + static_cast<size_t>(tok) * ld;
  // cos/sin once per (token, frequency); shared by all q and k heads
  __shared__ float s_cos[128], s_sin[128];
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    float f = (i < quarter) ? static_cast<float>(p.x) * inv_freq[i] : static_cast<float>(p.y) * inv_freq[i - quarter];
    s_cos[i] = cosf(f);
    s_sin[i] = sinf(f);
  }
  __syncthreads();
  const int total = 2 * nh * half;  // (q|k) x heads x pairs
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    int i = idx % half;
    int hh = idx / half;  // 0 .. 2*nh-1 (q heads then k heads; contiguous in memory)
    float c = s_cos[i], s = s_sin[i];
    T* h = row + hh * d;
    float x1 = to_f<T>(h[i]), x2 = to_f<T>(h[i + half]);
    float o1 = __fadd_rn(__fmul_rn(x1, c), __fmul_rn(-x2, s));
    float o2 = __fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, s));
    h[i] = from_f<T>(o1);
    h[i + half] = from_f<T>(o2);
  }
}

int rope_vision(int dtype, void* qkv, int ld, const int* pos_rc, const float* inv_freq, int n_tok, int nh, int d,
                cudaStream_t st) {
  if (n_tok <= 0) return 0;
  dim3 grid(n_tok), block(128);
  if (dtype == DT_BF16)
    rope_vision_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((__nv_bfloat16*)qkv, ld, (const int2*)pos_rc, inv_freq,
                                                             n_tok, nh, d);
  else
    rope_vision_kernel<__half><<<grid, block, 0, st>>>((__half*)qkv, ld, (const int2*)pos_rc, inv_freq, n_tok, nh, d);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ decoder RoPE + KV append
// qkv row = [q(nh*d) | k(nkv*d) | v(nkv*d)].  cos/sin are computed in fp32, cast to T, and the rotation is
// evaluated in T arithmetic with three roundings (mul, mul, add) like the eager reference.  q and k are rotated
// in place; rotated k and v are also written to the slot cache at index `pos`.  A token whose pos is outside
// [0, s_max) is still rotated but writes nothing to the cache (host-side callers reject it before launching): its
// row would land in the next kv head's or slot's rows, the same bound decode_attn_kernel enforces.
template <typename T>
__device__ __forceinline__ void rope_pair_T(float x1, float x2, float c, float s, float& o1, float& o2) {
  // o1 = x1*c + (-x2)*s ; o2 = x2*c + x1*s   (each product and the sum rounded to T)
  o1 = rnd<T>(rnd<T>(x1 * c) + rnd<T>(-x2 * s));
  o2 = rnd<T>(rnd<T>(x2 * c) + rnd<T>(x1 * s));
}

template <typename T>
__global__ void rope_kv_append_kernel(T* __restrict__ qkv, int ld, const int* __restrict__ tok_pos,
                                      const int* __restrict__ tok_slot, const float* __restrict__ inv_freq,
                                      T* __restrict__ kcache, T* __restrict__ vcache, int n_tok, int nh, int nkv,
                                      int d, int s_max) {
  int tok = blockIdx.x;
  if (tok >= n_tok) return;
  const int half = d >> 1;
  const int pos = tok_pos[tok];
  const int slot = tok_slot[tok];
  const bool in_cache = pos >= 0 && pos < s_max;
  T* row = qkv + static_cast<size_t>(tok) * ld;
  __shared__ float s_cos[128], s_sin[128];
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    float f = static_cast<float>(pos) * inv_freq[i];
    s_cos[i] = rnd<T>(cosf(f));
    s_sin[i] = rnd<T>(sinf(f));
  }
  __syncthreads();
  const int n_rot = (nh + nkv) * half;
  for (int idx = threadIdx.x; idx < n_rot; idx += blockDim.x) {
    int i = idx % half;
    int hh = idx / half;
    float c = s_cos[i], s = s_sin[i];
    T* h = row + hh * d;
    float x1 = to_f<T>(h[i]), x2 = to_f<T>(h[i + half]);
    float o1, o2;
    rope_pair_T<T>(x1, x2, c, s, o1, o2);
    h[i] = from_f<T>(o1);
    h[i + half] = from_f<T>(o2);
    if (hh >= nh && in_cache) {
      int kvh = hh - nh;
      T* kc = kcache + ((static_cast<size_t>(slot) * nkv + kvh) * s_max + pos) * d;
      kc[i] = from_f<T>(o1);
      kc[i + half] = from_f<T>(o2);
    }
  }
  if (!in_cache) return;
  const T* vrow = row + (nh + nkv) * d;
  for (int idx = threadIdx.x; idx < nkv * d; idx += blockDim.x) {
    int kvh = idx / d, i = idx % d;
    vcache[((static_cast<size_t>(slot) * nkv + kvh) * s_max + pos) * d + i] = vrow[idx];
  }
}

int rope_kv_append(int dtype, void* qkv, int ld, const int* tok_pos, const int* tok_slot, const float* inv_freq,
                   void* kcache, void* vcache, int n_tok, int nh, int nkv, int d, int s_max, cudaStream_t st) {
  if (n_tok <= 0) return 0;
  dim3 grid(n_tok), block(128);
  if (dtype == DT_BF16)
    rope_kv_append_kernel<__nv_bfloat16><<<grid, block, 0, st>>>((__nv_bfloat16*)qkv, ld, tok_pos, tok_slot, inv_freq,
                                                                (__nv_bfloat16*)kcache, (__nv_bfloat16*)vcache, n_tok,
                                                                nh, nkv, d, s_max);
  else
    rope_kv_append_kernel<__half><<<grid, block, 0, st>>>((__half*)qkv, ld, tok_pos, tok_slot, inv_freq,
                                                         (__half*)kcache, (__half*)vcache, n_tok, nh, nkv, d, s_max);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ embed + image splice
// out[t] = tok_feat_row[t] >= 0 ? T( feat[tok_feat_row[t]] + T(h_embed[hidx] + w_embed[widx]) ) : embed[ids[t]]
template <typename T>
__global__ void embed_splice_kernel(const long long* __restrict__ ids, const int* __restrict__ feat_row,
                                    const int* __restrict__ hidx, const int* __restrict__ widx,
                                    const T* __restrict__ embed, const T* __restrict__ feat, int ldf,
                                    const T* __restrict__ h_embed, const T* __restrict__ w_embed, T* __restrict__ out,
                                    int ldo, int n_tok, int H) {
  int t = blockIdx.x;
  if (t >= n_tok) return;
  T* o = out + static_cast<size_t>(t) * ldo;
  int fr = feat_row ? feat_row[t] : -1;
  if (fr >= 0) {
    const T* f = feat + static_cast<size_t>(fr) * ldf;
    const T* he = h_embed + static_cast<size_t>(hidx[t]) * H;
    const T* we = w_embed + static_cast<size_t>(widx[t]) * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      float pe = rnd<T>(to_f<T>(he[i]) + to_f<T>(we[i]));
      o[i] = from_f<T>(to_f<T>(f[i]) + pe);
    }
  } else {
    const T* e = embed + static_cast<size_t>(ids[t]) * H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) o[i] = e[i];
  }
}

int embed_splice(int dtype, const long long* ids, const int* feat_row, const int* hidx, const int* widx,
                 const void* embed, const void* feat, int ldf, const void* h_embed, const void* w_embed, void* out,
                 int ldo, int n_tok, int H, cudaStream_t st) {
  if (n_tok <= 0) return 0;
  dim3 grid(n_tok), block(128);
  if (dtype == DT_BF16)
    embed_splice_kernel<__nv_bfloat16><<<grid, block, 0, st>>>(
        ids, feat_row, hidx, widx, (const __nv_bfloat16*)embed, (const __nv_bfloat16*)feat, ldf,
        (const __nv_bfloat16*)h_embed, (const __nv_bfloat16*)w_embed, (__nv_bfloat16*)out, ldo, n_tok, H);
  else
    embed_splice_kernel<__half><<<grid, block, 0, st>>>(ids, feat_row, hidx, widx, (const __half*)embed,
                                                       (const __half*)feat, ldf, (const __half*)h_embed,
                                                       (const __half*)w_embed, (__half*)out, ldo, n_tok, H);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ greedy head
// Per row: token = argmax(float(logits)) (first index on ties), score = max softmax = 1 / sum exp(l - max),
// done = token in {eos, pad}; score forced to 0 when done; next input id = pad when done.
template <typename T>
__global__ void argmax_score_kernel(const T* __restrict__ logits, int ld, int V, long long* __restrict__ tok,
                                    float* __restrict__ score, unsigned char* __restrict__ done,
                                    long long* __restrict__ next_ids, int eos, int pad) {
  pdl_trigger();
  pdl_wait();
  int row = blockIdx.x;
  const T* l = logits + static_cast<size_t>(row) * ld;
  float m = -INFINITY;
  int mi = 0x7fffffff;
  float s = 0.f;  // running sum of exp(l - m)
  const int nv = V >> 3;
  // Chunks of CH 16-byte vectors per thread: all loads of a chunk are issued first, then the chunk maximum, then CH*8
  // independent exps against it — one rescale of the running sum per chunk instead of a dependent exp per element.
  constexpr int CH = 8;
  for (int i0 = threadIdx.x; i0 < nv; i0 += blockDim.x * CH) {
    uint4 u[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int i = i0 + c * blockDim.x;
      if (i < nv) u[c] = *reinterpret_cast<const uint4*>(l + static_cast<size_t>(i) * 8);
    }
    float cm = -INFINITY;
    int ci = 0x7fffffff;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int i = i0 + c * blockDim.x;
      if (i >= nv) break;
      const T* e = reinterpret_cast<const T*>(&u[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = to_f<T>(e[j]);
        if (v > cm) { cm = v; ci = i * 8 + j; }      // ascending index within the thread: first maximum wins
      }
    }
    if (cm == -INFINITY) continue;                    // all -inf (or empty): contributes nothing
    if (cm > m) { s *= __expf(m - cm); m = cm; mi = ci; }
    float add = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int i = i0 + c * blockDim.x;
      if (i >= nv) break;
      const T* e = reinterpret_cast<const T*>(&u[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) add += __expf(to_f<T>(e[j]) - m);
    }
    s += add;
  }
  for (int i = (nv << 3) + threadIdx.x; i < V; i += blockDim.x) {
    float v = to_f<T>(l[i]);
    if (v > m) { s = s * __expf(m - v) + 1.f; m = v; mi = i; }
    else s += __expf(v - m);
  }
  // block reduction of (m, mi, s)
  __shared__ float sm[32];
  __shared__ int si[32];
  __shared__ float ss[32];
  auto combine = [](float& m1, int& i1, float& s1, float m2, int i2, float s2) {
    if (m2 > m1 || (m2 == m1 && i2 < i1)) {
      s1 = s1 * __expf(m1 - m2) + s2;
      m1 = m2;
      i1 = i2;
    } else {
      s1 += s2 * __expf(m2 - m1);
    }
  };
  if (m == -INFINITY) s = 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    int i2 = __shfl_xor_sync(0xffffffffu, mi, o);
    float s2 = __shfl_xor_sync(0xffffffffu, s, o);
    if (m2 != -INFINITY) {
      if (m == -INFINITY) { m = m2; mi = i2; s = s2; }
      else combine(m, mi, s, m2, i2, s2);
    }
  }
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sm[warp] = m; si[warp] = mi; ss[warp] = s; }
  __syncthreads();
  if (warp == 0) {
    int nw = blockDim.x >> 5;
    m = lane < nw ? sm[lane] : -INFINITY;
    mi = lane < nw ? si[lane] : 0x7fffffff;
    s = lane < nw ? ss[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, m, o);
      int i2 = __shfl_xor_sync(0xffffffffu, mi, o);
      float s2 = __shfl_xor_sync(0xffffffffu, s, o);
      if (m2 != -INFINITY) {
        if (m == -INFINITY) { m = m2; mi = i2; s = s2; }
        else combine(m, mi, s, m2, i2, s2);
      }
    }
    if (lane == 0) {
      bool d = (mi == eos) || (mi == pad);
      tok[row] = mi;
      score[row] = d ? 0.f : 1.f / s;
      if (done) done[row] = d ? 1 : 0;
      if (next_ids) next_ids[row] = d ? pad : mi;
    }
  }
}

int argmax_score(int dtype, const void* logits, int ld, int rows, int V, long long* tok, float* score,
                 unsigned char* done, long long* next_ids, int eos, int pad, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (ld % 8) { set_error("argmax_score: logits pitch must be a multiple of 8"); return -1; }
  dim3 grid(rows), block(512);
  if (dtype == DT_BF16)
    launch_pdl(argmax_score_kernel<__nv_bfloat16>, grid, block, 0, st, (const __nv_bfloat16*)logits, ld, V, tok, score, done,
               next_ids, eos, pad);
  else
    launch_pdl(argmax_score_kernel<__half>, grid, block, 0, st, (const __half*)logits, ld, V, tok, score, done, next_ids, eos,
               pad);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ small dense head
// out[r, o] = act(T(x[r] . w[o] + b[o])); one warp per (row, output).  Used for the 6-wide bbox head:
// sig = T(sigmoid(T(lin))) ; box = trunc(float(sig) * bbox_size) as int64.
template <typename T>
__global__ void small_head_kernel(const T* __restrict__ x, int ldx, const T* __restrict__ w, const T* __restrict__ b,
                                  int rows, int H, int n_out, int sigmoid, float* __restrict__ out_f,
                                  long long* __restrict__ out_box, float box_scale) {
  pdl_trigger();
  pdl_wait();
  int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (gw >= rows * n_out) return;
  int r = gw / n_out, o = gw % n_out;
  const T* xr = x + static_cast<size_t>(r) * ldx;
  const T* wr = w + static_cast<size_t>(o) * H;
  float acc = 0.f;
  for (int i = lane; i < H; i += 32) acc += to_f<T>(xr[i]) * to_f<T>(wr[i]);
  acc = warp_sum(acc);
  if (lane == 0) {
    float v = rnd<T>(acc + (b ? to_f<T>(b[o]) : 0.f));
    if (sigmoid) v = rnd<T>(1.f / (1.f + expf(-v)));
    if (out_f) out_f[gw] = v;
    if (out_box) out_box[gw] = static_cast<long long>(v * box_scale);
  }
}

int small_head(int dtype, const void* x, int ldx, const void* w, const void* b, int rows, int H, int n_out,
               int sigmoid, float* out_f, long long* out_box, float box_scale, cudaStream_t st) {
  if (rows <= 0) return 0;
  int warps = rows * n_out;
  dim3 grid((warps + 3) / 4), block(128);
  if (dtype == DT_BF16)
    launch_pdl(small_head_kernel<__nv_bfloat16>, grid, block, 0, st, (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)w,
               (const __nv_bfloat16*)b, rows, H, n_out, sigmoid, out_f, out_box, box_scale);
  else
    launch_pdl(small_head_kernel<__half>, grid, block, 0, st, (const __half*)x, ldx, (const __half*)w, (const __half*)b, rows,
               H, n_out, sigmoid, out_f, out_box, box_scale);
  return launch_ok();
}

// ------------------------------------------------------------------------------------------ embedding rows
template <typename T>
__global__ void embed_rows_kernel(const long long* __restrict__ ids, const T* __restrict__ embed, T* __restrict__ out,
                                  int ldo, int n, int H) {
  pdl_trigger();
  pdl_wait();
  int t = blockIdx.x;
  if (t >= n) return;
  const uint4* e = reinterpret_cast<const uint4*>(embed + static_cast<size_t>(ids[t]) * H);
  uint4* o = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * ldo);
  for (int i = threadIdx.x; i < (H >> 3); i += blockDim.x) o[i] = e[i];
}

int embed_rows(int dtype, const long long* ids, const void* embed, void* out, int ldo, int n, int H, cudaStream_t st) {
  if (n <= 0) return 0;
  if (H % 8 || ldo % 8) { set_error("embed_rows: H and pitch must be multiples of 8"); return -1; }
  dim3 grid(n), block(128);
  if (dtype == DT_BF16)
    launch_pdl(embed_rows_kernel<__nv_bfloat16>, grid, block, 0, st, ids, (const __nv_bfloat16*)embed, (__nv_bfloat16*)out, ldo,
               n, H);
  else
    launch_pdl(embed_rows_kernel<__half>, grid, block, 0, st, ids, (const __half*)embed, (__half*)out, ldo, n, H);
  return launch_ok();
}

}  // namespace sb
