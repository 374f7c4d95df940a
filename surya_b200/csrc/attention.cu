// surya_b200 — attention kernels.
//
//  attn_varlen  : block-diagonal (per-sequence) flash attention over packed tokens, optional causal mask and GQA.
//                 Replaces flash_attn_varlen_func / SDPA in the recognition vision tower
//                 (surya/common/surya/encoder/__init__.py:136-178, 202-263, 266-411) and in decoder prefill
//                 (surya/common/surya/decoder/__init__.py:101-128, flash_attn_utils.py:106-154).
//                 Tensor-core path: mma.sync m16n8k16 (fp32 accumulate), online softmax in fp32 registers,
//                 P rounded to the storage type before the PV product (flash-attention semantics).
//                 Attention is < 1 % of the recognition FLOPs (SURVEY.md §8a a10), the tensor-core work is in the GEMMs.
//  decode_attn  : q_len = 1 attention over the slot KV cache fused with RoPE(q,k) and the in-place cache append
//                 (decoder/__init__.py:161-238 with DynamicCache.update -> no torch.cat, SURVEY.md §2.2 K10/K20).
//                 HBM-bound: streams K and V once, CUDA-core FMA.
#include "ops.cuh"
#include "sb_ptx.cuh"

namespace sb {

template <typename T> struct Mma;
template <> struct Mma<__nv_bfloat16> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};
template <> struct Mma<__half> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t smem_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_addr));
}

struct AttnKParams {
  const void* q; int ldq;
  const void* k; int ldk;
  const void* v; int ldv;
  void* out; int ldo;
  const int* seq_start;
  const int* seq_len;
  int q_tiles;      // q tiles per sequence (ceil(max_len / 64))
  int n_heads, group;  // group = n_heads / n_kv_heads
  int causal;
  float scale_log2;  // scale * log2(e)
};

template <typename T, int HD>
__global__ void __launch_bounds__(128) attn_varlen_kernel(const AttnKParams p) {
  constexpr int BQ = 64, BKV = 64, LDS = HD + 8, KS = HD / 16, DN = HD / 8;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  T* sQ = reinterpret_cast<T*>(smem_attn);
  T* sK = sQ + BQ * LDS;
  T* sV = sK + BKV * LDS;

  const int seq = blockIdx.x / p.q_tiles;
  const int qt = blockIdx.x % p.q_tiles;
  const int h = blockIdx.y;
  const int kvh = h / p.group;
  const int len = p.seq_len[seq];
  const int q0 = qt * BQ;
  if (q0 >= len) return;
  const int start = p.seq_start[seq];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;

  const T* qbase = reinterpret_cast<const T*>(p.q) + static_cast<size_t>(h) * HD;
  const T* kbase = reinterpret_cast<const T*>(p.k) + static_cast<size_t>(kvh) * HD;
  const T* vbase = reinterpret_cast<const T*>(p.v) + static_cast<size_t>(kvh) * HD;

  constexpr int VPR = HD / 8;  // uint4 per row
  // ---- load Q tile
  for (int i = tid; i < BQ * VPR; i += 128) {
    int r = i / VPR, c = i % VPR;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (q0 + r < len) val = *reinterpret_cast<const uint4*>(qbase + static_cast<size_t>(start + q0 + r) * p.ldq + c * 8);
    *reinterpret_cast<uint4*>(sQ + r * LDS + c * 8) = val;
  }
  __syncthreads();

  const int rbase = warp * 16;
  uint32_t aQ[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    aQ[ks][0] = *reinterpret_cast<const uint32_t*>(sQ + (rbase + g) * LDS + ks * 16 + 2 * t);
    aQ[ks][1] = *reinterpret_cast<const uint32_t*>(sQ + (rbase + g + 8) * LDS + ks * 16 + 2 * t);
    aQ[ks][2] = *reinterpret_cast<const uint32_t*>(sQ + (rbase + g) * LDS + ks * 16 + 8 + 2 * t);
    aQ[ks][3] = *reinterpret_cast<const uint32_t*>(sQ + (rbase + g + 8) * LDS + ks * 16 + 8 + 2 * t);
  }

  float O[DN][4];
#pragma unroll
  for (int i = 0; i < DN; ++i) { O[i][0] = O[i][1] = O[i][2] = O[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  const int kv_end = p.causal ? min(len, q0 + BQ) : len;
  const int n_kt = (kv_end + BKV - 1) / BKV;
  for (int kt = 0; kt < n_kt; ++kt) {
    const int k0 = kt * BKV;
    __syncthreads();  // previous tile fully consumed
    for (int i = tid; i < BKV * VPR; i += 128) {
      int r = i / VPR, c = i % VPR;
      uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
      if (k0 + r < len) {
        size_t tok = static_cast<size_t>(start + k0 + r);
        kv = *reinterpret_cast<const uint4*>(kbase + tok * p.ldk + c * 8);
        vv = *reinterpret_cast<const uint4*>(vbase + tok * p.ldv + c * 8);
      }
      *reinterpret_cast<uint4*>(sK + r * LDS + c * 8) = kv;
      *reinterpret_cast<uint4*>(sV + r * LDS + c * 8) = vv;
    }
    __syncthreads();

    float S[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      S[nt][0] = S[nt][1] = S[nt][2] = S[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (nt * 8 + g) * LDS + ks * 16 + 2 * t);
        uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (nt * 8 + g) * LDS + ks * 16 + 8 + 2 * t);
        Mma<T>::run(S[nt], aQ[ks], b0, b1);
      }
    }
    // ---- mask, scale (log2 domain), online softmax
    const int qi0 = q0 + rbase + g, qi1 = qi0 + 8;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int key = k0 + nt * 8 + 2 * t + (e & 1);
        int qi = (e < 2) ? qi0 : qi1;
        bool ok = key < len && (!p.causal || key <= qi);
        float sv = ok ? S[nt][e] * p.scale_log2 : -INFINITY;
        S[nt][e] = sv;
        if (e < 2) mx0 = fmaxf(mx0, sv); else mx1 = fmaxf(mx1, sv);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // rows with no visible key yet keep m = -inf; guard the subtraction against inf - inf
    const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
    const float c0 = exp2f(m0 - ms0), c1 = exp2f(m1 - ms1);
    m0 = mn0; m1 = mn1;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      S[nt][0] = exp2f(S[nt][0] - ms0);
      S[nt][1] = exp2f(S[nt][1] - ms0);
      S[nt][2] = exp2f(S[nt][2] - ms1);
      S[nt][3] = exp2f(S[nt][3] - ms1);
      rs0 += S[nt][0] + S[nt][1];
      rs1 += S[nt][2] + S[nt][3];
    }
    l0 = l0 * c0 + rs0;
    l1 = l1 * c1 + rs1;
#pragma unroll
    for (int dn = 0; dn < DN; ++dn) {
      O[dn][0] *= c0; O[dn][1] *= c0; O[dn][2] *= c1; O[dn][3] *= c1;
    }
    // ---- O += P V
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
      uint32_t aP[4];
      aP[0] = Mma<T>::pack(S[2 * kc][0], S[2 * kc][1]);
      aP[1] = Mma<T>::pack(S[2 * kc][2], S[2 * kc][3]);
      aP[2] = Mma<T>::pack(S[2 * kc + 1][0], S[2 * kc + 1][1]);
      aP[3] = Mma<T>::pack(S[2 * kc + 1][2], S[2 * kc + 1][3]);
      const int mid = lane >> 3, r = lane & 7;
#pragma unroll
      for (int dn = 0; dn < DN; dn += 2) {
        uint32_t bv[4];
        const T* addr = sV + (kc * 16 + (mid & 1) * 8 + r) * LDS + (dn + (mid >> 1)) * 8;
        ldmatrix_x4_trans(bv, smem_u32(addr));
        Mma<T>::run(O[dn], aP, bv[0], bv[1]);
        Mma<T>::run(O[dn + 1], aP, bv[2], bv[3]);
      }
    }
  }
  // ---- finalize
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
  T* obase = reinterpret_cast<T*>(p.out) + static_cast<size_t>(h) * HD;
  const int r0 = q0 + rbase + g, r1 = r0 + 8;
#pragma unroll
  for (int dn = 0; dn < DN; ++dn) {
    int col = dn * 8 + 2 * t;
    if (r0 < len)
      *reinterpret_cast<uint32_t*>(obase + static_cast<size_t>(start + r0) * p.ldo + col) =
          Mma<T>::pack(O[dn][0] * i0, O[dn][1] * i0);
    if (r1 < len)
      *reinterpret_cast<uint32_t*>(obase + static_cast<size_t>(start + r1) * p.ldo + col) =
          Mma<T>::pack(O[dn][2] * i1, O[dn][3] * i1);
  }
}

template <typename T, int HD>
static int launch_varlen(const AttnArgs& a, cudaStream_t st) {
  constexpr size_t SMEM = 3 * 64 * (HD + 8) * sizeof(T);
  auto kern = attn_varlen_kernel<T, HD>;
  static bool attr_set = false;
  if (!attr_set) {
    if (SMEM > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
    attr_set = true;
  }
  AttnKParams p;
  p.q = a.q; p.ldq = a.ldq; p.k = a.k; p.ldk = a.ldk; p.v = a.v; p.ldv = a.ldv; p.out = a.out; p.ldo = a.ldo;
  p.seq_start = a.seq_start; p.seq_len = a.seq_len;
  p.q_tiles = (a.max_len + 63) / 64;
  p.n_heads = a.n_heads; p.group = a.n_heads / a.n_kv_heads;
  p.causal = a.causal;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  dim3 grid(a.n_seq * p.q_tiles, a.n_heads), block(128);
  kern<<<grid, block, SMEM, st>>>(p);
  return launch_ok();
}

template <typename T>
static int dispatch_varlen(const AttnArgs& a, cudaStream_t st) {
  switch (a.head_dim) {
    case 32: return launch_varlen<T, 32>(a, st);
    case 64: return launch_varlen<T, 64>(a, st);
    case 80: return launch_varlen<T, 80>(a, st);
    case 96: return launch_varlen<T, 96>(a, st);
    case 128: return launch_varlen<T, 128>(a, st);
    default: set_error("attn_varlen: unsupported head_dim %d (32/64/80/96/128)", a.head_dim); return -1;
  }
}

int attn_varlen(const AttnArgs& a, cudaStream_t st) {
  if (a.n_seq <= 0 || a.max_len <= 0) return 0;
  if (a.n_kv_heads <= 0 || a.n_heads % a.n_kv_heads) {
    set_error("attn_varlen: n_heads must be a positive multiple of n_kv_heads"); return -1;
  }
  if (a.ldq % 8 || a.ldk % 8 || a.ldv % 8 || a.ldo % 2) { set_error("attn_varlen: pitches must be 16B multiples"); return -1; }
  // q / k / v rows are read as 16-byte vectors and out is stored as 4-byte pairs (the pitches are checked above)
  if ((reinterpret_cast<uintptr_t>(a.q) | reinterpret_cast<uintptr_t>(a.k) | reinterpret_cast<uintptr_t>(a.v)) % 16 ||
      reinterpret_cast<uintptr_t>(a.out) % 4) {
    set_error("attn_varlen: q, k and v must be 16B aligned and out 4B aligned"); return -1;
  }
  return a.dtype == DT_BF16 ? dispatch_varlen<__nv_bfloat16>(a, st) : dispatch_varlen<__half>(a, st);
}

// =========================================================================================== decode attention
struct DecodeKParams {
  const void* qkv; int ld;
  void* kcache; void* vcache;
  const int* slot; const int* pos;
  const float* inv_freq;
  void* out; int ldo;
  int n_heads, n_kv_heads, s_max;
  float scale;
};

// One CTA of 128 threads per (batch row, KV head).  The cache rows 0 .. pos-1 of a (slot, KV head) are contiguous, so they
// stream through a ring of DEC_STAGES shared-memory chunks of DEC_CK keys with 1-D bulk copies (cp.async.bulk completing on
// one mbarrier per stage): K chunks 0 .. nc-1, then V chunks 0 .. nc-1, nc = ceil(n_keys / DEC_CK).  Thread 0 requests the
// first DEC_STAGES chunks right after griddepcontrol.wait and refills a stage as soon as the CTA has consumed it, so the
// loads run under the RoPE step, the scores and the softmax, and the first V chunks are in flight before P.V starts.  The
// appended row (key pos) is never read back from global memory: the RoPE step keeps a copy in shared memory.  The ring holds
// DEC_STAGES * DEC_CK keys (20 KB at HD = 80), not the whole slab, so residency does not depend on the key count.
//
// Summation trees.  They fix the output bits and do not depend on how the work is spread over the threads
// (VPR = HD / 8, NKG = 128 / VPR):
//  - score s[g][j] = (fp32 chain acc = fmaf(q[g][x], k[j][x], acc), x = 0 .. HD-1 ascending, from 0.f) * scale.  The
//    16-bit products are exact in fp32, so q lives in shared memory as fp32, converted once;
//  - m_g = max over j of s[g][j] (order-free);
//  - l_g: 128 lanes t each sum __expf(s[g][j] - m_g) over j = t (mod 128) ascending from 0.f, then the xor butterfly 16, 8,
//    4, 2, 1 inside each warp, then ((w0 + w1) + w2) + w3;
//  - p[g][j] = rnd_T(__expf(s[g][j] - m_g)), kept as the fp32 value of the rounded number;
//  - out[g][d] = rnd_T(o / l_g) with o the sum over kg = 0 .. NKG-1, in order from 0.f, of the fp32 chains
//    fmaf(p[g][j], v[j][d], acc) over j = kg, kg + NKG, kg + 2 NKG, ... ascending from 0.f;
//  - RoPE: o1 = rnd(rnd(x1 c) + rnd(-x2 s)), o2 = rnd(rnd(x2 c) + rnd(x1 s)), c = rnd(cosf(pos inv_freq)), s likewise.
constexpr int DEC_CK = 32, DEC_STAGES = 4;

template <typename T, int HD, int G>
struct DecodeSmem {
  static constexpr int VPR = HD / 8, NKG = 128 / VPR, QS = HD + 4;  // QS: q row pitch in floats (conflict-free float4 reads)
  static constexpr int CHUNK = DEC_CK * HD * static_cast<int>(sizeof(T));
  static constexpr int RED = NKG * G * HD * 4;
  // [DEC_STAGES][DEC_CK][HD] T ring, reused as red [NKG][G][HD] fp32 once every chunk is consumed
  static constexpr int RING = DEC_STAGES * CHUNK > RED ? DEC_STAGES * CHUNK : RED;
  static constexpr int Q_OFF = RING;                                              // [G][QS] fp32 rotated queries
  static constexpr int KN_OFF = Q_OFF + G * QS * 4;                               // [HD] T appended K row (after RoPE)
  static constexpr int VN_OFF = KN_OFF + HD * static_cast<int>(sizeof(T));        // [HD] T appended V row
  static constexpr int BAR_OFF = VN_OFF + HD * static_cast<int>(sizeof(T));       // [DEC_STAGES] mbarriers
  static constexpr int SC_OFF = BAR_OFF + DEC_STAGES * 8;                         // [G][s_max + 1] fp32 scores, then p
  static_assert(CHUNK % 16 == 0 && RING % 16 == 0 && KN_OFF % 16 == 0 && VN_OFF % 16 == 0 && BAR_OFF % 8 == 0, "alignment");
  static size_t bytes(int s_max) { return SC_OFF + static_cast<size_t>(G) * (s_max + 1) * sizeof(float); }
};

template <typename T, int HD, int G>
__global__ void __launch_bounds__(128, G <= 4 ? 8 : 1) decode_attn_kernel(const DecodeKParams p) {
  using L = DecodeSmem<T, HD, G>;
  constexpr int HALF = HD / 2, VPR = L::VPR, NKG = L::NKG, QS = L::QS;
  extern __shared__ __align__(128) uint8_t smem_dec[];
  uint8_t* ring = smem_dec;
  float* red = reinterpret_cast<float*>(smem_dec);
  float* qf = reinterpret_cast<float*>(smem_dec + L::Q_OFF);
  T* knew = reinterpret_cast<T*>(smem_dec + L::KN_OFF);
  T* vnew = reinterpret_cast<T*>(smem_dec + L::VN_OFF);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_dec + L::BAR_OFF);
  float* sc = reinterpret_cast<float*>(smem_dec + L::SC_OFF);
  __shared__ float s_red[4][G];
  __shared__ float s_max_g[G], s_sum_g[G];

  pdl_trigger();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < DEC_STAGES; ++i) mbar_init(&full[i], 1);
    mbar_fence_init();
  }
  pdl_wait();  // every global read below (qkv, slot, pos and the cache rows) comes after it
  const int b = blockIdx.x, kvh = blockIdx.y;
  const int slot = p.slot[b];
  const int pos = p.pos[b];
  const int n_keys = pos + 1;
  if (pos < 0 || pos >= p.s_max) {
    // the cache row is full (host-side callers reject this before launching, recognition.py / layout.py): never write past
    // the slot — emit zeros so a caller that ignored the bound sees an obviously dead row instead of corrupting a neighbour
    T* orow0 = reinterpret_cast<T*>(p.out) + static_cast<size_t>(b) * p.ldo + (blockIdx.y * G) * HD;
    for (int i = threadIdx.x; i < G * HD; i += 128) orow0[i] = from_f<T>(0.f);
    return;
  }
  const T* row = reinterpret_cast<const T*>(p.qkv) + static_cast<size_t>(b) * p.ld;
  T* kc = reinterpret_cast<T*>(p.kcache) + (static_cast<size_t>(slot) * p.n_kv_heads + kvh) * p.s_max * HD;
  T* vc = reinterpret_cast<T*>(p.vcache) + (static_cast<size_t>(slot) * p.n_kv_heads + kvh) * p.s_max * HD;
  const int sp = p.s_max + 1;  // score row pitch: the G rows of a key fall in different banks
  const int nc = (n_keys + DEC_CK - 1) / DEC_CK;

  // stream step s < 2 nc loads K chunk s (s < nc) or V chunk s - nc into stage s % DEC_STAGES, phase (s / DEC_STAGES) & 1;
  // chunk c holds cache rows [c DEC_CK, min((c + 1) DEC_CK, pos)), none when it only holds the appended row
  auto issue = [&](int s) {
    const int c = s < nc ? s : s - nc;
    const uint32_t bytes = static_cast<uint32_t>(min(DEC_CK, pos - c * DEC_CK)) * HD * sizeof(T);
    uint64_t* bar = &full[s % DEC_STAGES];
    mbar_expect_tx(bar, bytes);
    if (bytes) bulk_load(ring + (s % DEC_STAGES) * L::CHUNK, (s < nc ? kc : vc) + static_cast<size_t>(c) * DEC_CK * HD, bytes, bar);
  };
  if (tid == 0)
    for (int s = 0; s < min(DEC_STAGES, 2 * nc); ++s) issue(s);

  // ---- RoPE on the G query heads and the new key; append k, v (and keep them for the key pos)
  for (int idx = tid; idx < (G + 1) * HALF; idx += 128) {
    int hh = idx / HALF, i = idx % HALF;
    const T* src = (hh < G) ? row + (kvh * G + hh) * HD : row + (p.n_heads + kvh) * HD;
    float f = static_cast<float>(pos) * p.inv_freq[i];
    float c = rnd<T>(cosf(f)), s = rnd<T>(sinf(f));
    float x1 = to_f<T>(src[i]), x2 = to_f<T>(src[i + HALF]);
    float o1 = rnd<T>(rnd<T>(x1 * c) + rnd<T>(-x2 * s));
    float o2 = rnd<T>(rnd<T>(x2 * c) + rnd<T>(x1 * s));
    if (hh < G) {
      qf[hh * QS + i] = o1;  // o1 / o2 are already rounded to T
      qf[hh * QS + i + HALF] = o2;
    } else {
      const T k1 = from_f<T>(o1), k2 = from_f<T>(o2);
      kc[static_cast<size_t>(pos) * HD + i] = k1;
      kc[static_cast<size_t>(pos) * HD + i + HALF] = k2;
      knew[i] = k1;
      knew[i + HALF] = k2;
    }
  }
  {
    const T* vsrc = row + (p.n_heads + p.n_kv_heads + kvh) * HD;
    for (int i = tid; i < HD; i += 128) {
      const T v = vsrc[i];
      vc[static_cast<size_t>(pos) * HD + i] = v;
      vnew[i] = v;
    }
  }
  __syncthreads();

  // ---- scores, one K chunk at a time: item it = (key it / G of the chunk, head it % G); 128 % G == 0, so a thread's head is fixed
  const int gs = tid % G;
  const float* qg = qf + gs * QS;
  float tmax = -INFINITY;
  for (int c = 0; c < nc; ++c) {
    const int st = c % DEC_STAGES;
    mbar_wait(&full[st], (c / DEC_STAGES) & 1);
    const T* kst = reinterpret_cast<const T*>(ring + st * L::CHUNK);
    const int c0 = c * DEC_CK, ck = min(DEC_CK, n_keys - c0);
    for (int it = tid; it < ck * G; it += 128) {
      const int jl = it / G, j = c0 + jl;
      const uint4* kr = reinterpret_cast<const uint4*>(j == pos ? knew : kst + jl * HD);
      float acc = 0.f;
#pragma unroll
      for (int c8 = 0; c8 < VPR; ++c8) {
        const uint4 u = kr[c8];
        const T* e = reinterpret_cast<const T*>(&u);
        const float4 qa = reinterpret_cast<const float4*>(qg + c8 * 8)[0];
        const float4 qb = reinterpret_cast<const float4*>(qg + c8 * 8)[1];
        acc = fmaf(qa.x, to_f<T>(e[0]), acc);
        acc = fmaf(qa.y, to_f<T>(e[1]), acc);
        acc = fmaf(qa.z, to_f<T>(e[2]), acc);
        acc = fmaf(qa.w, to_f<T>(e[3]), acc);
        acc = fmaf(qb.x, to_f<T>(e[4]), acc);
        acc = fmaf(qb.y, to_f<T>(e[5]), acc);
        acc = fmaf(qb.z, to_f<T>(e[6]), acc);
        acc = fmaf(qb.w, to_f<T>(e[7]), acc);
      }
      const float sv = acc * p.scale;
      sc[gs * sp + j] = sv;
      tmax = fmaxf(tmax, sv);
    }
    __syncthreads();  // stage st consumed
    if (tid == 0 && c + DEC_STAGES < 2 * nc) issue(c + DEC_STAGES);
  }
  for (int o = 16; o >= G; o >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
  if (lane < G) s_red[warp][lane] = tmax;
  __syncthreads();
  if (tid < G) s_max_g[tid] = fmaxf(fmaxf(s_red[0][tid], s_red[1][tid]), fmaxf(s_red[2][tid], s_red[3][tid]));
  __syncthreads();
  float tsum[G];
#pragma unroll
  for (int gq = 0; gq < G; ++gq) tsum[gq] = 0.f;
  for (int j = tid; j < n_keys; j += 128) {
#pragma unroll
    for (int gq = 0; gq < G; ++gq) {
      float pv = __expf(sc[gq * sp + j] - s_max_g[gq]);
      tsum[gq] += pv;
      sc[gq * sp + j] = rnd<T>(pv);
    }
  }
#pragma unroll
  for (int gq = 0; gq < G; ++gq) {
    float s = warp_sum(tsum[gq]);
    if (lane == 0) s_red[warp][gq] = s;
  }
  __syncthreads();
  if (tid < G) s_sum_g[tid] = s_red[0][tid] + s_red[1][tid] + s_red[2][tid] + s_red[3][tid];
  __syncthreads();

  // ---- O = P V, one V chunk at a time: thread = (key group kg, 8-wide dim chunk); jn walks j = kg (mod NKG) across the chunks
  const int chunk = tid % VPR, kg = tid / VPR;
  float acc[G][8];
#pragma unroll
  for (int gq = 0; gq < G; ++gq)
#pragma unroll
    for (int x = 0; x < 8; ++x) acc[gq][x] = 0.f;
  int jn = kg;
  for (int c = 0; c < nc; ++c) {
    const int s = nc + c, st = s % DEC_STAGES;
    mbar_wait(&full[st], (s / DEC_STAGES) & 1);
    if (kg < NKG) {
      const T* vst = reinterpret_cast<const T*>(ring + st * L::CHUNK);
      const int c0 = c * DEC_CK, c1 = min(c0 + DEC_CK, n_keys);
      for (; jn < c1; jn += NKG) {
        const uint4 u = reinterpret_cast<const uint4*>(jn == pos ? vnew : vst + (jn - c0) * HD)[chunk];
        const T* e = reinterpret_cast<const T*>(&u);
        float vf[8];
#pragma unroll
        for (int x = 0; x < 8; ++x) vf[x] = to_f<T>(e[x]);
#pragma unroll
        for (int gq = 0; gq < G; ++gq) {
          const float pg = sc[gq * sp + jn];
#pragma unroll
          for (int x = 0; x < 8; ++x) acc[gq][x] = fmaf(pg, vf[x], acc[gq][x]);
        }
      }
    }
    __syncthreads();  // stage st consumed
    if (tid == 0 && s + DEC_STAGES < 2 * nc) issue(s + DEC_STAGES);
  }
  // every issued chunk has been waited for and consumed: the ring is free for the partials
  if (kg < NKG) {
#pragma unroll
    for (int gq = 0; gq < G; ++gq)
#pragma unroll
      for (int x = 0; x < 8; ++x) red[(kg * G + gq) * HD + chunk * 8 + x] = acc[gq][x];
  }
  __syncthreads();
  T* orow = reinterpret_cast<T*>(p.out) + static_cast<size_t>(b) * p.ldo + (kvh * G) * HD;
  for (int i = tid; i < G * HD; i += 128) {
    float s = 0.f;
#pragma unroll
    for (int k2 = 0; k2 < NKG; ++k2) s += red[k2 * G * HD + i];
    orow[i] = from_f<T>(s / s_sum_g[i / HD]);
  }
}

template <typename T, int HD, int G>
static int launch_decode(const DecodeAttnArgs& a, cudaStream_t st) {
  const size_t smem = DecodeSmem<T, HD, G>::bytes(a.s_max);
  auto kern = decode_attn_kernel<T, HD, G>;
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      cudaGetLastError();  // clear it: the next launch_ok() would report this error as its own
      set_error("decode_attn: %zu bytes of shared memory exceed the device limit (s_max too large)", smem);
      return -3;
    }
    attr = smem;
  }
  DecodeKParams p;
  p.qkv = a.qkv; p.ld = a.ld; p.kcache = a.kcache; p.vcache = a.vcache; p.slot = a.slot; p.pos = a.pos;
  p.inv_freq = a.inv_freq; p.out = a.out; p.ldo = a.ldo;
  p.n_heads = a.n_heads; p.n_kv_heads = a.n_kv_heads; p.s_max = a.s_max; p.scale = a.scale;
  dim3 grid(a.batch, a.n_kv_heads), block(128);
  launch_pdl(kern, grid, block, smem, st, p);
  return launch_ok();
}

template <typename T, int HD>
static int dispatch_decode_g(const DecodeAttnArgs& a, cudaStream_t st) {
  int G = a.n_heads / a.n_kv_heads;
  switch (G) {
    case 1: return launch_decode<T, HD, 1>(a, st);
    case 2: return launch_decode<T, HD, 2>(a, st);
    case 4: return launch_decode<T, HD, 4>(a, st);
    case 8: return launch_decode<T, HD, 8>(a, st);
    default: set_error("decode_attn: unsupported GQA group %d (1/2/4/8)", G); return -1;
  }
}

template <typename T>
static int dispatch_decode(const DecodeAttnArgs& a, cudaStream_t st) {
  switch (a.head_dim) {
    case 64: return dispatch_decode_g<T, 64>(a, st);
    case 80: return dispatch_decode_g<T, 80>(a, st);
    case 128: return dispatch_decode_g<T, 128>(a, st);
    default: set_error("decode_attn: unsupported head_dim %d (64/80/128)", a.head_dim); return -1;
  }
}

int decode_attn(const DecodeAttnArgs& a, cudaStream_t st) {
  if (a.batch <= 0) return 0;
  if (a.n_kv_heads <= 0 || a.n_heads % a.n_kv_heads) {
    set_error("decode_attn: n_heads must be a positive multiple of n_kv_heads"); return -1;
  }
  // the cache rows are read with 16-byte bulk copies
  if ((reinterpret_cast<uintptr_t>(a.kcache) | reinterpret_cast<uintptr_t>(a.vcache)) % 16) {
    set_error("decode_attn: kcache and vcache must be 16B aligned"); return -1;
  }
  return a.dtype == DT_BF16 ? dispatch_decode<__nv_bfloat16>(a, st) : dispatch_decode<__half>(a, st);
}

}  // namespace sb
