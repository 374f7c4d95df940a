// surya_b200 — layout / table_rec engine: Donut-Swin encoder + ADETR box decoder behind the C ABI (sb_layout_*).
//
// The layer loops, the workspaces, the K/V caches and the greedy decode loop (one CUDA graph per 8 steps) live here so that
// nothing on the forward path depends on the host between the first and the last kernel.  Every decoder call, the greedy
// loop's steps, the predictors' single steps (sb_layout_step) and the table cell pass, goes through run_token: one statement of
// the decoder's op order.
//
// Reference: DonutSwinLayoutModel.forward / DonutSwinModel.forward (surya/layout/model/encoder.py:33-81,
// surya/table_rec/model/encoder.py:35-87), DonutSwinEncoder/Stage/Layer (surya/common/donut/encoder.py:534-931),
// SuryaADETRDecoderModel + layers (surya/common/adetr/decoder.py:360-652), SuryaLayoutDecoder / SuryaTableRecDecoder heads
// (surya/layout/model/decoder.py:95-126, surya/table_rec/model/decoder.py:121-155), per-step token logic
// (surya/layout/__init__.py:111-137, surya/table_rec/__init__.py:62-131).
#include "../../include/surya_b200.h"
#include "engine.cuh"

#include <cmath>
#include <vector>

using namespace sb;

namespace {
constexpr int GRAPH_GROUP = 8;
}

struct sb_layout_engine {
  sb_layout_config c;
  std::vector<const void*> w;
  size_t esz = 2;
  Arena arena;
  // encoder workspaces
  void *x = nullptr, *h = nullptr, *qkv = nullptr, *ao = nullptr, *mlp = nullptr;
  // decoder state (persistent: the step graphs point at these)
  void *dx = nullptr, *dn = nullptr, *dq = nullptr, *da = nullptr, *dcross = nullptr, *dres = nullptr, *dqkv = nullptr,
       *dm = nullptr, *dh = nullptr;
  void* enc = nullptr;                 // [B, Lk, enc_hidden]
  std::vector<void*> ckv, kc, vc;      // per decoder layer
  int* slot = nullptr;
  long long* tok = nullptr;            // [B, ncol]
  int* pos = nullptr;                  // [R]
  int* base = nullptr;                 // [1] + the row-decode state below, carved from the same block
  float* out_bbox = nullptr;           // [B, 6]
  float* out_head[4] = {nullptr, nullptr, nullptr, nullptr};
  unsigned char* done = nullptr;
  int Lk = 0;
  // sb_layout_decode_rows state (inside the `base` block): active-row count, row -> table map, per-token prefill arrays
  // (position, cache slot, K/V set; sequence starts and lengths for attn_varlen) and the sticky done flags
  int *n_active = nullptr, *row_table = nullptr, *t_pos = nullptr, *t_slot = nullptr, *t_kv = nullptr, *t_start = nullptr,
      *t_len = nullptr;
  unsigned char* sticky = nullptr;
  int R = 0, P = 0;                    // decoder rows, decoder activation rows (prefill tokens per chunk)
  // held cross K/V: sb_layout_cross_kv stamps held_gen = ++kv_gen; sb_layout_decode bumps kv_gen (it overwrites ckv)
  unsigned long long kv_gen = 0, held_gen = 0;
  int held_tables = 0;
  int* h_active = nullptr;             // pinned [2]: active counts of the last two step groups
  cudaEvent_t ev_active[2] = {nullptr, nullptr};
  // decode loop: GRAPH_GROUP steps per replay, and one step for the tail
  StepGraph g_group{"sb_layout_decode", GRAPH_GROUP}, g_one{"sb_layout_decode", 1};
  StepGraph g_rows{"sb_layout_decode_rows", GRAPH_GROUP}, g_rows_one{"sb_layout_decode_rows", 1};
  StepGraph g_pages{"sb_layout_decode_pages", GRAPH_GROUP}, g_pages_one{"sb_layout_decode_pages", 1};
  EngineStream stream;

  ~sb_layout_engine() {
    for (cudaEvent_t ev : ev_active)
      if (ev) cudaEventDestroy(ev);
    if (h_active) cudaFreeHost(h_active);
  }

  int ncol() const { return 6 + c.n_out_heads; }
  // ---- weight table (see include/surya_b200.h)
  const void* WF(int i) const { return w[i]; }
  int stage_base(int s) const {      // index of the stage's position table
    int idx = SB_LW_ENC_FIXED;
    for (int i = 0; i < s; ++i) idx += 1 + c.depths[i] * SB_LW_ENC_LAYER + (i < c.n_stages - 1 ? SB_LW_ENC_MERGE : 0);
    return idx;
  }
  const void* WL(int s, int l, int k) const { return w[stage_base(s) + 1 + l * SB_LW_ENC_LAYER + k]; }
  const void* WM(int s, int k) const { return w[stage_base(s) + 1 + c.depths[s] * SB_LW_ENC_LAYER + k]; }
  int dec_base() const { return stage_base(c.n_stages); }
  int n_tables() const { return c.kind == 1 ? 13 : 15; }
  const void* WT(int i) const { return w[dec_base() + i]; }
  const void* WD(int l, int k) const { return w[dec_base() + n_tables() + l * SB_LW_DEC_LAYER + k]; }
  const void* WX(int k) const { return w[dec_base() + n_tables() + c.dec_layers * SB_LW_DEC_LAYER + k]; }
  int n_weights() const { return dec_base() + n_tables() + c.dec_layers * SB_LW_DEC_LAYER + SB_LW_DEC_TAIL + (c.kind == 1 ? 5 : 3); }
};

// ------------------------------------------------------------------------------------------------ Swin encoder
static int run_encoder(sb_layout_engine* e, const void* pixels, int is_f32, int B, void* out, cudaStream_t st) {
  const sb_layout_config& c = e->c;
  const int dt = c.dtype;
  int H = c.img_h / c.patch, W = c.img_w / c.patch;
  const int K0 = c.in_ch * c.patch * c.patch;
  const int Kp = (K0 + 63) / 64 * 64;
  CK(patch_gather(dt, pixels, is_f32, e->h, B, c.in_ch, c.img_h, c.img_w, c.patch, Kp, st));
  long long rows = static_cast<long long>(B) * H * W;
  int C = c.embed_dim;
  CK(gemm_launch(weight_gemm(dt, e->h, Kp, e->WF(SB_LW_PE_W), Kp, e->x, C, static_cast<int>(rows), C, Kp, e->WF(SB_LW_PE_B)), st));
  CK(layernorm(dt, e->x, e->WF(SB_LW_PE_LN_W), e->WF(SB_LW_PE_LN_B), e->x, static_cast<int>(rows), C, 1e-5f, st));
  void* x = e->x;
  void* alt = e->ao;     // patch merging ping-pongs between the two C-wide buffers
  for (int s = 0; s < c.n_stages; ++s) {
    const int nh = c.heads[s];
    const int R = static_cast<int>(rows);
    CK(add_bcast_rows(dt, x, e->w[e->stage_base(s)], rows, H * W, C, st));
    for (int l = 0; l < c.depths[s]; ++l) {
      const int shift = (l % 2 == 1 && (H < W ? H : W) > c.window) ? c.window / 2 : 0;
      void* attn_out = (x == e->x) ? e->ao : e->x;   // any C-wide buffer that is not x
      CK(layernorm(dt, x, e->WL(s, l, SB_LWE_LN1_W), e->WL(s, l, SB_LWE_LN1_B), e->h, R, C, c.enc_ln_eps, st));
      CK(gemm_launch(weight_gemm(dt, e->h, C, e->WL(s, l, SB_LWE_QKV_W), C, e->qkv, 3 * C, R, 3 * C, C, e->WL(s, l, SB_LWE_QKV_B)), st));
      CK(swin_window_attn(dt, e->qkv, static_cast<const float*>(e->WL(s, l, SB_LWE_QKV_B)), e->WL(s, l, SB_LWE_RPB), attn_out, B, H, W, C, nh,
                          shift, st));
      // x = attn_out @ Wo^T + bo + x   (written over h first, then swapped in: the GEMM must not alias its residual's rows
      // with a different pitch; here both are [R, C] so in-place on x is the same read-then-write per element)
      CK(gemm_launch(weight_gemm(dt, attn_out, C, e->WL(s, l, SB_LWE_O_W), C, x, C, R, C, C, e->WL(s, l, SB_LWE_O_B), x, C), st));
      CK(layernorm(dt, x, e->WL(s, l, SB_LWE_LN2_W), e->WL(s, l, SB_LWE_LN2_B), e->h, R, C, c.enc_ln_eps, st));
      CK(gemm_launch(weight_gemm(dt, e->h, C, e->WL(s, l, SB_LWE_FC1_W), C, e->mlp, 4 * C, R, 4 * C, C, e->WL(s, l, SB_LWE_FC1_B),
                                 nullptr, 0, ACT_GELU_ERF), st));
      CK(gemm_launch(weight_gemm(dt, e->mlp, 4 * C, e->WL(s, l, SB_LWE_FC2_W), 4 * C, x, C, R, C, 4 * C, e->WL(s, l, SB_LWE_FC2_B), x,
                                 C), st));
    }
    if (s < c.n_stages - 1) {
      if ((H | W) & 1) {
        // the reference pads here (encoder.py:281-287) and then fails on its floor-sized stage position table (:730-735, 773-776)
        set_error("sb_layout_encode: stage %d has an odd %dx%d token grid (the reference's stage position table cannot follow it)", s, H, W);
        return -31;
      }
      CK(patch_merge_gather(dt, x, e->mlp, B, H, W, C, st));
      rows /= 4;
      H /= 2; W /= 2;
      CK(layernorm(dt, e->mlp, e->WM(s, 0), e->WM(s, 1), e->mlp, static_cast<int>(rows), 4 * C, 1e-5f, st));
      void* nx = (x == e->x) ? alt : e->x;
      CK(gemm_launch(weight_gemm(dt, e->mlp, 4 * C, e->WM(s, 2), 4 * C, nx, 2 * C, static_cast<int>(rows), 2 * C, 4 * C, nullptr), st));
      x = nx;
      C *= 2;
    }
  }
  CK(add_bcast_rows(dt, x, e->WF(SB_LW_ENC_POS), rows, H * W, C, st));
  if (cudaMemcpyAsync(out, x, static_cast<size_t>(rows) * C * e->esz, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
    cudaGetLastError();
    set_error("sb_layout_encode: copy-out failed");
    return -30;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------ ADETR decoder
// Batched prompt prefill of sb_layout_decode_rows: the B token rows are n_seq sequences of len tokens each; self-attention is
// RoPE + cache append at (t_pos, t_slot) and causal attention within each sequence, and nothing after the last layer runs.
struct Prefill { int n_seq, len; };

// One q_len = 1 call on the persistent state: embedding of e->tok rows -> layers -> heads into e->out_*.  kv_index: row b reads
// the cross K/V of table kv_index[b] (null: table b).  pf: the rows are prompt tokens (see Prefill) instead of decode steps.
static int run_token(sb_layout_engine* e, const long long* tok, const int* pos, int B, cudaStream_t st,
                     const int* kv_index = nullptr, const Prefill* pf = nullptr) {
  const sb_layout_config& c = e->c;
  const int dt = c.dtype, Hd = c.hidden, nh = c.n_heads, nkv = c.n_kv, hd = c.head_dim;
  const float scale = 1.0f / sqrtf(static_cast<float>(hd));
  const void* tables[15];
  for (int i = 0; i < e->n_tables(); ++i) tables[i] = e->WT(i);
  if (c.kind == 1) CK(label_embed(dt, tok, tables, e->dx, B, c.box_w, c.prop_w, c.bbox_size, c.vocab, st));
  else CK(bbox_embed_sum(dt, tok, tables, e->dx, B, Hd, c.bbox_size, st));
  const int QW = (nh + 2 * nkv) * hd, KVW = 2 * nkv * hd;
  for (int l = 0; l < c.dec_layers; ++l) {
    // cross attention over the cached encoder K/V
    CK(rmsnorm(dt, e->dx, Hd, e->WD(l, SB_LWD_CROSS_NORM), e->dn, Hd, B, Hd, c.rms_eps, nullptr, st, 1));
    CK(gemm_launch(weight_gemm(dt, e->dn, Hd, e->WD(l, SB_LWD_CQ_W), Hd, e->dq, nh * hd, B, nh * hd, Hd, nullptr), st));
    const uint8_t* kv = static_cast<const uint8_t*>(e->ckv[l]);
    CK(attn_single_query(dt, e->dq, nh * hd, kv, kv + static_cast<size_t>(nkv) * hd * e->esz, static_cast<long long>(e->Lk) * KVW, hd,
                         KVW, e->da, nh * hd, B, nh, nkv, hd, e->Lk, scale, st, kv_index));
    CK(gemm_launch(weight_gemm(dt, e->da, nh * hd, e->WD(l, SB_LWD_CO_W), nh * hd, e->dcross, Hd, B, Hd, nh * hd, e->WD(l, SB_LWD_CO_B),
                               e->dx, Hd), st));
    // causal self attention (RoPE + cache append fused into the attention kernel)
    CK(rmsnorm(dt, e->dcross, Hd, e->WD(l, SB_LWD_SELF_NORM), e->dn, Hd, B, Hd, c.rms_eps, nullptr, st, 1));
    CK(gemm_launch(weight_gemm(dt, e->dn, Hd, e->WD(l, SB_LWD_SQKV_W), Hd, e->dqkv, QW, B, QW, Hd, nullptr), st));
    if (pf) {
      CK(rope_kv_append(dt, e->dqkv, QW, e->t_pos, e->t_slot, static_cast<const float*>(e->WX(SB_LWX_INV_FREQ)), e->kc[l], e->vc[l],
                        B, nh, nkv, hd, c.s_max, st));
      const uint8_t* qkv = static_cast<const uint8_t*>(e->dqkv);
      AttnArgs a;
      a.dtype = dt; a.q = qkv; a.ldq = QW; a.k = qkv + static_cast<size_t>(nh) * hd * e->esz; a.ldk = QW;
      a.v = qkv + static_cast<size_t>(nh + nkv) * hd * e->esz; a.ldv = QW; a.out = e->da; a.ldo = nh * hd;
      a.seq_start = e->t_start; a.seq_len = e->t_len; a.n_seq = pf->n_seq; a.max_len = pf->len;
      a.n_heads = nh; a.n_kv_heads = nkv; a.head_dim = hd; a.causal = 1; a.scale = scale;
      CK(attn_varlen(a, st));
    } else {
      DecodeAttnArgs a;
      a.dtype = dt; a.qkv = e->dqkv; a.ld = QW; a.kcache = e->kc[l]; a.vcache = e->vc[l]; a.slot = e->slot; a.pos = pos;
      a.inv_freq = static_cast<const float*>(e->WX(SB_LWX_INV_FREQ));
      a.out = e->da; a.ldo = nh * hd; a.batch = B; a.n_heads = nh; a.n_kv_heads = nkv; a.head_dim = hd; a.s_max = c.s_max;
      a.scale = scale;
      CK(decode_attn(a, st));
    }
    const void* res_src = c.double_residual ? e->dx : e->dcross;
    CK(gemm_launch(weight_gemm(dt, e->da, nh * hd, e->WD(l, SB_LWD_SO_W), nh * hd, e->dres, Hd, B, Hd, nh * hd, e->WD(l, SB_LWD_SO_B),
                               res_src, Hd), st));
    // GeGLU MLP
    CK(rmsnorm(dt, e->dres, Hd, e->WD(l, SB_LWD_MLP_NORM), e->dn, Hd, B, Hd, c.rms_eps, nullptr, st, 1));
    CK(gemm_launch(weight_gemm(dt, e->dn, Hd, e->WD(l, SB_LWD_GU_W), Hd, e->dm, c.inter, B, 2 * c.inter, Hd, nullptr, nullptr, 0,
                               ACT_GELU_TANH, 1), st));
    GemmArgs down = weight_gemm(dt, e->dm, c.inter, e->WD(l, SB_LWD_DOWN_W), c.inter, e->dx, Hd, B, Hd, c.inter, nullptr, e->dres, Hd);
    down.allow_splitk = 1;
    CK(gemm_launch(down, st));
  }
  if (pf) return 0;        // the prompt's K/V are cached; its last token runs as the first decode step
  CK(rmsnorm(dt, e->dx, Hd, e->WX(SB_LWX_FINAL_NORM), e->dn, Hd, B, Hd, c.rms_eps, nullptr, st, 1));
  CK(layernorm(dt, e->dn, e->WX(SB_LWX_OUT_LN_W), e->WX(SB_LWX_OUT_LN_B), e->dh, B, Hd, c.dec_ln_eps, st));
  const int hb = e->dec_base() + e->n_tables() + c.dec_layers * SB_LW_DEC_LAYER + SB_LW_DEC_TAIL;
  if (c.kind == 1) {   // table: bbox (sigmoid), category, merges, colspan, is_header — all bias-free
    CK(small_head(dt, e->dh, Hd, e->w[hb + 0], nullptr, B, Hd, 6, 1, e->out_bbox, nullptr, 0.f, st));
    for (int k = 0; k < 4; ++k)
      CK(small_head(dt, e->dh, Hd, e->w[hb + 1 + k], nullptr, B, Hd, c.head_n[k], 0, e->out_head[k], nullptr, 0.f, st));
  } else {             // layout: bbox head with bias + sigmoid, class head
    CK(small_head(dt, e->dh, Hd, e->w[hb + 0], e->w[hb + 1], B, Hd, 6, 1, e->out_bbox, nullptr, 0.f, st));
    CK(small_head(dt, e->dh, Hd, e->w[hb + 2], nullptr, B, Hd, c.head_n[0], 0, e->out_head[0], nullptr, 0.f, st));
  }
  return 0;
}

// rule: LayoutPredictor's header/footer relabelling and its done flags (sb_layout_decode_pages); null for the plain greedy loop
static int run_next(sb_layout_engine* e, int B, int hist_T, long long* hist_tok, float* hist_bbox, float* const* hist_heads,
                    unsigned char* hist_done, cudaStream_t st, const PageRule* rule = nullptr) {
  const sb_layout_config& c = e->c;
  const float* heads[4];
  int hn[4], hm[4];
  for (int k = 0; k < c.n_out_heads; ++k) { heads[k] = e->out_head[k]; hn[k] = c.head_n[k]; hm[k] = 0; }
  if (c.kind == 1) hm[2] = 1;   // colspan: round(max(v, 1))
  return box_next_token(e->out_bbox, heads, hn, hm, c.n_out_heads, static_cast<float>(c.bbox_size), e->tok, e->done,
                        (c.kind == 1 || rule) ? 0 : -1, c.eos, c.pad, B, e->pos, e->base, hist_T, hist_tok, hist_bbox, hist_heads,
                        hist_done, st, rule ? *rule : PageRule());
}

// Pinned active-row counts and their events, created on first use by the loops that stop early.
static int ensure_active_count(sb_layout_engine* e, const char* who) {
  if (e->h_active) return 0;
  if (cudaHostAlloc(&e->h_active, 2 * sizeof(int), cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError(); e->h_active = nullptr; set_error("%s: pinned allocation failed", who); return -8;
  }
  for (cudaEvent_t& ev : e->ev_active)
    if (!ev && cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError(); ev = nullptr; set_error("%s: event creation failed", who); return -8;
    }
  return 0;
}

// The `left` steps after the first, as replays of `group` (GRAPH_GROUP steps) and `one`, each step ending in rows_done_count.
// Early exit: after each group the active-row count goes to pinned memory.  Group g+1 is enqueued before the count of group g
// is read, so the GPU never waits for the host; when that count is 0, group g+1's steps are extra and the loop stops.
// *ran += the steps enqueued.
static int replay_until_done(sb_layout_engine* e, StepGraph& group, StepGraph& one, int left, cudaStream_t st, int* ran,
                             const char* who) {
  const int groups = left / GRAPH_GROUP;
  bool stop = false;
  auto post = [&](int g) -> int {
    if (cudaMemcpyAsync(e->h_active + (g & 1), e->n_active, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaEventRecord(e->ev_active[g & 1], st) != cudaSuccess) {
      cudaGetLastError(); set_error("%s: active-count copy failed", who); return -5;
    }
    return 0;
  };
  auto all_done = [&](int g) { cudaEventSynchronize(e->ev_active[g & 1]); return e->h_active[g & 1] == 0; };
  for (int g = 0; g < groups && !stop; ++g) {
    CK(group.replay(1, st));
    *ran += GRAPH_GROUP;
    CK(post(g));
    if (g > 0 && all_done(g - 1)) stop = true;
  }
  if (!stop && left % GRAPH_GROUP) {
    if (groups > 0 && all_done(groups - 1)) stop = true;
    if (!stop) {
      CK(one.replay(left % GRAPH_GROUP, st));
      *ran += left % GRAPH_GROUP;
    }
  }
  return 0;
}

extern "C" {

int sb_layout_create(const sb_layout_config* cfg, const void* const* weights, int n_weights, sb_layout_engine** out) {
  if (!cfg || !weights || !out) { set_error("sb_layout_create: null argument"); return -1; }
  auto* e = new sb_layout_engine();
  e->c = *cfg;
  const sb_layout_config& c = e->c;
  if (c.n_stages < 1 || c.n_stages > 4 || c.n_out_heads < 1 || c.n_out_heads > 4 || c.head_dim != 64) {
    set_error("sb_layout_create: 1..4 stages, 1..4 output heads and head_dim 64 are supported");
    delete e;
    return -2;
  }
  if (c.patch <= 0 || c.img_h % c.patch || c.img_w % c.patch) {
    // the reference would zero pad the pixels (encoder.py:232-239) and then fail on its floor-sized position tables
    set_error("sb_layout_create: image size %dx%d is not a multiple of the patch size %d", c.img_h, c.img_w, c.patch);
    delete e;
    return -2;
  }
  if (n_weights != e->n_weights()) {
    set_error("sb_layout_create: expected %d weight pointers, got %d", e->n_weights(), n_weights);
    delete e;
    return -3;
  }
  for (int i = 0; i < n_weights; ++i)
    if (!weights[i]) { set_error("sb_layout_create: weight pointer %d is null", i); delete e; return -4; }
  e->w.assign(weights, weights + n_weights);
  const size_t es = e->esz;
  if (c.max_batch < 1 || c.max_rows < 0 || c.max_prefill_tokens < 0 || c.s_max < 1) {
    set_error("sb_layout_create: max_batch (%d) and s_max (%d) must be positive, max_rows (%d) and max_prefill_tokens (%d) not negative",
              c.max_batch, c.s_max, c.max_rows, c.max_prefill_tokens);
    delete e;
    return -2;
  }
  const size_t B = c.max_batch;
  // decoder rows (self-attention caches) and activation rows, never fewer than max_batch; 0 keeps the sizes sb_layout_decode has
  // always used
  const size_t R = static_cast<size_t>(c.max_rows) > B ? static_cast<size_t>(c.max_rows) : B;
  size_t P = R;
  if (static_cast<size_t>(c.max_prefill_tokens) > P) P = c.max_prefill_tokens;
  e->R = static_cast<int>(R);
  e->P = static_cast<int>(P);
  const size_t rows0 = B * (c.img_h / c.patch) * (c.img_w / c.patch);
  const size_t C0 = c.embed_dim;
  const int K0 = c.in_ch * c.patch * c.patch, Kp = (K0 + 63) / 64 * 64;
  const size_t hcols = C0 > static_cast<size_t>(Kp) ? C0 : Kp;
  int Hl = c.img_h / c.patch, Wl = c.img_w / c.patch;
  for (int s = 0; s < c.n_stages - 1; ++s) { Hl /= 2; Wl /= 2; }
  const size_t Lk = static_cast<size_t>(Hl) * Wl;
  const size_t Hd = c.hidden, QW = (c.n_heads + 2 * c.n_kv) * c.head_dim, KVW = 2 * c.n_kv * c.head_dim;
  const size_t cache = R * c.n_kv * c.s_max * c.head_dim * es;
  const size_t QH = static_cast<size_t>(c.n_heads) * c.head_dim;
  Arena& a = e->arena;
  a.add(e->x, rows0 * C0 * es); a.add(e->h, rows0 * hcols * es); a.add(e->qkv, rows0 * 3 * C0 * es); a.add(e->ao, rows0 * C0 * es);
  a.add(e->mlp, rows0 * 4 * C0 * es);
  a.add(e->dx, P * Hd * es); a.add(e->dn, P * Hd * es); a.add(e->dq, P * QH * es); a.add(e->da, P * QH * es);
  a.add(e->dcross, P * Hd * es); a.add(e->dres, P * Hd * es); a.add(e->dqkv, P * QW * es); a.add(e->dm, P * c.inter * es);
  a.add(e->dh, R * Hd * es);
  a.add(e->enc, B * Lk * c.enc_hidden * es);
  // `base` block: [0] history base, [1] active-row count, [2..3] spare, then row_table [R], five per-token arrays [P], sticky [R]
  const size_t state = (4 + R + 5 * P) * sizeof(int) + R;
  a.add(e->slot, R * sizeof(int)); a.add(e->tok, P * 10 * sizeof(long long)); a.add(e->pos, R * sizeof(int));
  a.add(e->base, state > 256 ? state : 256);
  a.add(e->out_bbox, R * 6 * sizeof(float)); a.add(e->done, R);
  for (int k = 0; k < 4; ++k) a.add(e->out_head[k], R * (k < c.n_out_heads ? c.head_n[k] : 1) * sizeof(float));
  e->ckv.resize(c.dec_layers); e->kc.resize(c.dec_layers); e->vc.resize(c.dec_layers);
  for (int l = 0; l < c.dec_layers; ++l) { a.add(e->ckv[l], B * Lk * KVW * es); a.add(e->kc[l], cache); a.add(e->vc[l], cache); }
  if (a.alloc() != cudaSuccess) {
    set_error("sb_layout_create: cudaMalloc(%zu) failed", a.bytes());
    delete e;
    return -5;
  }
  e->n_active = e->base + 1;
  e->row_table = e->base + 4;
  e->t_pos = e->row_table + R; e->t_slot = e->t_pos + P; e->t_kv = e->t_slot + P; e->t_start = e->t_kv + P; e->t_len = e->t_start + P;
  e->sticky = reinterpret_cast<unsigned char*>(e->t_len + P);
  std::vector<int> slots(R);
  for (size_t i = 0; i < R; ++i) slots[i] = static_cast<int>(i);
  cudaMemcpy(e->slot, slots.data(), R * sizeof(int), cudaMemcpyHostToDevice);
  e->Lk = static_cast<int>(Lk);
  *out = e;
  return 0;
}

void sb_layout_destroy(sb_layout_engine* e) { delete e; }

size_t sb_layout_workspace_bytes(const sb_layout_engine* e) { return e ? e->arena.bytes() : 0; }

int sb_layout_encode(sb_layout_engine* e, const void* pixels, int pixels_f32, int batch, void* enc_out, void* stream) {
  if (!e || !pixels || !enc_out) { set_error("sb_layout_encode: null argument"); return -1; }
  if (batch <= 0 || batch > e->c.max_batch) { set_error("sb_layout_encode: batch %d outside 1..%d", batch, e->c.max_batch); return -2; }
  return run_encoder(e, pixels, pixels_f32, batch, enc_out, static_cast<cudaStream_t>(stream));
}

// The greedy pass of sb_layout_decode, and with `rule` (sb_layout_decode_pages) LayoutPredictor's loop: the header/footer rule in
// the token step, sticky done flags and the early exit after the first group of steps at which every row is done (*n_run = the
// steps that ran).  Without a rule every one of the n_steps steps runs.
static int greedy_decode(sb_layout_engine* e, const char* who, const void* enc, int batch, const long long* prompt, int q_len,
                         int n_steps, long long* hist_tok, float* hist_bbox, float* const* hist_heads, unsigned char* hist_done,
                         int use_graph, void* stream, const PageRule* rule, int* n_run) {
  const sb_layout_config& c = e->c;
  if (batch <= 0 || batch > c.max_batch) { set_error("%s: batch %d outside 1..%d", who, batch, c.max_batch); return -2; }
  if (q_len < 1 || n_steps < 1 || q_len - 1 + n_steps > c.s_max) { set_error("%s: prompt + steps exceed s_max %d", who, c.s_max); return -3; }
  if (rule) CK(ensure_active_count(e, who));
  Hop hop(e->stream, static_cast<cudaStream_t>(stream), use_graph);
  if (hop.failed) { set_error("%s: could not create the engine stream", who); return -8; }
  const cudaStream_t st = hop.st;

  const int B = batch, ncol = e->ncol();
  const size_t es = e->esz;
  ++e->kv_gen;                     // the K/V held by sb_layout_cross_kv are overwritten below
  // encoder states -> persistent buffer; cross-attention K/V of every layer (SuryaADETRDecoderSdpaCrossAttention caches them at
  // the first call, adetr/decoder.py:150-194)
  if (cudaMemcpyAsync(e->enc, enc, static_cast<size_t>(B) * e->Lk * c.enc_hidden * es, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
    cudaGetLastError(); set_error("%s: encoder copy failed", who); return -4;
  }
  const int KVW = 2 * c.n_kv * c.head_dim;
  for (int l = 0; l < c.dec_layers; ++l)
    CK(gemm_launch(weight_gemm(c.dtype, e->enc, c.enc_hidden, e->WD(l, SB_LWD_CKV_W), c.enc_hidden, e->ckv[l], KVW, B * e->Lk, KVW,
                               c.enc_hidden, nullptr), st));
  // prompt: all but the last token, position by position (identical to the batched prefill under the causal mask)
  std::vector<int> hpos(B);
  for (int j = 0; j < q_len; ++j) {
    // gather column j of the prompt [B, q_len, ncol] into the token buffer
    if (cudaMemcpy2DAsync(e->tok, ncol * sizeof(long long), prompt + static_cast<size_t>(j) * ncol, static_cast<size_t>(q_len) * ncol * sizeof(long long),
                          ncol * sizeof(long long), B, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
      cudaGetLastError(); set_error("%s: prompt copy failed", who); return -5;
    }
    for (int b = 0; b < B; ++b) hpos[b] = j;
    if (cudaMemcpyAsync(e->pos, hpos.data(), B * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess) {
      cudaGetLastError(); set_error("%s: position copy failed", who); return -5;
    }
    if (j == q_len - 1) break;
    cudaStreamSynchronize(st);     // hpos is reused by the next iteration (pageable source)
    CK(run_token(e, e->tok, e->pos, B, st));
  }
  const int base = q_len - 1;
  if (cudaMemcpyAsync(e->base, &base, sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess) {
    cudaGetLastError(); set_error("%s: base copy failed", who); return -5;
  }
  if (rule && cudaMemsetAsync(e->sticky, 0, B, st) != cudaSuccess) {
    cudaGetLastError(); set_error("%s: done-flag reset failed", who); return -5;
  }
  cudaStreamSynchronize(st);       // host sources above are stack / vector memory

  auto body = [&](cudaStream_t s) -> int {
    CK(run_token(e, e->tok, e->pos, B, s));
    CK(run_next(e, B, n_steps, hist_tok, hist_bbox, hist_heads, hist_done, s, rule));
    return rule ? rows_done_count(e->done, e->sticky, e->n_active, B, s) : 0;
  };
  CK(body(st));                    // first step eagerly (sets kernel attributes before any capture)
  if (n_run) *n_run = 1;
  int left = n_steps - 1;
  if (left <= 0) return 0;
  StepGraph& group = rule ? e->g_pages : e->g_group;
  StepGraph& one = rule ? e->g_pages_one : e->g_one;
  if (!use_graph) {
    for (int i = 0; i < left; ++i) CK(body(st));
    if (n_run) *n_run = n_steps;
    return 0;
  }
  const StepGraph::Key key = {hist_tok, hist_bbox, hist_done, hist_heads ? hist_heads[0] : nullptr,
                              reinterpret_cast<const void*>(static_cast<uintptr_t>(n_steps)), rule ? rule->page_wh : nullptr};
  if (!group.hit(key, B) || !one.hit(key, B)) {
    CK(group.capture(key, B, st, body));
    CK(one.capture(key, B, st, body));
  }
  if (rule) return replay_until_done(e, group, one, left, st, n_run, who);
  CK(group.replay(left / GRAPH_GROUP, st));
  return one.replay(left % GRAPH_GROUP, st);
}

int sb_layout_decode(sb_layout_engine* e, const void* enc, int batch, const long long* prompt, int q_len, int n_steps,
                     long long* hist_tok, float* hist_bbox, float* const* hist_heads, unsigned char* hist_done, int use_graph,
                     void* stream) {
  if (!e || !enc || !prompt || !hist_tok) { set_error("sb_layout_decode: null argument"); return -1; }
  return greedy_decode(e, "sb_layout_decode", enc, batch, prompt, q_len, n_steps, hist_tok, hist_bbox, hist_heads, hist_done,
                       use_graph, stream, nullptr, nullptr);
}

int sb_layout_decode_pages(sb_layout_engine* e, const void* enc, int batch, const long long* prompt, int q_len, const int* page_wh,
                           int n_steps, long long* hist_tok, float* hist_bbox, float* hist_cls, unsigned char* hist_done,
                           int* n_run_host, void* stream) {
  if (!e || !enc || !prompt || !page_wh || !hist_tok || !hist_bbox || !hist_cls || !hist_done || !n_run_host) {
    set_error("sb_layout_decode_pages: null argument");
    return -1;
  }
  *n_run_host = 0;
  const sb_layout_config& c = e->c;
  if (c.kind != 0) { set_error("sb_layout_decode_pages: needs a layout engine (the page rule reads the layout class head)"); return -2; }
  // PageHeader / PageFooter are label ids 10 / 9 (surya/layout/model/config.py:16-34), after the special tokens
  if (c.special_tokens < 0 || c.special_tokens + 10 >= c.head_n[0]) {
    set_error("sb_layout_decode_pages: %d special tokens and %d classes leave no PageHeader class", c.special_tokens, c.head_n[0]);
    return -2;
  }
  PageRule rule;
  rule.page_wh = page_wh; rule.sticky = e->sticky; rule.dtype = c.dtype;
  rule.header = 10 + c.special_tokens; rule.footer = 9 + c.special_tokens; rule.skew_scaler = static_cast<float>(c.skew_scaler);
  float* heads[1] = {hist_cls};
  int ran = 0;
  CK(greedy_decode(e, "sb_layout_decode_pages", enc, batch, prompt, q_len, n_steps, hist_tok, hist_bbox, heads, hist_done, 1, stream,
                   &rule, &ran));
  *n_run_host = ran;
  return 0;
}


int sb_layout_cross_kv(sb_layout_engine* e, const void* enc, int n_tables, void* stream) {
  if (!e || !enc) { set_error("sb_layout_cross_kv: null argument"); return -1; }
  const sb_layout_config& c = e->c;
  if (n_tables <= 0 || n_tables > c.max_batch) {
    set_error("sb_layout_cross_kv: %d tables need max_batch >= %d (engine has %d)", n_tables, n_tables, c.max_batch);
    return -2;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int KVW = 2 * c.n_kv * c.head_dim;
  e->held_gen = 0;                 // a failed projection leaves nothing held
  for (int l = 0; l < c.dec_layers; ++l)
    CK(gemm_launch(weight_gemm(c.dtype, enc, c.enc_hidden, e->WD(l, SB_LWD_CKV_W), c.enc_hidden, e->ckv[l], KVW, n_tables * e->Lk, KVW,
                               c.enc_hidden, nullptr), st));
  e->held_gen = ++e->kv_gen;
  e->held_tables = n_tables;
  return 0;
}

int sb_layout_step(sb_layout_engine* e, const long long* tok, const int* pos, int batch, float* bbox, float* const* heads,
                   void* stream) {
  if (!e || !tok || !pos || !bbox || !heads) { set_error("sb_layout_step: null argument"); return -1; }
  const sb_layout_config& c = e->c;
  for (int k = 0; k < c.n_out_heads; ++k)
    if (!heads[k]) { set_error("sb_layout_step: head output %d is null", k); return -1; }
  if (e->held_gen == 0 || e->held_gen != e->kv_gen) {
    set_error("sb_layout_step: no cross K/V held (sb_layout_decode overwrote them, or sb_layout_cross_kv was not called)");
    return -3;
  }
  if (batch <= 0 || batch > e->held_tables) {
    set_error("sb_layout_step: batch %d outside 1..%d (the tables held by sb_layout_cross_kv)", batch, e->held_tables);
    return -2;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CK(run_token(e, tok, pos, batch, st));
  const size_t B = static_cast<size_t>(batch);
  bool ok = cudaMemcpyAsync(bbox, e->out_bbox, B * 6 * sizeof(float), cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  for (int k = 0; k < c.n_out_heads && ok; ++k)
    ok = cudaMemcpyAsync(heads[k], e->out_head[k], B * c.head_n[k] * sizeof(float), cudaMemcpyDeviceToDevice, st) == cudaSuccess;
  if (!ok) { cudaGetLastError(); set_error("sb_layout_step: output copy failed"); return -5; }
  return 0;
}

int sb_layout_decode_rows(sb_layout_engine* e, const int* row_table_host, int rows, const long long* prompt, int q_len, int n_steps,
                          long long* hist_tok, float* hist_bbox, float* const* hist_heads, unsigned char* hist_done,
                          int* n_run_host, void* stream) {
  if (!e || !row_table_host || !prompt || !hist_tok || !hist_done || !n_run_host) {
    set_error("sb_layout_decode_rows: null argument");
    return -1;
  }
  *n_run_host = 0;
  const sb_layout_config& c = e->c;
  if (c.kind != 1) { set_error("sb_layout_decode_rows: needs a table_rec engine (done is the category head)"); return -2; }
  if (e->held_gen == 0 || e->held_gen != e->kv_gen) {
    set_error("sb_layout_decode_rows: no cross K/V held (sb_layout_decode overwrote them, or sb_layout_cross_kv was not called)");
    return -3;
  }
  if (rows <= 0 || rows > e->R) { set_error("sb_layout_decode_rows: %d rows need max_rows >= %d (engine has %d)", rows, rows, e->R); return -2; }
  if (q_len < 1 || n_steps < 1 || q_len - 1 + n_steps > c.s_max) {
    set_error("sb_layout_decode_rows: a %d-token prompt and %d steps need s_max >= %d (engine has %d)", q_len, n_steps,
              q_len - 1 + n_steps, c.s_max);
    return -2;
  }
  if (q_len - 1 > e->P) {
    set_error("sb_layout_decode_rows: a %d-token prompt needs max_prefill_tokens >= %d (engine prefills %d tokens per chunk)", q_len,
              q_len - 1, e->P);
    return -2;
  }
  for (int r = 0; r < rows; ++r)
    if (row_table_host[r] < 0 || row_table_host[r] >= e->held_tables) {
      set_error("sb_layout_decode_rows: row %d maps to table %d, outside the %d held tables", r, row_table_host[r], e->held_tables);
      return -4;
    }
  CK(ensure_active_count(e, "sb_layout_decode_rows"));
  Hop hop(e->stream, static_cast<cudaStream_t>(stream), true);
  if (hop.failed) { set_error("sb_layout_decode_rows: could not create the engine stream"); return -8; }
  const cudaStream_t st = hop.st;
  const int ncol = e->ncol();
  const size_t tokb = static_cast<size_t>(ncol) * sizeof(long long);

  // host state, all copied before the one synchronisation below (the copies read pageable memory)
  const int nq = q_len - 1;                          // prompt tokens that only fill the self-attention caches
  const int per = nq > 0 ? e->P / nq : 0;            // rows per prefill chunk
  const int n_chunks = nq > 0 ? (rows + per - 1) / per : 0;
  std::vector<int> hstate(4 + rows);
  hstate[0] = q_len - 1;                             // history base: the step at position q_len-1 is history row 0
  hstate[1] = rows;
  for (int r = 0; r < rows; ++r) hstate[4 + r] = row_table_host[r];
  std::vector<int> hpos(rows, q_len - 1);
  std::vector<int> htok(static_cast<size_t>(n_chunks) * 5 * e->P);
  auto fail = [](const char* what) { cudaGetLastError(); set_error("sb_layout_decode_rows: %s failed", what); return -5; };
  if (cudaMemcpyAsync(e->base, hstate.data(), hstate.size() * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemsetAsync(e->sticky, 0, rows, st) != cudaSuccess)
    return fail("state copy");

  // batched prefill of positions 0 .. q_len-2, chunk by chunk (rows * nq tokens per chunk <= P)
  for (int ch = 0; ch < n_chunks; ++ch) {
    const int r0 = ch * per, n = rows - r0 < per ? rows - r0 : per, T = n * nq;
    int* h = htok.data() + static_cast<size_t>(ch) * 5 * e->P;
    for (int t = 0; t < T; ++t) {
      const int r = r0 + t / nq;
      h[t] = t % nq; h[e->P + t] = r; h[2 * e->P + t] = row_table_host[r];
    }
    for (int i = 0; i < n; ++i) { h[3 * e->P + i] = i * nq; h[4 * e->P + i] = nq; }
    if (cudaMemcpyAsync(e->t_pos, h, 5 * e->P * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpy2DAsync(e->tok, nq * tokb, prompt + static_cast<size_t>(r0) * q_len * ncol, q_len * tokb, nq * tokb, n,
                          cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return fail("prefill copy");
    const Prefill pf{n, nq};
    CK(run_token(e, e->tok, nullptr, T, st, e->t_kv, &pf));
  }
  // last prompt token of every row -> the first decode step
  if (cudaMemcpy2DAsync(e->tok, tokb, prompt + static_cast<size_t>(nq) * ncol, q_len * tokb, tokb, rows, cudaMemcpyDeviceToDevice,
                        st) != cudaSuccess ||
      cudaMemcpyAsync(e->pos, hpos.data(), rows * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return fail("prompt copy");
  cudaStreamSynchronize(st);       // host sources above are vector memory

  auto body = [&](cudaStream_t s) -> int {
    CK(run_token(e, e->tok, e->pos, rows, s, e->row_table));
    CK(run_next(e, rows, n_steps, hist_tok, hist_bbox, hist_heads, hist_done, s));
    return rows_done_count(e->done, e->sticky, e->n_active, rows, s);
  };
  CK(body(st));                    // first step eagerly (sets kernel attributes before any capture)
  int ran = 1;
  const int left = n_steps - 1;
  if (left > 0) {
    const StepGraph::Key key = {hist_tok, hist_bbox, hist_done, hist_heads ? hist_heads[0] : nullptr,
                                reinterpret_cast<const void*>(static_cast<uintptr_t>(n_steps))};
    if (!e->g_rows.hit(key, rows) || !e->g_rows_one.hit(key, rows)) {
      CK(e->g_rows.capture(key, rows, st, body));
      CK(e->g_rows_one.capture(key, rows, st, body));
    }
    CK(replay_until_done(e, e->g_rows, e->g_rows_one, left, st, &ran, "sb_layout_decode_rows"));
  }
  *n_run_host = ran;
  return 0;
}

}  // extern "C"
