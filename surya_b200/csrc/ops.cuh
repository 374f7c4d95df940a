// surya_b200 — host-side launchers for the non-GEMM kernels (ops.cu, attention.cu).
#pragma once
#include "gemm.cuh"

namespace sb {

int rmsnorm(int dtype, const void* x, int ldx, const void* w, void* y, int ldy, int rows, int H, float eps,
            const int* src_rows, cudaStream_t st, int mode = 0);
// rs[row] = rsqrt(mean_k x[row,k]^2 + eps): the per-row scale of a GEMM that folds the RMSNorm weight into W (gemm.cuh).
int row_rstd(int dtype, const void* x, int ldx, float* rs, int rows, int H, float eps, const int* src_rows, cudaStream_t st);

// Tail of a greedy decode step (ops.cu: decode_tail_kernel): argmax partial reduce, bbox head, bookkeeping, next embedding.
struct DecodeTailArgs {
  int rows = 0;
  const float* am_val = nullptr; const int* am_idx = nullptr; const float* am_sum = nullptr; int am_ld = 0, n_tiles = 0;
  const void* x = nullptr; int ldx = 0; int H = 0; float eps = 0.f;         // final hidden state BEFORE the final norm
  const void* bbox_w = nullptr; const void* bbox_b = nullptr; int n_box = 6; float bbox_size = 0.f;   // bbox_w has the norm weight folded in
  const void* embed = nullptr; void* x_next = nullptr; int ldx_next = 0;      // write embed[next_id] into x_next[row]
  long long* tok = nullptr; float* score = nullptr; long long* bbox = nullptr; float* bbox_sig = nullptr;
  unsigned char* done = nullptr; long long* next_ids = nullptr;
  int* step = nullptr; unsigned int* counter = nullptr;                       // device step counter of sb_rec_decode_steps
  long long* tok_hist = nullptr; float* score_hist = nullptr; long long* bbox_hist = nullptr; unsigned char* done_hist = nullptr;
  long long* ids_io = nullptr; int* pos_io = nullptr;
  int eos = 0, pad = 0;
};
int decode_tail(int dtype, const DecodeTailArgs& a, cudaStream_t st);

// Stop rules of the recognition decode loop evaluated on the device after a step (ops.cu: stop_rules_kernel).
int stop_rules(const long long* tok_hist, const unsigned char* done_hist, const int* step_dev, int step_host, int B, int* gen_count,
               long long* ring, unsigned char* row_done, int* n_valid, int* n_active, int max_tokens, int max_repeats,
               cudaStream_t st);

int gather_pad_rows(int dtype, const void* src, int src_is_f32, int lds, const int* perm, void* dst, int ldd, int rows,
                    int K, int Kp, cudaStream_t st);
int rope_vision(int dtype, void* qkv, int ld, const int* pos_rc, const float* inv_freq, int n_tok, int nh, int d,
                cudaStream_t st);
int rope_kv_append(int dtype, void* qkv, int ld, const int* tok_pos, const int* tok_slot, const float* inv_freq,
                   void* kcache, void* vcache, int n_tok, int nh, int nkv, int d, int s_max, cudaStream_t st);
int embed_splice(int dtype, const long long* ids, const int* feat_row, const int* hidx, const int* widx,
                 const void* embed, const void* feat, int ldf, const void* h_embed, const void* w_embed, void* out,
                 int ldo, int n_tok, int H, cudaStream_t st);
int argmax_score(int dtype, const void* logits, int ld, int rows, int V, long long* tok, float* score,
                 unsigned char* done, long long* next_ids, int eos, int pad, cudaStream_t st);
int small_head(int dtype, const void* x, int ldx, const void* w, const void* b, int rows, int H, int n_out,
               int sigmoid, float* out_f, long long* out_box, float box_scale, cudaStream_t st);
int embed_rows(int dtype, const long long* ids, const void* embed, void* out, int ldo, int n, int H, cudaStream_t st);

// Variable-length (block-diagonal) attention over packed sequences, tensor-core (mma.sync) flash kernel.
//   q/k/v: row-major token matrices with per-tensor row pitch and column offset of head 0; head h at col_off + h*d
//   seq_start[s], seq_len[s]: token range of sequence s (same for q and k); causal: key j <= query i (in-sequence)
//   n_kv_heads <= n_heads (GQA: kv head = h / (n_heads / n_kv_heads)); out[token, h*d + c], pitch ldo.
struct AttnArgs {
  int dtype = DT_BF16;
  const void* q = nullptr; int ldq = 0;
  const void* k = nullptr; int ldk = 0;
  const void* v = nullptr; int ldv = 0;
  void* out = nullptr;     int ldo = 0;
  const int* seq_start = nullptr;
  const int* seq_len = nullptr;
  int n_seq = 0, max_len = 0;
  int n_heads = 0, n_kv_heads = 0, head_dim = 0;
  int causal = 0;
  float scale = 1.f;
};
int attn_varlen(const AttnArgs& a, cudaStream_t st);

// k x k dense convolution (NHWC, implicit GEMM on wgmma); weight [Cout, k*k*Cin] with K ordered (r, s, c).
struct ConvArgs {
  int dtype = DT_F16;
  const void* in = nullptr;      // [n_img, H, W, Cin]
  const void* weight = nullptr;  // [Cout, ksize*ksize*Cin]
  const float* bias = nullptr;   // [Cout] fp32 (folded BN shift) or null
  const void* residual = nullptr;  // [n_img, Ho, Wo, Cout] or null
  void* out = nullptr;           // [n_img, Ho, Wo, Cout]
  int n_img = 0, H = 0, W = 0, Cin = 0, Cout = 0, ksize = 3, stride = 1, pad = 1, act = ACT_NONE;
};
int conv_igemm(const ConvArgs& a, cudaStream_t st);

// FusedMBConv (conv_fmb.cu): 3x3 expand conv + Hardswish + 1x1 project (+ shortcut) as one back-to-back wgmma GEMM kernel.
bool fmb_fused_ok(int Cin, int Cmid, int Cout, int ksize, int stride, int pad, int act1, int act2);
int fmb_fused(int dtype, const void* in, const void* w1, const float* bias1, const void* w2, const float* bias2,
              const void* residual, void* out, int n_img, int H, int W, int Cin, int Cmid, int Cout, int stride, cudaStream_t st);

// Fused decode head (det_head.cu): upsample + concat + fuse conv + ReLU + classifier + sigmoid in one wgmma kernel.
bool det_head_fused_ok(int n_src, int CS, int n_out, int cin, int cout, const int* hs, const int* ws, int HO, int WO);
int det_head_fused(int dtype, const void* const* srcs, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                   const void* fuse_w, const float* fuse_bias, const void* cls_w, const void* cls_b, void* logits, int B, int HO,
                   int WO, cudaStream_t st);

// Detection-path CUDA-core kernels (det_ops.cu).
int det_stem_conv(int dtype, const void* in, int in_f32, const float* w, const float* bias, void* out, int B, int H,
                  int W, int cout, cudaStream_t st);
int det_dwconv(int dtype, const void* in, const void* w, const float* bias, void* out, int B, int H, int W, int C, int ks,
               int stride, int pad, int act, cudaStream_t st);
int det_lite_mla(int dtype, const void* qkv_a, const void* qkv_b, void* out, int B, int HW, int heads, int dim, float eps,
                 cudaStream_t st);
int det_upsample_cat(int dtype, const void* const* src, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                     void* dst, int B, int HO, int WO, cudaStream_t st);
int det_classifier(int dtype, const void* x, const void* w, const void* b, void* out, long long P, int C, int HW, int n_out,
                   cudaStream_t st);
int det_upsample_nchw(int dtype, const void* in, float* out, int planes, int hs, int ws, int HO, int WO, cudaStream_t st);

int det_normalize_u8(int dtype, const unsigned char* in, void* out, int B, int H, int W, cudaStream_t st);
// Front half of the detection post-processing on the device (det_ops.cu): text-channel x4 bilinear map (16-bit), exact
// top-10 % mean -> dynamic thresholds, binarised mask.  hist: B x 16384 zeroed uint32 scratch (left zeroed); thr: B x 4 floats
// (text_threshold, low_text, top-10 % mean, scaling factor).
int det_text_front(int dtype, const void* logits, int n_labels, int B, int hs, int ws, int HO, int WO, void* map16,
                   unsigned char* mask, float* thr, unsigned int* hist, float text_threshold, float low_text, cudaStream_t st,
                   const int* chunk_tab = nullptr, int n_pages = 0, const int* page_tab = nullptr, int max_page_rows = 0);
// Page preparation (page_prep.cu): n_steps launches of the chained reduce / Lanczos jobs planned by surya_b200/page_prep.py.
int det_page_resize(const unsigned char* pages, unsigned char* scratch, unsigned char* out, const long long* desc, const int* tables,
                    int n_steps, const int* step_jobs, const long long* step_max_px, cudaStream_t st);
// Back half on the device (det_boxes.cu): connected components, keep filter and dilated row extents as per-page tables
// (layout in include/surya_b200.h, sb_det_text_boxes).
size_t det_text_boxes_scratch_bytes(int B, int H, int W, int max_points);
int det_text_boxes(int dtype, const void* map16, const unsigned char* mask, const float* thr, int B, int H, int W,
                   int max_boxes, int max_points, void* scratch, int* count, int* overflow, int* box, float* peak, int* points,
                   cudaStream_t st);

// Layout / table_rec kernels (layout_ops.cu).
int layernorm(int dtype, const void* x, const void* w, const void* b, void* y, int rows, int C, float eps, cudaStream_t st);
int patch_gather(int dtype, const void* in, int in_f32, void* out, int B, int Cin, int H, int W, int P, int Kp, cudaStream_t st);
int add_bcast_rows(int dtype, void* x, const void* tab, long long rows, int rows_per_batch, int C, cudaStream_t st);
int patch_merge_gather(int dtype, const void* x, void* y, int B, int H, int W, int C, cudaStream_t st);
int swin_window_attn(int dtype, const void* qkv, const float* qkv_bias, const void* bias_table, void* out, int B, int H, int W, int C,
                     int nh, int shift, cudaStream_t st);
int bbox_embed_sum(int dtype, const long long* boxes, const void* const* tables, void* out, int n, int Hd, int bbox_size,
                   cudaStream_t st);
// kv_index (device, may be null): query row b reads K/V set kv_index[b] instead of set b.
int attn_single_query(int dtype, const void* q, int ldq, const void* K, const void* V, long long bs, long long hs, long long ts,
                      void* out, int ldo, int B, int nh, int nkv, int head_dim, int n_keys, float scale, cudaStream_t st,
                      const int* kv_index = nullptr);
int label_embed(int dtype, const long long* boxes, const void* const* tables, void* out, int n, int box_w, int prop_w,
                int bbox_size, int vocab, cudaStream_t st);
// LayoutPredictor's header/footer rule inside box_next_token (off when page_wh is null): page_wh int32 [B, 2] = (w, h) of the
// image row b was preprocessed from; sticky (may be null) = rows already done, which the rule skips; header / footer = class
// tokens of PageHeader / PageFooter (label id + special_token_count); dtype = the model dtype the polygon is rounded to.
struct PageRule {
  const int* page_wh = nullptr;
  const unsigned char* sticky = nullptr;
  int dtype = DT_F16, header = -1, footer = -1;
  float skew_scaler = 0.f;
};
int box_next_token(const float* bbox, const float* const* heads, const int* head_n, const int* head_mode, int n_heads,
                   float bbox_size, long long* out, unsigned char* done, int done_head, int eos, int pad, int B, int* cache_pos,
                   const int* hist_base, int hist_T, long long* hist_tok, float* hist_bbox, float* const* hist_heads,
                   unsigned char* hist_done, cudaStream_t st, const PageRule& rule = PageRule());
// sticky[b] |= done[b]; n_active[0] = number of rows b < B with sticky[b] == 0 (table_rec early exit).
int rows_done_count(const unsigned char* done, unsigned char* sticky, int* n_active, int B, cudaStream_t st);

// Recognition crop preprocessing on the device (preproc.cu): uint8 crops -> Lanczos4 scale_to_fit -> cubic resize to x28 -> normalise ->
// merge-block-major fp32 tiles.  desc: n_crops x 9 int32 on the device; mean / std3: 3 host floats each.
int rec_preprocess(const unsigned char* crops, const int* desc, int n_crops, int max_nh, int max_nw, int max_hb, int max_wb, int any_stage1,
                   float* scratch, float* tiles, int ld_tiles, int patch, int merge, const float* mean, const float* std3, cudaStream_t st);

// ocr_error path (ocr_error_ops.cu): Embeddings.forward of DistilBERT over packed real tokens.
int embed_pos_layernorm(int dtype, const int* ids, const int* pos, const void* word, const void* ptab, const void* w, const void* b,
                        void* y, int rows, int C, float eps, cudaStream_t st);

// Single-token decode attention over the slot KV cache, fused with RoPE(q,k) and the in-place cache append.
//   qkv[b] = [q(nh*d) | k(nkv*d) | v(nkv*d)] for batch row b; slot[b], pos[b] (= number of cached tokens) on device.
//   cache layout: [slot][kv_head][s_max][d]; writes rotated k / v at index pos[b], then attends over 0..pos[b].
struct DecodeAttnArgs {
  int dtype = DT_BF16;
  const void* qkv = nullptr; int ld = 0;
  void* kcache = nullptr; void* vcache = nullptr;
  const int* slot = nullptr; const int* pos = nullptr;
  const float* inv_freq = nullptr;
  void* out = nullptr; int ldo = 0;
  int batch = 0, n_heads = 0, n_kv_heads = 0, head_dim = 0, s_max = 0;
  float scale = 1.f;
};
int decode_attn(const DecodeAttnArgs& a, cudaStream_t st);

}  // namespace sb
