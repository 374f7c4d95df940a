// surya_b200 — detection engine: executes the EfficientViT-seg op program over NHWC workspaces.
//
// Stands in for EfficientViTForSemanticSegmentation.forward (surya/detection/model/encoderdecoder.py:725-753):
// dense 3x3 convs -> conv_wgmma.cu, 1x1 / grouped 1x1 convs -> gemm_wgmma.cu, everything else -> det_ops.cu.
#include "../../include/surya_b200.h"
#include "engine.cuh"
#include "sb_ptx.cuh"

#include <vector>

using namespace sb;

struct BufDim { int H = 0, W = 0, C = 0; };

struct sb_det_engine {
  int dtype = DT_F16;
  std::vector<sb_det_op> ops;
  std::vector<const void*> w;
  std::vector<long long> buf_elems;
  std::vector<void*> bufs;
  std::vector<BufDim> dims;
  int max_batch = 0;
  Arena arena;
};

extern "C" {

int sb_det_create(int dtype, const sb_det_op* ops, int n_ops, const void* const* weights, int n_weights,
                  const long long* buf_elems, int n_bufs, int max_batch, sb_det_engine** out) {
  if (!ops || !weights || !buf_elems || !out) { set_error("sb_det_create: null argument"); return -1; }
  auto* e = new sb_det_engine();
  e->dtype = dtype;
  e->ops.assign(ops, ops + n_ops);
  e->w.assign(weights, weights + n_weights);
  e->buf_elems.assign(buf_elems, buf_elems + n_bufs);
  e->max_batch = max_batch;
  for (const auto& op : e->ops) {
    if (op.w >= n_weights || op.b >= n_weights) { set_error("sb_det_create: weight index out of range"); delete e; return -2; }
    if (op.dst >= n_bufs) { set_error("sb_det_create: buffer index out of range"); delete e; return -2; }
  }
  e->bufs.resize(n_bufs);
  for (int i = 0; i < n_bufs; ++i) e->arena.add(e->bufs[i], static_cast<size_t>(e->buf_elems[i]) * max_batch * 2);
  cudaError_t ce = e->arena.alloc();
  if (ce != cudaSuccess) {
    set_error("sb_det_create: cudaMalloc(%zu MiB) failed: %s", e->arena.bytes() >> 20, cudaGetErrorString(ce));
    delete e;
    return -3;
  }
  e->dims.resize(n_bufs);
  *out = e;
  return 0;
}

void sb_det_destroy(sb_det_engine* e) { delete e; }

size_t sb_det_workspace_bytes(const sb_det_engine* e) { return e ? e->arena.bytes() : 0; }

int sb_det_forward(sb_det_engine* e, const void* pixel_values, int in_f32, int B, int H, int W, void* logits, void* stream) {
  if (!e) { set_error("sb_det_forward: null engine"); return -1; }
  if (B > e->max_batch) { set_error("sb_det_forward: batch %d exceeds capacity %d", B, e->max_batch); return -2; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int dt = e->dtype;
  auto fits = [&](int buf, int h, int w, int c) -> bool {
    return static_cast<long long>(h) * w * c <= e->buf_elems[buf];
  };
  for (size_t i = 0; i < e->ops.size(); ++i) {
    const sb_det_op& op = e->ops[i];
    const int s0 = op.src[0];
    BufDim in = (s0 >= 0) ? e->dims[s0] : BufDim{H, W, op.cin};
    const void* in_ptr = (s0 >= 0) ? e->bufs[s0] : pixel_values;
    BufDim od;
    const void* res = op.res >= 0 ? e->bufs[op.res] : nullptr;
    switch (op.op) {
      case SB_DOP_STEM: {
        od = {H / 2, W / 2, op.cout};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small for %dx%dx%d", op.dst, od.H, od.W, od.C); return -4; }
        CK(det_stem_conv(dt, pixel_values, in_f32, static_cast<const float*>(e->w[op.w]), static_cast<const float*>(e->w[op.b]),
                         e->bufs[op.dst], B, H, W, op.cout, st));
        break;
      }
      case SB_DOP_CONV: {
        od = {(in.H + 2 * op.pad - op.k) / op.stride + 1, (in.W + 2 * op.pad - op.k) / op.stride + 1, op.cout};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        // FusedMBConv: 3x3 expand (Hardswish) directly followed by its 1x1 project -> one back-to-back GEMM kernel
        if (i + 1 < e->ops.size() && op.res < 0 && op.b >= 0) {
          const sb_det_op& pj = e->ops[i + 1];
          if (pj.op == SB_DOP_PW && pj.src[0] == op.dst && pj.cin == op.cout && pj.b >= 0 &&
              fmb_fused_ok(op.cin, op.cout, pj.cout, op.k, op.stride, op.pad, op.act, pj.act) && fits(pj.dst, od.H, od.W, pj.cout)) {
            CK(fmb_fused(dt, in_ptr, e->w[op.w], static_cast<const float*>(e->w[op.b]), e->w[pj.w], static_cast<const float*>(e->w[pj.b]),
                         pj.res >= 0 ? e->bufs[pj.res] : nullptr, e->bufs[pj.dst], B, in.H, in.W, op.cin, op.cout, pj.cout, op.stride, st));
            e->dims[op.dst] = od;
            e->dims[pj.dst] = {od.H, od.W, pj.cout};
            ++i;
            continue;
          }
        }
        ConvArgs a;
        a.dtype = dt; a.in = in_ptr; a.weight = e->w[op.w]; a.bias = op.b >= 0 ? static_cast<const float*>(e->w[op.b]) : nullptr;
        a.residual = res; a.out = e->bufs[op.dst]; a.n_img = B; a.H = in.H; a.W = in.W; a.Cin = op.cin; a.Cout = op.cout;
        a.ksize = op.k; a.stride = op.stride; a.pad = op.pad; a.act = op.act;
        CK(conv_igemm(a, st));
        break;
      }
      case SB_DOP_PW: {
        od = {in.H, in.W, op.cout};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        GemmArgs g;
        g.dtype = dt; g.A = in_ptr; g.lda = op.cin; g.W = e->w[op.w]; g.ldw = op.cin; g.C = e->bufs[op.dst]; g.ldc = op.cout;
        g.M = B * in.H * in.W; g.N = op.cout; g.K = op.cin;
        g.bias = op.b >= 0 ? static_cast<const float*>(e->w[op.b]) : nullptr;
        g.residual = res; g.ldr = op.cout; g.act = op.act;
        CK(gemm_launch(g, st));
        break;
      }
      case SB_DOP_DW: {
        od = {(in.H + 2 * op.pad - op.k) / op.stride + 1, (in.W + 2 * op.pad - op.k) / op.stride + 1, op.cout};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        CK(det_dwconv(dt, in_ptr, e->w[op.w], op.b >= 0 ? static_cast<const float*>(e->w[op.b]) : nullptr, e->bufs[op.dst], B,
                      in.H, in.W, op.cin, op.k, op.stride, op.pad, op.act, st));
        break;
      }
      case SB_DOP_GPW: {
        od = {in.H, in.W, op.cout};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        const int gk = op.cin / op.groups, gn = op.cout / op.groups;
        if (gn != 32 || gk > 64) { set_error("det: grouped 1x1 conv supports 32 outputs and <= 64 inputs per group"); return -5; }
        GemmArgs g;
        g.dtype = dt; g.A = in_ptr; g.lda = op.cin; g.W = e->w[op.w]; g.ldw = 64; g.C = e->bufs[op.dst]; g.ldc = op.cout;
        g.M = B * in.H * in.W; g.N = op.cout; g.K = 64;
        g.group_k = gk; g.group_n = gn; g.a_cols = op.cin;
        CK(gemm_launch(g, st));
        break;
      }
      case SB_DOP_MLA: {
        od = {in.H, in.W, 2 * op.heads * op.dim};
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        CK(det_lite_mla(dt, in_ptr, e->bufs[op.src[1]], e->bufs[op.dst], B, in.H * in.W, op.heads, op.dim, op.eps, st));
        break;
      }
      case SB_DOP_UPCAT: {
        const void* srcs[4]; int hs[4], ws[4];
        for (int j = 0; j < op.n_src; ++j) { srcs[j] = e->bufs[op.src[j]]; hs[j] = e->dims[op.src[j]].H; ws[j] = e->dims[op.src[j]].W; }
        od = {hs[0], ws[0], op.cout};
        // decode head: UPCAT -> 1x1 fuse conv (ReLU) -> classifier collapse into one kernel when the shapes are the default head's
        if (i + 2 < e->ops.size()) {
          const sb_det_op& fz = e->ops[i + 1];
          const sb_det_op& cl = e->ops[i + 2];
          if (fz.op == SB_DOP_PW && fz.src[0] == op.dst && fz.act == ACT_RELU && fz.res < 0 && fz.b >= 0 && cl.op == SB_DOP_CLS &&
              cl.src[0] == fz.dst && fz.cin == op.cout &&
              det_head_fused_ok(op.n_src, op.cin, cl.cout, fz.cin, fz.cout, hs, ws, od.H, od.W)) {
            CK(det_head_fused(dt, srcs, hs, ws, op.src_off, op.n_src, op.cin, e->w[fz.w], static_cast<const float*>(e->w[fz.b]),
                              e->w[cl.w], e->w[cl.b], logits, B, od.H, od.W, st));
            e->dims[op.dst] = od;
            e->dims[fz.dst] = {od.H, od.W, fz.cout};
            i += 2;
            continue;
          }
        }
        if (!fits(op.dst, od.H, od.W, od.C)) { set_error("det: buffer %d too small", op.dst); return -4; }
        CK(det_upsample_cat(dt, srcs, hs, ws, op.src_off, op.n_src, op.cin, e->bufs[op.dst], B, od.H, od.W, st));
        break;
      }
      case SB_DOP_CLS: {
        od = {in.H, in.W, op.cout};
        CK(det_classifier(dt, in_ptr, e->w[op.w], e->w[op.b], logits, static_cast<long long>(B) * in.H * in.W, op.cin,
                          in.H * in.W, op.cout, st));
        break;
      }
      default: set_error("det: unknown op %d", op.op); return -6;
    }
    if (op.dst >= 0) e->dims[op.dst] = od;
  }
  return 0;
}

int sb_det_upsample(int dtype, const void* logits, float* out, int planes, int hs, int ws, int HO, int WO, void* stream) {
  return det_upsample_nchw(dtype, logits, out, planes, hs, ws, HO, WO, static_cast<cudaStream_t>(stream));
}

int sb_det_normalize_u8(int dtype, const unsigned char* pages_nhwc, void* out_nchw, int B, int H, int W, void* stream) {
  if (!pages_nhwc || !out_nchw) { set_error("sb_det_normalize_u8: null argument"); return -1; }
  return det_normalize_u8(dtype, pages_nhwc, out_nchw, B, H, W, static_cast<cudaStream_t>(stream));
}

int sb_det_text_front(int dtype, const void* logits, int n_labels, int B, int hs, int ws, int HO, int WO, void* map16,
                      unsigned char* mask, float* thresholds, unsigned int* hist_scratch, float text_threshold, float low_text,
                      void* stream) {
  if (!logits || !map16 || !mask || !thresholds || !hist_scratch) { set_error("sb_det_text_front: null argument"); return -1; }
  return det_text_front(dtype, logits, n_labels, B, hs, ws, HO, WO, map16, mask, thresholds, hist_scratch, text_threshold,
                        low_text, static_cast<cudaStream_t>(stream));
}

int sb_det_text_front_stitched(int dtype, const void* logits, int n_labels, int n_chunks, int hs, int ws, int HO, int WO,
                               const int* chunk_tab, int n_pages, const int* page_tab, int max_page_rows, void* map16,
                               unsigned char* mask, float* thresholds, unsigned int* hist_scratch, float text_threshold,
                               float low_text, void* stream) {
  if (!logits || !chunk_tab || !page_tab || !map16 || !mask || !thresholds || !hist_scratch) {
    set_error("sb_det_text_front_stitched: null argument");
    return -1;
  }
  if (n_chunks < 0 || n_pages < 0 || max_page_rows < 0) { set_error("sb_det_text_front_stitched: negative count"); return -1; }
  return det_text_front(dtype, logits, n_labels, n_chunks, hs, ws, HO, WO, map16, mask, thresholds, hist_scratch, text_threshold,
                        low_text, static_cast<cudaStream_t>(stream), chunk_tab, n_pages, page_tab, max_page_rows);
}

int sb_det_page_resize(const unsigned char* pages, unsigned char* scratch, unsigned char* out, const long long* jobs,
                       const int* tables, int n_steps, const int* step_jobs, const long long* step_max_px, void* stream) {
  if (!pages || !out || !jobs || !tables || (n_steps > 0 && (!step_jobs || !step_max_px))) {
    set_error("sb_det_page_resize: null argument");
    return -1;
  }
  return det_page_resize(pages, scratch, out, jobs, tables, n_steps, step_jobs, step_max_px, static_cast<cudaStream_t>(stream));
}

int sb_det_text_boxes(int dtype, const void* map16, const unsigned char* mask, const float* thresholds, int B, int H, int W,
                      int max_boxes, int max_points, void* scratch, size_t scratch_bytes, int* count, int* overflow, int* box,
                      float* peak, int* points, void* stream) {
  if (!map16 || !mask || !thresholds || !scratch || !count || !overflow || !box || !peak || !points) {
    set_error("sb_det_text_boxes: null argument");
    return -1;
  }
  if (B <= 0 || H <= 0 || W <= 0 || max_boxes <= 0 || max_points < 2) {
    set_error("sb_det_text_boxes: non-positive size (B=%d H=%d W=%d max_boxes=%d max_points=%d)", B, H, W, max_boxes,
              max_points);
    return -1;
  }
  const size_t need = det_text_boxes_scratch_bytes(B, H, W, max_points);
  if (scratch_bytes < need) {
    set_error("sb_det_text_boxes: scratch of %zu bytes, %zu needed", scratch_bytes, need);
    return -1;
  }
  return det_text_boxes(dtype, map16, mask, thresholds, B, H, W, max_boxes, max_points, scratch, count, overflow, box, peak,
                        points, static_cast<cudaStream_t>(stream));
}

int sb_det_debug_copy(sb_det_engine* e, int buf, void* dst, size_t bytes, void* stream) {
  if (!e || buf < 0 || buf >= (int)e->bufs.size()) { set_error("sb_det_debug_copy: bad buffer"); return -1; }
  cudaError_t ce = cudaMemcpyAsync(dst, e->bufs[buf], bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
  if (ce != cudaSuccess) { cudaGetLastError(); set_error("sb_det_debug_copy: %s", cudaGetErrorString(ce)); return -2; }
  return 0;
}

int sb_conv2d_nhwc(int dtype, const void* in, const void* weight, const float* bias, const void* residual, void* out,
                   int n_img, int H, int W, int Cin, int Cout, int ksize, int stride, int pad, int act, void* stream) {
  ConvArgs a;
  a.dtype = dtype; a.in = in; a.weight = weight; a.bias = bias; a.residual = residual; a.out = out; a.n_img = n_img;
  a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.ksize = ksize; a.stride = stride; a.pad = pad; a.act = act;
  return conv_igemm(a, static_cast<cudaStream_t>(stream));
}

int sb_dwconv_nhwc(int dtype, const void* in, const void* w, const float* bias, void* out, int B, int H, int W, int C,
                   int ks, int stride, int pad, int act, void* stream) {
  return det_dwconv(dtype, in, w, bias, out, B, H, W, C, ks, stride, pad, act, static_cast<cudaStream_t>(stream));
}

int sb_det_stem_conv(int dtype, const void* in, int in_f32, const float* w, const float* bias, void* out, int B, int H, int W,
                     int cout, void* stream) {
  if (!in || !w || !bias || !out) { set_error("sb_det_stem_conv: null argument"); return -1; }
  return det_stem_conv(dtype, in, in_f32, w, bias, out, B, H, W, cout, static_cast<cudaStream_t>(stream));
}

int sb_det_fmb_fused(int dtype, const void* in, const void* w1, const float* bias1, const void* w2, const float* bias2,
                     const void* residual, void* out, int n_img, int H, int W, int Cin, int Cmid, int Cout, int stride,
                     void* stream) {
  if (!in || !w1 || !bias1 || !w2 || !bias2 || !out) { set_error("sb_det_fmb_fused: null argument"); return -1; }
  return fmb_fused(dtype, in, w1, bias1, w2, bias2, residual, out, n_img, H, W, Cin, Cmid, Cout, stride,
                   static_cast<cudaStream_t>(stream));
}

// the source list of an UPCAT op: 1..4 non-null maps with their sizes and channel offsets
static bool upcat_sources_ok(const void* const* srcs, const int* hs, const int* ws, const int* ch_off, int n_src) {
  if (!srcs || !hs || !ws || !ch_off || n_src < 1 || n_src > 4) return false;
  for (int i = 0; i < n_src; ++i)
    if (!srcs[i]) return false;
  return true;
}

int sb_det_head_fused(int dtype, const void* const* srcs, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                      const void* fuse_w, const float* fuse_bias, const void* cls_w, const void* cls_b, void* logits, int B,
                      int HO, int WO, void* stream) {
  if (!upcat_sources_ok(srcs, hs, ws, ch_off, n_src) || !fuse_w || !fuse_bias || !cls_w || !cls_b || !logits) {
    set_error("sb_det_head_fused: null argument or bad source count");
    return -1;
  }
  return det_head_fused(dtype, srcs, hs, ws, ch_off, n_src, CS, fuse_w, fuse_bias, cls_w, cls_b, logits, B, HO, WO,
                        static_cast<cudaStream_t>(stream));
}

int sb_det_upsample_cat(int dtype, const void* const* srcs, const int* hs, const int* ws, const int* ch_off, int n_src, int CS,
                        void* dst, int B, int HO, int WO, void* stream) {
  if (!upcat_sources_ok(srcs, hs, ws, ch_off, n_src) || !dst) {
    set_error("sb_det_upsample_cat: null argument or bad source count");
    return -1;
  }
  return det_upsample_cat(dtype, srcs, hs, ws, ch_off, n_src, CS, dst, B, HO, WO, static_cast<cudaStream_t>(stream));
}

int sb_det_classifier(int dtype, const void* x, const void* w, const void* b, void* out, long long P, int C, int HW, int n_out,
                      void* stream) {
  if (!x || !w || !b || !out) { set_error("sb_det_classifier: null argument"); return -1; }
  return det_classifier(dtype, x, w, b, out, P, C, HW, n_out, static_cast<cudaStream_t>(stream));
}

int sb_gemm_grouped(int dtype, const void* A, int lda, int a_cols, const void* W, int ldw, void* C, int ldc, int M, int N,
                    int Kpad, int group_k, int group_n, void* stream) {
  GemmArgs g;
  g.dtype = dtype; g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = Kpad;
  g.group_k = group_k; g.group_n = group_n; g.a_cols = a_cols;
  return gemm_launch(g, static_cast<cudaStream_t>(stream));
}

int sb_lite_mla(int dtype, const void* qkv_a, const void* qkv_b, void* out, int B, int HW, int heads, int dim, float eps,
                void* stream) {
  return det_lite_mla(dtype, qkv_a, qkv_b, out, B, HW, heads, dim, eps, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
