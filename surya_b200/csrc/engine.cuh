// surya_b200 — host scaffolding shared by the recognition, layout and detection engines: workspace arena, GEMMs over packed
// weights, the hop off the default stream and the cache of captured decode-step graphs.
#pragma once
#include "ops.cuh"

#include <array>
#include <functional>
#include <vector>

#define CK(x)                \
  do {                       \
    int rc_ = (x);           \
    if (rc_) return rc_;     \
  } while (0)

namespace sb {

inline size_t al256(size_t v) { return (v + 255) & ~size_t(255); }

// One zeroed cudaMalloc carved into buffers in declaration order, each starting on a 256-byte boundary.
class Arena {
 public:
  template <typename T>
  void add(T*& p, size_t n) {
    const size_t off = bytes_;
    bytes_ += al256(n);
    carve_.push_back([&p, off](uint8_t* base) { p = reinterpret_cast<T*>(base + off); });
  }
  cudaError_t alloc() {
    cudaError_t ce = cudaMalloc(&base_, bytes_);
    if (ce != cudaSuccess) { cudaGetLastError(); base_ = nullptr; return ce; }
    for (auto& f : carve_) f(base_);
    carve_.clear();
    cudaMemset(base_, 0, bytes_);
    return cudaSuccess;
  }
  size_t bytes() const { return bytes_; }
  ~Arena() { if (base_) cudaFree(base_); }

 private:
  uint8_t* base_ = nullptr;
  size_t bytes_ = 0;
  std::vector<std::function<void(uint8_t*)>> carve_;
};

// C = act(A W^T + bias) (+ residual) over an engine's packed weights, which are never written after packing: their tiles
// may be prefetched before the programmatic-dependency wait.  Callers set any other GemmArgs field by name.
inline GemmArgs weight_gemm(int dtype, const void* A, int lda, const void* W, int ldw, void* C, int ldc, int M, int N, int K,
                            const void* bias_f32, const void* residual = nullptr, int ldr = 0, int act = ACT_NONE,
                            int swiglu = 0) {
  GemmArgs a;
  a.dtype = dtype;
  a.A = A; a.lda = lda; a.W = W; a.ldw = ldw; a.C = C; a.ldc = ldc;
  a.M = M; a.N = N; a.K = K;
  a.bias = static_cast<const float*>(bias_f32);
  a.residual = residual; a.ldr = ldr; a.act = act; a.swiglu = swiglu;
  a.w_constant = 1;
  return a;
}

// An engine-owned stream and its two events, created on first use.
struct EngineStream {
  cudaStream_t own = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  ~EngineStream() {
    if (ev_in) cudaEventDestroy(ev_in);
    if (ev_out) cudaEventDestroy(ev_out);
    if (own) cudaStreamDestroy(own);
  }
};

// The legacy and per-thread default streams cannot be captured into a graph.  A graphed call made on one of them works on
// `st` = the engine stream, ordered after the caller's work; when the Hop goes out of scope, on every exit path, the
// caller's stream is ordered after the engine stream.  Otherwise `st` is the caller's stream.
struct Hop {
  cudaStream_t st;       // the stream to work on
  bool failed = false;   // the engine stream or its events could not be created
  Hop(EngineStream& es, cudaStream_t caller, bool graphed) : st(caller), es_(es), caller_(caller) {
    if (!graphed || (caller != nullptr && caller != cudaStreamLegacy && caller != cudaStreamPerThread)) return;
    if ((!es.own && cudaStreamCreateWithFlags(&es.own, cudaStreamNonBlocking) != cudaSuccess) ||
        (!es.ev_in && cudaEventCreateWithFlags(&es.ev_in, cudaEventDisableTiming) != cudaSuccess) ||
        (!es.ev_out && cudaEventCreateWithFlags(&es.ev_out, cudaEventDisableTiming) != cudaSuccess)) {
      cudaGetLastError();
      failed = true;
      return;
    }
    cudaEventRecord(es.ev_in, caller);
    cudaStreamWaitEvent(es.own, es.ev_in, 0);
    st = es.own;
    on_ = true;
  }
  ~Hop() {
    if (on_) { cudaEventRecord(es_.ev_out, es_.own); cudaStreamWaitEvent(caller_, es_.ev_out, 0); }
  }

 private:
  EngineStream& es_;
  cudaStream_t caller_;
  bool on_ = false;
};

// `k` calls of a decode-step body captured into one instantiated graph, cached under the pointers and batch it was captured
// with.  Launch accounting: launches made while capturing are not counted; each replay counts them once.
class StepGraph {
 public:
  using Key = std::array<const void*, 8>;
  StepGraph(const char* who, int k) : who_(who), k_(k) {}
  ~StepGraph() { invalidate(); }
  void invalidate() {
    if (exec_) cudaGraphExecDestroy(exec_);
    exec_ = nullptr;
  }
  bool hit(const Key& key, int batch) const { return exec_ && batch_ == batch && key_ == key; }
  template <typename Body>
  int capture(const Key& key, int batch, cudaStream_t st, Body&& body) {
    invalidate();
    cudaError_t ce = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) { cudaGetLastError(); set_error("%s: graph capture begin failed: %s", who_, cudaGetErrorString(ce)); return -6; }
    const long long before = launch_count();
    int rc = 0;
    for (int i = 0; i < k_ && !rc; ++i) rc = body(st);
    launches_ = launch_count() - before;
    count_launches(-launches_);  // captured, not executed
    cudaGraph_t graph = nullptr;
    ce = cudaStreamEndCapture(st, &graph);
    if (!rc && ce == cudaSuccess) ce = cudaGraphInstantiate(&exec_, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    if (rc || ce != cudaSuccess) {
      cudaGetLastError();
      exec_ = nullptr;
      set_error("%s: graph capture failed: rc=%d %s", who_, rc, cudaGetErrorString(ce));
      return -6;
    }
    key_ = key;
    batch_ = batch;
    return 0;
  }
  int replay(int n, cudaStream_t st) {
    for (int i = 0; i < n; ++i) {
      if (cudaGraphLaunch(exec_, st) != cudaSuccess) { cudaGetLastError(); set_error("%s: graph launch failed", who_); return -9; }
      count_launches(launches_);
    }
    return 0;
  }

 private:
  const char* who_;
  int k_;
  cudaGraphExec_t exec_ = nullptr;
  Key key_{};
  int batch_ = 0;
  long long launches_ = 0;
};

}  // namespace sb
