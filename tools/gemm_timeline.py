"""In-kernel timeline of one CTA of the wgmma GEMM (globaltimer stamps): where do the microseconds of a small
decode-step GEMM go?  Usage (GPU box): python tools/gemm_timeline.py"""
import ctypes
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from surya_b200 import _lib  # noqa: E402
from surya_b200._lib import c_int, c_void_p, check, ptr, stream_ptr  # noqa: E402


def run(M, N, K, bias=True, residual=False, swiglu=False, bn=0, reps=5, label=""):
    lib = _lib.load()
    dt = torch.bfloat16
    a = torch.randn(M, K, device="cuda").to(dt)
    w = (torch.randn(N, K, device="cuda") * 0.02).to(dt)
    n_out = N // 2 if swiglu else N
    c = torch.empty(M, n_out, device="cuda", dtype=dt)
    b = torch.randn(N, device="cuda") if bias else None
    r = torch.randn(M, n_out, device="cuda").to(dt) if residual else None
    tl = torch.zeros(64, dtype=torch.int64, device="cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    best = None
    for i in range(reps):
        flush.zero_()           # evict W / A from L2 like a real decode step does between reuses
        a.add_(0)               # re-touch the activations (L2-hot, as produced by the previous kernel)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        check(lib.sb_gemm_timeline(0, ptr(a), c_int(K), ptr(w), c_int(K), ptr(c), c_int(n_out), c_int(M), c_int(N), c_int(K),
                                   ptr(b), ptr(r), c_int(n_out if residual else 0), c_int(2 if swiglu else 0),
                                   c_int(1 if swiglu else 0), c_int(bn), ptr(tl), stream_ptr()), "sb_gemm_timeline")
        e1.record()
        torch.cuda.synchronize()
        t = tl.cpu().tolist()
        best = (e0.elapsed_time(e1) * 1e3, t)
    us, t = best
    kb = (K + 63) // 64
    t0 = t[0]
    land = [(t[2 + i] - t0) / 1e3 for i in range(min(kb, 38))]
    print(f"{label} M={M} N={N} K={K} bn={bn}: event {us:.1f} us | setup {(t[1]-t0)/1e3:.2f} | k-blocks land at "
          f"{', '.join(f'{x:.2f}' for x in land[:4])} ... {land[-1]:.2f} | acc ready {(t[40]-t0)/1e3:.2f} | "
          f"epilogue done {(t[41]-t0)/1e3:.2f} | exit {(t[42]-t0)/1e3:.2f}")


if __name__ == "__main__":
    run(16, 1024, 1024, bias=False, label="tiny (layout q_proj)")
    run(256, 1920, 1280, label="qkv")
    run(256, 1280, 1280, bias=False, residual=True, label="o_proj")
    run(256, 6848, 1280, bias=False, swiglu=True, label="gate_up")
    run(256, 1280, 3424, bias=False, residual=True, label="down")
    run(256, 65792, 1280, label="lm_head")
    for bn in (32, 64, 128, 256):
        run(256, 1920, 1280, bn=bn, label=f"qkv bn={bn}")
    run(40960, 3840, 1280, label="vision qkv")
    run(40960, 1280, 3424, residual=True, label="vision down")
