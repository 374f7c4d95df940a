"""Micro-benchmark (GPU box): the recognition decode step's GEMMs that take gemm_tn_kernel's decode variant, at their real
shapes (SYN-REC, B = 256, bf16), each timed INSIDE a CUDA graph of back-to-back launches with the weights rotated over more
than L2 holds (as tools/bench_decode_parts.py does): the plain variant ("plain"; "plain heuristic" = its own tile width) and
the decode variant (decode=1; "decode table" = its own tile width) at every tile width the decode variant takes.

Prints us per launch and the algorithmic GB/s ((A + W + C (+ residual)) bytes / time), then a markdown table."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from surya_b200 import ops  # noqa: E402

DT = torch.bfloat16
B, D, Q, I2, IP, V = 256, 1280, 1920, 6848, 3424, 65792
EPS = 1e-6


def timeit(fn, n=48, reps=5):
    for _ in range(3):
        fn(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(n):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (n * reps) * 1e3


def copies(N, K, cap=24):
    n = max(3, min(cap, int(300e6 // (N * K * 2))))
    return [torch.randn(N, K, device="cuda").to(DT) * 0.03 for _ in range(n)]


def main():
    name = torch.cuda.get_device_name()
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    print(f"# {name}, power limit / max SM clock: {pl}")
    x = torch.randn(B, D, device="cuda").to(DT)
    ao = torch.randn(B, D, device="cuda").to(DT)
    qkv = torch.empty(B, Q, device="cuda", dtype=DT)
    act_o = torch.empty(B, IP, device="cuda", dtype=DT)
    xo = torch.randn(B, D, device="cuda").to(DT)
    logits = torch.empty(B, V, device="cuda", dtype=DT)
    bq = torch.randn(Q, device="cuda") * 0.02
    bv = torch.randn(V, device="cuda") * 0.02
    rs = ops.row_rstd(x, EPS)
    wq, wo, wg = copies(Q, D), copies(D, D), copies(I2, D)
    wl = copies(V, D, cap=3)

    shapes = {
        "qkv": (lambda w, i, **k: ops.gemm(x, w[i % len(w)], bias=bq, out=qkv, rms_eps=EPS, **k), wq, (B * D + Q * D + B * Q) * 2, 48),
        "o-proj": (lambda w, i, **k: ops.gemm(ao, w[i % len(w)], residual=xo, out=xo, **k), wo, (B * D + D * D + 2 * B * D) * 2, 48),
        "gate/up": (lambda w, i, **k: ops.gemm(x, w[i % len(w)], act="silu", swiglu=True, out=act_o, rms_eps=EPS, **k), wg,
                    (B * D + I2 * D + B * IP) * 2, 48),
        "lm_head": (lambda w, i, **k: ops.gemm(x, w[i % len(w)], bias=bv, out=logits, rowscale=rs, argmax_only=True, **k), wl,
                    (B * D + V * D) * 2, 12),
    }
    rows = []

    def rec(shape, variant, bn, us, nbytes):
        gbs = nbytes / (us * 1e-6) / 1e9
        rows.append((shape, variant, bn, us, gbs))
        print(f"{shape:8s} {variant:16s} bn={bn:>4} {us:8.2f} us {gbs:7.0f} GB/s", flush=True)

    for shape, (fn, ws, nbytes, n) in shapes.items():
        rec(shape, "plain heuristic", "auto", timeit(lambda i: fn(ws, i), n=n), nbytes)
        bns = (128,) if shape == "lm_head" else (32, 64, 128)
        for bn in bns:
            rec(shape, "plain", bn, timeit(lambda i: fn(ws, i, force_bn=bn), n=n), nbytes)
            rec(shape, "decode", bn, timeit(lambda i: fn(ws, i, force_bn=bn, decode=1), n=n), nbytes)
        rec(shape, "decode table", "auto", timeit(lambda i: fn(ws, i, decode=1), n=n), nbytes)
    print("\n| GEMM | variant | BN | us per launch | algorithmic GB/s |\n|---|---|---:|---:|---:|")
    for s, v, bn, us, gbs in rows:
        print(f"| {s} | {v} | {bn} | {us:.2f} | {gbs:.0f} |")


if __name__ == "__main__":
    main()
