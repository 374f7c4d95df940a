"""Micro-benchmark (GPU box): every kernel of one recognition decode step (SYN-REC, B = 256, bf16) timed INSIDE a CUDA graph of
back-to-back launches (PDL on, weights rotated over > L2 worth of copies), plus whole decoder-layer sequences, so the step
time can be attributed.  Writes a markdown table to stdout."""
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from surya_b200 import ops  # noqa: E402

DT = torch.bfloat16
B, D, Q, I2, IP, V = 256, 1280, 1920, 6848, 3424, 65792
NH, NKV, HD, SMAX = 16, 4, 80, 256
EPS = 1e-6
HBM_BPS = 3.35e12  # H100 SXM data sheet


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


def card():
    """The card's name and power limit: part of every number below."""
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        limit = "power limit unknown"
    return f"{torch.cuda.get_device_name(0)}, {limit}"


def main():
    rows = []
    print(f"card: {card()}", flush=True)

    def rec(name, us, note=""):
        rows.append((name, us, note))
        print(f"{name:44s} {us:8.2f} us  {note}", flush=True)

    x = torch.randn(B, D, device="cuda").to(DT)
    ao = torch.randn(B, D, device="cuda").to(DT)
    act = torch.randn(B, IP, device="cuda").to(DT)
    qkv = torch.empty(B, Q, device="cuda", dtype=DT)
    act_o = torch.empty(B, IP, device="cuda", dtype=DT)
    xo = torch.empty(B, D, device="cuda", dtype=DT)
    logits = torch.empty(B, V, device="cuda", dtype=DT)
    bq = torch.randn(Q, device="cuda") * 0.02
    bv = torch.randn(V, device="cuda") * 0.02
    rs = ops.row_rstd(x, EPS)
    wq, wo, wg, wd = copies(Q, D), copies(D, D), copies(I2, D), copies(D, IP)
    wl = copies(V, D, cap=3)
    gnorm = torch.ones(D, device="cuda", dtype=DT)

    # ---- GEMMs
    for bn in (32, 64):
        rec(f"qkv plain bn{bn}", timeit(lambda i: ops.gemm(x, wq[i % len(wq)], bias=bq, out=qkv, force_bn=bn)))
        rec(f"qkv norm-inline bn{bn}", timeit(lambda i: ops.gemm(x, wq[i % len(wq)], bias=bq, out=qkv, force_bn=bn, rms_eps=EPS)))
        rec(f"qkv norm-rowscale bn{bn}", timeit(lambda i: ops.gemm(x, wq[i % len(wq)], bias=bq, out=qkv, force_bn=bn, rowscale=rs)))
    rec("o plain (heuristic) + residual", timeit(lambda i: ops.gemm(ao, wo[i % len(wo)], residual=xo, out=xo)))
    for bn in (96, 128):
        rec(f"gate_up plain bn{bn}", timeit(lambda i: ops.gemm(x, wg[i % len(wg)], act="silu", swiglu=True, out=act_o, force_bn=bn)))
        rec(f"gate_up norm-inline bn{bn}", timeit(lambda i: ops.gemm(x, wg[i % len(wg)], act="silu", swiglu=True, out=act_o, force_bn=bn, rms_eps=EPS)))
    rec("down split-K heuristic + residual", timeit(lambda i: ops.gemm(act, wd[i % len(wd)], residual=xo, out=xo, splitk=True)))
    rec("down plain bn32 + residual", timeit(lambda i: ops.gemm(act, wd[i % len(wd)], residual=xo, out=xo, force_bn=32)))
    rec("lm_head plain bn256 (writes logits)", timeit(lambda i: ops.gemm(x, wl[i % len(wl)], bias=bv, out=logits, force_bn=256), n=12))
    rec("lm_head norm-inline + argmax only", timeit(lambda i: ops.gemm(x, wl[i % len(wl)], bias=bv, out=logits, rms_eps=EPS, argmax_only=True), n=12))
    rec("lm_head norm-rowscale + argmax only", timeit(lambda i: ops.gemm(x, wl[i % len(wl)], bias=bv, out=logits, rowscale=rs, argmax_only=True), n=12))
    rec("lm_head norm-rowscale, logits + argmax", timeit(lambda i: ops.gemm(x, wl[i % len(wl)], bias=bv, out=logits, rowscale=rs, argmax={}), n=12))

    # ---- row kernels
    rec("rmsnorm 256 x 1280", timeit(lambda i: ops.rmsnorm(x, gnorm, EPS, out=xo)))
    rec("row_rstd 256 x 1280", timeit(lambda i: ops.row_rstd(x, EPS)))

    # ---- decode attention at several cache lengths (one layer's cache, 256 slots)
    kc = torch.randn(24, B, NKV, SMAX, HD, device="cuda").to(DT)          # 24 rotating copies ~ 1 GB: KV streams from HBM
    vc = torch.randn(24, B, NKV, SMAX, HD, device="cuda").to(DT)
    slot = torch.arange(B, dtype=torch.int32, device="cuda")
    inv = (1.0 / (10000.0 ** (torch.arange(0, HD, 2, device="cuda").float() / HD))).contiguous()
    qk = torch.randn(B, Q, device="cuda").to(DT)
    # KV bytes: every row reads keys 0 .. pos of its KV heads, K and V; the floor is those bytes at the data sheet's 3.35 TB/s
    def attn_case(name, pos):
        us = timeit(lambda i: ops.decode_attn(qk, kc[i % 24], vc[i % 24], slot, pos, inv, NH, NKV, HD, HD ** -0.5, out=ao))
        nbytes = NKV * int((pos.long() + 1).sum()) * HD * 2 * 2
        floor_us = nbytes / HBM_BPS * 1e6
        rec(name, us, f"{nbytes / 1e3 / us:.0f} GB/s of KV, {us / floor_us:.2f}x the {floor_us:.2f} us floor")

    for S in (46, 110, 173):
        attn_case(f"decode_attn S={S}", torch.full((B,), S, dtype=torch.int32, device="cuda"))
    # the benchmark's decode step: s_max = 256 with ragged positions across the 256 rows
    ragged = torch.randint(46, 173, (B,), generator=torch.Generator().manual_seed(0)).to(device="cuda", dtype=torch.int32)
    attn_case("decode_attn ragged 46..172", ragged)

    # ---- one decoder layer as the engine launches it (5 kernels) and the round-1 sequence (7 kernels)
    pos = torch.full((B,), 110, dtype=torch.int32, device="cuda")

    def layer_r2(i):
        ops.gemm(x, wq[i % len(wq)], bias=bq, out=qkv, rms_eps=EPS)
        ops.decode_attn(qkv, kc[i % 24], vc[i % 24], slot, pos, inv, NH, NKV, HD, HD ** -0.5, out=ao)
        ops.gemm(ao, wo[i % len(wo)], residual=x, out=x)
        ops.gemm(x, wg[i % len(wg)], act="silu", swiglu=True, out=act_o, rms_eps=EPS)
        ops.gemm(act_o, wd[i % len(wd)], residual=x, out=x, splitk=True)

    def layer_r1(i):
        ops.rmsnorm(x, gnorm, EPS, out=xo)
        ops.gemm(xo, wq[i % len(wq)], bias=bq, out=qkv)
        ops.decode_attn(qkv, kc[i % 24], vc[i % 24], slot, pos, inv, NH, NKV, HD, HD ** -0.5, out=ao)
        ops.gemm(ao, wo[i % len(wo)], residual=x, out=x)
        ops.rmsnorm(x, gnorm, EPS, out=xo)
        ops.gemm(xo, wg[i % len(wg)], act="silu", swiglu=True, out=act_o)
        ops.gemm(act_o, wd[i % len(wd)], residual=x, out=x, splitk=True)

    x.copy_(torch.randn(B, D, device="cuda").to(DT) * 0.1)
    rec("decoder layer, round-2 sequence (5 kernels)", timeit(layer_r2, n=24))
    x.copy_(torch.randn(B, D, device="cuda").to(DT) * 0.1)
    rec("decoder layer, round-1 sequence (7 kernels)", timeit(layer_r1, n=24))
    print("\n| kernel | us in graph | note |\n|---|---:|---|")
    for n, u, note in rows:
        print(f"| {n} | {u:.2f} | {note} |")


if __name__ == "__main__":
    main()
