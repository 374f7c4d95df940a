"""Micro-benchmark (GPU box): the GEMM launches of one recognition prefill at bench.py's workload (BASELINE config 2: 256 crops
of 48 x 512 -> 40 960 vision patches and 11 776 prompt tokens, SYN-REC, bf16), replayed over seeded weights and activations
of the engine's real shapes and epilogues (run_vision / run_decoder_prefill in rec_engine.cu).

Each path is one `force_bn` code of ops.gemm (0 = the launch heuristic, which is what the engine runs; 32 ... 256 = the plain
kernel at that tile width).  Every path runs each shape inside a CUDA graph of back-to-back launches; the paths alternate in
one process, `--rounds` times, and the best round per (shape, path) is kept.  The outputs of every path are compared with
torch.equal against the first path's on the same inputs (in-place residual launches start from the same residual).  One
difference from the engine: ops.gemm does not mark W as constant, so the weight prefetch before griddepcontrol.wait is off.

Prints per shape and in total: ms per prefill (launch time x launches per prefill), TFLOP/s, and, for forced tile widths, the
L2 -> SM bytes the tile plan requests (computed from the plan, not measured: every 128 x BN tile loads one 128-row A box and
one BN-row W box per 64-wide k-block), with the card's name, power limit and maximum SM clock read in the same run.
`--bench-json FILE` (a bench.py result line) adds the GEMM total against bench.py's prefill phase."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from surya_b200 import ops  # noqa: E402

DT = torch.bfloat16
NP, NT = 40960, 11776                   # vision patches, decoder prompt tokens (256 crops)
H, PD, I2, MH, Q = 1280, 592, 6848, 5120, 1920

# name, M, N, K, launches per prefill, epilogue
SHAPES = [
    ("vision patch embed", NP, H, PD, 1, ""),
    ("vision qkv", NP, 3 * H, H, 8, "bias"),
    ("vision proj", NP, H, H, 8, "bias+res"),
    ("vision gate/up", NP, I2, H, 8, "bias+swiglu"),
    ("vision down", NP, H, I2 // 2, 8, "bias+res"),
    ("merger 0", NP // 4, MH, MH, 1, "bias+gelu"),
    ("merger 2", NP // 4, H, MH, 1, "bias"),
    ("decoder qkv", NT, Q, H, 12, "bias+rowscale"),
    ("decoder o", NT, H, H, 12, "res"),
    ("decoder gate/up", NT, I2, H, 12, "rowscale+swiglu"),
    ("decoder down", NT, H, I2 // 2, 12, "res"),
]


def plan_l2_bytes(M, N, K, bn):
    """L2 -> SM bytes of the plain kernel's tile plan at a forced tile width (None for the heuristic)."""
    if bn == 0:
        return None
    return -(-M // 128) * -(-N // bn) * -(-K // 64) * (128 + bn) * 64 * 2


def make(M, N, K, epi, g):
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(DT)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(DT)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if "bias" in epi else None
    rs = torch.rand(M, device="cuda", generator=g) + 0.5 if "rowscale" in epi else None
    n_out = N // 2 if "swiglu" in epi else N
    res = (torch.randn(M, n_out, device="cuda", generator=g)).to(DT) if "res" in epi else None
    out = torch.empty(M, n_out, device="cuda", dtype=DT)
    act = "silu" if "swiglu" in epi else "gelu" if "gelu" in epi else "none"

    def run(code, dst=out):
        if res is not None:      # in place, as the engine adds the residual stream
            return ops.gemm(a, w, bias=bias, residual=dst, out=dst, force_bn=code)
        return ops.gemm(a, w, bias=bias, act=act, swiglu="swiglu" in epi, out=dst, rowscale=rs, force_bn=code)

    def fresh(code):
        dst = res.clone() if res is not None else torch.empty_like(out)
        return run(code, dst)

    if res is not None:
        out.copy_(res)
    return run, fresh


def time_graph(fn, n, reps=3):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (n * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--paths", default="auto=0,bn128=128", help="comma-separated name=force_bn")
    ap.add_argument("--bench-json", default=None)
    args = ap.parse_args()
    PATHS = {k: int(v) for k, v in (p.split("=") for p in args.paths.split(","))}
    paths = list(PATHS)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"# {gpu}", flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    best = {}
    equal = {}
    for name, M, N, K, count, epi in SHAPES:
        run, fresh = make(M, N, K, epi, g)
        ref = fresh(PATHS[paths[0]])
        for p in paths:
            equal[(name, p)] = torch.equal(fresh(PATHS[p]), ref)
        del ref
        n = max(2, min(20, int(2e12 // (2 * M * N * K))))
        for _ in range(args.rounds):
            for p in paths:
                ms = time_graph(lambda: run(PATHS[p]), n)
                best[(name, p)] = min(best.get((name, p), 1e30), ms)
        print(name, " ".join(f"{p}={best[(name, p)]:.4f}ms{'' if equal[(name, p)] else ' (DIFFERS)'}" for p in paths),
              flush=True)
        del run, fresh
        torch.cuda.empty_cache()

    print("\n| GEMM | M x N x K | per prefill | " + " | ".join(f"{p} ms (TFLOP/s)" for p in paths) +
          " | " + " | ".join(f"{p} plan L2 GB" for p in paths if PATHS[p]) + " |")
    print("|---|---|---:|" + "---:|" * (len(paths) + sum(1 for p in paths if PATHS[p])))
    tot = {p: 0.0 for p in paths}
    tot_l2 = {p: 0 for p in paths}
    flop_total = 0
    for name, M, N, K, count, epi in SHAPES:
        flop = 2.0 * M * N * K
        flop_total += flop * count
        cells = []
        for p in paths:
            ms = best[(name, p)]
            tot[p] += ms * count
            cells.append(f"{ms * count:.3f} ({flop / (ms * 1e9):.0f})")
        l2 = []
        for p in paths:
            b = plan_l2_bytes(M, N, K, PATHS[p])
            if b is not None:
                tot_l2[p] += b * count
                l2.append(f"{b * count / 1e9:.1f}")
        print(f"| {name} ({epi or 'plain'}) | {M}x{N}x{K} | x{count} | " + " | ".join(cells) + " | " + " | ".join(l2) + " |")
    print(f"| **total** | {flop_total / 1e12:.2f} TFLOP | | " +
          " | ".join(f"**{tot[p]:.2f}** ({flop_total / (tot[p] * 1e9):.0f})" for p in paths) + " | " +
          " | ".join(f"{tot_l2[p] / 1e9:.0f}" for p in paths if PATHS[p]) + " |")
    bad = [k for k, v in equal.items() if not v]
    print(f"\noutputs equal to {paths[0]}'s on every shape: {not bad}" + (f" (differ: {bad})" if bad else ""))
    if args.bench_json:
        line = [ln for ln in Path(args.bench_json).read_text().splitlines() if ln.startswith("{")][-1]
        pre = json.loads(line)["phases_ms"]["prefill(vision+decoder)"]
        print(f"GEMM total vs bench.py's prefill phase ({pre:.2f} ms): " +
              ", ".join(f"{p} {tot[p]:.2f} ms = {tot[p] / pre:.0%}" for p in paths))
    print(f"# {gpu}")
    if bad:
        sys.exit(1)


if __name__ == "__main__":
    main()
