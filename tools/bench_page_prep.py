"""Device page preparation against PIL on the host: per-page time of sb_det_page_resize (one page per launch chain, CUDA events)
for 816x1056, 1632x2112 and 2550x3300 pages into the processor size, PIL's thumbnail + resize for the same pages on one host
thread, and detect_text_pages throughput over a mixed-size batch at the default detection config.  Prints one JSON line."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import numpy as np
import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--pages", type=int, default=32)
    args = ap.parse_args()
    from PIL import Image

    from surya_b200.config import det_default
    from surya_b200.detection import DetEngine, detect_text_pages
    from surya_b200.page_prep import plan_pages
    from surya_b200.synth import det_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("bench_page_prep needs a CUDA device")
    size = (1024, 1024)
    cfg = det_default()
    eng = DetEngine(cfg, det_state_dict(cfg, 0), torch.float16, max_batch=16, max_hw=size)
    rng = np.random.default_rng(0)
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                 text=True).stdout.strip()}
    fwd = torch.empty((1, 3) + size, dtype=torch.float16, device="cuda").normal_()
    for _ in range(3):
        eng.forward(fwd)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        eng.forward(fwd)
    e1.record()
    torch.cuda.synchronize()
    res["forward_ms_per_chunk_1024"] = e0.elapsed_time(e1) / args.iters
    for w, h in [(816, 1056), (1632, 2112), (2550, 3300)]:
        page = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        plan = plan_pages([(w, h)], size)
        dev = torch.from_numpy(page.ravel()).cuda()
        out = eng.page_resize(dev, plan, size)
        for _ in range(3):
            eng.page_resize(dev, plan, size, out=out)
        e0.record()
        for _ in range(args.iters):
            eng.page_resize(dev, plan, size, out=out)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / args.iters
        best = 1e9
        for _ in range(3):
            t = time.perf_counter()
            im = Image.fromarray(page)
            im.thumbnail(size, Image.Resampling.LANCZOS)
            im.resize(size, Image.Resampling.LANCZOS)
            best = min(best, time.perf_counter() - t)
        res[f"{w}x{h}"] = {"chunks": len(plan.chunks), "device_resize_ms": round(dev_ms, 4), "pil_host_ms": round(best * 1e3, 2)}
    sizes = [(816, 1056), (1632, 2112), (2550, 3300), (1275, 1650), (600, 800)]
    pages = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in (sizes * (args.pages // len(sizes) + 1))[:args.pages]]
    detect_text_pages(eng, pages[:5], size)
    torch.cuda.synchronize()
    t = time.perf_counter()
    detect_text_pages(eng, pages, size)
    torch.cuda.synchronize()
    res["detect_text_pages_mixed_pages_per_s"] = round(len(pages) / (time.perf_counter() - t), 2)
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
