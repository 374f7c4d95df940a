"""Layout analysis of mixed-size pages: layout_pages (device preprocessing, encoder, the decode loop with the header/footer rule
and early exit, host post-processing) against the host path it replaces (cv2 cubic resize + normalisation of every page / slice
on the host, then layout_greedy's fixed 100-step loop), over the same seeded pages at B = 32, fp16, default layout config, with
synthetic weights.  The page mix: A4 at 96 and 192 dpi, and pages above 1500 px on both axes, which are sliced.  Prints one
JSON line with the card name and power limit, pages/s for both paths, the time split and the mean steps run."""
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


def _pages(n: int, seed: int):
    rng = np.random.default_rng(seed)
    kinds = [(794, 1123), (1588, 2246), (1800, 2400)]        # A4 at 96 / 192 dpi, and a page sliced in two
    out = []
    for i in range(n):
        w, h = kinds[i % 3]
        img = np.full((h, w, 3), 245, np.uint8)
        for _ in range(30):                                  # dark blocks on a light page
            x, y = int(rng.integers(0, w - 50)), int(rng.integers(0, h - 20))
            img[y:y + int(rng.integers(8, 200)), x:x + int(rng.integers(40, 600))] = int(rng.integers(0, 120))
        out.append(img)
    return out


def _host_path(eng, pages, B):
    import cv2

    from surya_b200 import layout_pages as LP
    from surya_b200.layout import layout_greedy

    H, W = eng.cfg.encoder.image_size
    px = []
    for p in pages:
        for x0, y0, sw, sh, _, _ in LP.slice_rects(p.shape[1], p.shape[0]):
            r = cv2.resize(p[y0:y0 + sh, x0:x0 + sw], (W, H), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1)
            r = (r.astype(np.float64) * (1 / 255)).astype(np.float32)
            px.append(torch.from_numpy((r - np.float32(0.5)) / np.float32(0.5)).to(torch.float16))
    for b0 in range(0, len(px), B):
        tok, bbox, cls, _ = layout_greedy(eng, torch.stack(px[b0:b0 + B]).cuda(), eng.cfg.decoder.max_boxes)
        tok.cpu()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=48)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()

    from surya_b200 import layout_pages as LP
    from surya_b200.config import layout_default
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_layout_state_dict, swin_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("bench_layout_pages needs a CUDA device")
    B = 32
    cfg = layout_default()
    # synthetic weights with the class rows of Text and PageHeader scaled up, so that every slice has boxes (the reference's
    # slice join raises on a first slice without any) and the header/footer rule runs
    sdd = adetr_layout_state_dict(cfg.decoder, 0)
    w = sdd["lm_head.weight"].clone()
    w[1 + cfg.decoder.special_token_count] *= 6.0
    w[10 + cfg.decoder.special_token_count] *= 3.0
    sdd["lm_head.weight"] = w
    eng = LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), sdd, torch.float16, max_batch=B)
    pages = _pages(args.pages, 0)
    res = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                 text=True).stdout.strip(), "pages": len(pages), "batch": B,
           "slices": sum(len(LP.slice_rects(p.shape[1], p.shape[0])) for p in pages)}
    LP.layout_pages(eng, pages, batch_size=B)                # warm-up: graphs, tap tables
    _host_path(eng, pages[:B], B)
    dev_t, host_t, split, steps = [], [], {}, []
    for _ in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run = LP.layout_pages(eng, pages, batch_size=B)
        dev_t.append(time.perf_counter() - t0)
        for k, v in run.timing.items():
            split[k] = split.get(k, 0.0) + v / args.iters
        steps += run.steps_run
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _host_path(eng, pages, B)
        torch.cuda.synchronize()
        host_t.append(time.perf_counter() - t0)
    res.update({"layout_pages_pages_per_s": len(pages) / min(dev_t), "host_preprocess_greedy_pages_per_s": len(pages) / min(host_t),
                "layout_pages_split_ms": {k: round(v * 1e3, 2) for k, v in split.items()},
                "mean_steps_run": float(np.mean(steps)), "max_steps": cfg.decoder.max_boxes})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
