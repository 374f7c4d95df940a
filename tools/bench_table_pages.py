"""Table recognition of pages: table_pages (layout, then the tables cropped and preprocessed on the device out of the resident
high-resolution page, both passes, geometry) against the same flow with the crop, cv2 cubic resize and normalisation on the
host feeding float32 pixel values to TableRecRunner.run.  A4 pages at 96 dpi for layout with 192-dpi copies for the crops,
default layout and table configs, fp16, synthetic weights with the layout's Table class row scaled up so that pages have
tables.  The two flows alternate in one process.  Prints one JSON line: the card, its power limit and maximum SM clock,
pages/s and tables/s of both flows, the per-phase times, the workload (tables, rows, columns, decode steps) and whether the
two flows' results are identical."""
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
    """(96-dpi page, 192-dpi copy) pairs: light pages with a few ruled blocks; the copy is the page upscaled 2x."""
    rng = np.random.default_rng(seed)
    lo, hi = [], []
    for _ in range(n):
        w, h = 794, 1123
        img = np.full((h, w, 3), 245, np.uint8)
        for _ in range(int(rng.integers(1, 4))):
            x, y = int(rng.integers(20, w - 320)), int(rng.integers(20, h - 260))
            bw, bh = int(rng.integers(200, 300)), int(rng.integers(120, 240))
            img[y:y + bh, x:x + bw] = 250
            img[y:y + bh:int(rng.integers(16, 30)), x:x + bw] = 40
            img[y:y + bh, x:x + bw:int(rng.integers(40, 90))] = 40
        lo.append(img)
        hi.append(np.ascontiguousarray(np.repeat(np.repeat(img, 2, 0), 2, 1)))
    return lo, hi


def _host_flow(tab, lay, pages, highres, batch, max_boxes):
    """layout_pages, the crop plan, then per table PIL's crop (zero fill past the page), cv2 INTER_CUBIC and the normalisation
    in float32 on the host, TableRecRunner.run and table_results."""
    import cv2

    from surya_b200 import table_pages as TP
    from surya_b200.layout_pages import layout_pages
    from surya_b200.table_rec import TableRecRunner, table_results

    t = {}
    t0 = time.perf_counter()
    layout = layout_pages(lay, pages, batch).results
    plan = TP.plan_tables(layout, [(p.shape[1], p.shape[0]) for p in pages], [(p.shape[1], p.shape[0]) for p in highres])
    t1 = time.perf_counter()
    H, W = tab.cfg.encoder.image_size
    px = []
    for tp in plan:
        page = highres[tp.page]
        x0, y0, x1, y1 = tp.crop
        crop = np.zeros((y1 - y0, x1 - x0, 3), np.uint8)
        sx0, sy0, sx1, sy1 = max(x0, 0), max(y0, 0), min(x1, page.shape[1]), min(y1, page.shape[0])
        crop[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = page[sy0:sy1, sx0:sx1]
        r = cv2.resize(crop, (W, H), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1)
        r = (r.astype(np.float64) * (1 / 255)).astype(np.float32)
        px.append(torch.from_numpy((r - np.float32(0.5)) / np.float32(0.5)))
    t2 = time.perf_counter()
    results = [[] for _ in pages]
    if plan:
        runner = TableRecRunner(tab, batch, max_boxes)
        out = runner.run(torch.stack(px), [tp.size for tp in plan])
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        res = [r for b in out for r in table_results(*b)]
        for tp, r in zip(plan, res):
            results[tp.page].append(r)
    else:
        t3 = time.perf_counter()
    t4 = time.perf_counter()
    t.update(layout=t1 - t0, host_preprocess=t2 - t1, model=t3 - t2, geometry=t4 - t3)
    return results, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=32)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--max-boxes", type=int, default=150)
    args = ap.parse_args()

    from surya_b200 import table_pages as TP
    from surya_b200.config import layout_default, table_default
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_layout_state_dict, adetr_table_state_dict, swin_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("bench_table_pages needs a CUDA device")
    B = 16
    lcfg, tcfg = layout_default(), table_default()
    sdd = adetr_layout_state_dict(lcfg.decoder, 0)
    w = sdd["lm_head.weight"].clone()
    w[13 + lcfg.decoder.special_token_count] *= 6.0               # Table
    sdd["lm_head.weight"] = w
    lay = LayoutEngine(lcfg, swin_state_dict(lcfg.encoder, 0), sdd, torch.float16, max_batch=B)
    tab = LayoutEngine(tcfg, swin_state_dict(tcfg.encoder, 0), adetr_table_state_dict(tcfg.decoder, 0), torch.float16, max_batch=B,
                       max_rows=512, max_prefill_tokens=4096)
    pages, highres = _pages(args.pages, 0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()

    def device():
        return TP.table_pages(tab, pages, lay, highres_pages=highres, batch_size=B, layout_batch_size=B, max_boxes=args.max_boxes)

    run = device()                                            # warm-up: graphs, tap tables
    _host_flow(tab, lay, pages, highres, B, args.max_boxes)
    dev_t, host_t, dev_split, host_split = [], [], {}, {}
    for _ in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run = device()
        dev_t.append(time.perf_counter() - t0)
        for k, v in list(run.timing.items()) + [("layout", sum(run.layout_timing.values()))]:
            dev_split[k] = dev_split.get(k, 0.0) + v / args.iters
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host, ht = _host_flow(tab, lay, pages, highres, B, args.max_boxes)
        host_t.append(time.perf_counter() - t0)
        for k, v in ht.items():
            host_split[k] = host_split.get(k, 0.0) + v / args.iters
    tables = [r for page in run.results for r in page]
    same = [[r.to_dict() for r in p] for p in run.results] == [[r.to_dict() for r in p] for p in host]
    print(json.dumps({
        "gpu": gpu, "pages": len(pages), "page_px": [794, 1123], "highres_px": [1588, 2246], "batch": B, "dtype": "fp16",
        "tables": len(tables), "tables_per_page": [len(p) for p in run.results], "rows": sum(len(r.rows) for r in tables),
        "cols": sum(len(r.cols) for r in tables), "decode_passes": len(run.steps_run), "decode_steps": sum(run.steps_run),
        "device_pages_per_s": len(pages) / min(dev_t), "device_tables_per_s": len(tables) / min(dev_t),
        "host_prep_pages_per_s": len(pages) / min(host_t), "host_prep_tables_per_s": len(tables) / min(host_t),
        "device_split_ms": {k: round(v * 1e3, 2) for k, v in dev_split.items()},
        "host_prep_split_ms": {k: round(v * 1e3, 2) for k, v in host_split.items()},
        "results_identical": same}))


if __name__ == "__main__":
    main()
