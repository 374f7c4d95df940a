"""Table recognition, both passes, 16 synthetic 768x768 pages through the default table config in fp16, batch_size 16 (needs a
CUDA device).  Two flows alternate in one process, each timed with CUDA events and a synchronise per phase:

  * device flow  TableRecRunner's steps: encoder, cross_kv once per table, the row/column pass and the cell pass through
                 LayoutEngine.decode_rows (shared K/V, batched prompt prefill, early exit)
  * ref shape    what TableRecPredictor does with the existing entry points: the row/column pass and then every row with its own
                 copy of its table's encoder states through LayoutEngine.run_loop in chunks of max_batch, the cell prompt fed
                 position by position, the full step budget (no early exit)

Reports per-phase milliseconds, pages/s, the workload (rows, columns, cell-prompt length, steps run: random weights set it),
the number of rows whose predictions differ between the flows, and the card, power limit and maximum SM clock.  Prints one JSON
line."""
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main(n_pages=16, runs=3, max_boxes=150):
    from bench import gpu_info
    from surya_b200.config import table_default
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_table_state_dict, layout_synthetic_pages, swin_state_dict
    from surya_b200.table_rec import (CATEGORY_COLUMN, CATEGORY_ROW, TableRecRunner, box_polygon, cell_prompts, pass_predictions,
                                      step_budget, table_query_prompt)

    if not torch.cuda.is_available():
        raise SystemExit("bench_table_flow needs a CUDA device")
    cfg = table_default()
    d = cfg.decoder
    eng = LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), adetr_table_state_dict(d, 0), dtype=torch.float16, max_batch=16,
                       max_rows=512, max_prefill_tokens=4096)
    x = layout_synthetic_pages(n_pages, cfg.encoder.image_size, seed=4).cuda()
    sizes = [(768, 768)] * n_pages
    sp = d.special_token_count
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def split(rowcol):
        rows, cols, idx = [], [], []
        for j, preds in enumerate(rowcol):
            for p in preds:
                item = {"polygon": box_polygon(p["bbox"]), "category": p["category"], "is_header": int(p["is_header"] == 1)}
                if p["category"] == CATEGORY_ROW:
                    rows.append(item)
                    idx.append(j)
                elif p["category"] == CATEGORY_COLUMN:
                    cols.append(item)
        return rows, cols, idx

    def device_flow():
        t = [ev() for _ in range(5)]
        t[0].record()
        enc = eng.encode(x)
        eng.cross_kv(enc)
        t[1].record()
        runner = TableRecRunner(eng, 16, max_boxes)
        runner.trace = []
        rowcol = runner._decode(list(range(n_pages)), table_query_prompt(sizes, d))
        t[2].record()
        rows, cols, idx = split(rowcol)
        prompts = cell_prompts(rows, cols, d)
        t[3].record()
        cells = []
        for r0 in range(0, len(rows), eng.max_rows):
            cells.extend(runner._decode(idx[r0:r0 + eng.max_rows], prompts[r0:r0 + eng.max_rows]))
        t[4].record()
        torch.cuda.synchronize()
        steps = [r["tok"].shape[0] for r in runner.trace]
        return [t[i].elapsed_time(t[i + 1]) for i in range(4)], rowcol, cells, (rows, cols, prompts, steps)

    def reference_shape():
        t = [ev() for _ in range(5)]
        t[0].record()
        enc = eng.encode(x)
        t[1].record()
        prompt = table_query_prompt(sizes, d)
        n = step_budget(max_boxes, prompt.shape[1])
        tok, bbox, _, done = eng.run_loop(enc, prompt.cuda(), n)
        rowcol = pass_predictions(tok.cpu(), bbox.cpu(), done.cpu(), n, sp)
        t[2].record()
        rows, cols, idx = split(rowcol)
        prompts = cell_prompts(rows, cols, d)
        t[3].record()
        cells = []
        n = step_budget(max_boxes, prompts.shape[1])
        for r0 in range(0, len(rows), eng.max_batch):
            sel = torch.tensor(idx[r0:r0 + eng.max_batch], device=enc.device)
            tok, bbox, _, done = eng.run_loop(enc[sel], prompts[r0:r0 + eng.max_batch].cuda(), n)
            cells.extend(pass_predictions(tok.cpu(), bbox.cpu(), done.cpu(), n, sp))
        t[4].record()
        torch.cuda.synchronize()
        return [t[i].elapsed_time(t[i + 1]) for i in range(4)], rowcol, cells

    device_flow()                   # warm-up: kernels, graphs, allocator
    reference_shape()
    dev_ms, ref_ms = [], []
    for _ in range(runs):
        ms, rc_d, cells_d, work = device_flow()
        dev_ms.append(ms)
        ms, rc_r, cells_r = reference_shape()
        ref_ms.append(ms)
    rows, cols, prompts, steps = work
    def differ(a, b):       # everything but the bbox floats, which the batched prefill may round differently
        strip = lambda t: [(p["category"], p["merges"], p["colspan"], p["is_header"], [int(v) for v in p["bbox"]]) for p in t]
        return strip(a) != strip(b)

    def bbox_err(xs, ys):
        return max([abs(u - v) for a, b in zip(xs, ys) if not differ(a, b) for p, q in zip(a, b) for u, v in zip(p["bbox"], q["bbox"])],
                   default=0.0)

    diff_rowcol = sum(differ(a, b) for a, b in zip(rc_d, rc_r))
    diff_cells = sum(differ(a, b) for a, b in zip(cells_d, cells_r)) + abs(len(cells_d) - len(cells_r))
    max_bbox = max(bbox_err(rc_d, rc_r), bbox_err(cells_d, cells_r))
    phases = ("encoder", "rowcol_pass", "host_prompt_build", "cell_pass")

    def summary(all_ms):
        tot = [sum(m) for m in all_ms]
        return {"ms": {p: [round(m[i], 2) for m in all_ms] for i, p in enumerate(phases)},
                "total_ms": [round(v, 2) for v in tot], "pages_per_s": [round(n_pages * 1e3 / v, 2) for v in tot]}

    print(json.dumps({"bench": "table_flow", "gpu": gpu_info(0), "pages": n_pages, "batch_size": 16, "dtype": "fp16",
                      "config": "table_default", "max_boxes": max_boxes,
                      "workload": {"rows": len(rows), "columns": len(cols), "cell_prompt_len": int(prompts.shape[1]) if len(rows) else 0,
                                   "steps_run_per_pass": steps,
                                   "step_budget": [step_budget(max_boxes, 3), step_budget(max_boxes, int(prompts.shape[1]) if len(rows) else 3)]},
                      "device_flow": summary(dev_ms), "reference_shape": summary(ref_ms),
                      "rows_differing": {"rowcol_tables": diff_rowcol, "cell_rows": diff_cells},
                      "max_bbox_diff_of_equal_rows": round(max_bbox, 4)}))


if __name__ == "__main__":
    main()
