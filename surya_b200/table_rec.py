"""Table recognition, both decode passes on the device: TableRecPredictor.batch_table_recognition
(surya/table_rec/__init__.py:134-236) up to the host geometry.

  * TableRecRunner      per image batch: encoder once, cross K/V held once per table (LayoutEngine.cross_kv), the row/column
                        pass, the row queries / columns / cell prompts on the host, then the cell pass of every predicted row
                        against its table's held K/V (LayoutEngine.decode_rows: batched prompt prefill, early exit).  Returns
                        the arguments the reference hands to decode_batch_predictions (:233), so a caller finishes with the
                        reference's own geometry: predictor.decode_batch_predictions(*batch, LabelShaper()).
  * query_label / box_polygon / prompt builders: the processor's and shaper's host arithmetic (processor.py:29-82,
                        shaper.py:12-52, 83-142), float64 like the reference, truncated to int64 like torch.tensor(.., long).

Works over any engine with LayoutEngine's surface (encode, cross_kv, decode_rows, cfg, max_batch, max_rows, s_max).  No import
of the reference and none of oracle/.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

BOX_DIM = 1024
CATEGORY_TABLE, CATEGORY_ROW, CATEGORY_COLUMN = 4, 1, 2       # surya/table_rec/model/config.py ID_TO_CATEGORY


def resize_polygon(polygon, orig_size, new_size):
    """SuryaTableRecProcessor.resize_polygon (processor.py:29-46), on a copy."""
    w_scaler = new_size[0] / orig_size[0]
    h_scaler = new_size[1] / orig_size[1]
    out = []
    for x, y in polygon:
        x, y = x * w_scaler, y * h_scaler
        out.append([min(max(x, 0), new_size[0]), min(max(y, 0), new_size[1])])
    return out


def box_polygon(box, skew_scaler=BOX_DIM // 2, skew_min=.001):
    """LabelShaper.convert_bbox_to_polygon (shaper.py:114-142)."""
    cx, cy, width, height = box[0], box[1], box[2], box[3]
    x1, y1, x2, y2 = cx - width / 2, cy - height / 2, cx + width / 2, cy + height / 2
    skew_x = math.floor((box[4] - skew_scaler) / 2)
    skew_y = math.floor((box[5] - skew_scaler) / 2)
    if abs(skew_x) < skew_min:
        skew_x = 0
    if abs(skew_y) < skew_min:
        skew_y = 0
    p = [x1 - skew_x, y1 - skew_y, x2 - skew_x, y1 + skew_y, x2 + skew_x, y2 + skew_y, x1 + skew_x, y2 - skew_y]
    return [[p[2 * i], p[2 * i + 1]] for i in range(4)]


def query_label(polygon, category: int, is_header: int, special: int) -> List[int]:
    """LabelShaper.convert_polygons_to_bboxes + dict_to_labels (shaper.py:83-112, 12-52) for one query item with colspan 0
    and merges 0, then torch.tensor(..., dtype=long)'s truncation."""
    (x1, y1), (x2, y2), (x3, y3), (x4, y4) = np.clip(polygon, 0, BOX_DIM)
    bbox = [(x1 + x2 + x3 + x4) / 4, (y1 + y2 + y3 + y4) / 4, (x2 + x3) / 2 - (x1 + x4) / 2, (y3 + y4) / 2 - (y2 + y1) / 2,
            (x3 + x4) / 2 - (x1 + x2) / 2 + BOX_DIM // 2, (y2 + y3) / 2 - (y1 + y4) / 2 + BOX_DIM // 2]
    bbox = [min(max(v, 0), BOX_DIM) for v in bbox]
    return [int(v) for v in bbox] + [category + special, special, 0, is_header + special]


def table_query_prompt(image_sizes: Sequence[Tuple[int, int]], cfg) -> torch.Tensor:
    """The row/column-pass prompt SuryaTableRecProcessor builds for whole images (processor.py:61-76):
    [bos x10], the whole-image 'Table' query, [query_end x10] -> int64 [n, 3, 10]."""
    rows = []
    for w, h in image_sizes:
        poly = resize_polygon([[0, 0], [w, 0], [w, h], [0, h]], (w, h), (BOX_DIM, BOX_DIM))
        rows.append([[cfg.bos_token_id] * 10, query_label(poly, CATEGORY_TABLE, 0, cfg.special_token_count),
                     [cfg.query_end_token_id] * 10])
    return torch.tensor(rows, dtype=torch.long)


def cell_prompts(row_items: List[dict], columns: List[dict], cfg) -> torch.Tensor:
    """Cell-pass prompts (processor.py:65-84 with convert_images=False): per row [bos], the row query, [query_end], then the
    label of every column -> int64 [rows, 3 + len(columns), 10]."""
    sp = cfg.special_token_count
    col_labels = [query_label(c["polygon"], c["category"], c["is_header"], sp) for c in columns]
    out = [[[cfg.bos_token_id] * 10, query_label(r["polygon"], r["category"], r["is_header"], sp), [cfg.query_end_token_id] * 10]
           + col_labels for r in row_items]
    return torch.tensor(out, dtype=torch.long).reshape(len(row_items), 3 + len(columns), 10)


def step_budget(max_boxes: int, q_len: int) -> int:
    """Decoder calls of one inference_loop (table_rec/__init__.py:59-125): the first call consumes the whole prompt of the token
    budget, every later call one token."""
    return max(1, max_boxes + 1 - q_len)


def pass_predictions(tok: torch.Tensor, bbox: torch.Tensor, done: torch.Tensor, n_steps: int, special: int) -> List[List[Dict]]:
    """Per-row prediction dicts of one inference_loop from the step histories (tok [n, rows, 10], bbox [n, rows, 6], done
    [n, rows], host tensors, n = steps that ran): a row keeps its steps before its first done step; when every row is done the
    loop breaks at the step where the last one became done (:98-122)."""
    n, rows = tok.shape[0], tok.shape[1]
    d = done.bool()
    first = [int(torch.nonzero(d[:, j])[0]) if bool(d[:, j].any()) else None for j in range(rows)]
    if any(f is None for f in first) and n < n_steps:
        raise _lib.SuryaB200Error(f"decode stopped after {n} of {n_steps} steps with rows still running")
    box = (bbox.float() * BOX_DIM).tolist()
    t = tok.tolist()
    out = []
    for j in range(rows):
        end = n if first[j] is None else first[j]
        out.append([{"bbox": box[s][j], "category": t[s][j][6] - special, "merges": t[s][j][7] - special,
                     "colspan": t[s][j][8], "is_header": t[s][j][9] - special} for s in range(end)])
    return out


class TableRecRunner:
    """TableRecPredictor.batch_table_recognition on the device up to decode_batch_predictions.

    One intended difference: for an image batch in which no table row is predicted the reference fails (torch.stack of an
    empty list, table_rec/__init__.py:220); here that batch gets empty cell predictions."""

    def __init__(self, engine, batch_size: int, max_boxes: int = 150):
        if batch_size < 1 or batch_size > engine.max_batch:
            raise _lib.SuryaB200Error(f"batch_size {batch_size} needs an engine with max_batch >= {batch_size} "
                                      f"(engine has {engine.max_batch})")
        self.engine, self.batch_size, self.max_boxes = engine, int(batch_size), int(max_boxes)
        self.cfg = engine.cfg.decoder
        self.trace: Optional[list] = None     # set to a list to keep every pass's inputs and step histories (host copies)

    def _decode(self, row_table: List[int], prompt: torch.Tensor) -> List[List[Dict]]:
        n_steps = step_budget(self.max_boxes, prompt.shape[1])
        tok, bbox, heads, done = self.engine.decode_rows(row_table, prompt, n_steps)
        tok, bbox, done = tok.cpu(), bbox.cpu(), done.cpu()
        if self.trace is not None:
            self.trace.append({"row_table": list(row_table), "prompt": prompt.cpu(), "n_steps": n_steps, "tok": tok, "bbox": bbox,
                               "heads": [h.cpu() for h in heads], "done": done})
        return pass_predictions(tok, bbox, done, n_steps, self.cfg.special_token_count)

    def run(self, pixel_values: torch.Tensor, image_sizes: Sequence[Tuple[int, int]]):
        """pixel_values float32 NCHW as SuryaTableRecProcessor makes them; image_sizes the original (w, h) of every image.
        Returns one (rowcol_predictions, cell_predictions, idx_map, orig_sizes) per image batch of batch_size images."""
        if pixel_values.shape[0] != len(image_sizes):
            raise _lib.SuryaB200Error(f"{pixel_values.shape[0]} images but {len(image_sizes)} sizes")
        eng, cfg = self.engine, self.cfg
        out = []
        for i in range(0, len(image_sizes), self.batch_size):
            sizes = [tuple(int(v) for v in s) for s in image_sizes[i:i + self.batch_size]]
            n = len(sizes)
            enc = eng.encode(pixel_values[i:i + n])
            eng.cross_kv(enc)
            if self.trace is not None:
                self.trace.append({"enc": enc.float().cpu()})
            rowcol = self._decode(list(range(n)), table_query_prompt(sizes, cfg))
            row_items, columns, idx_map = [], [], []
            for j, preds in enumerate(rowcol):
                for p in preds:
                    item = {"polygon": box_polygon(p["bbox"]), "category": p["category"], "is_header": int(p["is_header"] == 1)}
                    if p["category"] == CATEGORY_ROW:
                        row_items.append(item)
                        idx_map.append(j)
                    elif p["category"] == CATEGORY_COLUMN:
                        columns.append(item)
            cells: List[List[Dict]] = []
            if row_items:
                prompts = cell_prompts(row_items, columns, cfg)
                for r0 in range(0, len(row_items), eng.max_rows):
                    cells.extend(self._decode(idx_map[r0:r0 + eng.max_rows], prompts[r0:r0 + eng.max_rows]))
            out.append((rowcol, cells, idx_map, sizes))
        return out
