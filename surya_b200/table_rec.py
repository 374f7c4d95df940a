"""Table recognition, both decode passes on the device: TableRecPredictor.batch_table_recognition
(surya/table_rec/__init__.py:134-236) up to the host geometry.

  * TableRecRunner      per image batch: encoder once, cross K/V held once per table (LayoutEngine.cross_kv), the row/column
                        pass, the row queries / columns / cell prompts on the host, then the cell pass of every predicted row
                        against its table's held K/V (LayoutEngine.decode_rows: batched prompt prefill, early exit).  Returns
                        the arguments the reference hands to decode_batch_predictions (:233); run_batch is one image batch.
  * table_results       decode_batch_predictions (:239-387): the geometry that turns them into TableResults (TableCell /
                        TableRow / TableCol with the reference schema's fields, to_dict() = model_dump()).
  * query_label / box_polygon / prompt builders: the processor's and shaper's host arithmetic (processor.py:29-82,
                        shaper.py:12-52, 83-142), float64 like the reference, truncated to int64 like torch.tensor(.., long).

Works over any engine with LayoutEngine's surface (encode, cross_kv, decode_rows, cfg, max_batch, max_rows, s_max).  No import
of the reference and none of oracle/.
"""
from __future__ import annotations

import copy
import itertools
import math
import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .polygon import PolygonMethods

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
        self.steps_run: List[int] = []        # decode steps of every pass, in order

    def _decode(self, row_table: List[int], prompt: torch.Tensor) -> List[List[Dict]]:
        n_steps = step_budget(self.max_boxes, prompt.shape[1])
        tok, bbox, heads, done = self.engine.decode_rows(row_table, prompt, n_steps)
        tok, bbox, done = tok.cpu(), bbox.cpu(), done.cpu()
        self.steps_run.append(int(tok.shape[0]))
        if self.trace is not None:
            self.trace.append({"row_table": list(row_table), "prompt": prompt.cpu(), "n_steps": n_steps, "tok": tok, "bbox": bbox,
                               "heads": [h.cpu() for h in heads], "done": done})
        return pass_predictions(tok, bbox, done, n_steps, self.cfg.special_token_count)

    def run(self, pixel_values: torch.Tensor, image_sizes: Sequence[Tuple[int, int]]):
        """pixel_values float32 NCHW as SuryaTableRecProcessor makes them; image_sizes the original (w, h) of every image.
        Returns one (rowcol_predictions, cell_predictions, idx_map, orig_sizes) per image batch of batch_size images."""
        if pixel_values.shape[0] != len(image_sizes):
            raise _lib.SuryaB200Error(f"{pixel_values.shape[0]} images but {len(image_sizes)} sizes")
        return [self.run_batch(pixel_values[i:i + self.batch_size], image_sizes[i:i + self.batch_size])
                for i in range(0, len(image_sizes), self.batch_size)]

    def run_batch(self, pixel_values: torch.Tensor, image_sizes: Sequence[Tuple[int, int]], timing: Optional[Dict[str, float]] = None):
        """One image batch (at most batch_size images): encoder, row/column pass, cell pass.  Returns (rowcol_predictions,
        cell_predictions, idx_map, orig_sizes).  timing (optional): seconds added to its "encoder" and "passes" entries, with a
        device synchronise after each phase."""
        eng, cfg = self.engine, self.cfg
        sizes = [tuple(int(v) for v in s) for s in image_sizes]
        n = len(sizes)
        if n < 1 or n > self.batch_size or pixel_values.shape[0] != n:
            raise _lib.SuryaB200Error(f"a batch of {pixel_values.shape[0]} images with {n} sizes (batch_size {self.batch_size})")
        t0 = time.perf_counter()
        enc = eng.encode(pixel_values)
        eng.cross_kv(enc)
        if timing is not None:
            _sync(eng)
            t1 = time.perf_counter()
            timing["encoder"] = timing.get("encoder", 0.0) + t1 - t0
            t0 = t1
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
        if timing is not None:
            timing["passes"] = timing.get("passes", 0.0) + time.perf_counter() - t0
        return rowcol, cells, idx_map, sizes


def _sync(engine):
    if torch.device(engine.device).type == "cuda":
        torch.cuda.synchronize(engine.device)


# ------------------------------------------------------------------------------------------------ geometry
MERGE_UP, MERGE_DOWN, MERGE_BOTH = 1, 2, 3                   # surya/table_rec/model/config.py MERGE_KEYS
MERGE_VALUES = (MERGE_UP, MERGE_DOWN, MERGE_BOTH)


def _float_polygon(polygon) -> List[List[float]]:
    """PolygonBox's validator: a new list of float corners."""
    return [[float(x), float(y)] for x, y in polygon]


class _Polygon(PolygonMethods):
    """A bare PolygonBox."""

    def __init__(self, polygon):
        self.polygon = _float_polygon(polygon)


@dataclass
class TableCell(PolygonMethods):
    """surya/table_rec/schema.py TableCell."""
    polygon: List[List[float]]
    row_id: int
    colspan: int
    within_row_id: int
    cell_id: int
    is_header: bool
    rowspan: Optional[int] = None
    merge_up: bool = False
    merge_down: bool = False
    col_id: Optional[int] = None
    confidence: Optional[float] = None
    text_lines: Optional[List[dict]] = None

    def __post_init__(self):
        self.polygon = _float_polygon(self.polygon)

    def to_dict(self) -> dict:
        return {"polygon": [list(p) for p in self.polygon], "confidence": self.confidence, "row_id": self.row_id,
                "colspan": self.colspan, "within_row_id": self.within_row_id, "cell_id": self.cell_id, "is_header": self.is_header,
                "rowspan": self.rowspan, "merge_up": self.merge_up, "merge_down": self.merge_down, "col_id": self.col_id,
                "text_lines": self.text_lines, "bbox": self.bbox}


@dataclass
class TableRow(PolygonMethods):
    """surya/table_rec/schema.py TableRow."""
    polygon: List[List[float]]
    row_id: int
    is_header: bool
    confidence: Optional[float] = None

    def __post_init__(self):
        self.polygon = _float_polygon(self.polygon)

    def to_dict(self) -> dict:
        return {"polygon": [list(p) for p in self.polygon], "confidence": self.confidence, "row_id": self.row_id,
                "is_header": self.is_header, "bbox": self.bbox}


@dataclass
class TableCol(PolygonMethods):
    """surya/table_rec/schema.py TableCol."""
    polygon: List[List[float]]
    col_id: int
    is_header: bool
    confidence: Optional[float] = None

    def __post_init__(self):
        self.polygon = _float_polygon(self.polygon)

    def to_dict(self) -> dict:
        return {"polygon": [list(p) for p in self.polygon], "confidence": self.confidence, "col_id": self.col_id,
                "is_header": self.is_header, "bbox": self.bbox}


@dataclass
class TableResult:
    """surya/table_rec/schema.py TableResult; to_dict() is the reference's model_dump()."""
    cells: List[TableCell]
    unmerged_cells: List[TableCell]
    rows: List[TableRow]
    cols: List[TableCol]
    image_bbox: List[float]

    def to_dict(self) -> dict:
        return {"cells": [c.to_dict() for c in self.cells], "unmerged_cells": [c.to_dict() for c in self.unmerged_cells],
                "rows": [r.to_dict() for r in self.rows], "cols": [c.to_dict() for c in self.cols],
                "image_bbox": [float(v) for v in self.image_bbox]}


def _box_to_size(bbox, size) -> List[List[float]]:
    return resize_polygon(box_polygon(bbox), (BOX_DIM, BOX_DIM), size)


def table_results(rowcol, cells, idx_map, sizes) -> List[TableResult]:
    """TableRecPredictor.decode_batch_predictions (surya/table_rec/__init__.py:239-387) for one image batch, from what
    TableRecRunner.run_batch returns: columns and rows resized from BOX_DIM to the image, the spanning cells of every row, the
    row x column cells, the merge of cells across rows on a copy of the row grid, and the de-duplication by cell_id."""
    results = []
    for j, (img_predictions, size) in enumerate(zip(rowcol, sizes)):
        row_cells = [c for i, c in enumerate(cells) if idx_map[i] == j]
        rows, unmerged, columns = [], [], []
        cell_id = 0
        row_preds = [p for p in img_predictions if p["category"] == CATEGORY_ROW]
        col_preds = [p for p in img_predictions if p["category"] == CATEGORY_COLUMN]
        for z, p in enumerate(col_preds):
            columns.append(TableCol(polygon=_box_to_size(p["bbox"], size), col_id=z, is_header=p["is_header"] == 1))
        for z, p in enumerate(row_preds):
            row = TableRow(polygon=_box_to_size(p["bbox"], size), row_id=z, is_header=p["is_header"] == 1)
            rows.append(row)
            spanning = []
            for l, sc in enumerate(row_cells[z]):
                polygon = _box_to_size(sc["bbox"], size)
                colspan = max(1, int(sc["colspan"]))
                if colspan == 1 and sc["merges"] not in MERGE_VALUES:
                    continue                                    # a single-column cell that does not merge
                if _Polygon(polygon).height < row.height * .85:
                    continue                                    # a spanning cell must cover most of the row
                spanning.append(TableCell(polygon=polygon, row_id=z, rowspan=1, cell_id=cell_id, within_row_id=l, colspan=colspan,
                                          merge_up=sc["merges"] in (MERGE_UP, MERGE_BOTH), merge_down=sc["merges"] in (MERGE_DOWN, MERGE_BOTH),
                                          is_header=row.is_header or z == 0))
                cell_id += 1
            used = set()
            skip = 0
            for l, col in enumerate(columns):
                if skip:
                    skip -= 1
                    continue
                cell_polygon = row.intersection_polygon(col)
                cell_box = _Polygon(cell_polygon)
                added = False
                for zz, sc in enumerate(spanning):
                    col_width = sum(c.width for c in columns[l:l + sc.colspan])
                    if cell_box.intersection_pct(sc) > .9:
                        if sc.width > col_width * .85:
                            added = True
                            if zz not in used:
                                used.add(zz)
                                sc.col_id = l
                                unmerged.append(sc)
                                skip = sc.colspan - 1            # the columns the spanning cell covers
                        else:
                            used.add(zz)                         # too narrow for its colspan: never used
                if not added:
                    unmerged.append(TableCell(polygon=cell_polygon, row_id=z, rowspan=1, cell_id=cell_id, within_row_id=l, colspan=1,
                                              merge_up=False, merge_down=False, col_id=l,
                                              is_header=row.is_header or col.is_header or z == 0))
                    cell_id += 1
        grid = copy.deepcopy([[c for c in unmerged if c.row_id == r.row_id] for r in rows])
        for z, grid_row in enumerate(grid[1:]):
            prev = grid[z]
            for l, c in enumerate(grid_row):
                if l >= len(prev):
                    continue
                above = prev[l]
                if above.merge_down and c.merge_up and above.col_id == c.col_id and above.colspan == c.colspan:
                    above.merge(c)
                    above.rowspan += c.rowspan
                    grid_row[l] = above
        merged, seen = [], set()
        for c in itertools.chain.from_iterable(grid):
            if c.cell_id not in seen:
                seen.add(c.cell_id)
                merged.append(c)
        results.append(TableResult(cells=merged, unmerged_cells=unmerged, rows=rows, cols=columns,
                                   image_bbox=[0, 0, size[0], size[1]]))
    return results
