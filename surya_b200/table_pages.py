"""Table recognition of pages on the device: the reference's table_recognition CLI (surya/scripts/table_recognition.py:26-80)
from uint8 pages to TableResults.

  layout (optional)              layout_pages over the pages; every Table / TableOfContents box is a table
  crop plan (host)               rescale_bbox to the high-resolution page (int truncation), expand_bbox (x 0.99 / 1.01), then
                                 Image.crop's int(round(v)) of each coordinate (round half to even); the crop size is the
                                 table's size.  With skip_table_detection every high-resolution page is one table.
  SuryaTableRecProcessor images  sb_layout_preprocess, one bounded job per table over the resident high-resolution page: the part
                                 of an expanded box past the page reads 0 as Image.crop fills it, then the cubic resize and
                                 normalisation (surya/common/donut/processor.py:61-116)
  TableRecPredictor              TableRecRunner.run_batch (both passes), then table_results (decode_batch_predictions)

No import of the reference or of oracle/.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ._lib import SuryaB200Error
from .layout_pages import LayoutResult, _check_pages, layout_pages, plan_jobs
from .table_rec import TableRecRunner, TableResult, table_results

TABLE_LABELS = ("Table", "TableOfContents")
EXPANSION = 0.01                                            # expand_bbox's default expansion_factor


def rescale_bbox(bbox, lo_size, hi_size) -> List[int]:
    """surya.common.util.rescale_bbox: each coordinate times hi / lo, truncated by int()."""
    ws, hs = hi_size[0] / lo_size[0], hi_size[1] / lo_size[1]
    return [int(bbox[0] * ws), int(bbox[1] * hs), int(bbox[2] * ws), int(bbox[3] * hs)]


def expand_bbox(bbox) -> List[float]:
    """surya.common.util.expand_bbox: the low corner times 0.99, the high corner times 1.01, in double."""
    lo, hi = 1 - EXPANSION, 1 + EXPANSION
    return [bbox[0] * lo, bbox[1] * lo, bbox[2] * hi, bbox[3] * hi]


def crop_box(box) -> Tuple[int, int, int, int]:
    """Image._crop's integer box: int(round(v)), Python's round half to even on the double value."""
    return tuple(int(round(v)) for v in box)


@dataclass
class TablePlan:
    page: int                                    # index of the page the table is on
    box: List[float]                             # the expanded box in high-resolution page coordinates (the CLI's highres_bbox)
    crop: Tuple[int, int, int, int]              # the integer crop box; it may extend past the page
    size: Tuple[int, int]                        # crop (w, h): the table's orig_size


def plan_tables(layout: Optional[Sequence[LayoutResult]], lo_sizes: Sequence[Tuple[int, int]],
                hi_sizes: Sequence[Tuple[int, int]]) -> List[TablePlan]:
    """The tables of every page in page order.  layout None: each high-resolution page is one table (skip_table_detection).
    Sizes are (w, h).  A crop with no width or height after rounding raises: the reference fails on it inside cv2."""
    out = []
    for p, (lo, hi) in enumerate(zip(lo_sizes, hi_sizes)):
        if layout is None:
            out.append(TablePlan(p, [0, 0, hi[0], hi[1]], (0, 0, hi[0], hi[1]), (hi[0], hi[1])))
            continue
        for k, b in enumerate(x for x in layout[p].bboxes if x.label in TABLE_LABELS):
            box = expand_bbox(rescale_bbox(b.bbox, lo, hi))
            c = crop_box(box)
            w, h = c[2] - c[0], c[3] - c[1]
            if w <= 0 or h <= 0:
                raise SuryaB200Error(f"page {p}, table box {k} ({b.label} {b.bbox}): crop {c} of a {hi[0]}x{hi[1]} page is empty")
            out.append(TablePlan(p, box, c, (w, h)))
    return out


@dataclass
class TablePagesRun:
    results: List[List[TableResult]]                         # per page, its tables in layout box order
    table_boxes: List[List[List[float]]]                     # per page, the expanded boxes in high-resolution coordinates
    layout: Optional[List[LayoutResult]]                     # None with skip_table_detection
    timing: Dict[str, float] = field(default_factory=dict)  # seconds: upload, preprocess, encoder, passes, geometry
    layout_timing: Dict[str, float] = field(default_factory=dict)
    steps_run: List[int] = field(default_factory=list)      # decode steps of every pass, in order


def table_pages(table_engine, pages, layout_engine=None, highres_pages=None, skip_table_detection: bool = False,
                batch_size: int = 32, layout_batch_size: int = 32, max_boxes: int = 150,
                pixel_values: Optional[torch.Tensor] = None) -> TablePagesRun:
    """The table_recognition CLI on the device.  pages: uint8 [h, w, 3] RGB arrays (numpy or CPU tensors) that layout runs on;
    highres_pages: a list of the same length whose entries (None: the page itself) the tables are cropped from.  Tables are
    taken in page order and recognised in batches of batch_size, as TableRecPredictor batches the CLI's crops: per batch the
    high-resolution pages holding its tables are uploaded through a reused pinned staging buffer, one bounded
    sb_layout_preprocess job per table writes a reused device buffer, and TableRecRunner.run_batch decodes it.
    pixel_values (optional, [n_tables, 3, H, W] in table order) replaces the device preprocessing, e.g. by a host restatement."""
    if table_engine.kind != "table":
        raise SuryaB200Error("table_pages needs a table_rec engine")
    if not skip_table_detection and (layout_engine is None or layout_engine.kind != "layout"):
        raise SuryaB200Error("table_pages needs a layout engine unless skip_table_detection is set")
    runner = TableRecRunner(table_engine, batch_size, max_boxes)
    arrs = _check_pages(pages)
    if highres_pages is None:
        highres_pages = [None] * len(arrs)
    if len(highres_pages) != len(arrs):
        raise SuryaB200Error(f"{len(highres_pages)} high-resolution pages for {len(arrs)} pages")
    his = []
    for i, (a, h) in enumerate(zip(arrs, highres_pages)):
        try:
            his.append(a if h is None else _check_pages([h])[0])
        except SuryaB200Error as e:
            raise SuryaB200Error(f"high-resolution {str(e).replace('page 0', f'page {i}')}") from None
    lo_sizes = [(a.shape[1], a.shape[0]) for a in arrs]
    hi_sizes = [(a.shape[1], a.shape[0]) for a in his]

    layout, layout_timing = None, {}
    if not skip_table_detection:
        lrun = layout_pages(layout_engine, arrs, layout_batch_size)
        layout, layout_timing = lrun.results, lrun.timing
    plan = plan_tables(layout, lo_sizes, hi_sizes)
    if pixel_values is not None and pixel_values.shape[0] != len(plan):
        raise SuryaB200Error(f"{pixel_values.shape[0]} pixel values for {len(plan)} tables")

    eng = table_engine
    H, W = eng.cfg.encoder.image_size
    on_gpu = torch.device(eng.device).type == "cuda"
    sync = torch.cuda.synchronize if on_gpu else (lambda: None)
    t = {"upload": 0.0, "preprocess": 0.0, "encoder": 0.0, "passes": 0.0, "geometry": 0.0}
    results: List[List[TableResult]] = [[] for _ in arrs]
    boxes: List[List[List[float]]] = [[] for _ in arrs]
    for tp in plan:
        boxes[tp.page].append(tp.box)
    host = dev = px_buf = None    # staging and pixel buffers, grown to the largest batch and reused
    for b0 in range(0, len(plan), batch_size):
        batch = plan[b0:b0 + batch_size]
        t0 = time.perf_counter()
        if pixel_values is None:
            held = sorted({tp.page for tp in batch})
            offs = dict(zip(held, np.cumsum([0] + [his[p].nbytes for p in held[:-1]]).tolist()))
            total = int(sum(his[p].nbytes for p in held))
            if host is None or host.numel() < total:
                host = torch.empty(total, dtype=torch.uint8, pin_memory=on_gpu)
                dev = torch.empty(total, dtype=torch.uint8, device=eng.device)
            sync()                # the previous batch's upload has finished reading the staging buffer
            hv = host.numpy()
            for p in held:
                hv[offs[p]:offs[p] + his[p].nbytes] = his[p].reshape(-1)
            dev[:total].copy_(host[:total], non_blocking=True)
            sync()
        t1 = time.perf_counter()
        t["upload"] += t1 - t0
        n = len(batch)
        if pixel_values is None:
            rects = [(tp.crop[0], tp.crop[1], tp.size[0], tp.size[1]) for tp in batch]
            jobs, ti, tw = plan_jobs(rects, [offs[tp.page] for tp in batch], [hi_sizes[tp.page][0] for tp in batch], (H, W),
                                     page_h=[hi_sizes[tp.page][1] for tp in batch])
            if px_buf is None or px_buf.shape[0] < n:
                px_buf = torch.empty((n, 3, H, W), dtype=eng.dtype, device=eng.device)
            px = eng.preprocess(dev, jobs.to(eng.device), ti.to(eng.device), tw.to(eng.device), out=px_buf[:n])
        else:
            px = pixel_values[b0:b0 + n]
        sync()
        t["preprocess"] += time.perf_counter() - t1
        rowcol, cells, idx_map, sizes = runner.run_batch(px, [tp.size for tp in batch], timing=t)
        t2 = time.perf_counter()
        for tp, res in zip(batch, table_results(rowcol, cells, idx_map, sizes)):
            results[tp.page].append(res)
        t["geometry"] += time.perf_counter() - t2
    return TablePagesRun(results=results, table_boxes=boxes, layout=layout, timing=t, layout_timing=layout_timing,
                         steps_run=runner.steps_run)
