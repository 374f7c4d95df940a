"""Layout analysis of pages of any size on the device: LayoutPredictor.batch_layout_detection (surya/layout/__init__.py:40-226)
from uint8 pages to per-page results.

  ImageSlicer.slice / slice_count     pages above LAYOUT_SLICE_MIN on either axis are cut into at most 4 slices along their longer
                                      axis (surya/layout/slicer.py:19-66); each slice is a source rectangle of the resident page
  SuryaEncoderImageProcessor          sb_layout_preprocess: cubic resize of every page / slice to the encoder size, normalised, in
                                      the engine dtype (surya/common/donut/processor.py:61-116); the cubic taps come from here
  model + decode loop                 LayoutEngine.encode, then LayoutEngine.run_pages: the greedy loop with the header/footer rule
                                      and the early exit on the device (surya/layout/__init__.py:106-183)
  post-processing (host)              polygons from the model-dtype rows, softmax / top-k, confidence, positions, clean_boxes
                                      (:140-216), then ImageSlicer.join / merge_results (slicer.py:68-140)

The results are plain dataclasses with the fields of the reference's LayoutResult / LayoutBox (surya/layout/schema.py) and the
PolygonBox methods the slice join uses (surya/common/polygon.py, restated once in surya_b200/polygon.py).  No import of the reference or of oracle/.
"""
from __future__ import annotations

import math
import time
from dataclasses import dataclass, field
from functools import lru_cache
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ._lib import SuryaB200Error
from .pipeline import clean_keep
from .polygon import PolygonMethods

SLICE_MIN = (1500, 1500)          # settings.LAYOUT_SLICE_MIN (width, height)
SLICE_SIZE = (1200, 1200)         # settings.LAYOUT_SLICE_SIZE (width, height)
MAX_SLICES = 4                    # ImageSlicer(max_slices=4)
MERGE_TOLERANCE = 0.05            # ImageSlicer.merge_tolerance
MERGE_MARGIN = 0.05               # ImageSlicer.merge_margin
# surya/layout/model/config.py:16-34
ID_TO_LABEL = {0: "Blank", 1: "Text", 2: "TextInlineMath", 3: "Code", 4: "SectionHeader", 5: "Caption", 6: "Footnote",
               7: "Equation", 8: "ListItem", 9: "PageFooter", 10: "PageHeader", 11: "Picture", 12: "Figure", 13: "Table",
               14: "Form", 15: "TableOfContents", 16: "Handwriting"}
JOB_LEN = 8                       # int64 per job of sb_layout_preprocess


# ------------------------------------------------------------------------------------------------ results
@dataclass
class LayoutBox(PolygonMethods):
    polygon: List[List[float]]
    label: str
    position: int
    top_k: Optional[Dict[str, float]] = None
    confidence: Optional[float] = None


@dataclass
class LayoutResult:
    bboxes: List[LayoutBox]
    image_bbox: List[float]
    sliced: bool = False


# ------------------------------------------------------------------------------------------------ slicing plan
def _slice_size(dim: int, min_size: int) -> int:
    return max(min_size, dim // MAX_SLICES + 1)


def slice_count(w: int, h: int) -> int:
    """ImageSlicer.slice_count: the batching weight of a page (also for pages that are not sliced)."""
    if w > h:
        return math.ceil(w / _slice_size(w, SLICE_SIZE[0]))
    return math.ceil(h / _slice_size(h, SLICE_SIZE[1]))


def slice_rects(w: int, h: int) -> List[Tuple[int, int, int, int, int, int]]:
    """ImageSlicer.slice for one page of size (w, h): [(x0, y0, sw, sh, tile_x, tile_y)] in the reference's order."""
    if not (w > SLICE_MIN[0] or h > SLICE_MIN[1]):
        return [(0, 0, w, h, 0, 0)]
    out = []
    if w > h:
        size = _slice_size(w, SLICE_SIZE[0])
        for i, x in enumerate(range(0, w, size)):
            out.append((x, 0, min(x + size, w) - x, h, i, 0))
    else:
        size = _slice_size(h, SLICE_SIZE[1])
        for i, y in enumerate(range(0, h, size)):
            out.append((0, y, w, min(y + size, h) - y, 0, i))
    return out


def page_batches(counts: Sequence[int], batch_size: int) -> List[Tuple[int, int]]:
    """The page ranges of batch_layout_detection's batches (surya/layout/__init__.py:52-67)."""
    batches, start, end = [], 0, 1
    while end < len(counts):
        if sum(counts[start:end]) >= batch_size or sum(counts[start:end + 1]) > batch_size:
            batches.append((start, end))
            start = end
        end += 1
    if start < len(counts):
        batches.append((start, len(counts)))
    return batches


# ------------------------------------------------------------------------------------------------ preprocessing plan
@lru_cache(maxsize=256)
def cubic_axis(src: int, dst: int) -> Tuple[np.ndarray, np.ndarray]:
    """OpenCV's cubic taps for one axis, src -> dst pixels: coordinate f = (d + 0.5) * (1 / (dst / src)) - 0.5 and Keys weights
    (A = -0.75) in double, stored as float32; tap indices floor(f) - 1 .. floor(f) + 2 clamped to the axis.  int32 / float32
    [dst, 4]."""
    A = -0.75
    f = (np.arange(dst, dtype=np.float64) + 0.5) * (1.0 / (dst / src)) - 0.5
    s = np.floor(f)
    x = f - s
    c0 = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A
    c1 = ((A + 2) * x - (A + 3)) * x * x + 1
    c2 = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1
    w = np.stack([c0, c1, c2, 1.0 - c0 - c1 - c2], 1).astype(np.float32)
    idx = np.clip(s.astype(np.int64)[:, None] + np.arange(-1, 3)[None], 0, src - 1).astype(np.int32)
    idx.setflags(write=False)
    w.setflags(write=False)
    return idx, w


def plan_jobs(rects: Sequence[Tuple[int, int, int, int]], page_off: Sequence[int], page_w: Sequence[int], out_hw: Tuple[int, int],
              page_h: Optional[Sequence[int]] = None):
    """Job table and tap tables of sb_layout_preprocess.  rects[i] = (x0, y0, w, h) of the source rectangle of output i in the
    page that starts at byte page_off[i] of the packed pages and is page_w[i] pixels wide.  page_h (optional) gives page
    heights: a job with a non-zero height is bounded, its taps outside the page read 0 (PIL's crop fill), and its rectangle may
    extend past the page; without it every job has height 0 and must lie inside its page.  Returns (jobs int64 [n, 8],
    tap_idx int32 [rows, 4], tap_w float32 [rows, 4]) as CPU tensors; each (extent, out size) table appears once."""
    H, W = out_hw
    tables: Dict[Tuple[int, int], int] = {}
    idx_parts, w_parts = [], []
    rows = 0

    def table(src: int, dst: int) -> int:
        nonlocal rows
        key = (src, dst)
        if key not in tables:
            i, w = cubic_axis(src, dst)
            tables[key] = rows
            idx_parts.append(i)
            w_parts.append(w)
            rows += dst
        return tables[key]

    jobs = np.zeros((len(rects), JOB_LEN), np.int64)
    for n, (x0, y0, w, h) in enumerate(rects):
        jobs[n, :7] = (page_off[n], page_w[n], x0, y0, table(w, W), table(h, H), n)
        if page_h is not None:
            jobs[n, 7] = page_h[n]
    return (torch.from_numpy(jobs), torch.from_numpy(np.concatenate(idx_parts)), torch.from_numpy(np.concatenate(w_parts)))


# ------------------------------------------------------------------------------------------------ post-processing
def row_polygons(bbox: torch.Tensor, dtype: torch.dtype, bbox_size: int, skew_scaler: int, sizes: torch.Tensor) -> np.ndarray:
    """prediction_to_polygon (surya/layout/util.py:4-40) for many rows at once.  bbox: the sigmoid box outputs [n, 6] (fp32
    holding model-dtype values); the predictor's row is bbox * bbox_size in the model dtype (layout/__init__.py:127, 137), and
    every step up to the corners is a torch op in that dtype; the scaling to the image is Python float.  sizes [n, 2] = (w, h).
    Returns float64 [n, 4, 2]."""
    v = bbox.to(dtype) * bbox_size
    cx, cy, w, h = v[:, 0], v[:, 1], v[:, 2], v[:, 3]
    x1, y1, x2, y2 = cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2
    sx = torch.floor((v[:, 4] - skew_scaler) / 2)
    sy = torch.floor((v[:, 5] - skew_scaler) / 2)
    sx[torch.abs(sx) < 0.001] = 0
    sy[torch.abs(sy) < 0.001] = 0
    poly = torch.stack([x1 - sx, y1 - sy, x2 - sx, y1 + sy, x2 + sx, y2 + sy, x1 + sx, y2 - sy], 1).double().numpy().reshape(-1, 4, 2)
    scale = sizes.double().numpy() / bbox_size
    return poly * scale[:, None, :]


def slice_result(tok: torch.Tensor, bbox: torch.Tensor, cls: torch.Tensor, done: torch.Tensor, size: Tuple[int, int], dtype: torch.dtype,
                 cfg, top_k: int) -> LayoutResult:
    """One image's LayoutResult from its decode histories (host tensors over the steps that ran): tok [n, 7], bbox [n, 6], cls
    [n, label_count] (the logits after the header/footer rule), done [n].  A step counts while the image is not done (sticky,
    this step included), and its box is kept when its class is above the special tokens (surya/layout/__init__.py:140-216)."""
    special = cfg.special_token_count
    live = ~(torch.cumsum(done.to(torch.int64), 0) > 0)
    live &= tok[:, 6] > special
    steps = torch.nonzero(live).flatten()
    w, h = size
    boxes: List[LayoutBox] = []
    if steps.numel():
        polys = row_polygons(bbox[steps], dtype, cfg.bbox_size, cfg.skew_scaler, torch.tensor([[w, h]]).expand(len(steps), 2))
        probs, idx = torch.topk(torch.nn.functional.softmax(cls[steps].to(dtype), dim=-1), k=top_k, dim=-1)
        idx = idx - special
        for z, s in enumerate(steps.tolist()):
            top = {ID_TO_LABEL.get(int(l)): p.item() for l, p in zip(idx[z], probs[z]) if l > 0}
            label = ID_TO_LABEL[int(tok[s, 6]) - special]
            if label not in top:
                raise KeyError(label)      # the reference's top_k_dict[l] (layout/__init__.py:208)
            boxes.append(LayoutBox(polygon=[[float(x), float(y)] for x, y in polys[z]], label=label, position=z, top_k=top,
                                   confidence=top[label]))
    keep = clean_keep([b.polygon for b in boxes], [b.bbox for b in boxes])
    return LayoutResult(bboxes=[boxes[i] for i in keep], image_bbox=[0.0, 0.0, float(w), float(h)])


def merge_results(res1: LayoutResult, res2: LayoutResult, merge_dir: str) -> LayoutResult:
    """ImageSlicer.merge_results (surya/layout/slicer.py:84-140).  Mutates the boxes of both, as the reference does."""
    new_bbox = list(res1.image_bbox)
    remove = set()
    horiz = merge_dir == "width"
    k = 2 if horiz else 3
    new_bbox[k] += res2.image_bbox[k]
    max_position = max(b.position for b in res1.bboxes) + 1       # ValueError on a first slice without boxes, as the reference
    picture = ("Picture", "Figure")
    for i, b2 in enumerate(res2.bboxes):
        if horiz:
            b2.shift(x_shift=res1.image_bbox[2])
        else:
            b2.shift(y_shift=res1.image_bbox[3])
        b2.position += max_position
        for b1 in res1.bboxes:
            if horiz:
                inter = (b1.intersection_pct(b2, x_margin=MERGE_MARGIN) > MERGE_TOLERANCE or
                         b2.intersection_pct(b1, x_margin=MERGE_MARGIN) > MERGE_TOLERANCE)
                across = b1.y_overlap(b2) > b1.height // 2 or b2.y_overlap(b1) > b2.height // 2
            else:
                inter = (b1.intersection_pct(b2, y_margin=MERGE_MARGIN) > MERGE_TOLERANCE or
                         b2.intersection_pct(b1, y_margin=MERGE_MARGIN) > MERGE_TOLERANCE)
                across = b1.x_overlap(b2) > b1.width // 2 or b2.x_overlap(b1) > b2.width // 2
            same = b1.label == b2.label or (b1.label in picture and b2.label in picture)
            if inter and across and same:
                b1.merge(b2)
                remove.add(i)
    return LayoutResult(bboxes=res1.bboxes + [b for i, b in enumerate(res2.bboxes) if i not in remove], image_bbox=new_bbox, sliced=True)


def join(results: Sequence[LayoutResult], positions: Sequence[Tuple[int, int, int]]) -> List[LayoutResult]:
    """ImageSlicer.join (surya/layout/slicer.py:68-82): the slices of a page merged left to right / top to bottom."""
    out, cur = [], None
    for i, (res, (page, tx, _)) in enumerate(zip(results, positions)):
        if i == 0 or page != positions[i - 1][0]:
            if cur is not None:
                out.append(cur)
            cur = res
        else:
            cur = merge_results(cur, res, "width" if tx > 0 else "height")
    if cur is not None:
        out.append(cur)
    return out


# ------------------------------------------------------------------------------------------------ the flow
def _check_pages(pages) -> List[np.ndarray]:
    if len(pages) == 0:
        raise SuryaB200Error("layout_pages needs at least one page")
    out = []
    for i, p in enumerate(pages):
        a = p.numpy() if torch.is_tensor(p) else np.asarray(p)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
            raise SuryaB200Error(f"page {i}: expected uint8 [h, w, 3] RGB, got {a.dtype} {tuple(a.shape)}")
        out.append(np.ascontiguousarray(a))
    return out


@dataclass
class LayoutPagesRun:
    results: List[LayoutResult]
    timing: Dict[str, float] = field(default_factory=dict)
    steps_run: List[int] = field(default_factory=list)        # decode steps per batch (early exit: below max_boxes)


def layout_pages(engine, pages, batch_size: int = 32, top_k: int = 5, pixel_values: Optional[torch.Tensor] = None) -> LayoutPagesRun:
    """LayoutPredictor(pages, batch_size, top_k) on the device.  pages: uint8 [h, w, 3] RGB arrays (numpy or CPU tensors).
    Per batch of the reference's batching: the batch's pages are uploaded through a pinned staging buffer that is reused,
    then preprocessing, encoder, decode loop, and the host post-processing of the histories.  pixel_values (optional, [n_slices, 3, H, W] in the predictor's slice order) replaces
    the device preprocessing, e.g. by a host restatement.  Returns the per-page results and a timing breakdown (seconds)."""
    if engine.kind != "layout":
        raise SuryaB200Error("layout_pages needs a layout engine")
    if batch_size < 1 or batch_size > engine.max_batch:
        raise SuryaB200Error(f"batch_size {batch_size} outside 1..max_batch {engine.max_batch}")
    arrs = _check_pages(pages)
    cfg = engine.cfg.decoder
    H, W = engine.cfg.encoder.image_size
    t = {"upload": 0.0, "preprocess": 0.0, "encoder": 0.0, "decode": 0.0, "host_post": 0.0}
    on_gpu = torch.device(engine.device).type == "cuda"
    sync = torch.cuda.synchronize if on_gpu else (lambda: None)

    counts = [slice_count(a.shape[1], a.shape[0]) for a in arrs]
    results: List[LayoutResult] = []
    steps_run: List[int] = []
    done_slices = 0
    host = dev = None             # staging buffers, grown to the largest batch of pages and reused
    for p0, p1 in page_batches(counts, batch_size):
        t0 = time.perf_counter()
        offs = np.cumsum([0] + [arrs[p].nbytes for p in range(p0, p1)])
        if pixel_values is None:
            if host is None or host.numel() < offs[-1]:
                host = torch.empty(int(offs[-1]), dtype=torch.uint8, pin_memory=on_gpu)
                dev = torch.empty(int(offs[-1]), dtype=torch.uint8, device=engine.device)
            sync()                # the previous batch's upload has finished reading the staging buffer
            hv = host.numpy()
            for p, o in zip(range(p0, p1), offs[:-1]):
                hv[o:o + arrs[p].nbytes] = arrs[p].reshape(-1)
            dev[:int(offs[-1])].copy_(host[:int(offs[-1])], non_blocking=True)
            sync()
        t_up = time.perf_counter()
        t["upload"] += t_up - t0
        t0 = t_up
        rects, offs_b, widths, positions = [], [], [], []
        for p in range(p0, p1):
            ph, pw = arrs[p].shape[:2]
            for x0, y0, sw, sh, tx, ty in slice_rects(pw, ph):
                rects.append((x0, y0, sw, sh))
                offs_b.append(int(offs[p - p0]))
                widths.append(pw)
                positions.append((p - p0, tx, ty))
        n = len(rects)
        if n > engine.max_batch:
            raise SuryaB200Error(f"a batch of {n} slices exceeds max_batch {engine.max_batch}")
        if pixel_values is None:
            jobs, ti, tw = plan_jobs(rects, offs_b, widths, (H, W))
            px = engine.preprocess(dev, jobs.to(engine.device), ti.to(engine.device), tw.to(engine.device))
        else:
            px = pixel_values[done_slices:done_slices + n].to(engine.device, engine.dtype)
        done_slices += n
        sync()
        t1 = time.perf_counter()
        enc = engine.encode(px)
        sync()
        t2 = time.perf_counter()
        wh = torch.tensor([[r[2], r[3]] for r in rects], dtype=torch.int32)
        tok, bbox, cls, done = engine.run_pages(enc, wh, cfg.max_boxes)
        tok, bbox, cls, done = tok.cpu(), bbox.cpu(), cls.cpu(), done.cpu()
        t3 = time.perf_counter()
        steps_run.append(int(tok.shape[0]))
        per_slice = [slice_result(tok[:, j], bbox[:, j], cls[:, j], done[:, j], (r[2], r[3]), engine.dtype, cfg, top_k)
                     for j, r in enumerate(rects)]
        results.extend(join(per_slice, positions))
        t4 = time.perf_counter()
        t["preprocess"] += t1 - t0
        t["encoder"] += t2 - t1
        t["decode"] += t3 - t2
        t["host_post"] += t4 - t3
    return LayoutPagesRun(results=results, timing=t, steps_run=steps_run)
