"""BASELINE config 5: the `ocr_text` data flow (surya/scripts/ocr_text.py:32-38 -> RecognitionPredictor.__call__,
surya/recognition/__init__.py:773-942) on the CUDA engines: detect -> boxes -> crop -> width-sorted recognition.

  pages (uint8)  --H2D 3 B/px-->  normalise + EfficientViT + post-processing front half (device)
                 connected components, size / peak filter, dilated row extents (device; heatmap.py:33-60)
                 --D2H tables-->  min-area rectangles over two points per dilated row (host OpenCV; heatmap.py:61-107)
                 polygons      -> y-expansion, clamping, containment filter (heatmap.py:140-175, common/util.py:9-36)
                 line crops    -> polygon-masked slices (input/processing.py:57-101), sorted by width (recognition/__init__.py:848)
                 crops         -> RecognitionRunner (processor mirror on the host, engine prefill / decode on the device)

Multi-GPU: pages are independent, so every rank runs the whole flow on its contiguous share of the pages
(shard.page_slices) and the per-line results are all-gathered at the end; nothing is exchanged in between (dealing crops
across ranks would mean shipping pixels between GPUs for no gain — each rank already has ~1/G of the lines).
Host post-processing here is the minimum the data flow needs; detokenisation / text assembly stay with the reference.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import shard
from .detection import DetEngine, detect_text_boxes_host, detect_text_pages
from .recognition import RecEngine, RecognitionRunner

Y_EXPAND_MARGIN = 0.05      # settings.DETECTOR_BOX_Y_EXPAND_MARGIN
PAD_VALUE = 255             # settings.RECOGNITION_PAD_VALUE


@dataclass
class Line:
    page: int
    polygon: List[List[int]]
    confidence: float
    tokens: List[int] = field(default_factory=list)
    scores: List[float] = field(default_factory=list)
    boxes: Optional[np.ndarray] = None


def _bbox(poly):
    xs, ys = [p[0] for p in poly], [p[1] for p in poly]
    return [min(xs), min(ys), max(xs), max(ys)]


def clean_keep(polys: Sequence, bbs: Sequence) -> List[int]:
    """clean_boxes (surya/common/util.py:9-36): indices of the polygons kept, in order.  A polygon goes when its bbox is flat, or
    when it lies inside the bbox of another polygon that differs from it both as a polygon and as a bbox."""
    keep = []
    for i, (p, bb) in enumerate(zip(polys, bbs)):
        if bb[0] == bb[2] or bb[1] == bb[3]:
            continue
        contained = False
        for q, ob in zip(polys, bbs):
            if q == p or bb == ob:
                continue
            if bb[0] >= ob[0] and bb[1] >= ob[1] and bb[2] <= ob[2] and bb[3] <= ob[3]:
                contained = True
                break
        if not contained:
            keep.append(i)
    return keep


def page_polygons(boxes: Sequence[np.ndarray], confidences: Sequence[float], image_size: Tuple[int, int],
                  processor_size: Tuple[int, int]) -> Tuple[List[List[List[int]]], List[float]]:
    """get_and_clean_boxes + the vertical expansion of parallel_get_boxes (surya/detection/heatmap.py:125-175) on plain lists:
    rescale to the page size with int() truncation, clamp, drop degenerate / contained boxes (common/util.py:9-36), expand
    non-vertical boxes by 5 % of their height, clamp again.  Sizes are (width, height)."""
    pw, ph = processor_size
    iw, ih = image_size
    sx, sy = iw / pw, ih / ph
    polys = []
    for b in boxes:
        poly = [[int(float(x) * sx), int(float(y) * sy)] for x, y in b]
        poly = [[max(min(x, iw), 0), max(min(y, ih), 0)] for x, y in poly]
        polys.append(poly)
    bbs = [_bbox(p) for p in polys]
    out, conf = [], []
    for i in clean_keep(polys, bbs):
        p, bb = polys[i], bbs[i]
        w, h = bb[2] - bb[0], bb[3] - bb[1]
        if h < 3 * w:
            ym = Y_EXPAND_MARGIN * h
            p = [[int(p[0][0]), int(p[0][1] - ym)], [int(p[1][0]), int(p[1][1] - ym)], [int(p[2][0]), int(p[2][1] + ym)],
                 [int(p[3][0]), int(p[3][1] + ym)]]
            p = [[max(min(x, iw), 0), max(min(y, ih), 0)] for x, y in p]
        out.append(p)
        conf.append(float(confidences[i]))
    return out, conf


def slice_polygon(image: np.ndarray, poly: Sequence[Sequence[int]]) -> np.ndarray:
    """slice_and_pad_poly (surya/input/processing.py:64-101): bounding-box crop with everything outside the polygon set to the pad
    value.  image: float32 / uint8 HWC."""
    import cv2

    x0, y0, x1, y1 = _bbox(poly)
    crop = image[y0:y1, x0:x1].copy()
    h, w = crop.shape[:2]
    if y1 <= y0 or x1 <= x0 or len(poly) < 3 or h == 0 or w == 0:
        return crop
    mask = np.zeros((h, w), dtype=np.uint8)
    cv2.fillPoly(mask, [np.int32([(x - x0, y - y0) for x, y in poly])], 1)
    crop[mask == 0] = PAD_VALUE
    return crop


class OcrPipeline:
    """detect -> crop -> recognise over the CUDA engines.  `run(pages)` takes uint8 pages [N, H, W, 3] (H, W = the detection
    processor size), or a list of uint8 pages [h, w, 3] of any size with optional high-resolution pages to crop from, and returns
    (lines grouped per page, timing breakdown in seconds)."""

    def __init__(self, det: DetEngine, rec: RecEngine, rec_batch: int = 256, max_tokens: int = 128, det_chunk: int = 16,
                 workers: int = 16, math_mode: bool = True, preprocess: str = "host"):
        """workers: no longer used by any step.  The detection boxes are finished in the calling thread, because that measured
        faster than a thread pool once connected components and dilation moved to the device.
        preprocess: "host" — crops are resized / normalised / tiled by the OpenCV thread pool (the reference's processor code);
        "device" — uint8 crops go up as they are and sb_rec_preprocess does that work on the GPU (SURVEY §8 f2)."""
        if preprocess not in ("host", "device"):
            raise ValueError("preprocess must be 'host' or 'device'")
        self.det, self.rec, self.preprocess = det, rec, preprocess
        self.runner = RecognitionRunner(rec, batch_size=rec_batch, max_tokens=max_tokens)
        self.det_chunk, self.workers, self.math_mode = det_chunk, max(1, workers), math_mode

    def detect(self, pages_u8: torch.Tensor):
        """pinned uint8 [n, H, W, 3] -> per page (polygons, confidences)."""
        n, H, W, _ = pages_u8.shape
        boxes = detect_text_boxes_host(self.det, pages_u8, chunk=self.det_chunk)
        return [page_polygons(b, c, (W, H), (W, H)) for b, c in boxes]

    def detect_pages(self, pages: Sequence[np.ndarray], processor_size: Tuple[int, int]):
        """uint8 pages of any size -> per page (polygons, confidences) in page coordinates (detect_text_pages)."""
        return [(d.polygons, d.confidences) for d in detect_text_pages(self.det, pages, processor_size, chunk=self.det_chunk)]

    def run(self, pages, fixed_steps: bool = False, highres_pages: Optional[Sequence[np.ndarray]] = None,
            processor_size: Optional[Tuple[int, int]] = None):
        """pages: uint8 [N, H, W, 3] at the detection processor size, or a list of uint8 [h, w, 3] pages of any size (resized and
        split on the device; processor_size = (width, height), default the engine's max_hw).  With highres_pages (list form only;
        an entry may be None for a page without one), each page's polygons are scaled to its high-resolution page with int(p * scale) and the crops are cut from it
        (RecognitionPredictor.detect_and_slice_bboxes, surya/recognition/__init__.py:138-180); the returned line polygons stay in
        the coordinates of the page given to detection."""
        t = {}
        t0 = time.perf_counter()
        if isinstance(pages, np.ndarray):
            if highres_pages is not None:
                raise ValueError("highres_pages needs pages as a list")
            pages_t = torch.from_numpy(np.ascontiguousarray(pages))
            if torch.cuda.is_available() and not pages_t.is_pinned():
                pages_t = pages_t.pin_memory()
            t["pin_pages"] = time.perf_counter() - t0
            t0 = time.perf_counter()
            det = self.detect(pages_t)
        else:
            if highres_pages is not None and len(highres_pages) != len(pages):
                raise ValueError(f"{len(highres_pages)} high-resolution pages for {len(pages)} pages")
            if processor_size is None:
                processor_size = (self.det.max_hw[1], self.det.max_hw[0])
            det = self.detect_pages(pages, processor_size)
        t["detect(device + host boxes)"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        lines: List[Line] = []
        crops = []
        for pg, (polys, conf) in enumerate(det):
            # processor.image_processor converts the whole page with np.asarray(image, float32) before slicing; slicing / masking the
            # uint8 page first and converting only the crop gives the identical float values (integers, pad value 255) without
            # touching 12 MB per page; the device path keeps the crop as uint8
            img = pages[pg]
            cut = polys
            if highres_pages is not None and highres_pages[pg] is not None:
                img = highres_pages[pg]
                sx, sy = img.shape[1] / pages[pg].shape[1], img.shape[0] / pages[pg].shape[0]
                cut = [[[int(x * sx), int(y * sy)] for x, y in p] for p in polys]
            for p, q, c in zip(polys, cut, conf):
                crop = slice_polygon(img, q)
                if crop.shape[0] == 0 or crop.shape[1] == 0:
                    continue
                if self.preprocess != "device":
                    crop = crop.astype(np.float32)
                lines.append(Line(page=pg, polygon=p, confidence=c))
                crops.append(crop)
        order = sorted(range(len(crops)), key=lambda i: -crops[i].shape[1])     # longest first (recognition/__init__.py:848)
        t["crop + sort"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        if crops:
            if self.preprocess == "device":
                tiles, grids, seqs = self.runner.preprocess_device([crops[i] for i in order], self.math_mode)
            else:
                tiles, grids, seqs = self.runner.preprocess([crops[i] for i in order], self.math_mode)
            t["recognition host preprocessing"] = time.perf_counter() - t0
            t0 = time.perf_counter()
            tok, sc, bb = self.runner.run_preprocessed(tiles, grids, seqs, fixed_steps=fixed_steps)
            for j, i in enumerate(order):
                lines[i].tokens, lines[i].scores, lines[i].boxes = tok[j], sc[j], bb[j]
        t["recognition (device loop)"] = time.perf_counter() - t0
        per_page: List[List[Line]] = [[] for _ in range(len(pages))]
        for ln in lines:
            per_page[ln.page].append(ln)
        return per_page, t


def sharded_ocr(pipe: OcrPipeline, pages, max_tokens: int, device=None, fixed_steps: bool = False,
                highres_pages: Optional[Sequence[np.ndarray]] = None, processor_size: Optional[Tuple[int, int]] = None):
    """Every rank runs `pipe` on its contiguous share of `pages` (identical array or list on all ranks, or any whose pages this rank
    owns are valid; a list may hold pages of any size, with optional highres_pages as in OcrPipeline.run) and the per-line
    results are all-gathered: returns (lines per page for ALL pages, this rank's timings).
    Exchange format: per page up to `cap` lines of [polygon 8, confidence, n_tokens, tokens max_tokens] packed as int32 / fp32."""
    import torch.distributed as dist

    rank, n_ranks = shard.world()
    slices = shard.page_slices(len(pages), n_ranks)
    lo, hi = slices[rank]
    if hi <= lo:
        per_page, timings = [], {}
    elif isinstance(pages, np.ndarray):
        per_page, timings = pipe.run(pages[lo:hi], fixed_steps=fixed_steps)
    else:
        per_page, timings = pipe.run(list(pages[lo:hi]), fixed_steps=fixed_steps, processor_size=processor_size,
                                     highres_pages=None if highres_pages is None else list(highres_pages[lo:hi]))
    if n_ranks == 1:
        return per_page, timings
    dev = shard._collective_device(device)
    cap_local = max([len(p) for p in per_page], default=0)
    cap_t = torch.tensor([cap_local], dtype=torch.int32, device=dev)
    dist.all_reduce(cap_t, op=dist.ReduceOp.MAX)
    cap = max(1, int(cap_t.item()))
    share = max(h - l for l, h in slices)
    ints = torch.zeros((share, cap, 10 + max_tokens), dtype=torch.int32)
    flts = torch.zeros((share, cap, 1 + max_tokens), dtype=torch.float32)
    for i, page in enumerate(per_page):
        for j, ln in enumerate(page):
            n = min(len(ln.tokens), max_tokens)
            ints[i, j, :8] = torch.tensor([c for pt in ln.polygon for c in pt], dtype=torch.int32)
            ints[i, j, 8], ints[i, j, 9] = 1, n
            ints[i, j, 10:10 + n] = torch.tensor(ln.tokens[:n], dtype=torch.int32)
            flts[i, j, 0] = ln.confidence
            flts[i, j, 1:1 + n] = torch.tensor(ln.scores[:n], dtype=torch.float32)
    ints, flts = ints.to(dev), flts.to(dev)
    gi = [torch.empty_like(ints) for _ in range(n_ranks)]
    gf = [torch.empty_like(flts) for _ in range(n_ranks)]
    dist.all_gather(gi, ints)
    dist.all_gather(gf, flts)
    out: List[List[Line]] = []
    for r, (l, h) in enumerate(slices):
        gi_r, gf_r = gi[r].cpu(), gf[r].cpu()
        for i in range(h - l):
            page = []
            for j in range(cap):
                if int(gi_r[i, j, 8]) == 0:
                    continue
                n = int(gi_r[i, j, 9])
                poly = gi_r[i, j, :8].reshape(4, 2).tolist()
                page.append(Line(page=l + i, polygon=poly, confidence=float(gf_r[i, j, 0]), tokens=gi_r[i, j, 10:10 + n].tolist(),
                                 scores=gf_r[i, j, 1:1 + n].tolist()))
            out.append(page)
    return out, timings
