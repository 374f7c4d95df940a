"""Host planner of the detection page preparation: pages of any size -> processor-size chunks on the device.

Restates, for RGB uint8 pages, what DetectionPredictor does before its model call and after it:
  split_image / get_total_splits   pages taller than DETECTOR_IMAGE_CHUNK_HEIGHT are cut into chunks of processor height; the last
                                   chunk is padded by ImageOps.pad(..., color=255, centering=(0, 0)) (surya/detection/util.py:7-36)
  prepare_image                    img.thumbnail(size, LANCZOS) (reducing_gap=2.0), then img.resize(size, LANCZOS)
                                   (surya/detection/__init__.py:50-62)
  heatmap stitching                chunk heatmaps stacked per page, an appended chunk cut to its original row count when that is
                                   below the processor height (surya/detection/__init__.py:134-151)

PIL's Lanczos resample on 8-bit images is integer arithmetic once its weights are fixed: the weights are computed here in
double precision exactly as PIL does (support widened by the downscale factor, normalised, rounded to 22-bit fixed point),
cached per (source extent, box, destination extent), and the device kernel sb_det_page_resize only multiplies, adds, shifts and
clips.  The reduce step of `reducing_gap` is a box average with PIL's rounding, also integer.  So the device result equals PIL
byte for byte (tests/test_page_prep_cpu.py pins the geometry and oracle/page_prep_oracle.py's pixel passes to PIL).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from functools import lru_cache
from typing import List, Sequence, Tuple

import numpy as np

from ._lib import SuryaB200Error

CHUNK_HEIGHT = 1400          # settings.DETECTOR_IMAGE_CHUNK_HEIGHT
REDUCING_GAP = 2.0           # Image.thumbnail's default
LANCZOS_SUPPORT = 3.0
PRECISION_BITS = 22          # 32 - 8 - 2: fixed-point weights of PIL's 8-bit resample
# ImageOps.pad(color=255) on an RGB image: PIL reads a bare int as 0xAABBGGRR, so the padding is red, not white.
PAD_RGB = (255, 0, 0)

DEFAULT_MAX_PAGE_PIXELS = 64 << 20
DEFAULT_MAX_CHUNKS = 32

# job descriptor of sb_det_page_resize (int64 x DESC_LEN, include/surya_b200.h)
K_REDUCE, K_HORIZ, K_VERT = 0, 1, 2
DESC_LEN = 16


def thumbnail_size(w: int, h: int, tw: int, th: int) -> Tuple[int, int] | None:
    """Image.thumbnail's target size (preserve_aspect_ratio), or None when the page already fits."""
    if tw >= w and th >= h:
        return None
    aspect = w / h

    def round_aspect(number: float, key) -> int:
        return max(min(math.floor(number), math.ceil(number), key=key), 1)

    x, y = tw, th
    if x / y >= aspect:
        x = round_aspect(y * aspect, key=lambda n: abs(aspect - n / y))
    else:
        y = round_aspect(x / aspect, key=lambda n: 0 if n == 0 else abs(aspect - x / n))
    return x, y


def reduce_factors(w: int, h: int, tw: int, th: int, gap: float = REDUCING_GAP) -> Tuple[int, int]:
    """Image.resize's pre-reduce factors: int(extent / size / reducing_gap) or 1, per axis."""
    return int(w / tw / gap) or 1, int(h / th / gap) or 1


def is_split(h: int) -> bool:
    """split_image cuts (and pads) a page exactly when it is taller than DETECTOR_IMAGE_CHUNK_HEIGHT, whatever the processor
    height: with a processor taller than that, a page between the two becomes one chunk padded to the processor height."""
    return h > CHUNK_HEIGHT


def split_plan(h: int, ph: int) -> List[Tuple[int, int]]:
    """split_image: (first source row, row count) per chunk.  When is_split(h), a chunk shorter than ph is padded to ph rows."""
    if not is_split(h):
        return [(0, h)]
    return [(i * ph, min((i + 1) * ph, h) - i * ph) for i in range(math.ceil(h / ph))]


def stitch_rows(plan: Sequence[Tuple[int, int]], ph: int) -> List[int]:
    """Heatmap rows each chunk contributes to its page: the first chunk keeps all ph rows (also when it is padded), an appended
    chunk keeps its original row count when that is below ph."""
    return [ph if i == 0 else min(rows, ph) for i, (_, rows) in enumerate(plan)]


def _sinc(v: np.ndarray) -> np.ndarray:
    """sin(pi v) / (pi v), 1 at 0; sin through math.sin (the C library's, as in PIL), not NumPy's own vector sin."""
    x = v * math.pi
    sx = np.fromiter(map(math.sin, x.ravel().tolist()), dtype=np.float64, count=x.size).reshape(x.shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(v == 0.0, 1.0, sx / x)


@lru_cache(maxsize=512)
def lanczos_coeffs(in_size: int, in1: float, out_size: int) -> Tuple[int, np.ndarray, np.ndarray]:
    """PIL's precompute_coeffs + normalize_coeffs_8bpc for the box [0, in1) of an axis of in_size pixels resampled to out_size
    (in1 is the box edge as the C float PIL stores it).  Returns (ksize, bounds int32 [out_size, 2] = first tap, tap count,
    weights int32 [out_size, ksize]).  Vectorised over all taps with PIL's double-precision operations in PIL's order; the
    per-row normalising sum is a cumulative sum, i.e. left to right like the C loop (taps past the count add +0.0)."""
    scale = float(np.float32(in1)) / out_size
    filterscale = max(scale, 1.0)
    support = LANCZOS_SUPPORT * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)          # (int) truncates toward zero
    xmax = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size) - xmin
    taps = np.arange(ksize)[None, :]
    live = taps < xmax[:, None]
    arg = ((taps + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss
    w = np.where(live & (arg >= -3.0) & (arg < 3.0), _sinc(arg) * _sinc(arg / 3), 0.0)
    ww = np.cumsum(w, axis=1)[:, -1:]
    k = np.where(ww != 0.0, w / np.where(ww != 0.0, ww, 1.0), w)
    one = float(1 << PRECISION_BITS)
    kk = np.where(k < 0, np.trunc(-0.5 + k * one), np.trunc(0.5 + k * one))
    kk = np.where(live, kk, 0).astype(np.int32)
    return ksize, np.stack([xmin, xmax], axis=1).astype(np.int32), kk


@dataclass(frozen=True)
class Pass:
    """One step of the resize of one chunk image: kind K_REDUCE (box average by fx x fy) / K_HORIZ / K_VERT (Lanczos along one
    axis with lanczos_coeffs(*key))."""
    kind: int
    src: Tuple[int, int]      # (w, h)
    dst: Tuple[int, int]
    fx: int = 1
    fy: int = 1
    key: Tuple[int, float, int] | None = None


def _resample(src: Tuple[int, int], box: Tuple[float, float], size: Tuple[int, int]) -> List[Pass]:
    """Image.resize after its pre-reduce, box = (right, bottom) edges of the source box.  ImagingResampleInner runs a horizontal
    pass when the width or the box's x extent changes, then a vertical pass likewise; an image more than 100 times taller than
    wide that shrinks vertically is resized vertically first, as two separate resizes."""
    (iw, ih), (bx, by), (ow, oh) = src, (float(np.float32(box[0])), float(np.float32(box[1]))), size
    if ih > iw * 100 and oh < ih:
        return _resample_inner(src, (float(iw), by), (iw, oh)) + _resample_inner((iw, oh), (bx, float(oh)), size)
    return _resample_inner(src, (bx, by), size)


def _resample_inner(src: Tuple[int, int], box: Tuple[float, float], size: Tuple[int, int]) -> List[Pass]:
    (iw, ih), (bx, by), (ow, oh) = src, box, size
    out = []
    if ow != iw or bx != ow:
        out.append(Pass(K_HORIZ, (iw, ih), (ow, ih), key=(iw, bx, ow)))
        iw = ow
    if oh != ih or by != oh:
        out.append(Pass(K_VERT, (iw, ih), (iw, oh), key=(ih, by, oh)))
    return out


def chunk_passes(w: int, h: int, pw: int, ph: int) -> List[Pass]:
    """prepare_image on a w x h chunk image: thumbnail (pre-reduce + Lanczos) then the stretch to pw x ph.  An empty list means
    the chunk already is pw x ph."""
    passes: List[Pass] = []
    cur = (w, h)
    t = thumbnail_size(w, h, pw, ph)
    if t is not None and t != cur:
        fx, fy = reduce_factors(w, h, *t)
        box = (float(w), float(h))
        if fx > 1 or fy > 1:
            red = (-(-w // fx), -(-h // fy))
            passes.append(Pass(K_REDUCE, cur, red, fx, fy))
            cur, box = red, (w / fx, h / fy)
        passes += _resample(cur, box, t)
        cur = t
    if cur != (pw, ph):
        passes += _resample(cur, (float(cur[0]), float(cur[1])), (pw, ph))
    return passes


@dataclass
class PagePlan:
    """Everything sb_det_page_resize and the stitched text front need for a list of pages."""
    sizes: List[Tuple[int, int]]              # (w, h) per page
    page_off: np.ndarray                      # int64 [P + 1] byte offsets of the pages in the packed upload
    chunks: List[Tuple[int, int, int]]        # (page, first source row, source rows) per chunk
    chunk_tab: np.ndarray                     # int32 [n_chunks, 4]: page, first stitched row, rows kept, 0
    page_tab: np.ndarray                      # int32 [P, 2]: first row in the packed stitched map, stitched rows
    desc: np.ndarray                          # int64 [n_jobs, DESC_LEN], grouped by step
    step_jobs: List[int]
    step_max_px: List[int]
    tables: np.ndarray                        # int32: bounds and weights of every distinct axis
    scratch_bytes: int


def plan_pages(sizes: Sequence[Tuple[int, int]], processor_size: Tuple[int, int], max_chunks: int = DEFAULT_MAX_CHUNKS,
               max_page_pixels: int = DEFAULT_MAX_PAGE_PIXELS) -> PagePlan:
    """Plan the device resize of pages of the given (w, h) sizes into processor_size = (width, height) chunks.  Raises
    SuryaB200Error for a page beyond the capacity instead of truncating it."""
    pw, ph = processor_size
    page_off = np.zeros(len(sizes) + 1, dtype=np.int64)
    for i, (w, h) in enumerate(sizes):
        if w <= 0 or h <= 0:
            raise SuryaB200Error(f"page {i} is empty ({w}x{h})")
        if w * h > max_page_pixels:
            raise SuryaB200Error(f"page {i} has {w}x{h} pixels, more than the configured {max_page_pixels}")
        if len(split_plan(h, ph)) > max_chunks:
            raise SuryaB200Error(f"page {i} ({w}x{h}) needs {len(split_plan(h, ph))} chunks, more than the configured {max_chunks}")
        page_off[i + 1] = page_off[i] + w * h * 3
    chunks, chunk_tab, page_tab = [], [], []
    row = 0
    for p, (w, h) in enumerate(sizes):
        plan = split_plan(h, ph)
        kept = stitch_rows(plan, ph)
        page_tab.append((row, sum(kept)))
        off = 0
        for (r0, rows), k in zip(plan, kept):
            chunks.append((p, r0, rows))
            chunk_tab.append((p, row + off, k, 0))
            off += k
        row += sum(kept)
    # jobs: per chunk its passes chained through scratch, the last one into the output chunk
    tab_off = {}
    tables: List[np.ndarray] = []
    n_tab = 0
    steps: List[List[List[int]]] = []
    scratch = 0
    out_bytes = pw * ph * 3
    for c, (p, r0, rows) in enumerate(chunks):
        w, _ = sizes[p]
        hc = ph if is_split(sizes[p][1]) else rows       # chunks of a split page are padded to ph rows
        passes = chunk_passes(w, hc, pw, ph) or [Pass(K_REDUCE, (w, hc), (w, hc))]     # 1 x 1 box average = copy
        src = (int(page_off[p]) + r0 * w * 3, 1, rows)
        for j, ps in enumerate(passes):
            last = j == len(passes) - 1
            if last:
                dst = (c * out_bytes, 1)
            else:
                dst = (scratch, 0)
                scratch += ps.dst[0] * ps.dst[1] * 3
            ksize = coef = bnd = 0
            if ps.key is not None:
                if ps.key not in tab_off:
                    ksize, bounds, kk = lanczos_coeffs(*ps.key)
                    tab_off[ps.key] = (ksize, n_tab, n_tab + bounds.size)
                    tables += [bounds.ravel(), kk.ravel()]
                    n_tab += bounds.size + kk.size
                ksize, bnd, coef = tab_off[ps.key]
            d = [ps.kind, src[0], ps.src[0], ps.src[1], src[2], src[1], dst[0], ps.dst[0], ps.dst[1], dst[1], ps.fx, ps.fy, ksize,
                 coef, bnd, 0]
            while len(steps) <= j:
                steps.append([])
            steps[j].append(d)
            src = (dst[0], 0, ps.dst[1])
            if last:
                break
    desc = np.array([d for s in steps for d in s], dtype=np.int64).reshape(-1, DESC_LEN)
    return PagePlan(sizes=list(sizes), page_off=page_off, chunks=chunks, chunk_tab=np.array(chunk_tab, dtype=np.int32).reshape(-1, 4),
                    page_tab=np.array(page_tab, dtype=np.int32).reshape(-1, 2), desc=desc, step_jobs=[len(s) for s in steps],
                    step_max_px=[max(d[7] * d[8] for d in s) for s in steps],
                    tables=np.concatenate(tables) if tables else np.zeros(1, dtype=np.int32), scratch_bytes=scratch)
