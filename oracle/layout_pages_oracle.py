"""CPU ORACLE (test infrastructure, not product code) — LayoutPredictor's page flow restated for the device path's tests.

  * resize_cubic_u8 / process      SuryaEncoderImageProcessor.process_inner (surya/common/donut/processor.py:61-116) for one
                                   uint8 RGB image: cv2.resize(INTER_CUBIC) of the uint8 image (the processor's resample is
                                   Image.Resampling.BILINEAR == 2, which cv2 reads as INTER_CUBIC), x * (1/255) in double -> float32,
                                   (x - 0.5) / 0.5 in float32, cast to the model dtype.
  * rule_corners                   corners 0 and 2 of a predicted box as the predictor's polygon arithmetic yields them
                                   (surya/layout/util.py:4-40): a model of its rounding points, one float32 op rounded to the
                                   model dtype at a time, then the Python-float scaling to the image
  * next_token_pages               one step of the predictor's loop on the class / box outputs (surya/layout/__init__.py:122-183):
                                   argmax, done, the header/footer relabelling of rows not yet done, the next decoder input
  * stub_outputs / StubLayoutEngine  the deterministic stand-in decoder that oracle/make_layout_pages_golden.py runs under the
                                   reference's own LayoutPredictor, and a CPU engine with LayoutEngine's surface over the same
                                   outputs, so the repository's host flow can be checked against tests/golden/layout_pages.pt

OpenCV's uint8 INTER_CUBIC (opencv-python 4.13.0) does not take its generic fixed-point path (coefficients x 2048 in int16 and a
(v + 2^21) >> 22 vertical pass differ from cv2.resize on about 4 % of the values).  It follows the float model that
oracle/preproc_oracle.py documents for float32 input: double coordinate and Keys weights (A = -0.75), float32 accumulation tap
by tap, horizontal pass then vertical pass, then round half to even and clamp to 0..255.  That model leaves a residual of
values that are off by exactly one (about 5e-6 of them; OpenCV's SIMD summation order is not specified);
tests/test_layout_pages_cpu.py states the bound it pins.  The device kernel equals this restatement byte for byte.
Only tests/ and oracle/make_layout_pages_golden.py import this module.
"""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np
import torch

from oracle.preproc_oracle import axis_table

# surya/layout/model/config.py:16-34, kept here so that the oracle does not take it from the code under test
ID_TO_LABEL = {0: "Blank", 1: "Text", 2: "TextInlineMath", 3: "Code", 4: "SectionHeader", 5: "Caption", 6: "Footnote",
               7: "Equation", 8: "ListItem", 9: "PageFooter", 10: "PageHeader", 11: "Picture", 12: "Figure", 13: "Table",
               14: "Form", 15: "TableOfContents", 16: "Handwriting"}
LABEL_TO_ID = {v: k for k, v in ID_TO_LABEL.items()}
HEADER_FOOTER = ("PageHeader", "PageFooter")


def resize_cubic_u8(img: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(uint8 HWC, (dw, dh), INTER_CUBIC) in the float model above -> uint8 [dh, dw, 3]."""
    img = np.asarray(img)
    assert img.dtype == np.uint8
    h, w = img.shape[:2]
    xi, xw = axis_table(w, dw, "cubic")
    yi, yw = axis_table(h, dh, "cubic")
    src = img.astype(np.float32)
    rows = np.zeros((h, dw, img.shape[2]), np.float32)
    for j in range(4):
        rows = rows + src[:, xi[:, j], :] * xw[None, :, j, None]
    out = np.zeros((dh, dw, img.shape[2]), np.float32)
    for j in range(4):
        out = out + rows[yi[:, j]] * yw[:, j, None, None]
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def normalize(resized_u8: np.ndarray, dtype: torch.dtype) -> torch.Tensor:
    """process_inner after the resize: HWC uint8 -> CHW tensor in the model dtype."""
    x = resized_u8.transpose(2, 0, 1).astype(np.float32)
    x = (x.astype(np.float64) * (1 / 255)).astype(np.float32)
    mean = np.array([0.5, 0.5, 0.5], np.float32)
    x = ((x.T - mean) / mean).T
    return torch.tensor(x, dtype=dtype)


def process(img: np.ndarray, size: Tuple[int, int], dtype: torch.dtype) -> torch.Tensor:
    """One image (uint8 HWC) -> pixel values [3, H, W] in `dtype`; size = (H, W)."""
    return normalize(resize_cubic_u8(img, size[1], size[0]), dtype)


def _rd(v, dtype) -> float:
    """A float32 value rounded to the model dtype, as a torch op on 16-bit CPU tensors stores its float result."""
    return float(torch.tensor(np.float32(v), dtype=torch.float32).to(dtype))


def rule_corners(bbox, size: Tuple[int, int], dtype: torch.dtype, bbox_size: int, skew_scaler: int):
    """Corner 0 (left, top) and corner 2 (right, bottom) of a box in image pixels.  bbox: the six sigmoid outputs (model-dtype
    values).  Rounding points: the decoder-input row v = bbox * bbox_size; half extents v / 2; edges centre -/+ half; skew
    floor((v - skew_scaler) / 2); corners edge -/+ skew; each a float32 op rounded to `dtype`.  The scale to the image,
    size / bbox_size, and the product are double."""
    f = np.float32
    v = [_rd(f(b) * f(bbox_size), dtype) for b in bbox]
    hw, hh = _rd(f(v[2]) / f(2), dtype), _rd(f(v[3]) / f(2), dtype)
    left, right = _rd(f(v[0]) - f(hw), dtype), _rd(f(v[0]) + f(hw), dtype)
    top, bottom = _rd(f(v[1]) - f(hh), dtype), _rd(f(v[1]) + f(hh), dtype)
    sx = float(np.floor(_rd(f(_rd(f(v[4]) - f(skew_scaler), dtype)) / f(2), dtype)))
    sy = float(np.floor(_rd(f(_rd(f(v[5]) - f(skew_scaler), dtype)) / f(2), dtype)))
    ws, hs = size[0] / bbox_size, size[1] / bbox_size
    c0 = (_rd(f(left) - f(sx), dtype) * ws, _rd(f(top) - f(sy), dtype) * hs)
    c2 = (_rd(f(right) + f(sx), dtype) * ws, _rd(f(bottom) + f(sy), dtype) * hs)
    return c0, c2


def rule_fires(bbox, token: int, size: Tuple[int, int], dtype: torch.dtype, cfg) -> bool:
    """The header/footer test of surya/layout/__init__.py:161-168 for one row: a PageHeader / PageFooter whose corner 0 lies
    before 0.8 and corner 2 after 0.2 of the image on both axes."""
    if ID_TO_LABEL.get(int(token) - cfg.special_token_count) not in HEADER_FOOTER:
        return False
    (x0, y0), (x2, y2) = rule_corners([float(b) for b in bbox], size, dtype, cfg.bbox_size, cfg.skew_scaler)
    w, h = size
    return y0 < h * .8 and y2 > h * .2 and x0 < w * .8 and x2 > w * .2


def next_token_pages(bbox: torch.Tensor, cls: torch.Tensor, sizes: Sequence[Tuple[int, int]], sticky: torch.Tensor,
                     dtype: torch.dtype, cfg):
    """One loop step for a batch (CPU tensors): bbox [B, 6] and cls [B, C] fp32 holding model-dtype values; sticky [B] bool =
    rows done before this step.  Returns (tokens int64 [B, 7], modified class logits [B, C], done [B] bool, rule count)."""
    cls = cls.clone()
    B = bbox.shape[0]
    tok = torch.zeros((B, 7), dtype=torch.int64)
    tok[:, :6] = (bbox * cfg.bbox_size).clamp(0, cfg.bbox_size).to(torch.int64)
    t = cls.argmax(-1)
    done = (t == cfg.eos_token_id) | (t == cfg.pad_token_id)
    fired = 0
    for b in range(B):
        tb = int(t[b])
        if not (sticky[b] or done[b]) and rule_fires(bbox[b], tb, sizes[b], dtype, cfg):
            cls[b, tb] = 0
            tb = int(cls[b].argmax(-1))
            fired += 1
        tok[b, 6] = tb
    return tok, cls, done, fired


# ------------------------------------------------------------------------------------------------ stub decoder
# Cases of tests/golden/layout_pages.pt: pages (w, h) in the predictor's order, the batch size, the fixture-page seeds.
LAYOUT_PAGES_CASE = {"pages": [(816, 1056), (3100, 1700), (1700, 2600), (600, 400), (1632, 2112), (1600, 1600)], "batch_size": 4,
                     "seed": 40, "special": 3, "label_count": 20, "eos": 1, "pad": 0}
STUB_CYCLE = 8


def fixture_page(w: int, h: int, seed: int) -> np.ndarray:
    """A light page with dark blocks, uint8 [h, w, 3]."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 240, np.uint8)
    for _ in range(12):
        x, y = int(rng.integers(0, w - 8)), int(rng.integers(0, h - 8))
        img[y:y + int(rng.integers(4, h // 4 + 5)), x:x + int(rng.integers(4, w // 3 + 5))] = rng.integers(0, 120, 3)
    return img


def stub_outputs(row: int, step: int, prev_class: int, special: int = 3, label_count: int = 20, eos: int = 1):
    """The stand-in decoder's outputs for image row `row` (in the predictor's order over the whole call), at `step`, fed class
    `prev_class`: (box sigmoid [6], class logits [label_count]) as float64 lists, before the cast to the model dtype.
    Per step of an 8-step cycle: a Text box mid-page; a PageHeader mid-page (relabelled to SectionHeader); a PageHeader at the
    top (kept); a PageFooter mid-page whose runner-up is the pause token (relabelled, then dropped as a special token); a Text
    box at the right edge and one at the left edge (merged across a width-wise cut); a Figure at the bottom edge and a Picture
    at the top edge (merged across a height-wise cut).  Rows stop at row-dependent steps; rows 2, 7, 12, ... never stop."""
    stop = None if row % 5 == 2 else 4 + (row * 5) % 17
    logits = [-4.0 + 0.125 * j for j in range(label_count)]
    k = step % STUB_CYCLE
    jit = (row % 5) * 6 + (prev_class % 3) * 2          # the fed class shifts the box: relabelling changes later rows
    boxes = {0: (300 + jit, 500, 200, 60), 1: (512, 480 + jit, 300, 70), 2: (512, 30 + jit // 4, 500, 40),
             3: (500 + jit, 600, 260, 50), 4: (962, 450, 124, 100), 5: (62, 450 + jit // 4, 124, 100),
             6: (450, 962, 100, 124), 7: (450 + jit // 4, 62, 100, 124)}
    labels = {0: "Text", 1: "PageHeader", 2: "PageHeader", 3: "PageFooter", 4: "Text", 5: "Text", 6: "Figure", 7: "Picture"}
    cx, cy, w, h = boxes[k]
    bbox = [cx / 1024, cy / 1024, w / 1024, h / 1024, 0.5, 0.5]
    if stop is not None and step >= stop:
        logits[eos] = 9.0
        return bbox, logits
    logits[LABEL_TO_ID[labels[k]] + special] = 6.0
    if k == 1:
        logits[LABEL_TO_ID["SectionHeader"] + special] = 3.0
    if k == 3:
        logits[2] = 3.0                                   # the pause token: the relabelled box is not a layout class
    return bbox, logits


class StubLayoutEngine:
    """A CPU object with the surface layout_pages uses (kind, max_batch, cfg, dtype, device, encode, run_pages).  encode hands
    out the rows' order numbers; run_pages decodes stub_outputs with next_token_pages and stops after the first group of 8
    steps at which every row is done, as sb_layout_decode_pages does."""

    kind = "layout"

    def __init__(self, cfg, dtype=torch.float16, max_batch: int = 32):
        self.cfg, self.dtype, self.max_batch, self.device = cfg, dtype, max_batch, torch.device("cpu")
        self.rows_seen = 0
        self.rule_count = 0

    def encode(self, px: torch.Tensor) -> torch.Tensor:
        ids = torch.arange(self.rows_seen, self.rows_seen + px.shape[0])
        self.rows_seen += px.shape[0]
        return ids

    def run_pages(self, enc, page_wh, n_steps):
        d = self.cfg.decoder
        B, C = enc.shape[0], d.label_count
        sizes = [tuple(int(v) for v in r) for r in torch.as_tensor(page_wh).reshape(B, 2).tolist()]
        hist = {"tok": [], "bbox": [], "cls": [], "done": []}
        sticky = torch.zeros(B, dtype=torch.bool)
        prev = [d.bos_token_id] * B
        for s in range(n_steps):
            outs = [stub_outputs(int(enc[b]), s, prev[b], d.special_token_count, C, d.eos_token_id) for b in range(B)]
            bbox = torch.tensor([o[0] for o in outs]).to(self.dtype).float()
            cls = torch.tensor([o[1] for o in outs]).to(self.dtype).float()
            tok, cm, dn, fired = next_token_pages(bbox, cls, sizes, sticky, self.dtype, d)
            self.rule_count += fired
            for k, v in (("tok", tok), ("bbox", bbox), ("cls", cm), ("done", dn.to(torch.uint8))):
                hist[k].append(v)
            sticky |= dn
            prev = tok[:, 6].tolist()
            if bool(sticky.all()) and (s + 1) % 8 == 1:
                break
        return tuple(torch.stack(hist[k]) for k in ("tok", "bbox", "cls", "done"))
