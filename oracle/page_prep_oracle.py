"""NumPy restatement of the detection page preparation (PIL's thumbnail + resize on RGB uint8 pages, the tall-page split and the
heatmap stitching of DetectionPredictor), the CPU reference of sb_det_page_resize and the stitched text front.

The geometry (thumbnail size, pre-reduce factors, boxes, split plan, Lanczos weights) comes from surya_b200.page_prep, which
the device path uses too; this module restates the pixel arithmetic PIL applies on top of it:
  reduce     box average over fx x fy blocks (partial blocks at the right / bottom edge average the pixels they have):
             ((sum + n // 2) * m) >> 24 with m = uint32(float32(2**32) / float32(256 n))
  resample   per output pixel sum of uint8 source * int32 weight + 2**21, arithmetic shift by 22, clip to 0..255;
             horizontal pass into a uint8 image, then the vertical pass over it
tests/test_page_prep_cpu.py checks the composition against PIL byte for byte.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

from surya_b200.page_prep import (K_HORIZ, K_REDUCE, K_VERT, PAD_RGB, PRECISION_BITS, chunk_passes, is_split, lanczos_coeffs,
                                  split_plan, stitch_rows)


def reduce_box(img: np.ndarray, fx: int, fy: int) -> np.ndarray:
    h, w, _ = img.shape
    oh, ow = -(-h // fy), -(-w // fx)
    pad = np.zeros((oh * fy, ow * fx, 3), dtype=np.uint64)
    pad[:h, :w] = img
    s = pad.reshape(oh, fy, ow, fx, 3).sum(axis=(1, 3))
    ny = np.minimum(fy, h - np.arange(oh) * fy)
    nx = np.minimum(fx, w - np.arange(ow) * fx)
    n = (ny[:, None] * nx[None, :]).astype(np.uint64)
    m = (np.float32(2.0 ** 32) / (np.float32(256) * n.astype(np.float32))).astype(np.uint64)
    return (((s + (n // 2)[..., None]) * m[..., None]) >> np.uint64(24)).astype(np.uint8)


def _resample_axis(img: np.ndarray, key, axis: int) -> np.ndarray:
    ksize, bounds, kk = lanczos_coeffs(*key)
    src = np.moveaxis(img, axis, 0).astype(np.int64)            # resampled axis first
    n_in = src.shape[0]
    idx = np.minimum(bounds[:, :1] + np.arange(ksize)[None, :], n_in - 1)      # taps past the count carry weight 0
    acc = np.full((bounds.shape[0],) + src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for t in range(ksize):
        wt = np.where(t < bounds[:, 1], kk[:, t], 0).astype(np.int64)
        acc += src[idx[:, t]] * wt.reshape((-1,) + (1,) * (src.ndim - 1))
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def run_passes(img: np.ndarray, passes) -> np.ndarray:
    for ps in passes:
        if ps.kind == K_REDUCE:
            img = reduce_box(img, ps.fx, ps.fy)
        elif ps.kind == K_HORIZ:
            img = _resample_axis(img, ps.key, 1)
        else:
            assert ps.kind == K_VERT
            img = _resample_axis(img, ps.key, 0)
    return img


def prepare_image(img: np.ndarray, processor_size: Tuple[int, int]) -> np.ndarray:
    """DetectionPredictor.prepare_image's pixels (before the processor's normalisation): thumbnail + stretch, uint8 HWC."""
    h, w, _ = img.shape
    return run_passes(np.ascontiguousarray(img), chunk_passes(w, h, *processor_size))


def split_page(img: np.ndarray, ph: int) -> Tuple[List[np.ndarray], List[int]]:
    """split_image: the chunk images (the short last one padded by ImageOps.pad) and their original row counts."""
    if not is_split(img.shape[0]):
        return [img], [img.shape[0]]
    plan = split_plan(img.shape[0], ph)
    chunks = []
    for r0, rows in plan:
        c = np.empty((ph, img.shape[1], 3), dtype=np.uint8)
        c[:] = PAD_RGB
        c[:rows] = img[r0:r0 + rows]
        chunks.append(c)
    return chunks, [rows for _, rows in plan]


def stitch(chunk_maps: Sequence[np.ndarray], heights: Sequence[int], ph: int) -> np.ndarray:
    """batch_detection's stacking of one page's chunk heatmaps [ph, W]: appended chunks are cut to their original rows."""
    kept = stitch_rows([(0, r) for r in heights], ph)
    return np.vstack([m[:k] for m, k in zip(chunk_maps, kept)])



# ------------------------------------------------------------------------------------------------ reference fixture (stub model)
PAGE_SIZES_CASES = [
    # processor (width, height), pages (width, height): smaller than the processor, not split, just above 1400 rows, many chunks
    # with a short last one; then a processor taller than 1400 rows: a page between 1400 and its height (one padded chunk)
    {"processor": (256, 256), "pages": [(200, 180), (300, 900), (260, 1401), (240, 1800)]},
    {"processor": (256, 1536), "pages": [(300, 1450), (200, 1000), (180, 3100)]},
]
IMAGENET_MEAN = np.array((0.485, 0.456, 0.406))
IMAGENET_STD = np.array((0.229, 0.224, 0.225))


def fixture_page(w: int, h: int, seed: int) -> np.ndarray:
    """White page with dark bars of text-line shape (deterministic from the seed)."""
    rng = np.random.default_rng(seed)
    p = np.full((h, w, 3), 255, np.uint8)
    for _ in range(max(4, h * w // 30000)):
        bh, bw = int(rng.integers(6, 24)), int(rng.integers(20, max(21, w // 2)))
        y, x = int(rng.integers(0, max(1, h - bh))), int(rng.integers(0, max(1, w - bw)))
        p[y:y + bh, x:x + bw] = rng.integers(0, 90, 3)
    return p


def pixels_u8(pixel_values) -> np.ndarray:
    """The uint8 NCHW image a normalised NCHW batch encodes ((u8 / 255 - mean) / std is one-to-one on 0..255)."""
    x = np.asarray(pixel_values, dtype=np.float64)
    u = (x * IMAGENET_STD[None, :, None, None] + IMAGENET_MEAN[None, :, None, None]) * 255.0
    r = np.rint(u)
    assert np.abs(u - r).max() < 1e-3, "pixel values do not encode a uint8 image"
    return r.astype(np.uint8)


class DarknessStub:
    """Deterministic stand-in for the detection model (what DetectionPredictor touches: config.num_labels, dtype, device, to(),
    model(pixel_values=...).logits): both label maps are the 4 x 4 average-pooled darkness of the uint8 page the pixel values
    encode, so pages with dark bars yield text lines and the maps do not depend on last-bit differences of the normalisation."""

    def __init__(self, record: list | None = None):
        import torch

        self.record = record                    # when given, collects the uint8 batches the model is called on
        self.config = type("Cfg", (), {"num_labels": 2})()
        self.dtype, self.device = torch.float32, torch.device("cpu")

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def __call__(self, pixel_values):
        import torch
        import torch.nn.functional as F

        u8 = pixels_u8(pixel_values.float().numpy())
        if self.record is not None:
            self.record.append(u8)
        u8 = torch.from_numpy(u8).double()
        dark = 1.0 - u8.mean(1, keepdim=True) / 255.0
        pooled = F.avg_pool2d(dark, 4).float()
        return type("Out", (), {"logits": torch.cat([pooled, pooled], 1)})()
