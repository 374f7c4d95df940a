"""Detection page preparation on the CPU: the NumPy restatement (oracle/page_prep_oracle.py) of PIL's thumbnail + resize, the
tall-page split with ImageOps.pad and the heatmap stitching, all against PIL itself, byte for byte; and the job tables
surya_b200.page_prep plans for sb_det_page_resize, run through a NumPy interpreter of the kernel."""
import math

import numpy as np
import pytest
from PIL import Image, ImageOps

from oracle import page_prep_oracle as O
from surya_b200 import page_prep as pp
from surya_b200._lib import SuryaB200Error

# (width, height): upscaling only, identity, one axis or both down, pre-reduce in one axis (>= 4x) and in both, odd / prime,
# 1-pixel-wide and 1-pixel-tall, tall and narrow (PIL's vertical-first path), a 4000-px-tall page
SIZES = [(300, 200), (1024, 1024), (768, 512), (1100, 700), (816, 1056), (1632, 2112), (4100, 900), (4099, 4111), (997, 1009),
         (1, 500), (500, 1), (1, 1), (3, 4000), (600, 4000), (2549, 1023)]
PROCESSOR_SIZES = [(1024, 1024), (768, 512), (512, 1536)]      # the last is taller than the 1400-row split threshold


def _page(w, h, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img[: h // 2] = (np.arange(w)[None, :, None] * 7 % 256).astype(np.uint8)      # smooth half: exercises the clip less
    return img


def pil_prepare(img, size):
    im = Image.fromarray(img)
    im.thumbnail(size, Image.Resampling.LANCZOS)
    return np.asarray(im.resize(size, Image.Resampling.LANCZOS))


def pil_split(img, ph):
    """split_image's rule (surya/detection/util.py) with PIL's crop and ImageOps.pad."""
    im = Image.fromarray(img)
    h = img.shape[0]
    if h <= pp.CHUNK_HEIGHT:
        return [img], [h]
    out, heights = [], []
    for i in range(math.ceil(h / ph)):
        bottom = min((i + 1) * ph, h)
        c = im.crop((0, i * ph, img.shape[1], bottom))
        if bottom - i * ph < ph:
            c = ImageOps.pad(c, (img.shape[1], ph), color=255, centering=(0, 0))
        out.append(np.asarray(c))
        heights.append(bottom - i * ph)
    return out, heights


@pytest.mark.parametrize("processor_size", PROCESSOR_SIZES)
@pytest.mark.parametrize("wh", SIZES)
def test_prepare_image_equals_pil(wh, processor_size):
    img = _page(*wh, seed=wh[0] * 7 + wh[1])
    got = O.prepare_image(img, processor_size)
    ref = pil_prepare(img, processor_size)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_thumbnail_size_leaves_fitting_pages():
    assert pp.thumbnail_size(1024, 1024, 1024, 1024) is None
    assert pp.thumbnail_size(300, 200, 1024, 1024) is None
    for w, h in SIZES:
        im = Image.new("RGB", (w, h))
        im.thumbnail((1024, 1024), Image.Resampling.LANCZOS)
        assert (pp.thumbnail_size(w, h, 1024, 1024) or (w, h)) == im.size


@pytest.mark.parametrize("h,ph", [(1024, 1024), (1400, 1024), (1401, 1024), (2048, 1024), (3300, 1024), (4000, 1024), (1450, 1536),
                                  (1400, 1536), (3100, 1536)])
def test_split_and_pad_equal_pil(h, ph):
    img = _page(37, h, seed=h)
    got, gh = O.split_page(img, ph)
    ref, rh = pil_split(img, ph)
    assert gh == rh and len(got) == len(ref)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)


def test_stitch_cuts_only_appended_short_chunks():
    maps = [np.full((8, 4), i, np.float32) for i in range(3)]
    assert O.stitch(maps, [8, 8, 3], 8).shape == (19, 4)
    assert O.stitch(maps[:1], [5], 8).shape == (8, 4)          # a padded first chunk keeps all its rows
    assert pp.stitch_rows(pp.split_plan(3300, 1024), 1024) == [1024, 1024, 1024, 228]
    assert pp.stitch_rows(pp.split_plan(1450, 1536), 1536) == [1536]


def _interpret(plan, packed, pw, ph):
    """NumPy interpreter of sb_det_page_resize over a plan's job table."""
    scratch = np.zeros(max(plan.scratch_bytes, 1), np.uint8)
    out = np.zeros(len(plan.chunks) * ph * pw * 3, np.uint8)
    tab = plan.tables
    for d in plan.desc:
        kind, soff, sw, sh, valid, spage, doff, dw, dh, dout, fx, fy, ks, coef, bnd = (int(v) for v in d[:15])
        src = (packed if spage else scratch)[soff:soff + sw * min(sh, valid) * 3].reshape(min(sh, valid), sw, 3)
        img = np.empty((sh, sw, 3), np.uint8)
        img[:] = pp.PAD_RGB
        img[:src.shape[0]] = src
        if kind == pp.K_REDUCE:
            res = O.reduce_box(img, fx, fy)
        else:
            n = dw if kind == pp.K_HORIZ else dh
            bounds = tab[bnd:bnd + 2 * n].reshape(n, 2)
            kk = tab[coef:coef + n * ks].reshape(n, ks)
            a = np.moveaxis(img, 1 if kind == pp.K_HORIZ else 0, 0).astype(np.int64)
            acc = np.full((n,) + a.shape[1:], 1 << 21, np.int64)
            for i in range(n):
                t0, c = bounds[i]
                acc[i] += np.tensordot(kk[i, :c].astype(np.int64), a[t0:t0 + c], axes=(0, 0))
            res = np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), 0, 1 if kind == pp.K_HORIZ else 0)
        assert res.shape == (dh, dw, 3)
        (out if dout else scratch)[doff:doff + res.size] = res.ravel()
    return out.reshape(-1, ph, pw, 3)


@pytest.mark.parametrize("processor_size", PROCESSOR_SIZES)
def test_job_tables_reproduce_pil(processor_size):
    pw, ph = processor_size
    sizes = [(816, 1056), (1300, 3300), (640, 1500), (300, 200), (pw, ph), (2100, 97), (5, 2900), (300, 1450)]
    pages = [_page(w, h, seed=i) for i, (w, h) in enumerate(sizes)]
    plan = pp.plan_pages(sizes, processor_size)
    packed = np.concatenate([p.ravel() for p in pages])
    got = _interpret(plan, packed, pw, ph)
    ref = [pil_prepare(c, processor_size) for p in pages for c in pil_split(p, ph)[0]]
    assert got.shape[0] == len(ref)
    for c, r in enumerate(ref):
        assert np.array_equal(got[c], r), f"chunk {c} ({plan.chunks[c]})"
    rows = [sum(pp.stitch_rows(pp.split_plan(h, ph), ph)) for _, h in sizes]
    assert plan.page_tab[:, 1].tolist() == rows
    assert plan.page_tab[:, 0].tolist() == np.concatenate([[0], np.cumsum(rows)[:-1]]).tolist()


def test_capacity_is_checked():
    with pytest.raises(SuryaB200Error):
        pp.plan_pages([(100, 100), (9000, 9000)], (1024, 1024), max_page_pixels=64 << 20)
    with pytest.raises(SuryaB200Error):
        pp.plan_pages([(100, 20000)], (1024, 1024), max_chunks=8)
    with pytest.raises(SuryaB200Error):
        pp.plan_pages([(0, 10)], (1024, 1024))
