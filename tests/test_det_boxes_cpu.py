"""Device text-box tables (sb_det_text_boxes) on the CPU: the NumPy restatement of the tables (tests/det_boxes_ref.py) followed by
the product's host finish (text_boxes_from_tables) must give text_boxes_from_front's boxes and confidences byte for byte.  The
three facts the device tables rest on are pinned against OpenCV directly: components numbered in raster order, cv2.dilate's rows
from the source row extents, and minAreaRect over two points per dilated row."""
import cv2
import numpy as np
import pytest

from det_boxes_ref import as_16bit, assert_same, dilated_rows, ks_of, raster_labels, synth_map, text_box_tables
from surya_b200.detection import text_boxes_from_front, text_boxes_from_tables


def finish(line_map, mask, tt, **cap):
    t = text_box_tables(line_map, mask, tt, **cap)
    assert not t["overflow"]
    return text_boxes_from_tables(t["box"], t["peak"], t["points"], t["count"])


def branches(t):
    """(number of boxes that take the diamond fix-up, set of ks parities) of one page's tables."""
    diamonds = 0
    for k in range(t["count"]):
        off, n = t["box"][k, 4:6]
        r = cv2.boxPoints(cv2.minAreaRect(t["points"][off:off + n].astype(np.int64)))
        bw, bh = np.linalg.norm(r[0] - r[1]), np.linalg.norm(r[1] - r[2])
        diamonds += abs(1 - max(bw, bh) / (min(bw, bh) + 1e-5)) <= 0.1
    return diamonds, {int(k) % 2 for k in t["box"][:t["count"], 6]}


def check_page(m16, low, tt):
    mask = (np.asarray(m16, dtype=np.float32) > np.float32(low)).astype(np.uint8)
    ref = text_boxes_from_front(m16, mask, float(tt), float(low))
    assert_same(finish(m16, mask, tt), ref)
    return ref


@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_tables_then_host_finish_equal_text_boxes_from_front(kind):
    rng = np.random.default_rng(11 if kind == "fp16" else 12)
    n_boxes = diamonds = 0
    parity = set()
    for i in range(110):
        H, W = int(rng.integers(20, 200)), int(rng.integers(20, 200))
        m16 = as_16bit(synth_map(rng, H, W), kind)
        low = np.float32(rng.uniform(0.3, 0.45))
        tt = np.float32(rng.uniform(0.45, 0.8))
        boxes, _ = check_page(m16, low, tt)
        n_boxes += len(boxes)
        d, p = branches(text_box_tables(m16, (np.asarray(m16, np.float32) > low).astype(np.uint8), tt))
        diamonds += d
        parity |= p
    assert n_boxes > 200 and parity == {0, 1} and diamonds > 0


def test_crafted_components():
    """Border-touching lines, 1-px-wide and 1-px-tall lines, areas 9 and 10, a peak exactly at the text threshold, a U-shape and a
    spiral whose later branches join earlier roots, near-squares (diamond branch), odd and even ks."""
    H, W = 120, 160
    m = np.full((H, W), 0.1, np.float32)
    m[0:6, 0:50] = 0.9                  # top-left corner
    m[H - 4:H, W - 70:W] = 0.8          # bottom-right corner
    m[30:90, W - 1] = 0.7               # 1 px wide, on the right border
    m[20, 60:120] = 0.75                # 1 px tall
    m[50, 10:19] = 0.9                  # area 9: dropped
    m[54, 10:20] = 0.9                  # area 10: kept
    m[60:70, 30:40] = 0.65              # square: diamond branch, ks = 4
    m[75:100, 40:65] = 0.7              # square, ks = 6
    m[40:43, 60:70] = 0.6               # peak exactly text_threshold (0.6 as a 16-bit value)
    u = np.zeros((20, 30), bool)        # U-shape: two arms from the top meet at the bottom
    u[:, :4] = u[:, -4:] = u[-4:, :] = True
    m[95:115, 100:130][u] = 0.85
    sp = np.zeros((40, 40), bool)       # spiral: each ring's left side turns into the next ring's top side
    for r in range(0, 20, 4):
        sp[r, r:40 - r] = sp[r:40 - r, 39 - r] = sp[39 - r, r:40 - r] = True
        sp[r + 4:40 - r, r] = True
        sp[r + 4, r:r + 4] = True
    m[30:70, 100:140][sp] = 0.95
    for kind in ("fp16", "bf16"):
        m16 = as_16bit(m, kind)
        tt = np.float32(np.asarray(m16, np.float32)[41, 61])
        boxes, conf = check_page(m16, np.float32(0.35), tt)
        mask = (np.asarray(m16, np.float32) > 0.35).astype(np.uint8)
        t = text_box_tables(m16, mask, tt)
        assert t["count"] == len(boxes) == 10
        diamonds, parity = branches(t)
        assert diamonds >= 2 and parity == {0, 1}
        assert tt in t["peak"][:t["count"]]
        lab, n = raster_labels(mask)
        assert n == 11                  # the area-9 line is the only one dropped


def test_empty_and_full_masks():
    for kind in ("fp16", "bf16"):
        m = as_16bit(np.full((64, 96), 0.2, np.float32), kind)
        assert check_page(m, np.float32(0.35), np.float32(0.6)) == ([], [])
        m = as_16bit(np.full((64, 96), 0.7, np.float32), kind)
        boxes, conf = check_page(m, np.float32(0.35), np.float32(0.6))
        assert len(boxes) == 1 and conf == [np.float32(1.0)]


def test_overflow_is_flagged():
    rng = np.random.default_rng(3)
    m = synth_map(rng, 128, 128)
    m[10:14, 5:100] = m[40:44, 5:100] = 0.9
    m16 = as_16bit(m, "fp16")
    mask = (m16.astype(np.float32) > 0.35).astype(np.uint8)
    full = text_box_tables(m16, mask, 0.6)
    assert full["count"] >= 2 and not full["overflow"]
    assert text_box_tables(m16, mask, 0.6, max_boxes=full["count"] - 1)["overflow"]
    used = int(full["box"][full["count"] - 1, 4] + full["box"][full["count"] - 1, 5])
    assert text_box_tables(m16, mask, 0.6, max_points=used - 1)["overflow"]
    assert not text_box_tables(m16, mask, 0.6, max_boxes=full["count"], max_points=used)["overflow"]


def _noisy_masks(seed, n, lo=5, hi=80):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        H, W = rng.integers(lo, hi, 2)
        yield (rng.uniform(size=(H, W)) < rng.uniform(0.2, 0.75)).astype(np.uint8)


def test_fact_raster_order_labels():
    """cv2.connectedComponentsWithStats(connectivity=4) numbers components in raster order of their first pixel."""
    for mask in list(_noisy_masks(1, 300)) + list(_noisy_masks(2, 3, 900, 1100)):
        cnt, lab, _, _ = cv2.connectedComponentsWithStats(mask, connectivity=4)
        ref, n = raster_labels(mask)
        assert n == cnt - 1 and np.array_equal(lab, ref)


def _components(seed, n, min_area=1):
    for mask in _noisy_masks(seed, n):
        H, W = mask.shape
        cnt, lab, st, _ = cv2.connectedComponentsWithStats(mask, connectivity=4)
        for k in range(1, cnt):
            x, y, w, h, area = (int(v) for v in st[k])
            if area < min_area:
                continue
            ks = ks_of(w, h)
            sx, sy, ex, ey = max(0, x - ks), max(0, y - ks), min(W, x + w + ks), min(H, y + h + ks)
            comp = lab[sy:ey, sx:ex] == k
            seg = cv2.dilate(comp.astype(np.uint8), cv2.getStructuringElement(cv2.MORPH_RECT, (ks, ks)))
            rows = comp[y - sy:y - sy + h, x - sx:x - sx + w]
            lo = np.argmax(rows, axis=1) + x
            hi = w - 1 - np.argmax(rows[:, ::-1], axis=1) + x
            yield H, W, x, y, h, ks, sx, sy, seg, lo, hi


def test_fact_dilation_from_row_extents():
    """cv2.dilate's leftmost / rightmost pixel per row follows from the source rows' extents; only image borders clip."""
    n = 0
    for H, W, x, y, h, ks, sx, sy, seg, lo, hi in _components(4, 400):
        yi, xi = np.nonzero(seg)
        y0d, xl, xr = dilated_rows(lo, hi, y, y + h - 1, ks, H, W)
        assert np.array_equal(np.unique(yi) + sy, np.arange(y0d, y0d + len(xl)))
        for r, Y in enumerate(range(y0d, y0d + len(xl))):
            xs = xi[yi == Y - sy] + sx
            assert xs.min() == xl[r] and xs.max() == xr[r]
        n += 1
    assert n > 5000


def test_fact_min_area_rect_over_row_extents():
    """minAreaRect over (xl, Y), (xr, Y) per dilated row gives the boxPoints of minAreaRect over every dilated pixel."""
    n = 0
    for H, W, x, y, h, ks, sx, sy, seg, lo, hi in _components(5, 300, min_area=10):
        yi, xi = np.nonzero(seg)
        ref = cv2.boxPoints(cv2.minAreaRect(np.column_stack((xi + sx, yi + sy)))).tobytes()
        y0d, xl, xr = dilated_rows(lo, hi, y, y + h - 1, ks, H, W)
        Y = np.arange(y0d, y0d + len(xl))
        ext = np.stack([np.column_stack((xl, Y)), np.column_stack((xr, Y))], 1).reshape(-1, 2)
        for dt in (np.int64, np.int32):
            assert cv2.boxPoints(cv2.minAreaRect(ext.astype(dt))).tobytes() == ref
        n += 1
    assert n > 1000
