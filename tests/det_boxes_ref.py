"""NumPy restatement of sb_det_text_boxes' per-page tables (include/surya_b200.h), independent of OpenCV and of the kernels:
scipy's 4-connected labelling numbered in raster order of each component's first pixel, area / bounding box / peak per component,
the keep filter of surya/detection/heatmap.py:43-60, and cv2.dilate's output per row from the source row extents."""
import cv2
import numpy as np
import torch
from scipy import ndimage

MIN_AREA = 10
FOUR = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], dtype=bool)


def raster_labels(mask: np.ndarray):
    """Labels 1..n of the 4-connected components of `mask`, numbered in raster order of their first pixel."""
    lab, n = ndimage.label(mask != 0, structure=FOUR)
    if n == 0:
        return lab, 0
    flat = lab.ravel()
    nz = np.flatnonzero(flat)
    first = np.full(n + 1, flat.size, dtype=np.int64)
    np.minimum.at(first, flat[nz], nz)
    order = np.argsort(first[1:], kind="stable")        # old label - 1 in raster order of first pixels
    remap = np.zeros(n + 1, dtype=np.int32)
    remap[order + 1] = np.arange(1, n + 1, dtype=np.int32)
    return remap[lab], n


def ks_of(w: int, h: int) -> int:
    return int(np.sqrt(min(w, h))) + 1


def dilated_rows(rows_lo, rows_hi, y0: int, y1: int, ks: int, H: int, W: int):
    """Leftmost / rightmost pixel of every row of cv2.dilate(component, ones(ks, ks)) with the default anchor ks // 2, from the
    source rows' extents (rows_lo / rows_hi indexed by y - y0).  Returns (first dilated row, xl array, xr array)."""
    a = ks // 2
    lead = ks - 1 - a
    y0d, y1d = max(0, y0 - lead), min(H - 1, y1 + a)
    xl, xr = [], []
    for Y in range(y0d, y1d + 1):
        s0, s1 = max(y0, Y - a), min(y1, Y - a + ks - 1)
        xl.append(max(0, int(rows_lo[s0 - y0:s1 - y0 + 1].min()) - lead))
        xr.append(min(W - 1, int(rows_hi[s0 - y0:s1 - y0 + 1].max()) + a))
    return y0d, np.array(xl), np.array(xr)


def text_box_tables(line_map: np.ndarray, mask: np.ndarray, text_threshold: float, max_boxes: int = 1024,
                    max_points: int = 65536):
    """One page's tables: {"count", "overflow", "box" [max_boxes, 7], "peak" [max_boxes], "points" [max_points, 2]}; rows past
    count / the last point stay zero.  line_map: 16-bit (fp16 or bf16 widened to fp32) or fp32 map."""
    H, W = mask.shape
    lm = np.asarray(line_map, dtype=np.float32)
    lab, n = raster_labels(mask)
    box = np.zeros((max_boxes, 7), dtype=np.int32)
    peak = np.zeros(max_boxes, dtype=np.float32)
    points = np.zeros((max_points, 2), dtype=np.int32)
    count, used, overflow = 0, 0, 0
    tt = np.float32(text_threshold)
    objs = ndimage.find_objects(lab)
    areas = np.bincount(lab.ravel(), minlength=n + 1)
    for k in range(1, n + 1):
        if areas[k] < MIN_AREA:
            continue
        sl = objs[k - 1]
        comp = lab[sl] == k
        line_max = lm[sl][comp].max()
        if line_max < tt:
            continue
        y0, x0 = sl[0].start, sl[1].start
        h, w = comp.shape
        ks = ks_of(w, h)
        lo = np.argmax(comp, axis=1) + x0
        hi = w - 1 - np.argmax(comp[:, ::-1], axis=1) + x0
        y0d, xl, xr = dilated_rows(lo, hi, y0, y0 + h - 1, ks, H, W)
        rows = len(xl)
        if count < max_boxes and used + 2 * rows <= max_points:
            Y = np.arange(y0d, y0d + rows)
            pts = points[used:used + 2 * rows]
            pts[0::2, 0], pts[0::2, 1], pts[1::2, 0], pts[1::2, 1] = xl, Y, xr, Y
            box[count] = (xl.min(), y0d, xr.max(), y0d + rows - 1, used, 2 * rows, ks)
            peak[count] = line_max
        else:
            overflow = 1
        count += 1
        used += 2 * rows
    return {"count": count, "overflow": overflow, "box": box, "peak": peak, "points": points}


def as_16bit(m: np.ndarray, kind: str) -> np.ndarray:
    """The map as the pipeline hands it to the host finish: float16, or bf16 widened to float32."""
    if kind == "fp16":
        return m.astype(np.float16)
    return torch.from_numpy(m.astype(np.float32)).to(torch.bfloat16).float().numpy()


def synth_map(rng, H, W):
    """Background noise below low_text, text-line rectangles (some cut by the page border), ragged after a blur, plus speckles."""
    m = rng.uniform(0.0, 0.3, (H, W)).astype(np.float32)
    for _ in range(int(rng.integers(0, 12))):
        h, w = int(rng.integers(1, 20)), int(rng.integers(1, W))
        y, x = int(rng.integers(-h // 2, H)), int(rng.integers(-w // 2, W))
        m[max(0, y):y + h, max(0, x):x + w] = rng.uniform(0.4, 0.98)
    if rng.uniform() < 0.5:
        m = cv2.GaussianBlur(m, (5, 5), 0)
    n_sp = int(rng.integers(0, 40))
    m[rng.integers(0, H, n_sp), rng.integers(0, W, n_sp)] = rng.uniform(0.4, 0.9, n_sp)
    return m


def assert_same(got, ref):
    gb, gc = got
    rb, rc = ref
    assert len(gb) == len(rb) and len(gc) == len(rc)
    for p, q in zip(gb, rb):
        assert p.dtype == q.dtype == np.float32 and p.shape == q.shape and p.tobytes() == q.tobytes()
    for p, q in zip(gc, rc):
        assert type(p) is type(q) and np.float32(p).tobytes() == np.float32(q).tobytes()
