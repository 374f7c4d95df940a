"""CPU tests of the layout page flow (surya_b200/layout_pages.py): the preprocessing restatement against cv2, the slicing plan,
the header/footer rule's polygon arithmetic at its boundaries, the slice join, and the host flow over a CPU stand-in engine
against the predictor's post-processing written step by step."""
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import layout_pages_oracle as O
from oracle.preproc_oracle import axis_table
from surya_b200 import layout_pages as LP
from surya_b200.config import layout_default

# The float model of OpenCV's uint8 cubic resize leaves values off by exactly one (oracle/layout_pages_oracle.py); measured
# 5e-6 of the values over the sizes below with opencv-python 4.13.0.
MAX_OFF_BY_ONE_FRACTION = 2e-5


def _page(h, w, seed):
    import cv2

    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return cv2.GaussianBlur(img, (0, 0), 1.5) if min(h, w) > 16 else img


def test_cubic_resize_restatement_vs_cv2():
    import cv2

    rng = np.random.default_rng(7)
    sizes = [(30, 30), (4000, 60), (45, 3900), (1056, 816), (2112, 1632), (768, 768), (300, 500)]
    sizes += [tuple(int(v) for v in rng.integers(30, 4001, 2)) for _ in range(4)]
    total = off = 0
    for i, (h, w) in enumerate(sizes):
        img = _page(h, w, i)
        for dw, dh in ((768, 768), (256, 256)):
            got = O.resize_cubic_u8(img, dw, dh)
            ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_CUBIC)
            d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
            assert d.max() <= 1, (h, w, dw)
            total += d.size
            off += int((d > 0).sum())
    assert off / total <= MAX_OFF_BY_ONE_FRACTION, off / total


def test_cubic_tap_tables_equal_the_oracle_axis_table():
    for src, dst in ((30, 768), (768, 768), (1200, 768), (4000, 768), (3, 256), (1, 768)):
        idx, w = LP.cubic_axis(src, dst)
        ri, rw = axis_table(src, dst, "cubic")
        assert np.array_equal(idx, ri) and np.array_equal(w, rw)


def test_slicer_plan():
    # ImageSlicer.slice / slice_count with LAYOUT_SLICE_MIN 1500, LAYOUT_SLICE_SIZE 1200, 4 slices at most
    assert LP.slice_rects(1500, 1500) == [(0, 0, 1500, 1500, 0, 0)]
    assert LP.slice_count(1400, 900) == 2                 # weight of an unsliced page, as the reference batches it
    assert LP.slice_rects(1501, 900) == [(0, 0, 1200, 900, 0, 0), (1200, 0, 301, 900, 1, 0)]
    assert LP.slice_rects(1700, 1700) == [(0, 0, 1700, 1200, 0, 0), (0, 1200, 1700, 500, 0, 1)]
    r = LP.slice_rects(2000, 6000)
    assert [x[1] for x in r] == [0, 1501, 3002, 4503] and r[-1][3] == 6000 - 4503 and LP.slice_count(2000, 6000) == 4
    for w, h in ((3300, 2550), (1600, 5000), (9000, 1000)):
        rects = LP.slice_rects(w, h)
        assert len(rects) == LP.slice_count(w, h) <= 4
        along = 2 if w > h else 3
        assert sum(x[along] for x in rects) == (w if w > h else h)
    # batch_layout_detection's batching
    assert LP.page_batches([1, 1, 1], 2) == [(0, 2), (2, 3)]
    assert LP.page_batches([2, 4, 1, 1], 4) == [(0, 1), (1, 2), (2, 4)]
    assert LP.page_batches([5], 4) == [(0, 1)]


def _row(cx, cy, w, h, sx=512, sy=512):
    return torch.tensor([cx, cy, w, h, sx, sy], dtype=torch.float64) / 1024


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_row_polygons_follow_the_rounding_points(dtype):
    """The host flow's vectorised polygons give the corners the oracle's one-op-at-a-time rounding model gives (the fixture
    test below pins both to the reference's own polygons)."""
    cfg = layout_default().decoder
    g = torch.Generator().manual_seed(3)
    bbox = torch.rand((300, 6), generator=g).to(dtype).float()
    sizes = torch.randint(50, 5000, (300, 2), generator=g)
    got = LP.row_polygons(bbox, dtype, cfg.bbox_size, cfg.skew_scaler, sizes)
    for i in range(300):
        c0, c2 = O.rule_corners(bbox[i].tolist(), tuple(sizes[i].tolist()), dtype, cfg.bbox_size, cfg.skew_scaler)
        assert tuple(got[i][0]) == c0 and tuple(got[i][2]) == c2


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_rule_at_the_boundaries(dtype):
    """A header whose lower edge lands next to 0.2 of the page height (204.8 of 1024): the model-dtype rounding of the row and of
    the corner decides the outcome, so it differs from the same test in float64 for some boxes."""
    cfg = layout_default().decoder
    header = 10 + cfg.special_token_count
    outcomes, differs = set(), 0
    for H in (997, 1000, 1013, 1500):
        for y2 in np.linspace(200.0, 210.0, 161):
            # centre in [64, 128) and the edge in [128, 256): the edge's sum is rounded to the coarser step of the dtype
            bbox = _row(512, y2 - 100, 300, 200).to(dtype).float()
            fires = O.rule_fires(bbox, header, (1000, H), dtype, cfg)
            poly = LP.row_polygons(bbox[None], dtype, cfg.bbox_size, cfg.skew_scaler, torch.tensor([[1000, H]]))[0]
            assert fires == bool(poly[0][1] < H * .8 and poly[2][1] > H * .2 and poly[0][0] < 800 and poly[2][0] > 200)
            b = bbox.double() * 1024
            exact = (b[1] + b[3] / 2) * H / 1024 > H * .2
            differs += int(fires != bool(exact))
            outcomes.add(fires)
        # left edge next to 0.8 of the width (819.2 of 1024), with a centre on the coarse grid of [512, 1024)
        for w in range(180, 231):
            bbox = _row(920, 512, w, 200).to(dtype).float()
            fires = O.rule_fires(bbox, header, (1000, H), dtype, cfg)
            b = bbox.double() * 1024
            differs += int(fires != bool((b[0] - b[2] / 2) * 1000 / 1024 < 1000 * .8))
            outcomes.add(fires)
    assert outcomes == {True, False} and differs > 0
    # footers fire by the same test; other labels never do, whatever the box
    assert O.rule_fires(_row(512, 512, 300, 80).to(dtype).float(), 9 + cfg.special_token_count, (1000, 1000), dtype, cfg)
    assert not O.rule_fires(_row(512, 512, 300, 80).to(dtype).float(), 4, (1000, 1000), dtype, cfg)
    # near the edges the rule does not fire
    assert not O.rule_fires(_row(512, 40, 900, 60).to(dtype).float(), header, (1000, 1000), dtype, cfg)
    assert not O.rule_fires(_row(512, 990, 900, 60).to(dtype).float(), header, (1000, 1000), dtype, cfg)


def _box(x0, y0, x1, y1, label="Text", pos=0):
    return LP.LayoutBox(polygon=[[x0, y0], [x1, y0], [x1, y1], [x0, y1]], label=label, position=pos)


def test_join_merges_across_slices():
    a = LP.LayoutResult([_box(10, 10, 100, 50), _box(1150, 300, 1199, 400, "Picture", 1)], [0, 0, 1200, 900])
    b = LP.LayoutResult([_box(0, 310, 80, 395, "Figure"), _box(5, 600, 90, 700, "Table", 1)], [0, 0, 400, 900])
    out = LP.join([a, b], [(0, 0, 0), (0, 1, 0)])
    assert len(out) == 1 and out[0].sliced and out[0].image_bbox == [0, 0, 1600, 900]
    assert [x.label for x in out[0].bboxes] == ["Text", "Picture", "Table"]
    assert out[0].bboxes[1].bbox == [1150, 300, 1280, 400] and out[0].bboxes[2].position == 3
    # height-wise: the lower slice's boxes are shifted by the first slice's height
    c = LP.LayoutResult([_box(100, 1100, 400, 1199)], [0, 0, 800, 1200])
    d = LP.LayoutResult([_box(110, 0, 390, 60), _box(0, 500, 10, 600)], [0, 0, 800, 300])
    out = LP.join([c, d, LP.LayoutResult([_box(1, 1, 5, 5)], [0, 0, 50, 50])], [(0, 0, 0), (0, 0, 1), (1, 0, 0)])
    assert len(out) == 2 and out[0].image_bbox == [0, 0, 800, 1500]
    assert out[0].bboxes[0].bbox == [100, 1100, 400, 1260] and out[0].bboxes[1].bbox == [0, 1700, 10, 1800]
    # the reference takes max() over the first slice's positions: an empty first slice raises
    with pytest.raises(ValueError):
        LP.join([LP.LayoutResult([], [0, 0, 10, 10]), d], [(0, 0, 0), (0, 0, 1)])


GOLDEN = Path(__file__).resolve().parent / "golden" / "layout_pages.pt"


def _golden():
    g = torch.load(GOLDEN)
    case = g["case"]
    pages = [O.fixture_page(w, h, case["seed"] + i) for i, (w, h) in enumerate(case["pages"])]
    px = torch.frombuffer(bytearray(zlib.decompress(g["pixels_f16_zlib"])), dtype=torch.float16).reshape(g["pixels_shape"])
    return g, pages, px


def test_slicer_plan_vs_reference_fixture():
    g, pages, _ = _golden()
    sizes, positions = [], []
    for i, p in enumerate(pages):
        for x0, y0, sw, sh, tx, ty in LP.slice_rects(p.shape[1], p.shape[0]):
            sizes.append((sw, sh))
            positions.append((i, tx, ty))
    assert sizes == g["slice_sizes"] and positions == g["tile_positions"]
    assert {tx for _, tx, _ in positions} != {0} and {ty for _, _, ty in positions} != {0}      # cuts along both axes


def test_preprocessing_vs_reference_processor_fixture():
    """The restatement against what SuryaEncoderImageProcessor + the predictor's fp16 cast produced: equal except where the
    cubic resize is off by one (the stated bound)."""
    g, pages, px = _golden()
    H, W = px.shape[2:]
    k, diff_n, total = 0, 0, 0
    for p in pages:
        for x0, y0, sw, sh, _, _ in LP.slice_rects(p.shape[1], p.shape[0]):
            got = O.process(p[y0:y0 + sh, x0:x0 + sw], (H, W), torch.float16)
            d = (got.float() - px[k].float()).abs()
            assert d.max() <= 2 / 255 + 1e-3
            diff_n += int((d > 0).sum())
            total += d.numel()
            k += 1
    assert diff_n / total <= MAX_OFF_BY_ONE_FRACTION


def test_host_flow_vs_reference_fixture():
    """layout_pages over the stub engine, fed the reference processor's pixel values, reproduces every LayoutResult that the
    reference's LayoutPredictor produced over the same stub decoder: header/footer relabelling (also to a special token, whose
    box is dropped), rows that stop at different steps or never, polygons, top-k, confidence, positions, clean_boxes and the
    width- and height-wise slice joins."""
    g, pages, px = _golden()
    cfg = layout_default()
    eng = O.StubLayoutEngine(cfg, dtype=torch.float16, max_batch=g["case"]["batch_size"])
    run = LP.layout_pages(eng, pages, batch_size=g["case"]["batch_size"], pixel_values=px)
    assert eng.rule_count > 0 and any(n < cfg.decoder.max_boxes for n in run.steps_run)
    assert any(n == cfg.decoder.max_boxes for n in run.steps_run)
    assert len(run.results) == len(g["results"])
    for got, want in zip(run.results, g["results"]):
        assert got.image_bbox == want["image_bbox"] and got.sliced == want["sliced"]
        assert [(b.polygon, b.label, b.position, b.top_k, b.confidence) for b in got.bboxes] == \
               [(b["polygon"], b["label"], b["position"], b["top_k"], b["confidence"]) for b in want["boxes"]]
    # the joins merged boxes across the cuts in both directions
    spans = {"x": False, "y": False}
    for (w, h), res in zip(g["case"]["pages"], g["results"]):
        for x0, y0, sw, sh, tx, ty in LP.slice_rects(w, h)[1:]:
            for b in res["boxes"]:
                xs, ys = [p[0] for p in b["polygon"]], [p[1] for p in b["polygon"]]
                spans["x"] |= tx > 0 and min(xs) < x0 < max(xs)
                spans["y"] |= ty > 0 and min(ys) < y0 < max(ys)
    assert spans == {"x": True, "y": True}


def test_errors_are_loud():
    from surya_b200._lib import SuryaB200Error

    cfg = layout_default()
    eng = O.StubLayoutEngine(cfg, max_batch=4)
    with pytest.raises(SuryaB200Error, match="at least one page"):
        LP.layout_pages(eng, [], batch_size=4)
    with pytest.raises(SuryaB200Error, match="uint8"):
        LP.layout_pages(eng, [np.zeros((10, 10, 3), np.float32)], batch_size=4)
    with pytest.raises(SuryaB200Error, match="uint8"):
        LP.layout_pages(eng, [np.zeros((10, 10, 4), np.uint8)], batch_size=4)
    with pytest.raises(SuryaB200Error, match="max_batch"):
        LP.layout_pages(eng, [np.zeros((10, 10, 3), np.uint8)], batch_size=5)
