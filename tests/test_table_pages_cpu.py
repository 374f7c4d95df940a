"""CPU tests of the table page flow (surya_b200/table_pages.py, table_rec.table_results) against tests/golden/table_pages.pt, which
the reference's own table_recognition CLI wrote over stub models: the crop plan, the preprocessing restatement of the crops
(zero fill past the page included), the geometry of decode_batch_predictions, and the whole host flow over CPU stand-in
engines, dict for dict against the CLI's results.json."""
import json
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import layout_pages_oracle as LPO
from oracle import table_pages_oracle as T
from surya_b200 import layout_pages as LP
from surya_b200 import table_pages as TP
from surya_b200._lib import SuryaB200Error
from surya_b200.config import layout_default, table_tiny
from surya_b200.table_rec import table_results

GOLDEN = Path(__file__).resolve().parent / "golden" / "table_pages.pt"
MAX_OFF_BY_ONE_FRACTION = 2e-5         # the bound tests/test_layout_pages_cpu.py pins the cubic restatement to against cv2


@pytest.fixture(scope="module")
def golden():
    g = torch.load(GOLDEN, weights_only=False)
    lo, hi = T.case_pages(g["case"])
    return g, lo, hi


def _pixels(run):
    return torch.frombuffer(bytearray(zlib.decompress(run["pixels_f16_zlib"])), dtype=torch.float16).reshape(run["pixels_shape"])


def _layout(run):
    return [LP.LayoutResult([LP.LayoutBox(polygon=b["polygon"], label=b["label"], position=b["position"], top_k=b["top_k"],
                                          confidence=b["confidence"]) for b in r["boxes"]], r["image_bbox"], r["sliced"])
            for r in run["layout"]]


def _sizes(case):
    return [lo for _, lo, _ in case["pages"]], [hi for _, _, hi in case["pages"]]


def test_fixture_covers_the_cases(golden):
    g, _, _ = golden
    d = g["detect"]
    per_page = [sum(b["label"] in TP.TABLE_LABELS for b in r["boxes"]) for r in d["layout"]]
    assert 0 in per_page and max(per_page) >= 2 and any(r["sliced"] for r in d["layout"])
    assert len(d["crop_boxes"]) > d["table_batch_size"]
    hi = [s for _, _, s in g["case"]["pages"]]
    assert any(b[2] > hi[0][0] and b[3] > hi[0][1] for b in d["crop_boxes"][:2])            # past the right and bottom edges
    assert any(v % 1 == 0.5 for b in d["crop_boxes"] for v in b)                            # .5 coordinates
    cells = [c for v in d["results_json"].values() for t in v for c in t["cells"]]
    assert any(c["colspan"] > 1 for c in cells) and any(c["rowspan"] > 1 for c in cells)
    merges = {(c["merge_up"], c["merge_down"]) for v in d["results_json"].values() for t in v for c in t["unmerged_cells"]}
    assert merges == {(False, False), (True, False), (False, True), (True, True)}
    rows = [r for v in d["results_json"].values() for t in v for r in t["rows"] + t["cols"]]
    assert {r["is_header"] for r in rows} == {True, False}


def test_crop_rounding_is_round_half_to_even():
    assert TP.expand_bbox([150, 150, 50, 50]) == [148.5, 148.5, 50.5, 50.5]
    assert TP.crop_box([148.5, 49.5, 50.5, 151.5]) == (148, 50, 50, 152)
    assert TP.rescale_bbox([75.9, 10.0, 125.5, 99.99], (1000, 800), (2000, 1200)) == [151, 15, 251, 149]


def test_crop_plan_vs_reference_fixture(golden):
    g, _, _ = golden
    lo, hi = _sizes(g["case"])
    plan = TP.plan_tables(_layout(g["detect"]), lo, hi)
    assert [tp.box for tp in plan] == g["detect"]["crop_boxes"]
    got = [(tp.size[0], tp.size[1]) for tp in plan]
    want = [(int(t["image_bbox"][2]), int(t["image_bbox"][3])) for v in g["detect"]["results_json"].values() for t in v]
    assert sorted(got) == sorted(want)
    skip = TP.plan_tables(None, lo, hi)
    assert [tp.crop for tp in skip] == [(0, 0, w, h) for w, h in hi]


def test_crop_zero_fill_is_pil_crop(golden):
    from PIL import Image

    g, _, hi = golden
    lo_s, hi_s = _sizes(g["case"])
    for tp in TP.plan_tables(_layout(g["detect"]), lo_s, hi_s):
        want = np.asarray(Image.fromarray(hi[tp.page]).crop(tp.box))
        assert np.array_equal(T.crop_zero_fill(hi[tp.page], tp.crop), want)
    page = hi[0][:10, :10]
    assert np.array_equal(T.crop_zero_fill(page, (-3, -2, 6, 12)), np.asarray(Image.fromarray(page).crop((-3, -2, 6, 12))))


@pytest.mark.parametrize("which", ["detect", "skip"])
def test_preprocessing_vs_reference_processor_fixture(golden, which):
    """PIL's zero-filled crop, the cubic restatement and the normalisation against what SuryaTableRecProcessor produced (after
    the predictor's fp16 cast): equal except where the cubic resize is off by one.  The job-table restatement of the bounded
    jobs the flow writes equals the crop restatement byte for byte."""
    g, lo, hi = golden
    run = g[which]
    px = _pixels(run)
    lo_s, hi_s = _sizes(g["case"])
    plan = TP.plan_tables(None if which == "skip" else _layout(run), lo_s, hi_s)
    assert len(plan) == px.shape[0]
    H, W = px.shape[2:]
    diff_n = total = 0
    for k, tp in enumerate(plan):
        got = LPO.process(T.crop_zero_fill(hi[tp.page], tp.crop), (H, W), torch.float16)
        d = (got.float() - px[k].float()).abs()
        assert d.max() <= 2 / 255 + 1e-3
        diff_n += int((d > 0).sum())
        total += d.numel()
        jobs, ti, tw = LP.plan_jobs([(tp.crop[0], tp.crop[1], tp.size[0], tp.size[1])], [0], [hi_s[tp.page][0]], (H, W),
                                    page_h=[hi_s[tp.page][1]])
        assert torch.equal(T.preprocess_jobs(hi[tp.page], jobs, ti, tw, (H, W), torch.float16)[0], got)
    assert diff_n / total <= MAX_OFF_BY_ONE_FRACTION


@pytest.mark.parametrize("which", ["detect", "skip"])
def test_geometry_vs_reference_fixture(golden, which):
    """table_results over the pass predictions the reference handed to decode_batch_predictions gives its TableResults."""
    g, _, _ = golden
    run = g[which]
    got = []
    for d in run["decodes"]:
        got.extend(r.to_dict() for r in table_results(d["rowcol"], d["cells"], d["idx_map"], d["orig_sizes"]))
    want = [{k: v for k, v in t.items() if k not in ("page", "table_idx")} for v in run["results_json"].values() for t in v]
    key = lambda t: (t["image_bbox"], len(t["rows"]))              # noqa: E731  (results.json groups the tables by name)
    assert sorted(json.loads(json.dumps(got)), key=key) == sorted(want, key=key)
    assert json.loads(json.dumps(got)) == got                         # floats and plain types, as model_dump gives them


def _results_json(case, run):
    """The CLI's results.json from a TablePagesRun."""
    out, pnum, prev = {}, [], None
    for name, _, _ in case["pages"]:
        pnum.append(0 if name != prev else pnum[-1] + 1)
        prev = name
    for p, ((name, _, _), res) in enumerate(zip(case["pages"], run.results)):
        for i, r in enumerate(res):
            out.setdefault(name, []).append(dict(r.to_dict(), page=pnum[p] + 1, table_idx=i))
    return json.loads(json.dumps(out))


@pytest.mark.parametrize("which", ["detect", "skip"])
def test_host_flow_vs_reference_fixture(golden, which):
    """table_pages over the CPU stand-in engines (layout and table stubs with LayoutEngine's surface, preprocessing by the
    job-table restatement) reproduces the CLI's results.json, its layout results and crop boxes."""
    g, lo, hi = golden
    run = g[which]
    lay = T.StubPagesLayoutEngine(layout_default(), dtype=torch.float16, max_batch=run["layout_batch_size"])
    tab = T.StubTableEngine(table_tiny(), dtype=torch.float16, max_batch=run["table_batch_size"])
    skip = which == "skip"
    res = TP.table_pages(tab, lo, None if skip else lay, highres_pages=hi, skip_table_detection=skip,
                         batch_size=run["table_batch_size"], layout_batch_size=run["layout_batch_size"])
    assert _results_json(g["case"], res) == run["results_json"]
    if skip:
        assert res.layout is None
    else:
        assert [[b["polygon"] for b in r["boxes"]] for r in run["layout"]] == [[b.polygon for b in r.bboxes] for r in res.layout]
        assert [b for page in res.table_boxes for b in page] == run["crop_boxes"]
    px = torch.cat(tab.encoded)
    want = _pixels(run)
    assert px.shape == want.shape and float((px.float() - want.float()).abs().max()) <= 2 / 255 + 1e-3
    assert len(tab.encoded) == -(-px.shape[0] // run["table_batch_size"]) and set(res.timing) == {"upload", "preprocess", "encoder", "passes", "geometry"}


def test_errors_are_loud(golden):
    g, lo, hi = golden
    tab = T.StubTableEngine(table_tiny(), max_batch=8)
    lay = T.StubPagesLayoutEngine(layout_default(), max_batch=4)
    with pytest.raises(SuryaB200Error, match="high-resolution"):
        TP.table_pages(tab, lo, lay, highres_pages=hi[:-1], batch_size=8, layout_batch_size=4)
    with pytest.raises(SuryaB200Error, match="uint8"):
        TP.table_pages(tab, [p.astype(np.float32) for p in lo], lay, batch_size=8, layout_batch_size=4)
    with pytest.raises(SuryaB200Error, match="uint8"):
        TP.table_pages(tab, lo, lay, highres_pages=[None, hi[1][..., :2], None, None, None], batch_size=8, layout_batch_size=4)
    with pytest.raises(SuryaB200Error, match="layout engine"):
        TP.table_pages(tab, lo, None, batch_size=8)
    with pytest.raises(SuryaB200Error, match="table_rec engine"):
        TP.table_pages(lay, lo, lay, batch_size=8)
    with pytest.raises(SuryaB200Error, match="max_batch"):
        TP.table_pages(tab, lo, skip_table_detection=True, batch_size=9)
    with pytest.raises(SuryaB200Error, match="pixel values"):
        TP.table_pages(tab, lo, skip_table_detection=True, batch_size=8, pixel_values=torch.zeros(2, 3, 256, 256))
    # a table box that rounds to an empty crop: the reference fails inside cv2
    thin = LP.LayoutResult([LP.LayoutBox(polygon=[[10, 5], [10.2, 5], [10.2, 50], [10, 50]], label="Table", position=0)], [0, 0, 100, 100])
    with pytest.raises(SuryaB200Error, match="page 0, table box 0"):
        TP.plan_tables([thin], [(100, 100)], [(100, 100)])
