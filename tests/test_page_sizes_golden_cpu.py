"""The host flow over pages of mixed sizes against tests/golden/det_page_sizes.pt, the reference DetectionPredictor's own
output over a deterministic stub model (oracle/make_page_sizes_golden.py): the split plan, the ImageOps.pad padding and the PIL
resize (the uint8 images the predictor's pixel_values encode), the heatmap stitching (stitched heatmap size), and the polygons,
confidences and image_bbox of parallel_get_boxes in page coordinates — all exactly."""
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import det_oracle as D
from oracle import page_prep_oracle as O
from surya_b200 import page_prep as pp
from surya_b200.synth import det_normalize

GOLDEN = Path(__file__).resolve().parent / "golden" / "det_page_sizes.pt"


def _host_flow(pages, processor_size):
    """split + prepare_image (NumPy restatement), processor normalisation, stub model, ×4 bilinear upsample, stitching,
    dynamic thresholds, boxes, rescale to the page."""
    from surya_b200.detection import text_boxes_from_front
    from surya_b200.pipeline import page_polygons

    pw, ph = processor_size
    chunks, results = [], []
    for img in pages:
        parts, heights = O.split_page(img, ph)
        u8 = np.stack([O.prepare_image(c, processor_size) for c in parts])
        chunks.append(u8.transpose(0, 3, 1, 2))
        logits = O.DarknessStub()(det_normalize(u8)).logits
        heat = F.interpolate(logits, size=[ph, pw], mode="bilinear", align_corners=False).float().numpy()[:, 0]
        m = O.stitch(list(heat), heights, ph)
        tt, low, _ = D.dynamic_thresholds(m)
        boxes, conf = text_boxes_from_front(m, (m > low).astype(np.uint8), float(tt), float(low))
        polys, conf = page_polygons(boxes, conf, (img.shape[1], img.shape[0]), (pw, m.shape[0]))
        results.append({"heatmap_size": (pw, m.shape[0]), "image_bbox": [0.0, 0.0, float(img.shape[1]), float(img.shape[0])],
                        "polygons": [[[float(v) for v in pt] for pt in p] for p in polys], "confidences": [float(c) for c in conf]})
    return np.concatenate(chunks, 0), results


@pytest.mark.parametrize("case", range(len(O.PAGE_SIZES_CASES)))
def test_host_flow_reproduces_reference_predictor(case):
    g = torch.load(GOLDEN, weights_only=False)["cases"][case]
    assert g["processor"] == O.PAGE_SIZES_CASES[case]["processor"] and g["pages"] == O.PAGE_SIZES_CASES[case]["pages"]
    pages = [O.fixture_page(w, h, seed=s) for (w, h), s in zip(g["pages"], g["seeds"])]
    ref_chunks = np.frombuffer(zlib.decompress(g["chunks_u8_zlib"]), np.uint8).reshape(g["chunks_shape"])
    chunks, results = _host_flow(pages, g["processor"])
    assert chunks.shape == ref_chunks.shape and np.array_equal(chunks, ref_chunks)
    plan = pp.plan_pages([(p.shape[1], p.shape[0]) for p in pages], g["processor"])
    assert len(plan.chunks) == ref_chunks.shape[0]
    assert [int(r) for r in plan.page_tab[:, 1]] == [r["heatmap_size"][1] for r in g["results"]]
    assert sum(len(r["polygons"]) for r in g["results"]) > 0
    for got, ref in zip(results, g["results"]):
        assert got == ref
