"""ORACLE TOOLING — the reference's DetectionPredictor over pages of mixed sizes, with a deterministic stub model.

    SURYA_REFERENCE=<checkout> python -m oracle.make_page_sizes_golden     # writes tests/golden/det_page_sizes.pt

The reference's UNMODIFIED DetectionPredictor.__call__ (split_image + ImageOps.pad, prepare_image's PIL thumbnail + resize, its
SegformerImageProcessor, the ×4 upsample, the heatmap stitching and parallel_get_boxes) runs on the CPU over
oracle.page_prep_oracle.DarknessStub.  Per case and page the fixture keeps the uint8 images its pixel_values encode (zlib),
the stitched heatmap size, the polygons, the confidences and image_bbox; tests/test_page_sizes_golden_cpu.py reproduces them
with the repository's host flow.
"""
from __future__ import annotations

import zlib

import numpy as np
import torch

from oracle.make_golden import GOLDEN, ref_shim  # noqa: E402  (make_golden puts the repository on sys.path)


def make_page_sizes_golden():
    from oracle import page_prep_oracle as O
    from surya_b200 import dropin

    ref_shim.install()
    from PIL import Image
    from surya.detection import DetectionPredictor
    from surya.detection.processor import SegformerImageProcessor

    g = {"cases": []}
    for ci, case in enumerate(O.PAGE_SIZES_CASES):
        pw, ph = case["processor"]
        proc = SegformerImageProcessor(size={"height": ph, "width": pw})
        seen = []
        stub = O.DarknessStub(record=seen)
        Stock = type("StockDetectionPredictor", (DetectionPredictor,), {"model_loader_cls": dropin.loader_for(stub, proc)})
        pred = Stock(device="cpu", dtype=torch.float32)
        pred.disable_tqdm = True
        pages = [O.fixture_page(w, h, seed=100 * ci + i) for i, (w, h) in enumerate(case["pages"])]
        res = pred([Image.fromarray(p) for p in pages], batch_size=6, include_maps=True)
        chunks = np.concatenate(seen, 0)                        # [n_chunks, 3, ph, pw] in the predictor's order
        out = {"processor": (pw, ph), "pages": list(case["pages"]), "seeds": [100 * ci + i for i in range(len(pages))],
               "chunks_shape": tuple(chunks.shape), "chunks_u8_zlib": zlib.compress(chunks.tobytes(), 9), "results": []}
        for r in res:
            out["results"].append({"heatmap_size": tuple(r.heatmap.size), "image_bbox": [float(v) for v in r.image_bbox],
                                   "polygons": [[[float(v) for v in pt] for pt in b.polygon] for b in r.bboxes],
                                   "confidences": [float(b.confidence) for b in r.bboxes]})
        g["cases"].append(out)
        print(f"case {ci}: {len(pages)} pages -> {chunks.shape[0]} chunks, lines per page {[len(r['polygons']) for r in out['results']]}")
    torch.save(g, GOLDEN / "det_page_sizes.pt")


if __name__ == "__main__":
    make_page_sizes_golden()
