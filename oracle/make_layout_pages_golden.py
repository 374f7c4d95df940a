"""ORACLE TOOLING — the reference's LayoutPredictor over pages of mixed sizes, with a deterministic stub model.

    SURYA_REFERENCE=<checkout> python -m oracle.make_layout_pages_golden     # writes tests/golden/layout_pages.pt

The reference's UNMODIFIED LayoutPredictor.batch_layout_detection (ImageSlicer.slice / join, its SuryaEncoderImageProcessor,
the decode loop with the header/footer rule and the stop rule, prediction_to_polygon, top-k, clean_boxes) runs on the CPU in
fp16 over a stub model whose decoder answers oracle.layout_pages_oracle.stub_outputs for (row order number, step, fed class).
The fixture keeps the case, the pixel values the processor produced (fp16, zlib), each image's size and tile position, and the
full LayoutResults; tests/test_layout_pages_cpu.py reproduces them with the repository's slicer, preprocessing restatement and
host flow.
"""
from __future__ import annotations

import zlib

import numpy as np
import torch

from oracle.make_golden import GOLDEN, ref_shim  # noqa: E402  (make_golden puts the repository on sys.path)


def make_layout_pages_golden():
    from oracle import layout_pages_oracle as O
    from surya_b200 import dropin
    from surya_b200.config import layout_default

    ref_shim.install()
    from PIL import Image
    from surya.common.donut.processor import SuryaEncoderImageProcessor
    from surya.layout import LayoutPredictor
    from surya.settings import settings

    case = O.LAYOUT_PAGES_CASE
    d = layout_default().decoder
    seen, sizes = [], []

    class _Ns:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    dec_cfg = _Ns(**d.__dict__)
    state = {"rows": 0, "step": 0}

    class _Inner:
        def _setup_cache(self, config, batch, device, dtype):
            state["step"] = 0

        def _clear_cache(self):
            pass

    class _Decoder:
        config = dec_cfg
        model = _Inner()

        def __call__(self, input_boxes=None, encoder_hidden_states=None, cache_position=None, use_cache=True, prefill=False, **kw):
            if prefill:
                state["step"] = 0
            prev = input_boxes[:, -1, 6].tolist()
            outs = [O.stub_outputs(int(r), state["step"], int(p), d.special_token_count, d.label_count, d.eos_token_id)
                    for r, p in zip(encoder_hidden_states.tolist(), prev)]
            state["step"] += 1
            bbox = torch.tensor([o[0] for o in outs], dtype=torch.float16)[:, None]
            cls = torch.tensor([o[1] for o in outs], dtype=torch.float16)[:, None]
            return {"bbox_logits": bbox, "class_logits": cls}

    class _Model:
        device, dtype = torch.device("cpu"), torch.float16
        config = _Ns(decoder=dec_cfg)
        decoder = _Decoder()

        def encoder(self, pixel_values=None, **kw):
            seen.append(pixel_values.clone())
            n = pixel_values.shape[0]
            ids = torch.arange(state["rows"], state["rows"] + n)
            state["rows"] += n
            return (ids,)

        def to(self, *a, **k):
            return self

        def eval(self):
            return self

    proc = SuryaEncoderImageProcessor(max_size=settings.LAYOUT_IMAGE_SIZE)
    Stock = type("StockLayoutPredictor", (LayoutPredictor,), {"model_loader_cls": dropin.loader_for(_Model(), proc)})
    pred = Stock(device="cpu", dtype=torch.float16)
    pred.disable_tqdm = True
    pages = [O.fixture_page(w, h, case["seed"] + i) for i, (w, h) in enumerate(case["pages"])]
    # the slices the predictor cuts, from its own slicer
    from surya.layout.slicer import ImageSlicer
    slicer = ImageSlicer(settings.LAYOUT_SLICE_MIN, settings.LAYOUT_SLICE_SIZE)
    imgs = [Image.fromarray(p) for p in pages]
    slices, positions = slicer.slice(imgs)
    res = pred(imgs, batch_size=case["batch_size"], top_k=5)
    px = torch.cat(seen, 0)
    assert px.dtype == torch.float16 and px.shape[0] == len(slices)
    g = {"case": dict(case), "pixels_shape": tuple(px.shape), "pixels_f16_zlib": zlib.compress(px.numpy().tobytes(), 9),
         "slice_sizes": [tuple(s.size) for s in slices], "tile_positions": [tuple(p) for p in positions], "results": []}
    for r in res:
        g["results"].append({"image_bbox": [float(v) for v in r.image_bbox], "sliced": bool(r.sliced),
                             "boxes": [{"polygon": [[float(v) for v in pt] for pt in b.polygon], "label": b.label,
                                        "position": int(b.position), "top_k": {k: float(v) for k, v in b.top_k.items()},
                                        "confidence": float(b.confidence)} for b in r.bboxes]})
    torch.save(g, GOLDEN / "layout_pages.pt")
    print(f"{len(pages)} pages -> {len(slices)} images, boxes per page {[len(r['boxes']) for r in g['results']]}, "
          f"sliced {[r['sliced'] for r in g['results']]}, {len(g['pixels_f16_zlib'])} bytes of pixels")


if __name__ == "__main__":
    make_layout_pages_golden()
