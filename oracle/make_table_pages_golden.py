"""ORACLE TOOLING — the reference's table_recognition CLI over pages with a high-resolution copy, with deterministic stub models.

    SURYA_REFERENCE=<checkout> python -m oracle.make_table_pages_golden     # writes tests/golden/table_pages.pt

The reference's UNMODIFIED table_recognition_cli callback (surya/scripts/table_recognition.py:26-127) runs on the CPU twice,
without and with skip_table_detection.  Three names of its module are replaced: CLILoader by a loader that hands out the
case's pages, their high-resolution copies, names and a temporary result path (save_images False); LayoutPredictor and
TableRecPredictor by subclasses whose model_loader_cls (surya_b200.dropin.loader_for) returns stub models.  The layout stub
answers oracle.table_pages_oracle.layout_outputs, the table stub table_outputs, each by (row, step) only.  The layout
predictor keeps its SuryaEncoderImageProcessor and slicer; the table predictor keeps the real SuryaTableRecProcessor with a real
SuryaEncoderImageProcessor at the tiny table config's encoder size, the code the device flow replaces.

The fixture keeps, per run: the results.json the CLI wrote, every LayoutResult, every expanded crop box (the CLI's
highres_bbox, recorded from Image.crop), the arguments of every decode_batch_predictions call, and the pixel values the table processor produced (fp16 after the predictor's cast,
zlib), which tests/test_table_pages_cpu.py reproduces with the repository's crop plan, preprocessing restatement and host flow.
"""
from __future__ import annotations

import copy
import json
import tempfile
import zlib
from pathlib import Path

import torch

from oracle.make_golden import GOLDEN, ref_shim  # noqa: E402  (make_golden puts the repository on sys.path)


class _Ns:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _layout_model(T, d):
    """The stub layout model: the encoder hands out the rows' order numbers, the decoder answers T.layout_outputs."""
    state = {"rows": 0, "step": 0}
    dec_cfg = _Ns(**d.__dict__)

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
            outs = [T.layout_outputs(int(r), state["step"], d.special_token_count, d.label_count, d.eos_token_id)
                    for r in encoder_hidden_states.tolist()]
            state["step"] += 1
            bbox = torch.tensor([o[0] for o in outs], dtype=torch.float16)[:, None]
            cls = torch.tensor([o[1] for o in outs], dtype=torch.float16)[:, None]
            return {"bbox_logits": bbox, "class_logits": cls}

    class _Model:
        device, dtype = torch.device("cpu"), torch.float16
        config = _Ns(decoder=dec_cfg)
        decoder = _Decoder()

        def encoder(self, pixel_values=None, **kw):
            n = pixel_values.shape[0]
            ids = torch.arange(state["rows"], state["rows"] + n)
            state["rows"] += n
            return (ids,)

        def to(self, *a, **k):
            return self

        def eval(self):
            return self

    return _Model()


def _table_model(T, d, seen):
    """The stub table model: the encoder records its pixel values and hands out the tables' order numbers; the decoder keys
    every row at its prefill by (table, row query) and answers T.table_outputs."""
    state = {"tables": 0, "keys": [], "step": 0}
    dec_cfg = _Ns(**d.__dict__)

    class _Inner:
        def _setup_cache(self, config, batch, device, dtype):
            state["step"] = 0

    class _Decoder:
        config = dec_cfg
        model = _Inner()

        def __call__(self, input_ids=None, encoder_hidden_states=None, cache_position=None, use_cache=True, prefill=False, **kw):
            if prefill:
                state["step"] = 0
                state["keys"] = [(int(t), T.prompt_row_cy(p, d.special_token_count))
                                 for t, p in zip(encoder_hidden_states.tolist(), input_ids)]
            outs = [T.table_head_logits(T.table_outputs(t, cy, state["step"]), d) for t, cy in state["keys"]]
            state["step"] += 1
            names = ("bbox", "category", "merges", "colspan", "is_header")
            return {"box_property_logits": {k: torch.tensor([o[i] for o in outs], dtype=torch.float32)[:, None]
                                            for i, k in enumerate(names)}}

    class _Model:
        device, dtype = torch.device("cpu"), torch.float16
        config = _Ns(decoder=dec_cfg)
        decoder = _Decoder()

        def encoder(self, pixel_values=None, **kw):
            seen.append(pixel_values.clone())
            n = pixel_values.shape[0]
            ids = torch.arange(state["tables"], state["tables"] + n)
            state["tables"] += n
            return _Ns(last_hidden_state=ids)

        def to(self, *a, **k):
            return self

    return _Model()


def run_cli(skip_table_detection: bool):
    from oracle import table_pages_oracle as T
    from surya_b200 import dropin
    from surya_b200.config import layout_default, table_tiny

    ref_shim.install()
    from PIL import Image
    import surya.scripts.table_recognition as cli
    from surya.common.donut.processor import SuryaEncoderImageProcessor
    from surya.layout import LayoutPredictor
    from surya.settings import settings
    from surya.table_rec import TableRecPredictor
    from surya.table_rec.processor import SuryaTableRecProcessor
    from surya.table_rec.shaper import LabelShaper

    case = T.TABLE_PAGES_CASE
    lo, hi = T.case_pages(case)
    tcfg = table_tiny()
    th, tw = tcfg.encoder.image_size
    seen, layouts, crops = [], [], []
    tmp = tempfile.TemporaryDirectory()

    class _Loader:
        def __init__(self, filepath, cli_options, highres=False):
            self.images = [Image.fromarray(p) for p in lo]
            self.highres_images = [_CropRecorder.wrap(Image.fromarray(p)) for p in hi]
            self.names = [n for n, _, _ in case["pages"]]
            self.result_path = tmp.name
            self.save_images = False

    class _CropRecorder(Image.Image):
        """A PIL image whose crop() records its box before cropping as PIL does."""

        @classmethod
        def wrap(cls, im):
            im.__class__ = cls
            return im

        def crop(self, box=None):
            crops.append([float(v) for v in box])
            return Image.Image.crop(self, box)

    lay_proc = SuryaEncoderImageProcessor(max_size=settings.LAYOUT_IMAGE_SIZE)
    Lay = type("StubLayoutPredictor", (LayoutPredictor,), {"model_loader_cls": dropin.loader_for(_layout_model(T, layout_default().decoder),
                                                                                                  lay_proc)})
    orig_layout_call = LayoutPredictor.__call__

    def layout_call(self, images, *a, **k):
        res = orig_layout_call(self, images, *a, **k)
        layouts.extend(res)
        return res

    Lay.__call__ = layout_call

    proc = SuryaTableRecProcessor.__new__(SuryaTableRecProcessor)
    ip = SuryaEncoderImageProcessor(max_size={"height": th, "width": tw})
    ip.do_align_long_axis = False
    proc.image_processor, proc.box_size, proc.special_token_count, proc.shaper = ip, (1024, 1024), 5, LabelShaper()
    proc.token_pad_id, proc.token_eos_id, proc.token_bos_id, proc.token_query_end_id = 0, 1, 1, 4
    decodes = []

    def decode_batch_predictions(self, rowcol, cells, orig_sizes, idx_map, shaper):
        decodes.append({"rowcol": copy.deepcopy(rowcol), "cells": copy.deepcopy(cells), "idx_map": list(idx_map),
                        "orig_sizes": [tuple(s) for s in orig_sizes]})
        return TableRecPredictor.decode_batch_predictions(self, rowcol, cells, orig_sizes, idx_map, shaper)

    Tab = type("StubTableRecPredictor", (TableRecPredictor,), {"model_loader_cls": dropin.loader_for(_table_model(T, tcfg.decoder, seen), proc),
                                                               "decode_batch_predictions": decode_batch_predictions})

    saved = (cli.CLILoader, cli.LayoutPredictor, cli.TableRecPredictor)
    cli.CLILoader, cli.LayoutPredictor, cli.TableRecPredictor = _Loader, Lay, Tab
    try:
        cli.table_recognition_cli.callback(input_path="unused", skip_table_detection=skip_table_detection)
        results = json.loads((Path(tmp.name) / "results.json").read_text())
    finally:
        cli.CLILoader, cli.LayoutPredictor, cli.TableRecPredictor = saved
        tmp.cleanup()
    px = torch.cat(seen, 0)
    assert px.dtype == torch.float16
    return {"results_json": results, "crop_boxes": crops, "decodes": decodes,
            "layout": [{"image_bbox": [float(v) for v in r.image_bbox], "sliced": bool(r.sliced),
                        "boxes": [{"polygon": [[float(v) for v in pt] for pt in b.polygon], "label": b.label, "position": int(b.position),
                                   "top_k": {k: float(v) for k, v in b.top_k.items()}, "confidence": float(b.confidence)}
                                  for b in r.bboxes]} for r in layouts],
            "table_batch_size": Tab(device="cpu").get_batch_size(), "layout_batch_size": Lay(device="cpu").get_batch_size(),
            "pixels_shape": tuple(px.shape), "pixels_f16_zlib": zlib.compress(px.numpy().tobytes(), 9)}


def make_table_pages_golden():
    from oracle import table_pages_oracle as T

    g = {"case": dict(T.TABLE_PAGES_CASE), "detect": run_cli(False), "skip": run_cli(True),
         "meta": {"reference": "VikParuchuri/surya@80e9a7e table_recognition_cli, CPU, fp16 stub models", "torch": str(torch.__version__)}}
    torch.save(g, GOLDEN / "table_pages.pt")
    for k in ("detect", "skip"):
        r = g[k]
        print(f"{k}: {len(r['crop_boxes'])} crops, tables per page {[len(v) for v in r['results_json'].values()]}, "
              f"pixels {r['pixels_shape']} -> {len(r['pixels_f16_zlib'])} bytes, batch {r['table_batch_size']}")


if __name__ == "__main__":
    GOLDEN.mkdir(parents=True, exist_ok=True)
    make_table_pages_golden()
