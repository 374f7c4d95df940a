"""ORACLE TOOLING — the table recognition flow golden from the reference's own predictor.

    SURYA_REFERENCE=<checkout> python -m oracle.make_table_flow_golden     # writes tests/golden/table_flow.pt

Kept beside oracle/make_golden.py (whose output directory and reference import it shares) so that the other goldens'
generator stays as it was.
"""
from __future__ import annotations

import copy
import sys
import time

import torch

from oracle.make_golden import GOLDEN, ref_shim  # noqa: E402  (make_golden puts the repository on sys.path)


def make_table_flow_golden():
    """The reference's UNMODIFIED TableRecPredictor.batch_table_recognition (surya/table_rec/__init__.py:134-236) on the CPU over
    its own table_rec modules (tiny config, seed 0 weights), with a synthetic loader and a processor whose image half hands out
    seeded pages (layout_oracle.table_flow_pages; the query / column arithmetic is the reference processor's).  A wrapper around
    inference_loop records every pass's prompt ids, decoder-call count and predictions; decode_batch_predictions is wrapped to
    record its arguments, and the final TableResults are kept as plain dicts: tests/golden/table_flow.pt."""
    from oracle import ref_predictors as RP
    from oracle import table_flow_oracle as L
    from surya_b200 import dropin
    from surya_b200.config import table_tiny
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    RP.install_predictors()
    from PIL import Image
    from surya.settings import settings
    from surya.table_rec import TableRecPredictor
    from surya.table_rec.processor import SuryaTableRecProcessor
    from surya.table_rec.shaper import LabelShaper

    case = L.TABLE_FLOW_CASE
    cfg = table_tiny()
    sde, sdd = swin_state_dict(cfg.encoder, case["seed"]), adetr_table_state_dict(cfg.decoder, case["seed"])
    enc, dec = ref_shim.build_reference_table_models(cfg, sde, sdd)

    class _Model:          # the attributes batch_table_recognition / inference_loop use on self.model
        device, dtype = torch.device("cpu"), torch.float32

        def __init__(self):
            self.encoder, self.decoder = enc, dec
            self.config = type("Cfg", (), {"encoder": enc.config, "decoder": dec.config})()

        def to(self, *a, **k):
            return self

    class _Pages:          # stand-in for SuryaEncoderImageProcessor (the Donut resize is out of the device flow)
        def __call__(self, images, **kw):
            return {"pixel_values": [L.table_flow_pages([im.size], cfg.encoder.image_size)[0].numpy() for im in images]}

    proc = SuryaTableRecProcessor.__new__(SuryaTableRecProcessor)
    proc.image_processor, proc.box_size, proc.special_token_count, proc.shaper = _Pages(), (1024, 1024), 5, LabelShaper()
    proc.token_pad_id, proc.token_eos_id, proc.token_bos_id, proc.token_query_end_id = 0, 1, 1, 4

    passes, decodes = [], []
    Stock = type("StockTableRecPredictor", (TableRecPredictor,), {"model_loader_cls": dropin.loader_for(_Model(), proc)})
    pred = Stock(device="cpu", dtype=torch.float32)
    pred.disable_tqdm = True
    orig_loop, orig_decode, orig_call = pred.inference_loop, pred.decode_batch_predictions, dec.forward
    calls = [0]

    def loop(encoder_hidden_states, batch_input_ids, current_batch_size, batch_size):
        calls[0] = 0
        ids = batch_input_ids.clone()
        res = orig_loop(encoder_hidden_states, batch_input_ids, current_batch_size, batch_size)
        passes.append({"input_ids": ids, "calls": calls[0], "predictions": copy.deepcopy(res)})
        return res

    def count(*a, **k):
        calls[0] += 1
        return orig_call(*a, **k)

    def decode(rowcol, cells, orig_sizes, idx_map, shaper):
        decodes.append({"idx_map": list(idx_map), "orig_sizes": [tuple(s) for s in orig_sizes]})
        return orig_decode(rowcol, cells, orig_sizes, idx_map, shaper)

    pred.inference_loop, pred.decode_batch_predictions, dec.forward = loop, decode, count
    old_max = settings.TABLE_REC_MAX_BOXES
    settings.TABLE_REC_MAX_BOXES = case["max_boxes"]
    t0 = time.time()
    try:
        images = [Image.new("RGB", s, "white") for s in case["sizes"]]
        results = pred(images, batch_size=case["batch_size"])
    finally:
        settings.TABLE_REC_MAX_BOXES = old_max
        dec.forward = orig_call

    def cell(c):
        return {k: getattr(c, k) for k in ("polygon", "row_id", "rowspan", "cell_id", "within_row_id", "colspan", "merge_up",
                                           "merge_down", "col_id", "is_header")}

    res = [{"cells": [cell(c) for c in r.cells], "unmerged_cells": [cell(c) for c in r.unmerged_cells],
            "rows": [{"polygon": x.polygon, "row_id": x.row_id, "is_header": x.is_header} for x in r.rows],
            "cols": [{"polygon": x.polygon, "col_id": x.col_id, "is_header": x.is_header} for x in r.cols],
            "image_bbox": list(r.image_bbox)} for r in results]
    g = {"passes": passes, "decodes": decodes, "results": res,
         "meta": dict(case, kind="table_flow", config="table_tiny", image_size=list(cfg.encoder.image_size), torch=str(torch.__version__),
                      reference="VikParuchuri/surya@80e9a7e TableRecPredictor.batch_table_recognition, fp32 CPU")}
    torch.save(g, GOLDEN / "table_flow.pt")
    print(f"[golden] table_flow: {time.time() - t0:.1f}s {len(passes)} passes, calls {[p['calls'] for p in passes]}, "
          f"prompt lengths {[p['input_ids'].shape[1] for p in passes]}, idx_map {[d['idx_map'] for d in decodes]}")


if __name__ == "__main__":
    GOLDEN.mkdir(parents=True, exist_ok=True)
    torch.set_num_threads(8)
    make_table_flow_golden()
