"""CPU ORACLE (test infrastructure, not product code) — table recognition's two-pass flow.

  * TABLE_FLOW_CASE / table_flow_pages   the seeded case of tests/golden/table_flow.pt and its input pages
  * table_pass                           one TableRecPredictor.inference_loop in fp32 (early break included)
  * table_flow                           TableRecPredictor.batch_table_recognition (surya/table_rec/__init__.py:134-236) up to
                                         decode_batch_predictions, over oracle.layout_oracle's Swin encoder and ADETR decoder
  * OracleTableEngine                    LayoutEngine's cross_kv / decode_rows surface on the CPU, so that
                                         surya_b200.table_rec.TableRecRunner runs without a GPU

Pinned by tests/golden/table_flow.pt (oracle/make_table_flow_golden.py).
"""
from __future__ import annotations

from typing import List

import torch

from . import layout_oracle as L

SD = L.SD


# The seeded case of tests/golden/table_flow.pt (tiny table config, seed 0 weights): five images of mixed sizes in batches of 3,
# widths 644 and 748 hit the query prompt's float64 rounding, and a 24-box budget keeps the CPU passes short.
TABLE_FLOW_CASE = {"seed": 0, "sizes": [(644, 500), (748, 390), (300, 300), (1024, 700), (512, 640)], "batch_size": 3, "max_boxes": 24}


def table_flow_pages(image_sizes, image_size=(256, 256)) -> torch.Tensor:
    """Seeded stand-in for the Donut processor's resize + normalise of table images (the device flow starts from its output):
    one synthetic page per original (w, h), seeded by the size.  oracle/make_table_flow_golden.py's processor hands these to
    the reference predictor, and the tests regenerate them with this same function."""
    from surya_b200.synth import layout_synthetic_pages

    return torch.cat([layout_synthetic_pages(1, image_size, seed=10007 * int(w) + int(h)) for w, h in image_sizes], 0)


def table_pass(sd_dec: SD, cfg, enc: torch.Tensor, ids: torch.Tensor, n_steps: int):
    """One TableRecPredictor.inference_loop (table_rec/__init__.py:34-132) in fp32: the whole prompt as the first call, then
    one token per call; stops after the first call at which every row is done (done is sticky).  Returns per-step histories
    tok [n, B, 10], bbox [n, B, 6], heads (category, merges, colspan, is_header: [n, B, k]), done [n, B] for the n calls made."""
    with torch.inference_mode():
        st = L.AdetrState(cfg.num_hidden_layers)
        pos = torch.arange(ids.shape[1])
        all_done = torch.zeros(ids.shape[0], dtype=torch.bool)
        toks, bbs, hs, dones = [], [], [], []
        for _ in range(n_steps):
            out = L.adetr_forward(sd_dec, cfg, ids, enc, pos, st)
            pos = pos[-1:] + 1
            tok, done = L.table_next_tokens(out, cfg)
            toks.append(tok)
            bbs.append(out["bbox"][:, -1].float().clone())
            hs.append([out[k][:, -1].float().clone() for k in ("category", "merges", "colspan", "is_header")])
            dones.append(done)
            all_done = all_done | done
            if bool(all_done.all()):
                break
            ids = tok.unsqueeze(1)
    heads = [torch.stack([h[i] for h in hs]) for i in range(4)]
    return torch.stack(toks), torch.stack(bbs), heads, torch.stack(dones).to(torch.uint8)


def _predictions(tok, bbox, done, special):
    """inference_loop's per-call prediction dicts (:80-122): appended for the rows not yet done, nothing at the breaking call."""
    n, B = tok.shape[0], tok.shape[1]
    preds = [[] for _ in range(B)]
    all_done = torch.zeros(B, dtype=torch.bool)
    for s in range(n):
        all_done = all_done | done[s].bool()
        if bool(all_done.all()):
            break
        for j in range(B):
            if not all_done[j]:
                t = tok[s, j].tolist()
                preds[j].append({"bbox": (bbox[s, j] * 1024).tolist(), "category": t[6] - special, "merges": t[7] - special,
                                 "colspan": t[8], "is_header": t[9] - special})
    return preds


def table_flow(sd_enc: SD, sd_dec: SD, cfg, pixel_values: torch.Tensor, image_sizes, batch_size: int, max_boxes: int):
    """TableRecPredictor.batch_table_recognition (table_rec/__init__.py:134-236) up to decode_batch_predictions, fp32: per
    image batch the encoder, the row/column pass, the row queries and columns of every table of the batch, and the cell pass
    of every row over its own table's encoder states.  Returns [(rowcol_predictions, cell_predictions, idx_map, orig_sizes)]
    per image batch.  The prompt arithmetic is surya_b200.table_rec's (pinned against the reference processor's ids)."""
    from surya_b200.table_rec import box_polygon, cell_prompts, step_budget, table_query_prompt

    d = cfg.decoder
    sp = d.special_token_count
    out = []
    for i in range(0, len(image_sizes), batch_size):
        sizes = [tuple(s) for s in image_sizes[i:i + batch_size]]
        enc = L.swin_forward(sd_enc, cfg.encoder, pixel_values[i:i + batch_size])
        ids = table_query_prompt(sizes, d)
        tok, bbox, _, done = table_pass(sd_dec, d, enc, ids, step_budget(max_boxes, ids.shape[1]))
        rowcol = _predictions(tok, bbox, done, sp)
        rows, cols, idx_map = [], [], []
        for j, preds in enumerate(rowcol):
            for p in preds:
                item = {"polygon": box_polygon(p["bbox"]), "category": p["category"], "is_header": int(p["is_header"] == 1)}
                if p["category"] == 1:
                    rows.append(item)
                    idx_map.append(j)
                elif p["category"] == 2:
                    cols.append(item)
        cells = []
        if rows:
            ids = cell_prompts(rows, cols, d)
            for r0 in range(0, len(rows), batch_size):
                e = enc[torch.tensor(idx_map[r0:r0 + batch_size])]
                q = ids[r0:r0 + batch_size]
                tok, bbox, _, done = table_pass(sd_dec, d, e, q, step_budget(max_boxes, q.shape[1]))
                cells.extend(_predictions(tok, bbox, done, sp))
        out.append((rowcol, cells, idx_map, sizes))
    return out


class OracleTableEngine:
    """LayoutEngine's table_rec flow surface (encode, cross_kv, decode_rows) computed by oracle.layout_oracle in fp32 on the
    CPU, so that surya_b200.table_rec.TableRecRunner runs without a GPU."""

    def __init__(self, cfg, sd_enc, sd_dec, max_batch: int = 16, max_rows: int = 64, s_max: int | None = None):
        self.cfg, self.sde, self.sdd = cfg, sd_enc, sd_dec
        self.kind, self.device, self.dtype = "table", torch.device("cpu"), torch.float32
        self.max_batch, self.max_rows = max_batch, max_rows
        self.s_max = s_max if s_max is not None else cfg.decoder.max_boxes + 72
        self.held = None
        self.calls: List[tuple] = []

    def encode(self, pixel_values):
        return L.swin_forward(self.sde, self.cfg.encoder, pixel_values.float())

    def cross_kv(self, enc):
        if not 1 <= enc.shape[0] <= self.max_batch:
            raise RuntimeError(f"{enc.shape[0]} tables need max_batch >= {enc.shape[0]}")
        self.held = enc.float()
        return self

    def decode_rows(self, row_table, prompt, n_steps):
        rows, q = prompt.shape[0], prompt.shape[1]
        table = torch.tensor([int(t) for t in row_table], dtype=torch.long)
        assert self.held is not None and rows <= self.max_rows and q - 1 + n_steps <= self.s_max
        assert int(table.min()) >= 0 and int(table.max()) < self.held.shape[0]
        self.calls.append((rows, q, n_steps))
        return table_pass(self.sdd, self.cfg.decoder, self.held[table], prompt.cpu(), n_steps)
