"""CPU ORACLE (test infrastructure, not product code) — the table_recognition CLI's page flow restated for the device path's tests.

  * TABLE_PAGES_CASE / case_pages    the pages of tests/golden/table_pages.pt: low-resolution pages that layout runs on and
                                     high-resolution copies of another size that the tables are cropped from
  * crop_zero_fill                   PIL's Image.crop for a box that may extend past the page: the outside reads 0
  * preprocess_jobs                  sb_layout_preprocess restated from its job table (bounded jobs included): the cubic model of
                                     oracle/layout_pages_oracle.py over the tap tables, page taps outside a bounded job's page read 0
  * layout_outputs / table_outputs   the deterministic stand-in decoders that oracle/make_table_pages_golden.py runs under the
                                     reference's own LayoutPredictor and TableRecPredictor: outputs depend on (row, step) only
  * StubPagesLayoutEngine / StubTableEngine   CPU objects with LayoutEngine's surface over the same outputs, whose preprocess()
                                     is preprocess_jobs, so the repository's host flow runs without a GPU

Only tests/ and oracle/make_table_pages_golden.py import this module.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from oracle import layout_pages_oracle as LPO

# Pages in the CLI's order: (name, low-resolution (w, h), high-resolution (w, h)).  Page 0 has a table at .5 crop coordinates and
# one past the right and bottom edges; page 1 has no table; page 2 is tall enough to be cut in two slices by layout, with a
# full-width table at its bottom; 10 tables in all, so the reference's CPU table batch of 8 mixes pages.
TABLE_PAGES_CASE = {"pages": [("doc", (1024, 1024), (2048, 2048)), ("doc", (900, 700), (1800, 1400)),
                              ("doc", (1024, 2000), (1536, 3000)), ("scan", (1000, 800), (2000, 1600)),
                              ("scan", (1024, 768), (1700, 1275))],
                    "seed": 70, "max_boxes": 150}

# Layout boxes per image row (slice order over the call), in the decoder's 1024 grid: (label, cx, cy, w, h).
LAYOUT_SCRIPT = {
    0: [("Text", 512, 40, 800, 40), ("Table", 250, 250, 350, 300), ("TableOfContents", 787, 812, 474, 424)],
    1: [("Text", 300, 300, 200, 100), ("Text", 600, 600, 200, 100)],
    2: [("Table", 512, 600, 800, 400)],
    3: [("Table", 512, 700, 1024, 648)],
    4: [("Table", 256, 200, 400, 300), ("TableOfContents", 768, 200, 400, 300), ("Table", 512, 700, 900, 400)],
    5: [("Table", 300, 300, 500, 400), ("Table", 800, 300, 300, 400), ("Text", 512, 800, 1000, 100)],
}


def case_pages(case=TABLE_PAGES_CASE) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """(pages, highres_pages): uint8 [h, w, 3] light pages with dark blocks, seeded per page."""
    lo = [LPO.fixture_page(w, h, case["seed"] + 2 * i) for i, (_, (w, h), _) in enumerate(case["pages"])]
    hi = [LPO.fixture_page(w, h, case["seed"] + 2 * i + 1) for i, (_, _, (w, h)) in enumerate(case["pages"])]
    return lo, hi


def crop_zero_fill(page: np.ndarray, box: Sequence[int]) -> np.ndarray:
    """Image.crop(box) of an integer box: the pixels of the box, 0 where it lies outside the page."""
    x0, y0, x1, y1 = box
    h, w = page.shape[:2]
    out = np.zeros((y1 - y0, x1 - x0, page.shape[2]), np.uint8)
    sx0, sy0, sx1, sy1 = max(x0, 0), max(y0, 0), min(x1, w), min(y1, h)
    if sx1 > sx0 and sy1 > sy0:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = page[sy0:sy1, sx0:sx1]
    return out


def preprocess_jobs(pages: np.ndarray, jobs: torch.Tensor, tap_idx: torch.Tensor, tap_w: torch.Tensor, out_hw: Tuple[int, int],
                    dtype: torch.dtype) -> torch.Tensor:
    """sb_layout_preprocess on the CPU from its arguments: pages uint8 (flat), jobs int64 [n, 8], tap tables [rows, 4].  Per job
    the taps (relative to the rectangle, plus x0 / y0) gather the page; in a bounded job (page height > 0) a tap outside the
    page reads 0.  Then the float model of the cubic resize and the normalisation.  -> [n, 3, H, W] in `dtype`."""
    H, W = out_hw
    pages = np.asarray(pages).reshape(-1)
    ti, tw = tap_idx.numpy(), tap_w.numpy()
    out = torch.empty((jobs.shape[0], 3, H, W), dtype=dtype)
    for off, pw, x0, y0, xt, yt, o, ph in jobs.tolist():
        xi, xw = ti[xt:xt + W] + x0, tw[xt:xt + W]
        yi, yw = ti[yt:yt + H] + y0, tw[yt:yt + H]
        rows_n = ph if ph else int(yi.max()) + 1
        page = pages[off:off + pw * rows_n * 3].reshape(rows_n, pw, 3)
        xin = (xi >= 0) & (xi < pw) if ph else np.ones_like(xi, bool)
        yin = (yi >= 0) & (yi < ph) if ph else np.ones_like(yi, bool)
        rows = np.zeros((H, 4, W, 3), np.float32)          # the four source rows of every output row, resized horizontally
        for r in range(4):
            sel = page[np.clip(yi[:, r], 0, rows_n - 1)].astype(np.float32)    # [H, pw, 3]
            acc = np.zeros((H, W, 3), np.float32)
            for t in range(4):
                v = sel[:, np.clip(xi[:, t], 0, pw - 1), :] * (yin[:, r, None, None] & xin[None, :, t, None])
                acc = acc + v * xw[None, :, t, None]
            rows[:, r] = acc
        res = np.zeros((H, W, 3), np.float32)
        for r in range(4):
            res = res + rows[:, r] * yw[:, r, None, None]
        u8 = np.clip(np.rint(res), 0, 255).astype(np.uint8)
        out[o] = LPO.normalize(u8, dtype)
    return out


# ------------------------------------------------------------------------------------------------ stub decoders
def layout_outputs(row: int, step: int, special: int = 3, label_count: int = 20, eos: int = 1):
    """The stand-in layout decoder for image row `row` at `step`: (box sigmoid [6], class logits [label_count]) as float lists;
    LAYOUT_SCRIPT's boxes one per step, then eos.  Every value is exact in fp16 and bf16."""
    logits = [-4.0 + 0.125 * j for j in range(label_count)]
    script = LAYOUT_SCRIPT.get(row, [])
    if step >= len(script):
        logits[eos] = 9.0
        return [0.5, 0.5, 0.0625, 0.0625, 0.5, 0.5], logits
    label, cx, cy, w, h = script[step]
    logits[LPO.LABEL_TO_ID[label] + special] = 6.0
    return [cx / 1024, cy / 1024, w / 1024, h / 1024, 0.5, 0.5], logits


TABLE_COLS = 3


def table_rows(table: int) -> int:
    return 2 + table % 4


def _row_cy(z: int) -> int:
    return 64 + 128 * z


def table_outputs(table: int, row_cy, step: int):
    """The stand-in table decoder: (bbox [6] in the 1024 grid, category, merges, colspan, is_header) for the row/column pass of
    table `table` (row_cy None) or the cell pass of its row whose query centre is row_cy; category None = eos.
    Row/column pass: TABLE_COLS full-height columns (column 0 a header on even tables), then table_rows(table) full-width rows
    of 128 (row 0 a header).  Cell pass, by row number z mod 4:
      0: a 2-column spanning cell over columns 0-1, and a merge_down cell in column 2
      1: the same spanning cell, and a merge_up cell in column 2 (merges with row 0's)
      2: a spanning cell too short for the row (dropped), a merge_both cell in column 1, a single cell without merge (skipped)
      3: a 2-column cell only one column wide (rejected), and a merge_up cell in column 1 (merges with row 2's)"""
    if row_cy is None:
        items = [((170 + 340 * c, 512, 340, 1024), 2, 0, 1, int(c == 0 and table % 2 == 0)) for c in range(TABLE_COLS)]
        items += [((510, _row_cy(z), 1020, 128), 1, 0, 1, int(z == 0)) for z in range(table_rows(table))]
    else:
        z = (int(row_cy) - 64) // 128
        cy = _row_cy(z)
        items = {0: [((340, cy, 680, 128), 3, 0, 2, 0), ((850, cy, 340, 128), 3, 2, 1, 0)],
                 1: [((340, cy, 680, 128), 3, 0, 2, 0), ((850, cy, 340, 128), 3, 1, 1, 0)],
                 2: [((510, cy, 1020, 64), 3, 0, 3, 0), ((510, cy, 340, 128), 3, 3, 1, 0), ((170, cy, 340, 128), 3, 0, 1, 0)],
                 3: [((170, cy, 340, 128), 3, 0, 2, 0), ((510, cy, 340, 128), 3, 1, 1, 0)]}[z % 4]
    if step >= len(items):
        return [512, 512, 16, 16, 512, 512], None, 0, 1, 0
    (cx, cy, w, h), cat, merges, colspan, header = items[step]
    return [cx, cy, w, h, 512, 512], cat, merges, colspan, header


def table_head_logits(out, cfg):
    """table_outputs -> (bbox sigmoid [6], category, merges, colspan, is_header head outputs) as float lists."""
    bbox, cat, merges, colspan, header = out
    sp = cfg.special_token_count

    def onehot(n, k):
        v = [0.0] * n
        v[k] = 5.0
        return v

    category = onehot(cfg.category_count, cfg.eos_token_id if cat is None else cat + sp)
    return ([b / 1024 for b in bbox], category, onehot(cfg.merge_count, merges + sp), [float(colspan)],
            onehot(cfg.header_count, header + sp))


def prompt_row_cy(prompt_row: torch.Tensor, special: int):
    """The row key of a decoder prompt [q, 10]: None for the row/column pass's Table query, else the row query's centre y."""
    return None if int(prompt_row[1, 6]) - special == 4 else int(prompt_row[1, 1])


# ------------------------------------------------------------------------------------------------ CPU engines
class StubPagesLayoutEngine(LPO.StubLayoutEngine):
    """oracle.layout_pages_oracle.StubLayoutEngine over layout_outputs, with preprocess_jobs as its preprocess."""

    def preprocess(self, pages_dev, jobs, tap_idx, tap_w, out=None):
        px = preprocess_jobs(pages_dev.numpy(), jobs, tap_idx, tap_w, tuple(self.cfg.encoder.image_size), self.dtype)
        if out is not None:
            out.copy_(px)
            return out
        return px

    def run_pages(self, enc, page_wh, n_steps):
        d = self.cfg.decoder
        B, C = enc.shape[0], d.label_count
        sizes = [tuple(int(v) for v in r) for r in torch.as_tensor(page_wh).reshape(B, 2).tolist()]
        hist = {"tok": [], "bbox": [], "cls": [], "done": []}
        sticky = torch.zeros(B, dtype=torch.bool)
        for s in range(n_steps):
            outs = [layout_outputs(int(enc[b]), s, d.special_token_count, C, d.eos_token_id) for b in range(B)]
            bbox = torch.tensor([o[0] for o in outs]).to(self.dtype).float()
            cls = torch.tensor([o[1] for o in outs]).to(self.dtype).float()
            tok, cm, dn, fired = LPO.next_token_pages(bbox, cls, sizes, sticky, self.dtype, d)
            self.rule_count += fired
            for k, v in (("tok", tok), ("bbox", bbox), ("cls", cm), ("done", dn.to(torch.uint8))):
                hist[k].append(v)
            sticky |= dn
            if bool(sticky.all()) and (s + 1) % 8 == 1:
                break
        return tuple(torch.stack(hist[k]) for k in ("tok", "bbox", "cls", "done"))


class StubTableEngine:
    """A CPU object with the surface TableRecRunner and table_pages use (kind, cfg, dtype, device, max_batch, max_rows, s_max,
    preprocess, encode, cross_kv, decode_rows) over table_outputs.  encode hands out the tables' order numbers; decode_rows
    stops at the step where every row is done."""

    kind = "table"

    def __init__(self, cfg, dtype=torch.float16, max_batch: int = 32, max_rows: int = 64):
        self.cfg, self.dtype, self.device = cfg, dtype, torch.device("cpu")
        self.max_batch, self.max_rows, self.s_max = max_batch, max_rows, cfg.decoder.max_boxes + 72
        self.tables_seen = 0
        self.held = None
        self.encoded: List[torch.Tensor] = []       # every pixel batch encode() was given

    def preprocess(self, pages_dev, jobs, tap_idx, tap_w, out=None):
        px = preprocess_jobs(pages_dev.numpy(), jobs, tap_idx, tap_w, tuple(self.cfg.encoder.image_size), self.dtype)
        if out is not None:
            out.copy_(px)
            return out
        return px

    def encode(self, px):
        self.encoded.append(px.clone())
        ids = torch.arange(self.tables_seen, self.tables_seen + px.shape[0])
        self.tables_seen += px.shape[0]
        return ids

    def cross_kv(self, enc):
        if not 1 <= enc.shape[0] <= self.max_batch:
            raise RuntimeError(f"{enc.shape[0]} tables need max_batch >= {enc.shape[0]}")
        self.held = enc
        return self

    def decode_rows(self, row_table, prompt, n_steps):
        d = self.cfg.decoder
        rows = prompt.shape[0]
        keys = [(int(self.held[int(t)]), prompt_row_cy(prompt[r], d.special_token_count)) for r, t in enumerate(row_table)]
        toks, bbs, heads, dones = [], [], [[], [], [], []], []
        all_done = torch.zeros(rows, dtype=torch.bool)
        for s in range(n_steps):
            outs = [table_head_logits(table_outputs(t, cy, s), d) for t, cy in keys]
            bbox = torch.tensor([o[0] for o in outs], dtype=torch.float32)
            hs = [torch.tensor([o[k + 1] for o in outs], dtype=torch.float32) for k in range(4)]
            cat = hs[0].argmax(-1)
            done = (cat == d.eos_token_id) | (cat == d.pad_token_id)
            tok = torch.cat([(bbox * d.bbox_size).clamp(0, d.bbox_size).to(torch.long), cat[:, None], hs[1].argmax(-1)[:, None],
                             torch.round(hs[2].clamp(min=1)).to(torch.long), hs[3].argmax(-1)[:, None]], 1)
            toks.append(tok)
            bbs.append(bbox)
            for k in range(4):
                heads[k].append(hs[k])
            dones.append(done.to(torch.uint8))
            all_done |= done
            if bool(all_done.all()):
                break
        return torch.stack(toks), torch.stack(bbs), [torch.stack(h) for h in heads], torch.stack(dones)
