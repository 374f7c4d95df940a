"""Table recognition's two-pass flow on the CPU, against tests/golden/table_flow.pt: what the reference's own
TableRecPredictor.batch_table_recognition passed to decode_batch_predictions, and every decode pass it ran (prompt ids,
decoder calls, predictions).  The fp32 oracle restatement, and TableRecRunner's host bookkeeping over the oracle engine."""
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


@pytest.fixture(scope="module")
def case():
    from oracle import table_flow_oracle as L
    from surya_b200.config import table_tiny
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    g = torch.load(GOLDEN / "table_flow.pt", weights_only=False)
    m = g["meta"]
    cfg = table_tiny()
    sde, sdd = swin_state_dict(cfg.encoder, m["seed"]), adetr_table_state_dict(cfg.decoder, m["seed"])
    px = L.table_flow_pages(m["sizes"], cfg.encoder.image_size)
    torch.set_num_threads(max(1, min(16, len(__import__("os").sched_getaffinity(0)))))
    return g, cfg, sde, sdd, px


def _golden_batches(g):
    """Per image batch: (rowcol_predictions, cell_predictions, idx_map, orig_sizes) as the reference passed them on."""
    out, k = [], 0
    for d in g["decodes"]:
        rowcol = g["passes"][k]["predictions"]
        k += 1
        cells = []
        while len(cells) < len(d["idx_map"]):
            cells.extend(g["passes"][k]["predictions"])
            k += 1
        out.append((rowcol, cells, d["idx_map"], d["orig_sizes"]))
    assert k == len(g["passes"])
    return out


def _assert_same(got, want, tol):
    assert len(got) == len(want)
    for (rc, cells, idx, sizes), (rc_w, cells_w, idx_w, sizes_w) in zip(got, want):
        assert idx == idx_w and [tuple(s) for s in sizes] == [tuple(s) for s in sizes_w]
        for a, b in ((rc, rc_w), (cells, cells_w)):
            assert [len(p) for p in a] == [len(p) for p in b]
            for pa, pb in zip(a, b):
                for x, y in zip(pa, pb):
                    assert {k: v for k, v in x.items() if k != "bbox"} == {k: v for k, v in y.items() if k != "bbox"}
                    diff = max(abs(u - v) for u, v in zip(x["bbox"], y["bbox"]))
                    assert diff <= tol, diff


def test_golden_covers_the_flow(case):
    """The fixture exercises what the flow has to get right: tables with rows and columns, rows that stop early and rows
    that run the whole budget in both passes, a whole pass that breaks early, and non-empty cell predictions."""
    from surya_b200.table_rec import step_budget

    g = case[0]
    mx = g["meta"]["max_boxes"]
    assert len(g["decodes"]) >= 2
    first, k = set(), 0           # index of every batch's row/column pass; the cell passes follow it
    for d in g["decodes"]:
        first.add(k)
        k += 1
        n = 0
        while n < len(d["idx_map"]):
            n += len(g["passes"][k]["predictions"])
            k += 1
    rowcol = [p for i, p in enumerate(g["passes"]) if i in first]
    cells = [p for i, p in enumerate(g["passes"]) if i not in first]
    full = [t for p in rowcol for t in p["predictions"]]
    both = [t for t in full if sum(x["category"] == 1 for x in t) >= 2 and any(x["category"] == 2 for x in t)]
    assert len(both) >= 2
    for kind in (rowcol, cells):
        lens = [(len(t), step_budget(mx, p["input_ids"].shape[1])) for p in kind for t in p["predictions"]]
        assert any(n < b for n, b in lens) and any(n == b for n, b in lens)
    assert any(p["calls"] < step_budget(mx, p["input_ids"].shape[1]) for p in g["passes"])
    assert any(len(t) > 0 for p in cells for t in p["predictions"])
    assert any(p["input_ids"].shape[1] > 3 for p in cells)
    for p in g["passes"]:       # the reference's step budget: max(1, max_boxes + 1 - q_len) decoder calls
        assert p["calls"] <= step_budget(mx, p["input_ids"].shape[1])
        if all(len(t) == step_budget(mx, p["input_ids"].shape[1]) for t in p["predictions"][:1]):
            assert p["calls"] == step_budget(mx, p["input_ids"].shape[1])


def test_prompt_builders_match_the_reference_processor(case):
    """Query prompts from the original sizes (incl. widths 644 / 748, where 644 * (1024 / 644) < 1024) and the cell prompts from
    the reference's own row/column predictions reproduce the ids the reference processor built, exactly."""
    from surya_b200.table_rec import CATEGORY_COLUMN, CATEGORY_ROW, box_polygon, cell_prompts, table_query_prompt

    g, cfg = case[0], case[1]
    d = cfg.decoder
    sizes = [tuple(s) for s in g["meta"]["sizes"]]
    assert 644 in [w for w, _ in sizes] and 748 in [w for w, _ in sizes]
    k = 0
    for batch in _golden_batches(g):
        rowcol, cells, idx, orig = batch
        q = table_query_prompt(orig, d)
        assert torch.equal(q, g["passes"][k]["input_ids"])
        k += 1
        rows = [{"polygon": box_polygon(p["bbox"]), "category": p["category"], "is_header": int(p["is_header"] == 1)}
                for t in rowcol for p in t if p["category"] == CATEGORY_ROW]
        cols = [{"polygon": box_polygon(p["bbox"]), "category": p["category"], "is_header": int(p["is_header"] == 1)}
                for t in rowcol for p in t if p["category"] == CATEGORY_COLUMN]
        ids = cell_prompts(rows, cols, d)
        r0 = 0
        while r0 < len(rows):
            want = g["passes"][k]["input_ids"]
            assert torch.equal(ids[r0:r0 + want.shape[0]], want)
            r0 += want.shape[0]
            k += 1
    assert table_query_prompt([(644, 500)], d)[0, 1, :4].tolist() == [511, 512, 1023, 1024]


def test_oracle_flow_vs_reference_predictor(case):
    from oracle import table_flow_oracle as L

    g, cfg, sde, sdd, px = case
    m = g["meta"]
    got = L.table_flow(sde, sdd, cfg, px, m["sizes"], m["batch_size"], m["max_boxes"])
    _assert_same(got, _golden_batches(g), 1e-5 * 1024)


def test_runner_over_oracle_engine_vs_reference_predictor(case):
    """TableRecRunner's bookkeeping (histories -> prediction dicts, stop rule, row queries, columns, cell prompts) over the fp32
    oracle engine: every token, count, index and size equals what the reference predictor passed on, and the bbox floats agree
    to fp32 rounding (the oracle's op order is not the reference modules').  Against the oracle's own restatement of the flow,
    whose decoder arithmetic is the same, the result is identical bit for bit."""
    from oracle import table_flow_oracle as L
    from oracle.table_flow_oracle import OracleTableEngine
    from surya_b200.table_rec import TableRecRunner

    g, cfg, sde, sdd, px = case
    m = g["meta"]
    eng = OracleTableEngine(cfg, sde, sdd, max_batch=m["batch_size"], max_rows=m["batch_size"])
    got = TableRecRunner(eng, m["batch_size"], max_boxes=m["max_boxes"]).run(px, m["sizes"])
    _assert_same(got, _golden_batches(g), 1e-5 * 1024)
    _assert_same(got, L.table_flow(sde, sdd, cfg, px, m["sizes"], m["batch_size"], m["max_boxes"]), 0.0)
    assert any(rows > 1 for rows, _, _ in eng.calls)
    # cell-pass row chunks other than the reference's (its image batch size) change nothing it would see
    eng5 = OracleTableEngine(cfg, sde, sdd, max_batch=m["batch_size"], max_rows=5)
    _assert_same(TableRecRunner(eng5, m["batch_size"], max_boxes=m["max_boxes"]).run(px, m["sizes"]), _golden_batches(g), 1e-5 * 1024)


def test_runner_returns_empty_cells_for_a_batch_without_rows(case):
    """The one intended difference from the reference (which fails on torch.stack([])): no predicted row -> no cell pass."""
    from surya_b200.table_rec import TableRecRunner

    class _NoRows:
        max_batch, max_rows, s_max = 4, 8, 222

        def __init__(self, cfg):
            self.cfg = cfg

        def encode(self, px):
            return px

        def cross_kv(self, enc):
            return self

        def decode_rows(self, row_table, prompt, n_steps):
            n = len(row_table)
            tok = torch.zeros((2, n, 10), dtype=torch.long)
            tok[0, :, 6] = 5 + 2            # a column
            tok[1, :, 6] = 1                # eos
            done = torch.tensor([[0] * n, [1] * n], dtype=torch.uint8)
            return tok, torch.full((2, n, 6), 0.5), [], done

    cfg = case[1]
    out = TableRecRunner(_NoRows(cfg), 2, max_boxes=24).run(torch.zeros(2, 3, 4, 4), [(100, 80), (90, 90)])
    (rowcol, cells, idx, sizes), = out
    assert [len(t) for t in rowcol] == [1, 1] and rowcol[0][0]["category"] == 2 and cells == [] and idx == []
