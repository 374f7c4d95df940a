"""Table recognition's two-pass flow on the device: the row -> K/V-set cross-attention, LayoutEngine.cross_kv /
decode_rows (held K/V, batched prompt prefill, early exit) and TableRecRunner against the fp32 oracle."""
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("group", [1, 2, 4])
def test_indexed_single_query_attention_is_bit_identical(built_lib, dtype, group):
    """Many-to-one, out-of-order index == the plain kernel over stacked copies of the K/V sets; no index == today."""
    from surya_b200 import ops

    nkv, hd, n_keys, S = 4, 64, 576, 3
    nh = nkv * group
    g = torch.Generator(device="cuda").manual_seed(group)
    kv = torch.randn((S * n_keys, 2 * nkv * hd), generator=g, device="cuda").to(dtype)
    idx = torch.tensor([2, 0, 2, 1, 1, 2, 0], dtype=torch.int32, device="cuda")
    B = idx.numel()
    q = torch.randn((B, nh * hd), generator=g, device="cuda").to(dtype)
    got = ops.attn_single_query(q, kv, n_keys, nh, nkv, hd, hd ** -0.5, kv_index=idx)
    stacked = kv.view(S, n_keys, -1)[idx.long()].reshape(B * n_keys, -1).contiguous()
    want = ops.attn_single_query(q, stacked, n_keys, nh, nkv, hd, hd ** -0.5)
    assert torch.equal(got, want)
    ident = ops.attn_single_query(q[:S], kv, n_keys, nh, nkv, hd, hd ** -0.5, kv_index=torch.arange(S, dtype=torch.int32, device="cuda"))
    assert torch.equal(ident, ops.attn_single_query(q[:S], kv, n_keys, nh, nkv, hd, hd ** -0.5))
    with pytest.raises(Exception):
        ops.attn_single_query(q, kv, n_keys, nh, nkv, hd, hd ** -0.5, kv_index=idx + 1)       # 3 is not a set: host check


def _tiny_engine(**kw):
    from surya_b200.config import table_tiny
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_table_state_dict, layout_synthetic_pages, swin_state_dict

    cfg = table_tiny()
    sde, sdd = swin_state_dict(cfg.encoder, 0), adetr_table_state_dict(cfg.decoder, 0)
    eng = LayoutEngine(cfg, sde, sdd, dtype=torch.float16, **kw)
    x = layout_synthetic_pages(3, cfg.encoder.image_size, seed=31).cuda()
    return cfg, sde, sdd, eng, eng.encode(x)


def test_decode_rows_one_token_prompt_equals_decode_over_stacked_copies(built_lib):
    """Shared K/V + early exit without the prefill: rows on a many-to-one map give bit-identical histories to sb_layout_decode
    over stacked copies of their tables' encoder states, for every step decode_rows ran; when every row stops early it runs
    fewer steps than the budget, and at least through the step at which the last row became done."""
    cfg, _, _, eng, enc = _tiny_engine(max_batch=8, max_rows=8)
    d = cfg.decoder
    table = [2, 0, 1, 2, 2, 0]
    rows = len(table)
    g = torch.Generator().manual_seed(3)
    prompt = torch.randint(0, 1025, (rows, 1, 10), generator=g)
    prompt[:, 0, 6:] = torch.randint(5, 10, (rows, 4), generator=g)
    budget = 60
    want = [t.clone() for t in _flat(eng.run_loop(enc[torch.tensor(table)], prompt.cuda(), budget))]
    eng.cross_kv(enc)
    got = _flat(eng.decode_rows(table, prompt, budget))
    n = got[0].shape[0]
    for a, b in zip(got, want):
        assert torch.equal(a, b[:n])
    done = want[-1].bool().cpu()
    first = [int(torch.nonzero(done[:, r])[0]) if done[:, r].any() else None for r in range(rows)]
    if all(f is not None for f in first):
        assert max(first) < n
    if all(f is not None and f < budget - 16 for f in first):
        assert n < budget
    print(f"decode_rows: {n} of {budget} steps, first done {first}")


def test_early_exit_stops_before_the_budget(built_lib):
    """Rows whose next category is eos from the first step: the loop stops after one or two groups of steps."""
    cfg, _, sdd, eng, enc = _tiny_engine(max_batch=4)
    d = cfg.decoder
    # find prompts that finish: run the full budget once, keep rows that reach done early, and check the early-exit run
    g = torch.Generator().manual_seed(5)
    prompt = torch.randint(0, 1025, (4, 1, 10), generator=g)
    prompt[:, 0, 6:] = 5
    budget = 120
    eng.cross_kv(enc)
    full = [t.clone() for t in _flat(eng.run_loop(enc[torch.tensor([0, 1, 2, 0])], prompt.cuda(), budget))]
    eng.cross_kv(enc)
    got = _flat(eng.decode_rows([0, 1, 2, 0], prompt, budget))
    n = got[0].shape[0]
    for a, b in zip(got, full):
        assert torch.equal(a, b[:n])
    done = full[-1].bool().cpu()
    if bool(done.any(0).all()):
        last = max(int(torch.nonzero(done[:, r])[0]) for r in range(4))
        assert last < n and n <= last + 1 + 2 * 8
        assert n < budget or last >= budget - 17


def test_batched_prefill_vs_reference_cellpass_golden(built_lib):
    """7-token cell prompt prefilled in one pass (rows x 6 GEMM rows) against the reference's batched prefill, within the
    tolerances test_engine_nonsquare_encoder_and_cellpass_prompt_vs_reference_golden uses for the position-by-position path."""
    from surya_b200.config import LayoutConfig, SwinConfig, table_decoder
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    g = torch.load(GOLDEN / "table_nonsquare_cellpass.pt")
    enc_cfg = SwinConfig(image_size=tuple(g["meta"]["image_size"]), depths=(2, 2, 2, 2), encoder_length=128)
    cfg = LayoutConfig(encoder=enc_cfg, decoder=table_decoder(2))
    sde, sdd = swin_state_dict(enc_cfg, g["meta"]["seed"]), adetr_table_state_dict(cfg.decoder, g["meta"]["seed"])
    for max_prefill in (6, 12):          # one row per chunk, and both rows in one chunk
        eng = LayoutEngine(cfg, sde, sdd, dtype=torch.float16, max_batch=2, max_prefill_tokens=max_prefill)
        eng.cross_kv(g["encoder"].to(torch.float16).cuda())
        tok, bbox, heads, done = eng.decode_rows([0, 1], g["prompt"], 1)
        got = {"bbox": bbox[0], "category": heads[0][0], "merges": heads[1][0], "colspan": heads[2][0], "is_header": heads[3][0]}
        for k, v in got.items():
            err = (v.cpu() - g["heads"][k][:, 0]).abs().max().item()
            assert err < 1e-2 * max(1.0, g["heads"][k].abs().max().item()), (max_prefill, k, err)
        eng.close()


def test_row_chunking_changes_rounding_only(built_lib):
    """A row decoded alone and among 64 others: the GEMMs pick their kernels by row count, so the bits may differ; the first
    step's head outputs (prefill included) agree to fp16 rounding."""
    cfg, _, _, eng, enc = _tiny_engine(max_batch=4, max_rows=72, max_prefill_tokens=128)
    g = torch.Generator().manual_seed(9)
    rows = 65
    prompt = torch.randint(0, 1025, (rows, 6, 10), generator=g)
    prompt[:, 0], prompt[:, 2] = cfg.decoder.bos_token_id, cfg.decoder.query_end_token_id
    prompt[:, 1:, 6:] = torch.randint(5, 10, (rows, 5, 4), generator=g)
    table = [r % 3 for r in range(rows)]
    eng.cross_kv(enc)
    many = [t.clone() for t in _flat(eng.decode_rows(table, prompt, 1))]
    for r in (0, 37, 64):
        one = _flat(eng.decode_rows([table[r]], prompt[r:r + 1], 1))
        for a, b in zip(one[1:-1], many[1:-1]):
            assert (a[0, 0] - b[0, r]).abs().max().item() < 2e-2


def test_capacity_and_argument_errors(built_lib):
    from surya_b200 import _lib

    cfg, _, _, eng, enc = _tiny_engine(max_batch=2, max_rows=4, s_max=40, max_prefill_tokens=8)
    prompt = torch.full((2, 3, 10), 5, dtype=torch.long)
    with pytest.raises(_lib.SuryaB200Error, match="max_batch >= 3"):
        eng.cross_kv(enc)                                       # 3 tables, max_batch 2
    eng.cross_kv(enc[:2])
    with pytest.raises(_lib.SuryaB200Error, match="s_max >= 41"):
        eng.decode_rows([0, 1], prompt, 39)
    with pytest.raises(_lib.SuryaB200Error, match="max_rows >= 5"):
        eng.decode_rows([0] * 5, prompt[[0] * 5], 4)
    with pytest.raises(_lib.SuryaB200Error, match="max_prefill_tokens >= 9"):
        eng.decode_rows([0], torch.full((1, 10, 10), 5, dtype=torch.long), 4)
    with pytest.raises(_lib.SuryaB200Error, match="outside the 2 held tables"):
        eng.decode_rows([0, 2], prompt, 4)
    with pytest.raises(_lib.SuryaB200Error, match="outside the 2 held tables"):
        eng.decode_rows([-1, 0], prompt, 4)
    eng.decode_rows([1, 0], prompt, 4)                          # valid call after the refusals
    eng.run_loop(enc[:2], prompt.cuda(), 4)                     # overwrites the held K/V
    with pytest.raises(_lib.SuryaB200Error, match="no cross K/V held"):
        eng.decode_rows([0, 1], prompt, 4)
    eng.cross_kv(enc[:2])
    eng.decode_rows([0, 1], prompt, 4)


def _flat(res):
    tok, bbox, heads, done = res
    return [tok, bbox] + list(heads) + [done]


def _runner_vs_oracle(cfg, sde, sdd, x, sizes, batch_size, max_boxes, check_rows, **kw):
    from oracle import layout_oracle as L
    from surya_b200.layout import LayoutEngine
    from surya_b200.table_rec import TableRecRunner, step_budget

    eng = LayoutEngine(cfg, sde, sdd, dtype=torch.float16, max_batch=batch_size, **kw)
    runner = TableRecRunner(eng, batch_size, max_boxes=max_boxes)
    runner.trace = []
    out = runner.run(x.cuda(), sizes)
    d = cfg.decoder
    sd32 = {k: v.to(torch.float16).float() for k, v in sdd.items()}
    worst, enc, n_pass = {}, None, 0
    torch.set_num_threads(max(1, min(64, len(__import__("os").sched_getaffinity(0)))))
    for rec in runner.trace:
        if "enc" in rec:
            enc = rec["enc"]
            continue
        n_pass += 1
        sel = list(range(min(check_rows, len(rec["row_table"]))))
        tok, heads, done = rec["tok"][:, sel], [h[:, sel] for h in rec["heads"]], rec["done"][:, sel]
        assert rec["tok"].shape[0] <= step_budget(max_boxes, rec["prompt"].shape[1])
        st = L.AdetrState(d.num_hidden_layers)
        ids, pos = rec["prompt"][sel], torch.arange(rec["prompt"].shape[1])
        e = enc[torch.tensor([rec["row_table"][i] for i in sel])]
        with torch.inference_mode():
            for s in range(tok.shape[0]):
                ref = L.adetr_forward(sd32, d, ids, e, pos, st)
                pos = pos[-1:] + 1
                got = dict(zip(("category", "merges", "colspan", "is_header"), [h[s] for h in heads]), bbox=rec["bbox"][s, sel])
                for k in ref:
                    worst[k] = max(worst.get(k, 0.0), (ref[k][:, -1] - got[k]).abs().max().item())
                ref_tok, ref_done = L.table_next_tokens({k: v.unsqueeze(1) for k, v in got.items()}, d)
                assert torch.equal(ref_tok, tok[s]) and torch.equal(ref_done, done[s].bool())
                ids = tok[s].unsqueeze(1)
    print(f"runner vs oracle: {n_pass} passes, head errs " + str({k: round(v, 5) for k, v in worst.items()}))
    assert all(v < 3e-2 for v in worst.values()), worst
    return out, runner


def test_runner_vs_oracle_tiny(built_lib):
    from oracle import table_flow_oracle as L
    from surya_b200.config import table_tiny
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    case = L.TABLE_FLOW_CASE
    cfg = table_tiny()
    sde, sdd = swin_state_dict(cfg.encoder, case["seed"]), adetr_table_state_dict(cfg.decoder, case["seed"])
    x = L.table_flow_pages(case["sizes"], cfg.encoder.image_size)
    out, _ = _runner_vs_oracle(cfg, sde, sdd, x, case["sizes"], case["batch_size"], case["max_boxes"], 64, max_rows=4)
    assert len(out) == 2 and sum(len(b[2]) for b in out) > 0


def test_runner_vs_oracle_default_config(built_lib):
    """Default table config, 16 pages of 768x768 in one image batch, the full 150-box budget; the first rows of every pass are
    teacher-forced through the fp32 oracle."""
    from surya_b200.config import table_default
    from surya_b200.synth import adetr_table_state_dict, layout_synthetic_pages, swin_state_dict

    cfg = table_default()
    sde, sdd = swin_state_dict(cfg.encoder, 0), adetr_table_state_dict(cfg.decoder, 0)
    x = layout_synthetic_pages(16, cfg.encoder.image_size, seed=6)
    sizes = [(768 + 37 * i, 768 - 11 * i) for i in range(16)]
    _runner_vs_oracle(cfg, sde, sdd, x, sizes, 16, 150, 2, max_rows=256, max_prefill_tokens=4096)
