import sys, time, torch
sys.path.insert(0, str(__import__("pathlib").Path(__file__).resolve().parent.parent))
from surya_b200.config import layout_default, table_default
from surya_b200.layout import LayoutEngine, layout_greedy, table_greedy
from surya_b200.synth import adetr_layout_state_dict, adetr_table_state_dict, layout_synthetic_pages, swin_state_dict, table_query_tokens
for kind in ("layout", "table"):
    cfg = layout_default() if kind == "layout" else table_default()
    sdd = adetr_layout_state_dict(cfg.decoder, 0) if kind == "layout" else adetr_table_state_dict(cfg.decoder, 0)
    x = layout_synthetic_pages(16, cfg.encoder.image_size, seed=1).half().cuda()
    for group in (1, 4, 8, 16):
        LayoutEngine.GRAPH_GROUP = group
        eng = LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), sdd, dtype=torch.float16)
        enc = eng.encode(x)
        n = 100 if kind == "layout" else 150
        prompt = torch.full((16, 1, 7), 1, dtype=torch.int64, device="cuda") if kind == "layout" else table_query_tokens(cfg.decoder, 16).cuda()
        ts = []
        for rep in range(4):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            eng.run_loop(enc, prompt, n)
            torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
        print(kind, "group", group, " ".join(f"{t:.1f}" for t in ts), "ms per call ->", f"{ts[-1] / n * 1e3:.0f} us/step", flush=True)
        del eng
