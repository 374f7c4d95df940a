"""Host behaviour the recognition and layout engines share around their kernels: launch accounting of graph-replayed loops,
the hop off the default stream, re-capture of the cached step graphs when what they were captured with changes, and the
workspace sizes of the engines the tests build.  Every comparison is bit for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# sb_*_workspace_bytes of the engines built below: the arenas' buffer lists, each rounded up to 256 bytes
REC_TINY_WORKSPACE = 23505152       # tiny_rec, max_slots 8, s_max 256, max_patches 4096, max_tokens 1024
LAYOUT_TINY_WORKSPACE = 21991936    # layout_tiny, max_batch 2
TABLE_TINY_WORKSPACE = 22434304     # table_tiny, max_batch 2
DET_TINY_WORKSPACE = 37650432       # det_tiny, max_batch 2, 256 x 256


class _Rec:
    """A tiny recognition engine after one prefill of three crops, with persistent decode buffers (stable pointers)."""

    def __init__(self):
        from surya_b200.config import tiny_rec
        from surya_b200.recognition import RecEngine, RecognitionRunner, build_prefill_plan
        from surya_b200.synth import rec_state_dict, rec_synthetic_crops

        cfg = tiny_rec()
        self.eng = RecEngine(cfg, rec_state_dict(cfg, seed=0), dtype=torch.float16, max_slots=8, s_max=256, max_patches=4096,
                             max_tokens=1024)
        tiles, grids, seqs = RecognitionRunner(self.eng, batch_size=4, max_tokens=8).preprocess(rec_synthetic_crops(3, 48, 512, seed=7))
        slots = self.eng.alloc_slots(3)
        out = self.eng.prefill(torch.from_numpy(np.concatenate(tiles, 0)).cuda(), build_prefill_plan(cfg, np.array(grids), seqs, slots))
        self.ids0, self.tok0 = out["next_ids"].clone(), out["tok"].clone()
        self.pos0 = torch.tensor([len(s) for s in seqs], dtype=torch.int32, device="cuda")
        self.slot = torch.tensor(slots, dtype=torch.int32, device="cuda")
        self.ids, self.pos = torch.empty_like(self.ids0), torch.empty_like(self.pos0)
        self.max_pos = max(len(s) for s in seqs)

    def hist(self, n, B=3):
        return {"tok": torch.zeros((n, B), dtype=torch.int64, device="cuda"),
                "score": torch.zeros((n, B), dtype=torch.float32, device="cuda"),
                "bbox": torch.zeros((n, B, 6), dtype=torch.int64, device="cuda"),
                "done": torch.zeros((n, B), dtype=torch.uint8, device="cuda")}

    def sched(self):
        B = self.ids0.numel()
        ring = torch.zeros((B, 40), dtype=torch.int64, device="cuda")
        ring[:, 0] = self.tok0
        return {"gen": torch.ones(B, dtype=torch.int32, device="cuda"), "ring": ring,
                "done": torch.zeros(B, dtype=torch.uint8, device="cuda"), "valid": torch.zeros(B, dtype=torch.int32, device="cuda"),
                "active": torch.zeros(1, dtype=torch.int32, device="cuda")}

    def run(self, n, use_graph, hist=None, B=3):
        """decode_steps(n) from the post-prefill state (the KV rows it writes are rewritten by every run); returns the
        histories plus ids / pos after the run, and the launch-count delta."""
        from surya_b200 import _lib

        hist = hist if hist is not None else self.hist(n, B)
        ids, pos = self.ids[:B], self.pos[:B]
        ids.copy_(self.ids0[:B])
        pos.copy_(self.pos0[:B])
        before = _lib.launch_count()
        self.eng.decode_steps(ids, self.slot[:B], pos, n, hist=hist, use_graph=use_graph, max_pos=self.max_pos)
        launches = _lib.launch_count() - before
        torch.cuda.synchronize()
        return [t.clone() for t in (*hist.values(), ids, pos)], launches


def _layout(kind):
    from surya_b200.config import layout_tiny, table_tiny
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import (adetr_layout_state_dict, adetr_table_state_dict, layout_synthetic_pages, swin_state_dict,
                                  table_query_tokens)

    if kind == "layout":
        cfg = layout_tiny()
        sde, sdd = swin_state_dict(cfg.encoder, 0), adetr_layout_state_dict(cfg.decoder, 0)
        prompt = torch.full((2, 1, 7), cfg.decoder.bos_token_id, dtype=torch.int64, device="cuda")
    else:
        cfg = table_tiny()
        sde, sdd = swin_state_dict(cfg.encoder, 1), adetr_table_state_dict(cfg.decoder, 1)
        prompt = table_query_tokens(cfg.decoder, 2).cuda()
    eng = LayoutEngine(cfg, sde, sdd, dtype=torch.float16, max_batch=2)
    enc = eng.encode(layout_synthetic_pages(2, cfg.encoder.image_size, seed=7).cuda())
    return eng, enc, prompt


def _loop(eng, enc, prompt, n, use_graph):
    from surya_b200 import _lib

    before = _lib.launch_count()
    tok, bbox, heads, done = eng.run_loop(enc, prompt, n, use_graph=use_graph)
    launches = _lib.launch_count() - before
    torch.cuda.synchronize()
    return [t.clone() for t in (tok, bbox, *heads, done)], launches


def _equal(a, b):
    assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_rec_launch_accounting_is_the_same_with_and_without_graphs(built_lib):
    r = _Rec()
    per = {}
    for n in (5, 6):
        eager, le = r.run(n, False)
        for _ in range(2):                      # the first graphed call captures, the second replays the cached graph
            got, lg = r.run(n, True)
            _equal(got, eager)
            assert lg == le, (n, lg, le)
        per[n] = le
    assert per[6] - per[5] > 0
    r.eng.close()


@pytest.mark.parametrize("kind", ["layout", "table"])
def test_layout_launch_accounting_is_the_same_with_and_without_graphs(built_lib, kind):
    eng, enc, prompt = _layout(kind)
    per = {}
    for n in (11, 12):                          # 1 eager step + one replay of the 8-step graph + 2 or 3 single-step replays
        eager, le = _loop(eng, enc, prompt, n, False)
        for _ in range(2):
            got, lg = _loop(eng, enc, prompt, n, True)
            _equal(got, eager)
            assert lg == le, (n, lg, le)
        per[n] = le
    assert per[12] - per[11] > 0
    eng.close()


def test_rec_graphs_on_default_and_user_streams_agree(built_lib):
    """On torch's default stream the engine captures on a stream of its own; on a user stream it captures there."""
    r = _Rec()
    eager, _ = r.run(6, False)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        user, _ = r.run(6, True, hist=r.hist(6))
    torch.cuda.current_stream().wait_stream(side)
    default, _ = r.run(6, True, hist=r.hist(6))   # new history pointers: captured again, now through the hop
    _equal(user, eager)
    _equal(default, eager)
    r.eng.close()


def test_rec_graph_recaptured_for_new_histories_batch_and_sched(built_lib):
    r = _Rec()
    n = 6
    h = r.hist(n)
    eager, _ = r.run(n, False)
    _equal(r.run(n, True, hist=h)[0], eager)
    _equal(r.run(n, True, hist=r.hist(n))[0], eager)           # new history tensors, same batch
    eager2, _ = r.run(n, False, B=2)
    _equal(r.run(n, True, hist=r.hist(n, 2), B=2)[0], eager2)  # new batch
    # stop rules switched on and off under the same pointers: the step graph gains and loses the stop-rules kernel
    s_eager, s_graph = r.sched(), r.sched()
    r.eng.set_sched(s_eager, 100, 40)
    want, _ = r.run(n, False, hist=h)
    r.eng.set_sched(None)
    _equal(r.run(n, True, hist=h)[0], eager)
    r.eng.set_sched(s_graph, 100, 40)
    _equal(r.run(n, True, hist=h)[0], want)
    for k in s_eager:
        assert torch.equal(s_graph[k], s_eager[k]), k
    assert int(s_graph["valid"].max()) > 0
    r.eng.set_sched(None)
    frozen = {k: v.clone() for k, v in s_graph.items()}
    _equal(r.run(n, True, hist=h)[0], eager)
    for k in s_graph:
        assert torch.equal(s_graph[k], frozen[k]), k
    r.eng.close()


@pytest.mark.parametrize("kind", ["layout", "table"])
def test_layout_graph_recaptured_for_new_histories_and_batch(built_lib, kind):
    eng, enc, prompt = _layout(kind)
    n = 11
    eager, _ = _loop(eng, enc, prompt, n, False)
    _equal(_loop(eng, enc, prompt, n, True)[0], eager)
    old = eng._nhist                     # kept alive, so the next histories get other pointers
    eng._nhist = None
    _equal(_loop(eng, enc, prompt, n, True)[0], eager)
    assert eng._nhist["tok"].data_ptr() != old["tok"].data_ptr()
    eager1, _ = _loop(eng, enc[1:], prompt[1:], n, False)
    _equal(_loop(eng, enc[1:], prompt[1:], n, True)[0], eager1)         # new batch
    eng.close()


def test_workspace_bytes(built_lib):
    from surya_b200.config import det_tiny
    from surya_b200.detection import DetEngine
    from surya_b200.synth import det_state_dict

    r = _Rec()
    assert r.eng.workspace_bytes == REC_TINY_WORKSPACE
    r.eng.close()
    for kind, want in (("layout", LAYOUT_TINY_WORKSPACE), ("table", TABLE_TINY_WORKSPACE)):
        eng, _, _ = _layout(kind)
        assert eng.workspace_bytes == want, kind
        eng.close()
    cfg = det_tiny()
    det = DetEngine(cfg, det_state_dict(cfg, seed=0), torch.float16, max_batch=2, max_hw=(256, 256))
    assert det.workspace_bytes == DET_TINY_WORKSPACE
    det.close()
