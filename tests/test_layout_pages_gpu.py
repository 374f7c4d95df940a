"""GPU tests of the layout page flow: sb_layout_preprocess against its restatement (and cv2 within the stated bound), the
header/footer rule in box_next_token, sb_layout_decode_pages against the predictor's loop run step by step over the model
surface, and layout_pages from uint8 pages against the same flow fed host-preprocessed pixel values."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import layout_pages_oracle as O

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


def _page(h, w, seed):
    import cv2

    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return cv2.GaussianBlur(img, (0, 0), 1.5)


def _engine(cfg, dtype=torch.float16, max_batch=8, boost=None):
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_layout_state_dict, swin_state_dict

    sdd = adetr_layout_state_dict(cfg.decoder, 0)
    if boost:
        w = sdd["lm_head.weight"].clone()
        for row, f in boost.items():
            w[row] *= f
        sdd["lm_head.weight"] = w
    return LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), sdd, dtype=dtype, max_batch=max_batch)


@pytest.mark.parametrize("dtype", DTYPES)
def test_preprocess_equals_restatement(built_lib, dtype):
    """Whole pages, slices read out of a resident page, and small upscaled pages: byte-identical to the restatement; within the
    stated bound of cv2.resize."""
    import cv2

    from surya_b200 import layout_pages as LP
    from surya_b200.config import layout_tiny

    cfg = layout_tiny()
    eng = _engine(cfg, dtype)
    H, W = cfg.encoder.image_size
    pages = [_page(1056, 816, 0), _page(2600, 1700, 1), _page(40, 30, 2), _page(300, 3100, 3)]
    offs = np.cumsum([0] + [p.nbytes for p in pages])
    dev = torch.from_numpy(np.concatenate([p.reshape(-1) for p in pages])).cuda()
    rects, po, pw, want = [], [], [], []
    for i, p in enumerate(pages):
        h, w = p.shape[:2]
        for x0, y0, sw, sh, _, _ in LP.slice_rects(w, h):
            rects.append((x0, y0, sw, sh))
            po.append(int(offs[i]))
            pw.append(w)
            want.append(O.process(p[y0:y0 + sh, x0:x0 + sw], (H, W), dtype))
    assert len(rects) > len(pages)                          # slices were cut
    jobs, ti, tw = LP.plan_jobs(rects, po, pw, (H, W))
    got = eng.preprocess(dev, jobs.cuda(), ti.cuda(), tw.cuda()).cpu()
    assert torch.equal(got, torch.stack(want))
    # against cv2: the resized bytes recovered from the fp16 output are within one of cv2's
    if dtype == torch.float16:
        u8 = torch.round((got.float() * 0.5 + 0.5) * 255).to(torch.uint8).numpy()
        off = total = 0
        for k, (x0, y0, sw, sh) in enumerate(rects):
            page = pages[[i for i in range(len(pages)) if offs[i] == po[k]][0]]
            ref = cv2.resize(page[y0:y0 + sh, x0:x0 + sw], (W, H), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1)
            d = np.abs(u8[k].astype(np.int16) - ref.astype(np.int16))
            assert d.max() <= 1
            off += int((d > 0).sum())
            total += d.size
        assert off / total <= 2e-5
    eng.close()


def _next_pages(bbox, cls, wh, sticky, dtype, hist_cls=None, page=True):
    from surya_b200 import _lib, ops
    from surya_b200.config import layout_default

    d = layout_default().decoder
    lib = _lib.load()
    B, C = cls.shape
    out = torch.empty((B, 7), dtype=torch.int64, device="cuda")
    done = torch.empty((B,), dtype=torch.uint8, device="cuda")
    hp = (ctypes.c_void_p * 1)(cls.data_ptr())
    hn = (ctypes.c_int * 1)(C)
    hm = (ctypes.c_int * 1)(0)
    hh = (ctypes.c_void_p * 1)(hist_cls.data_ptr()) if hist_cls is not None else None
    pos = torch.zeros(B, dtype=torch.int32, device="cuda")
    base = torch.zeros(1, dtype=torch.int32, device="cuda")
    if not page:
        _lib.check(lib.sb_box_next_token(_lib.ptr(bbox), hp, hn, hm, ctypes.c_int(1), ctypes.c_float(1024.0), _lib.ptr(out), _lib.ptr(done),
                                         ctypes.c_int(0), ctypes.c_int(d.eos_token_id), ctypes.c_int(d.pad_token_id), ctypes.c_int(B),
                                         _lib.ptr(pos), _lib.ptr(base), ctypes.c_int(1), None, None, hh, None, _lib.stream_ptr()))
        return out, done
    _lib.check(lib.sb_box_next_token_pages(_lib.ptr(bbox), hp, hn, hm, ctypes.c_int(1), ctypes.c_float(1024.0), _lib.ptr(out), _lib.ptr(done),
                                           ctypes.c_int(0), ctypes.c_int(d.eos_token_id), ctypes.c_int(d.pad_token_id), ctypes.c_int(B),
                                           _lib.ptr(pos), _lib.ptr(base), ctypes.c_int(1), None, None, hh, None, _lib.ptr(wh),
                                           _lib.ptr(sticky), ctypes.c_int(ops.dt_code(dtype)), ctypes.c_int(10 + d.special_token_count),
                                           ctypes.c_int(9 + d.special_token_count), ctypes.c_float(d.skew_scaler), _lib.stream_ptr()),
               "sb_box_next_token_pages")
    return out, done


@pytest.mark.parametrize("dtype", DTYPES)
def test_box_next_token_page_rule(built_lib, dtype):
    from surya_b200.config import layout_default

    d = layout_default().decoder
    g = torch.Generator().manual_seed(11)
    B, C = 512, d.label_count
    header, footer = 10 + d.special_token_count, 9 + d.special_token_count
    bbox = torch.rand((B, 6), generator=g).to(dtype).float()
    bbox[:, 1] = (torch.arange(B) % 64).float() / 64         # rows from the top edge to the bottom edge
    bbox = bbox.to(dtype).float()
    cls = torch.randn((B, C), generator=g)
    cls[:, header] += 4 * (torch.arange(B) % 2 == 0)
    cls[:, footer] += 4 * (torch.arange(B) % 4 == 1)
    cls[::7, d.eos_token_id] += 9                            # rows done at this step: no rule
    cls[5] = -1.0                                            # zeroing the argmax leaves ties at 0 behind: first index wins
    cls[5, header], cls[5, 7], cls[5, 9] = 3.0, 0.0, 0.0
    bbox[5] = torch.tensor([0.5, 0.5, 0.3, 0.3, 0.5, 0.5]).to(dtype).float()
    cls = cls.to(dtype).float()
    sticky = (torch.arange(B) % 9 == 3)
    wh = torch.randint(200, 4000, (B, 2), generator=g, dtype=torch.int32)
    sizes = [tuple(r) for r in wh.tolist()]
    tok, cm, done, fired = O.next_token_pages(bbox, cls, sizes, sticky, dtype, d)
    assert fired > 20 and cm[5, header] == 0 and tok[5, 6] == 7      # the zeroed logit ties with 7 and 9: the first wins
    hist = torch.zeros((1, B, C), device="cuda")
    got, gdone = _next_pages(bbox.cuda(), cls.cuda(), wh.cuda(), sticky.to(torch.uint8).cuda(), dtype, hist)
    assert torch.equal(got.cpu(), tok) and torch.equal(gdone.cpu().bool(), done) and torch.equal(hist[0].cpu(), cm)
    # where the rule cannot fire (every row already done), the page entry is today's kernel bit for bit: every token column,
    # done and the head history
    hist_plain, hist_page = torch.zeros((1, B, C), device="cuda"), torch.zeros((1, B, C), device="cuda")
    plain, pdone = _next_pages(bbox.cuda(), cls.cuda(), None, None, dtype, hist_plain, page=False)
    same, sdone = _next_pages(bbox.cuda(), cls.cuda(), wh.cuda(), torch.ones(B, dtype=torch.uint8, device="cuda"), dtype, hist_page)
    assert torch.equal(plain, same) and torch.equal(pdone, sdone) and torch.equal(hist_plain, hist_page)
    assert torch.equal(plain.cpu()[:, 6], cls.argmax(-1)) and torch.equal(hist_plain[0].cpu(), cls)
    # the page entry needs a page size
    with pytest.raises(Exception):
        _next_pages(bbox.cuda(), cls.cuda(), None, None, dtype)


def _mirror_loop(eng, enc, sizes, n_steps):
    """LayoutPredictor's loop over the model surface (decode_step), with the rule and stop restated on the host."""
    d = eng.cfg.decoder
    B = enc.shape[0]
    eng.setup_cache(B)
    tokens = torch.full((B, 7), d.bos_token_id, dtype=torch.int64, device="cuda")
    sticky = torch.zeros(B, dtype=torch.bool)
    hist, fired_total = [], 0
    for s in range(n_steps):
        bbox, cls = eng.decode_step(tokens, enc, s)
        tok, cm, dn, fired = O.next_token_pages(bbox.cpu(), cls.cpu(), sizes, sticky, eng.dtype, d)
        fired_total += fired
        hist.append((tok, bbox.cpu(), cm, dn))
        sticky |= dn
        if bool(sticky.all()):
            break
        tokens = tok.cuda()
    return hist, fired_total


@pytest.mark.parametrize("which,boost", [("tiny", {13: 6.0, 12: 6.0}), ("tiny", {0: 0.0, 1: 30.0}), ("default", {13: 4.0, 12: 4.0})])
def test_run_pages_equals_the_predictor_loop(built_lib, which, boost):
    from surya_b200.config import layout_default, layout_tiny
    from surya_b200.synth import layout_synthetic_pages

    cfg = layout_tiny() if which == "tiny" else layout_default()
    B = 6
    eng = _engine(cfg, torch.float16, max_batch=B, boost=boost)
    x = layout_synthetic_pages(B, cfg.encoder.image_size, seed=4).cuda()
    enc = eng.encode(x)
    sizes = [(816, 1056), (1700, 1200), (300, 3000), (1200, 1200), (2000, 700), (640, 640)]
    n_steps = 40
    tok, bbox, cls, done = [t.cpu() for t in eng.run_pages(enc, torch.tensor(sizes), n_steps)]
    hist, fired = _mirror_loop(eng, enc, sizes, n_steps)
    n_ref = len(hist)
    assert n_ref <= tok.shape[0] <= n_steps
    for s, (t, b, c, dn) in enumerate(hist):
        assert torch.equal(tok[s], t), s
        assert torch.equal(bbox[s], b) and torch.equal(cls[s], c) and torch.equal(done[s].bool(), dn), s
    if boost.get(1):
        # every row ends at once: the loop stops after the first group of steps that saw it
        assert n_ref < n_steps and tok.shape[0] <= n_ref + 16 and tok.shape[0] < n_steps
    else:
        assert fired >= 3, fired
    eng.close()


def test_layout_pages_device_equals_host_preprocessed(built_lib):
    from surya_b200 import layout_pages as LP
    from surya_b200.config import layout_tiny

    cfg = layout_tiny()
    H, W = cfg.encoder.image_size
    eng = _engine(cfg, torch.float16, max_batch=8, boost={13: 5.0, 12: 5.0})
    sizes = [(816, 1056), (1632, 2112), (1600, 1600), (3000, 900), (200, 150)]
    pages = [_page(h, w, i) for i, (w, h) in enumerate(sizes)]
    run = LP.layout_pages(eng, pages, batch_size=8)
    px = []
    for p0, p1 in LP.page_batches([LP.slice_count(w, h) for w, h in sizes], 8):
        for p in range(p0, p1):
            for x0, y0, sw, sh, _, _ in LP.slice_rects(*sizes[p]):
                px.append(O.process(pages[p][y0:y0 + sh, x0:x0 + sw], (H, W), torch.float16))
    ref = LP.layout_pages(eng, pages, batch_size=8, pixel_values=torch.stack(px))
    assert len(run.results) == len(pages) and any(r.sliced for r in run.results)
    assert run.results == ref.results and run.steps_run == ref.steps_run
    assert sum(len(r.bboxes) for r in run.results) > 0
    assert set(run.timing) == {"upload", "preprocess", "encoder", "decode", "host_post"}
    eng.close()


def test_errors_are_loud(built_lib):
    from surya_b200 import _lib
    from surya_b200 import layout_pages as LP
    from surya_b200.config import layout_tiny, table_tiny
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    cfg = layout_tiny()
    eng = _engine(cfg, torch.float16, max_batch=4)
    with pytest.raises(_lib.SuryaB200Error, match="at least one page"):
        LP.layout_pages(eng, [], batch_size=4)
    with pytest.raises(_lib.SuryaB200Error, match="uint8"):
        LP.layout_pages(eng, [np.zeros((64, 64, 3), np.float32)], batch_size=4)
    with pytest.raises(_lib.SuryaB200Error, match="uint8"):
        LP.layout_pages(eng, [np.zeros((64, 64), np.uint8)], batch_size=4)
    with pytest.raises(_lib.SuryaB200Error, match="max_batch"):
        LP.layout_pages(eng, [np.zeros((64, 64, 3), np.uint8)], batch_size=5)
    enc = eng.encode(torch.zeros((4, 3) + tuple(cfg.encoder.image_size), device="cuda"))
    with pytest.raises(_lib.SuryaB200Error, match="max_batch"):
        eng.run_pages(torch.cat([enc, enc[:1]]), torch.full((5, 2), 100), 8)
    with pytest.raises(_lib.SuryaB200Error, match="page_wh"):
        eng.run_pages(enc, torch.full((3, 2), 100), 8)
    # the C entry refuses a table engine and a null page size
    tcfg = table_tiny()
    teng = LayoutEngine(tcfg, swin_state_dict(tcfg.encoder, 0), adetr_table_state_dict(tcfg.decoder, 0), dtype=torch.float16, max_batch=4)
    with pytest.raises(_lib.SuryaB200Error, match="layout engine"):
        teng.run_pages(enc, torch.full((4, 2), 100), 8)
    n_run = ctypes.c_int(0)
    buf = torch.zeros(1 << 16, device="cuda")
    rc = teng.lib.sb_layout_decode_pages(teng._h, _lib.ptr(enc), ctypes.c_int(1), _lib.ptr(buf), ctypes.c_int(1), _lib.ptr(buf),
                                         ctypes.c_int(4), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf), ctypes.byref(n_run),
                                         _lib.stream_ptr())
    assert rc != 0
    rc = eng.lib.sb_layout_decode_pages(eng._h, _lib.ptr(enc), ctypes.c_int(1), _lib.ptr(buf), ctypes.c_int(1), None,
                                        ctypes.c_int(4), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf), ctypes.byref(n_run),
                                        _lib.stream_ptr())
    assert rc != 0
    teng.close()
    eng.close()
