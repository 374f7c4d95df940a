"""GPU tests of the table page flow: bounded sb_layout_preprocess jobs (crops that extend past the page read 0, as PIL's crop
fills them) against the job-table restatement, and table_pages from uint8 pages against the same flow fed host-preprocessed
pixel values."""
import numpy as np
import pytest
import torch

from oracle import layout_pages_oracle as LPO
from oracle import table_pages_oracle as T

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]


def _page(h, w, seed):
    import cv2

    rng = np.random.default_rng(seed)
    return cv2.GaussianBlur(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (0, 0), 1.5)


def _table_engine(cfg, dtype=torch.float16, max_batch=8):
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_table_state_dict, swin_state_dict

    return LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), adetr_table_state_dict(cfg.decoder, 0), dtype=dtype, max_batch=max_batch,
                        max_rows=512, max_prefill_tokens=4096)


def _layout_engine(cfg, table_boost, max_batch=8):
    """Synthetic layout weights with the class row of Table scaled up, so that tables are found."""
    from surya_b200.layout import LayoutEngine
    from surya_b200.synth import adetr_layout_state_dict, swin_state_dict

    sdd = adetr_layout_state_dict(cfg.decoder, 0)
    w = sdd["lm_head.weight"].clone()
    w[LPO.LABEL_TO_ID["Table"] + cfg.decoder.special_token_count] *= table_boost
    sdd["lm_head.weight"] = w
    return LayoutEngine(cfg, swin_state_dict(cfg.encoder, 0), sdd, dtype=torch.float16, max_batch=max_batch)


@pytest.mark.parametrize("dtype", DTYPES)
def test_bounded_jobs_equal_restatement(built_lib, dtype):
    """Crops inside the page, across the right edge, the bottom edge, both, with negative x0 / y0, 1-px crops and a crop wholly
    outside the page: byte-identical to the restatement and to PIL's zero-filled crop resized by the restatement.  A bounded
    job inside its page equals the same job with page height 0."""
    from surya_b200 import layout_pages as LP
    from surya_b200.config import table_tiny

    cfg = table_tiny()
    eng = _table_engine(cfg, dtype)
    H, W = cfg.encoder.image_size
    pages = [_page(300, 400, 0), _page(1100, 850, 1)]
    offs = np.cumsum([0] + [p.nbytes for p in pages])
    flat = np.concatenate([p.reshape(-1) for p in pages])
    dev = torch.from_numpy(flat).cuda()
    crops = [(0, 10, 20, 300, 200), (0, 350, 40, 420, 120), (0, 50, 250, 200, 330), (0, 330, 260, 410, 315), (0, -7, -3, 80, 60),
             (0, -20, 100, 401, 310), (1, 5, 6, 6, 7), (1, 849, 1099, 850, 1100), (1, 900, 50, 960, 90), (1, -40, -30, -10, -5),
             (1, 100, 1000, 900, 1150), (1, 0, 0, 850, 1100)]
    rects = [(x0, y0, x1 - x0, y1 - y0) for _, x0, y0, x1, y1 in crops]
    po = [int(offs[p]) for p, *_ in crops]
    pw = [pages[p].shape[1] for p, *_ in crops]
    ph = [pages[p].shape[0] for p, *_ in crops]
    jobs, ti, tw = LP.plan_jobs(rects, po, pw, (H, W), page_h=ph)
    got = eng.preprocess(dev, jobs.cuda(), ti.cuda(), tw.cuda()).cpu()
    assert torch.equal(got, T.preprocess_jobs(flat, jobs, ti, tw, (H, W), dtype))
    for k, (p, x0, y0, x1, y1) in enumerate(crops):
        assert torch.equal(got[k], LPO.process(T.crop_zero_fill(pages[p], (x0, y0, x1, y1)), (H, W), dtype)), crops[k]
    assert float(got[9].float().min()) == float(got[9].float().max()) == -1.0          # wholly outside: all black
    inside = [k for k, (p, x0, y0, x1, y1) in enumerate(crops) if x0 >= 0 and y0 >= 0 and x1 <= pw[k] and y1 <= ph[k]]
    assert len(inside) >= 4
    j0, ti0, tw0 = LP.plan_jobs([rects[k] for k in inside], [po[k] for k in inside], [pw[k] for k in inside], (H, W))
    assert torch.equal(eng.preprocess(dev, j0.cuda(), ti0.cuda(), tw0.cuda()).cpu(), got[inside])
    eng.close()


def _host_pixels(eng, run, pages, highres, skip):
    """The tables' pixel values restated on the host (PIL's zero-filled crop, cubic model, normalisation) in the engine dtype."""
    from surya_b200 import table_pages as TP

    his = [p if h is None else h for p, h in zip(pages, highres)]
    plan = TP.plan_tables(None if skip else run.layout, [(p.shape[1], p.shape[0]) for p in pages],
                          [(p.shape[1], p.shape[0]) for p in his])
    H, W = eng.cfg.encoder.image_size
    return torch.stack([LPO.process(T.crop_zero_fill(his[tp.page], tp.crop), (H, W), eng.dtype) for tp in plan])


@pytest.mark.parametrize("which,skip", [("tiny", False), ("tiny", True), ("default", False), ("default", True)])
def test_table_pages_device_equals_host_preprocessed(built_lib, which, skip):
    """table_pages with device preprocessing equals the same flow fed host-preprocessed pixel values, bit for bit in every
    TableResult.to_dict(), over pages with and without a high-resolution copy, in batches that mix pages."""
    from surya_b200 import table_pages as TP
    from surya_b200.config import layout_default, layout_tiny, table_default, table_tiny

    lcfg, tcfg = (layout_tiny(), table_tiny()) if which == "tiny" else (layout_default(), table_default())
    lay = _layout_engine(lcfg, 12.0 if which == "tiny" else 6.0)       # the tiny model stops at once below x 12
    tab = _table_engine(tcfg, torch.float16, max_batch=4)
    pages = [_page(700, 540, 3), _page(1000, 700, 4), _page(500, 900, 5)]
    highres = [_page(1400, 1080, 6), None, _page(1000, 1800, 7)]
    kw = dict(highres_pages=highres, skip_table_detection=skip, batch_size=3, layout_batch_size=4, max_boxes=24)
    dev = TP.table_pages(tab, pages, None if skip else lay, **kw)
    n = sum(len(r) for r in dev.results)
    assert n >= (3 if skip else 4), [len(r) for r in dev.results]       # tables found, more than one batch
    assert sum(len(b) for b in dev.table_boxes) == n
    px = _host_pixels(tab, dev, pages, highres, skip)
    host = TP.table_pages(tab, pages, None if skip else lay, pixel_values=px, **kw)
    assert [[r.to_dict() for r in page] for page in dev.results] == [[r.to_dict() for r in page] for page in host.results]
    assert dev.table_boxes == host.table_boxes and dev.steps_run == host.steps_run
    lay.close()
    tab.close()


def test_errors_are_loud(built_lib):
    from surya_b200 import table_pages as TP
    from surya_b200._lib import SuryaB200Error
    from surya_b200.config import layout_tiny, table_tiny

    lay = _layout_engine(layout_tiny(), 6.0, max_batch=2)
    tab = _table_engine(table_tiny(), max_batch=2)
    pages = [_page(200, 150, 8), _page(220, 160, 9)]
    with pytest.raises(SuryaB200Error, match="max_batch"):
        TP.table_pages(tab, pages, skip_table_detection=True, batch_size=3)
    with pytest.raises(SuryaB200Error, match="max_batch"):
        TP.table_pages(tab, pages, lay, batch_size=2, layout_batch_size=3)
    with pytest.raises(SuryaB200Error, match="high-resolution"):
        TP.table_pages(tab, pages, lay, highres_pages=[None], batch_size=2, layout_batch_size=2)
    with pytest.raises(SuryaB200Error, match="uint8"):
        TP.table_pages(tab, [p.astype(np.int16) for p in pages], skip_table_detection=True, batch_size=2)
    with pytest.raises(SuryaB200Error, match="table_rec engine"):
        TP.table_pages(lay, pages, lay, batch_size=2, layout_batch_size=2)
    with pytest.raises(SuryaB200Error, match="layout engine"):
        TP.table_pages(tab, pages, tab, batch_size=2)
    lay.close()
    tab.close()
