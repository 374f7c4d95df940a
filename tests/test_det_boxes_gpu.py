"""Text-box tables on the device (sb_det_text_boxes, SURVEY §8 f1 second half) against the NumPy restatement
(tests/det_boxes_ref.py), and detect_text_boxes_host / OcrPipeline against the host path (detect_text_front_host +
text_boxes_from_front), byte for byte."""
import numpy as np
import pytest
import torch

from det_boxes_ref import assert_same, synth_map, text_box_tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny_engine(built_lib):
    from surya_b200.config import det_tiny
    from surya_b200.detection import DetEngine
    from surya_b200.synth import det_state_dict

    cfg = det_tiny()
    eng = DetEngine(cfg, det_state_dict(cfg, 0), torch.float16, max_batch=8, max_hw=(256, 256))
    yield eng
    eng.close()


def _spiral(H, W, step=4):
    """One component: each ring's left side turns into the next ring's top side."""
    sp = np.zeros((H, W), bool)
    r = 0
    while r + step < min(H, W) - r:
        sp[r, r:W - r] = sp[r:H - r, W - 1 - r] = sp[H - 1 - r, r:W - r] = True
        sp[r + step:H - r, r] = True
        sp[r + step, r:r + step] = True
        r += step
    return sp


def _crafted(H, W, seed):
    """Lines crossing the 32-px tiles in both directions, ragged text lines, and a U-shape opening upward over a tile border."""
    rng = np.random.default_rng(seed)
    m = synth_map(rng, H, W)
    m[31:34, 5:W - 5] = 0.9                       # crosses every vertical tile border, on a horizontal one
    m[5:H - 5, 63:65] = 0.8                       # crosses every horizontal tile border, on a vertical one
    u = np.zeros((70, 90), bool)
    u[:, :3] = u[:, -3:] = u[-3:, :] = True
    m[H // 2 - 35:H // 2 + 35, W // 2 - 45:W // 2 + 45][u] = 0.85
    return m


def _device_tables(eng, maps, low, tt, dtype, max_boxes=1024, max_points=65536):
    m16 = torch.from_numpy(np.stack(maps)).to(dtype).cuda()
    front = {"map": m16, "mask": (m16.float() > low).to(torch.uint8),
             "thr": torch.tensor([[tt, low, 0.0, 1.0]] * len(maps), dtype=torch.float32, device="cuda")}
    out = eng.text_boxes(front, max_boxes, max_points)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, m16.float().cpu().numpy(), front["mask"].cpu().numpy()


def _assert_tables_equal(got, b, ref):
    assert int(got["count"][b]) == ref["count"] and int(got["overflow"][b]) == ref["overflow"]
    if ref["overflow"]:
        return
    c = ref["count"]
    assert np.array_equal(got["box"][b, :c], ref["box"][:c])
    assert got["peak"][b, :c].tobytes() == ref["peak"][:c].tobytes()
    used = int(ref["box"][c - 1, 4] + ref["box"][c - 1, 5]) if c else 0
    assert np.array_equal(got["points"][b, :used], ref["points"][:used])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,W", [(1024, 1024), (384, 512), (1000, 777)])
def test_device_tables_equal_restatement(tiny_engine, H, W, dtype):
    low, tt = 0.35, 0.6
    maps = [_crafted(H, W, 1), np.where(_spiral(H, W), 0.9, 0.1).astype(np.float32),
            np.where((np.arange(H)[:, None] + np.arange(W)[None, :]) % 2 == 0, 0.9, 0.1).astype(np.float32),
            synth_map(np.random.default_rng(H + W), H, W)]
    got, m, mask = _device_tables(tiny_engine, maps, low, tt, dtype)
    counts = []
    for b in range(len(maps)):
        ref = text_box_tables(m[b], mask[b], tt)
        _assert_tables_equal(got, b, ref)
        counts.append(ref["count"])
    assert counts[1] == 1 and counts[2] == 0


def test_tables_are_deterministic(tiny_engine):
    maps = [_crafted(1024, 1024, s) for s in range(4)]
    a, _, _ = _device_tables(tiny_engine, maps, 0.35, 0.6, torch.float16)
    b, _, _ = _device_tables(tiny_engine, maps, 0.35, 0.6, torch.float16)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def _host_path(eng, pages, chunk):
    from surya_b200.detection import detect_text_front_host, text_boxes_from_front

    front = detect_text_front_host(eng, pages, chunk=chunk)
    maps = front["map"] if front["map"].dtype != torch.bfloat16 else front["map"].float()
    return [text_boxes_from_front(maps[b].numpy(), front["mask"][b].numpy(), float(front["thr"][b, 0]),
                                  float(front["thr"][b, 1])) for b in range(len(maps))]


def _assert_pages_equal(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert_same(g, r)


def test_boxes_host_equals_front_path_tiny(tiny_engine):
    from surya_b200.detection import detect_text_boxes_host
    from surya_b200.synth import det_synthetic_pages

    pages = torch.from_numpy(det_synthetic_pages(5, 256, seed=31, text_like=True)).pin_memory()
    ref = _host_path(tiny_engine, pages, 2)
    _assert_pages_equal(detect_text_boxes_host(tiny_engine, pages, chunk=2), ref)


def test_overflowing_pages_take_the_host_path(built_lib):
    """Capacities too small for some pages: those are flagged and finished on the host, with the same result."""
    from surya_b200.config import det_default
    from surya_b200.detection import DetEngine, _front_pipeline, detect_text_boxes_host
    from surya_b200.synth import det_state_dict, det_synthetic_pages

    cfg = det_default()
    eng = DetEngine(cfg, det_state_dict(cfg, seed=0), torch.float16, max_batch=4, max_hw=(512, 512))
    pages = torch.from_numpy(det_synthetic_pages(8, 512, seed=9, text_like=True)).pin_memory()
    ref = _host_path(eng, pages, 4)
    full = _front_pipeline(eng, pages, 4, None, 0.6, 0.35, True, (1024, 65536))
    count, box = full["count"].numpy().copy(), full["box"].numpy().copy()
    assert not full["overflow"].numpy().any()
    used = [int(box[b, c - 1, 4] + box[b, c - 1, 5]) if c else 0 for b, c in enumerate(count)]
    caps = [{"max_points": max(2, sorted(set(used))[0])}]          # the pages with more points overflow
    if len(set(count)) > 1:
        caps.append({"max_boxes": max(1, sorted(set(count))[0])})
    assert len(set(used)) > 1, used
    for cap in caps:
        tabs = _front_pipeline(eng, pages, 4, None, 0.6, 0.35, True, (cap.get("max_boxes", 1024), cap.get("max_points", 65536)))
        flagged = tabs["overflow"].numpy().astype(bool)
        assert 0 < flagged.sum() < len(pages), (cap, count, used)
        _assert_pages_equal(detect_text_boxes_host(eng, pages, chunk=4, **cap), ref)
    eng.close()


@pytest.mark.parametrize("text_like", [True, False])
def test_boxes_host_equals_front_path_default_b32(built_lib, text_like):
    from surya_b200.config import det_default
    from surya_b200.detection import DetEngine, detect_text_boxes_host
    from surya_b200.synth import det_state_dict, det_synthetic_pages

    cfg = det_default()
    eng = DetEngine(cfg, det_state_dict(cfg, seed=0), torch.float16, max_batch=16, max_hw=(1024, 1024))
    pages = torch.from_numpy(det_synthetic_pages(32, 1024, seed=3, text_like=text_like)).pin_memory()
    ref = _host_path(eng, pages, 16)
    got = detect_text_boxes_host(eng, pages, chunk=16)
    _assert_pages_equal(got, ref)
    eng.close()


def test_ocr_pipeline_lines_equal_host_box_path(built_lib):
    from surya_b200.config import det_tiny, tiny_rec
    from surya_b200.detection import DetEngine
    from surya_b200.pipeline import OcrPipeline, page_polygons
    from surya_b200.recognition import RecEngine
    from surya_b200.synth import det_state_dict, det_synthetic_pages, rec_state_dict

    S = 256
    dcfg, rcfg = det_tiny(), tiny_rec()
    det = DetEngine(dcfg, det_state_dict(dcfg, 0), torch.float16, max_batch=4, max_hw=(S, S))
    rec = RecEngine(rcfg, rec_state_dict(rcfg, 0), dtype=torch.float16, max_slots=9, s_max=256, max_patches=8192, max_tokens=2048)
    pages = det_synthetic_pages(5, S, seed=77, text_like=True)
    pipe = OcrPipeline(det, rec, rec_batch=8, max_tokens=6, det_chunk=2, workers=2)
    per_page, _ = pipe.run(pages, fixed_steps=True)
    pipe.detect = lambda p: [page_polygons(b, c, (S, S), (S, S)) for b, c in _host_path(det, p, 2)]
    ref_page, _ = pipe.run(pages, fixed_steps=True)
    assert sum(len(p) for p in per_page) >= 5
    for got, ref in zip(per_page, ref_page):
        assert [(ln.polygon, ln.confidence, ln.tokens) for ln in got] == [(ln.polygon, ln.confidence, ln.tokens) for ln in ref]
    rec.close()
    det.close()
