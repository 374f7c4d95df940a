"""Pages of any size on the device: sb_det_page_resize against PIL byte for byte, sb_det_text_front_stitched against a NumPy stitch
of per-chunk sb_det_text_front outputs bit for bit, detect_text_pages against the host flow (PIL resize, engine forward,
NumPy stitch, text_boxes_from_front, rescale), and OcrPipeline on list pages with high-resolution crops."""
import numpy as np
import pytest
import torch

from test_page_prep_cpu import PROCESSOR_SIZES, SIZES, _page, pil_prepare, pil_split

pytestmark = pytest.mark.gpu


def _engine(kind, max_hw, dtype=torch.float16, max_batch=8):
    from surya_b200.config import det_default, det_tiny
    from surya_b200.detection import DetEngine
    from surya_b200.synth import det_state_dict

    cfg = det_tiny() if kind == "tiny" else det_default()
    return DetEngine(cfg, det_state_dict(cfg, 0), dtype, max_batch=max_batch, max_hw=max_hw)


def _text_page(w, h, seed):
    """White page with dark bars of text-line shape, so that the detector's maps have structure at any size."""
    rng = np.random.default_rng(seed)
    p = np.full((h, w, 3), 255, np.uint8)
    for _ in range(max(4, h * w // 40000)):
        bh, bw = int(rng.integers(6, 30)), int(rng.integers(20, max(21, w // 2)))
        y, x = int(rng.integers(0, max(1, h - bh))), int(rng.integers(0, max(1, w - bw)))
        p[y:y + bh, x:x + bw] = rng.integers(0, 90, 3)
    return p


def _thresholds(m16, text_threshold=0.6, low_text=0.35):
    """get_dynamic_thresholds over a 16-bit map with the device's roundings: the top-k sum is exact in float64 (16-bit values),
    the rest in float32."""
    flat = np.sort(m16.astype(np.float64).ravel())[::-1]
    k = len(flat) - int(len(flat) * 0.9)
    avg = np.float32(flat[:k].sum() / k)
    sf = np.sqrt(np.float32(min(max(avg / np.float32(0.7), np.float32(0)), np.float32(1))))
    tt = np.float32(min(max(np.float32(text_threshold) * sf, np.float32(0.15)), np.float32(0.8)))
    lt = np.float32(min(max(np.float32(low_text) * sf, np.float32(0.1)), np.float32(0.6)))
    return tt, lt


def _upload(pages, psize):
    from surya_b200.page_prep import plan_pages

    plan = plan_pages([(p.shape[1], p.shape[0]) for p in pages], psize)
    packed = torch.from_numpy(np.concatenate([p.ravel() for p in pages])).cuda()
    return plan, packed


@pytest.fixture(scope="module")
def big_tiny(built_lib):
    eng = _engine("tiny", (1024, 1024))
    yield eng
    eng.close()


@pytest.mark.parametrize("processor_size", PROCESSOR_SIZES)
def test_device_resize_equals_pil(big_tiny, processor_size):
    pages = [_page(w, h, seed=w * 7 + h) for w, h in SIZES] + [_page(1300, 3300, 5), _page(640, 1500, 6), _page(300, 1450, 7)]
    plan, packed = _upload(pages, processor_size)
    got = big_tiny.page_resize(packed, plan, processor_size).cpu().numpy()
    ref = [pil_prepare(c, processor_size) for p in pages for c in pil_split(p, processor_size[1])[0]]
    assert got.shape[0] == len(ref)
    for c, r in enumerate(ref):
        assert np.array_equal(got[c], r), f"chunk {c} {plan.chunks[c]}"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_normalised_input_equals_normalised_pil(built_lib, dtype):
    eng = _engine("tiny", (1024, 1024), dtype)
    pages = [_page(816, 1056, 1), _page(2100, 1500, 2)]
    plan, packed = _upload(pages, (1024, 1024))
    got = eng.normalize_u8(eng.page_resize(packed, plan, (1024, 1024)))
    ref = np.stack([pil_prepare(c, (1024, 1024)) for p in pages for c in pil_split(p, 1024)[0]])
    assert torch.equal(got, eng.normalize_u8(torch.from_numpy(ref).cuda()))
    eng.close()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_stitched_front_equals_numpy_stitch(built_lib, dtype):
    from oracle.page_prep_oracle import stitch

    S = 256
    eng = _engine("tiny", (S, S), dtype)
    pages = [_text_page(300, 1401, 1), _text_page(200, 180, 2), _text_page(256, 1800, 3), _text_page(500, 900, 4)]
    plan, packed = _upload(pages, (S, S))
    logits = eng.forward(eng.normalize_u8(eng.page_resize(packed, plan, (S, S))))
    front = eng.text_front_stitched(logits, plan, (S, S))
    per_chunk = eng.text_front(logits, (S, S))
    maps = per_chunk["map"].float().cpu().numpy()
    smap, smask, sthr = front["map"].float().cpu().numpy(), front["mask"].cpu().numpy(), front["thr"].cpu().numpy()
    c = 0
    for p, img in enumerate(pages):
        heights = pil_split(img, S)[1]
        ref = stitch(list(maps[c:c + len(heights)]), heights, S)
        c += len(heights)
        r0, rows = plan.page_tab[p]
        assert rows == ref.shape[0]
        assert np.array_equal(smap[r0:r0 + rows], ref)
        tt, lt = _thresholds(ref)
        assert sthr[p, 0] == tt and sthr[p, 1] == lt
        assert np.array_equal(smask[r0:r0 + rows], (ref > lt).astype(np.uint8))
    eng.close()


def _host_flow(eng, pages, psize):
    """DetectionPredictor's flow with PIL on the host: split + prepare_image, forward, per-chunk front, NumPy stitch, host boxes."""
    from oracle.page_prep_oracle import stitch
    from surya_b200.detection import text_boxes_from_front
    from surya_b200.pipeline import page_polygons

    pw, ph = psize
    out = []
    for img in pages:
        chunks, heights = pil_split(img, ph)
        x = torch.from_numpy(np.stack([pil_prepare(c, psize) for c in chunks])).cuda()
        maps = eng.text_front(eng.forward(eng.normalize_u8(x)), (ph, pw))["map"].float().cpu().numpy()
        m = stitch(list(maps), heights, ph)
        tt, lt = _thresholds(m)
        boxes, conf = text_boxes_from_front(m, (m > lt).astype(np.uint8), float(tt), float(lt))
        out.append(page_polygons(boxes, conf, (img.shape[1], img.shape[0]), (pw, m.shape[0])))
    return out


@pytest.mark.parametrize("kind,psize,sizes", [
    ("tiny", (256, 256), [(180, 240), (400, 1300), (300, 1401), (256, 1800), (520, 700)]),
    ("default", (1024, 1024), [(816, 1056), (1000, 1450), (1275, 3300), (700, 600)]),
])
def test_detect_text_pages_equals_host_flow(built_lib, kind, psize, sizes):
    from surya_b200.detection import detect_text_pages

    eng = _engine(kind, (psize[1], psize[0]), max_batch=4)
    pages = [_text_page(w, h, seed=i) for i, (w, h) in enumerate(sizes)]
    got = detect_text_pages(eng, pages, psize, chunk=5)
    ref = _host_flow(eng, pages, psize)
    assert sum(len(g.polygons) for g in got) > 0
    for g, (polys, conf), (w, h) in zip(got, ref, sizes):
        assert g.polygons == polys and g.confidences == conf
        assert g.image_bbox == [0, 0, w, h]
    eng.close()


def test_ocr_pipeline_highres_pages(built_lib):
    from surya_b200.config import tiny_rec
    from surya_b200.pipeline import OcrPipeline, slice_polygon
    from surya_b200.recognition import RecEngine
    from surya_b200.synth import rec_state_dict

    S = 256
    det = _engine("tiny", (S, S), max_batch=4)
    rcfg = tiny_rec()
    rec = RecEngine(rcfg, rec_state_dict(rcfg, 0), dtype=torch.float16, max_slots=9, s_max=1024, max_patches=16384, max_tokens=4096)
    pages = [_text_page(w, h, seed=10 + i) for i, (w, h) in enumerate([(300, 400), (256, 1500), (200, 180)])]
    high = [np.ascontiguousarray(np.repeat(np.repeat(p, 2, 0), 2, 1)) for p in pages]
    pipe = OcrPipeline(det, rec, rec_batch=8, max_tokens=6, det_chunk=4, workers=2)
    per_page, _ = pipe.run(pages, fixed_steps=True, highres_pages=high, processor_size=(S, S))
    lines = [ln for pg in per_page for ln in pg]
    assert len(lines) >= 3
    det_pages = pipe.detect_pages(pages, (S, S))
    crops, meta = [], []
    for pg, (polys, conf) in enumerate(det_pages):
        for p, c in zip(polys, conf):
            crop = slice_polygon(high[pg], [[int(x * 2.0), int(y * 2.0)] for x, y in p])
            if crop.shape[0] and crop.shape[1]:
                crops.append(crop.astype(np.float32))
                meta.append((pg, p, c))
    order = sorted(range(len(crops)), key=lambda i: -crops[i].shape[1])
    tiles, grids, seqs = pipe.runner.preprocess([crops[i] for i in order], pipe.math_mode)
    tok, sc, _ = pipe.runner.run_preprocessed(tiles, grids, seqs, fixed_steps=True)
    ref = [None] * len(crops)
    for j, i in enumerate(order):
        ref[i] = (meta[i][0], meta[i][1], meta[i][2], tok[j], sc[j])
    assert [(ln.page, ln.polygon, ln.confidence, ln.tokens, ln.scores) for ln in lines] == ref
    rec.close()
    det.close()


def test_over_capacity_and_empty(built_lib):
    from surya_b200._lib import SuryaB200Error
    from surya_b200.detection import detect_text_pages

    eng = _engine("tiny", (256, 256), max_batch=2)
    assert detect_text_pages(eng, [], (256, 256)) == []
    with pytest.raises(SuryaB200Error):
        detect_text_pages(eng, [_text_page(100, 100, 0), _text_page(64, 5000, 1)], (256, 256), max_chunks=4)
    with pytest.raises(SuryaB200Error):
        detect_text_pages(eng, [_text_page(3000, 3000, 0)], (256, 256), max_page_pixels=1 << 20)
    with pytest.raises(SuryaB200Error):
        detect_text_pages(eng, [_text_page(100, 100, 0)], (512, 512))
    got = detect_text_pages(eng, [_text_page(100, 100, 0)], (256, 256))       # the engine is still usable
    assert len(got) == 1
    torch.cuda.synchronize()
    eng.close()
