"""Detection boxes on the device vs on the host (needs a CUDA device): 32 synthetic 1024x1024 text pages through the default detection
config.  Reports the card, CUDA-event time of sb_det_text_boxes per page, host-finish time per page, device-to-host bytes per
page for both paths, and host-to-host pages/s of detection to boxes through the old path (detect_text_front_host + thread-pool
text_boxes_from_front) and the new one (detect_text_boxes_host), alternated in one process.  Prints one JSON line."""
import json
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main(B=32, S=1024, runs=3, workers=16):
    from bench import gpu_info
    from surya_b200.config import det_default
    from surya_b200.detection import (DEFAULT_MAX_BOXES, DEFAULT_MAX_POINTS, DetEngine, detect_text_boxes_host,
                                      detect_text_front_host, text_boxes_from_front, text_boxes_from_tables)
    from surya_b200.synth import det_state_dict, det_synthetic_pages

    if not torch.cuda.is_available():
        raise SystemExit("bench_det_boxes needs a CUDA device")
    cfg = det_default()
    eng = DetEngine(cfg, det_state_dict(cfg, 0), torch.float16, max_batch=16, max_hw=(S, S))
    pages = torch.from_numpy(det_synthetic_pages(B, S, seed=1234, text_like=True)).pin_memory()

    # box kernels alone, on a resident front of all B pages
    xn = eng.normalize_u8(pages.cuda())
    front = eng.text_front(eng.forward(xn), (S, S))
    tabs = eng.text_boxes(front)
    torch.cuda.synchronize()
    reps = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        eng.text_boxes(front, out=tabs)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms_per_page = e0.elapsed_time(e1) / reps / B

    host = {k: v.cpu().numpy() for k, v in tabs.items()}
    text_boxes_from_tables(host["box"][0], host["peak"][0], host["points"][0], int(host["count"][0]))    # imports OpenCV
    t0 = time.perf_counter()
    for b in range(B):
        text_boxes_from_tables(host["box"][b], host["peak"][b], host["points"][b], int(host["count"][b]))
    finish_ms_per_page = (time.perf_counter() - t0) * 1e3 / B

    def old():
        f = detect_text_front_host(eng, pages, chunk=16)
        maps, masks, thr = f["map"].numpy(), f["mask"].numpy(), f["thr"].numpy()
        with ThreadPoolExecutor(max_workers=workers) as ex:
            return list(ex.map(lambda b: text_boxes_from_front(maps[b], masks[b], float(thr[b, 0]), float(thr[b, 1])), range(B)))

    def new():
        return detect_text_boxes_host(eng, pages, chunk=16)

    paths = {f"front + host boxes ({workers}-thread pool)": old, "device boxes + host finish": new}
    for fn in paths.values():       # warm-up: staging buffers, thread pools
        fn()
    times = {k: [] for k in paths}
    for _ in range(runs):
        for k, fn in paths.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            times[k].append(time.perf_counter() - t0)
    print(json.dumps({
        "gpu": gpu_info(torch.cuda.current_device()), "pages": B, "size": S,
        "boxes_per_page": float(host["count"].mean()), "overflowed_pages": int(host["overflow"].sum()),
        "box_kernels_ms_per_page": round(kernel_ms_per_page, 4), "host_finish_ms_per_page": round(finish_ms_per_page, 4),
        "d2h_bytes_per_page": {"front (map + mask + thresholds)": 3 * S * S + 16,
                               "box tables": DEFAULT_MAX_BOXES * 32 + DEFAULT_MAX_POINTS * 8 + 8},
        "detection_to_boxes_pages_per_s": {k: [round(B / t, 1) for t in v] for k, v in times.items()},
    }))
    eng.close()


if __name__ == "__main__":
    main()
