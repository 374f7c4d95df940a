"""Detection forward only (GPU box): BASELINE config 3 (32 pages 1024^2, fp16) resident forward, CUDA-event timed; prints ms
per forward and pages/s.  Environment switches of the kernels under test are read by the library (SB_DET_FUSED_HEAD, SB_FMB_FUSED)."""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def main(B=32, size=1024, reps=6):
    from surya_b200.config import det_default
    from surya_b200.detection import DetEngine
    from surya_b200.synth import det_normalize, det_state_dict, det_synthetic_pages

    cfg = det_default()
    eng = DetEngine(cfg, det_state_dict(cfg, 0), torch.float16, max_batch=B, max_hw=(size, size))
    x = det_normalize(det_synthetic_pages(B, size, seed=3, text_like=True)).cuda().half()
    for _ in range(3):
        out = eng.forward(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = eng.forward(x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print(f"detection forward B={B} {size}x{size}: {ms:.3f} ms  {B / ms * 1e3:.1f} pages/s  checksum {out.float().sum().item():.4f}")


if __name__ == "__main__":
    main()
