"""Dump decode_attn outputs and caches (GPU) for a fixed seeded grid, one .npy per array, so two builds can be compared
byte for byte: run it on each build with its own output directory and `cmp` the files.

Grid: dtype x head_dim {64, 80, 128} x GQA group {1, 2, 4, 8} x s_max {256, 512, 1536}.  Each case is one launch over rows
at pos 0, 127, 128, 129, 4 NKG - 1, 4 NKG + 1 (NKG = 128 / (head_dim / 8), the key groups of the P.V sum), s_max - 1 and
four ragged positions, in shuffled slots of a cache with two KV heads.  16-bit arrays are stored as int16 bit patterns.

    python tools/dump_decode_attn.py OUT_DIR
"""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from surya_b200 import ops  # noqa: E402

NKV = 2


def run_case(dtype, d, G, s_max, seed):
    nh = G * NKV
    g = torch.Generator(device="cuda").manual_seed(seed)
    nkg4 = 4 * (128 // (d // 8))
    ragged = torch.randint(0, s_max, (4,), generator=torch.Generator().manual_seed(seed)).tolist()
    poses = [0, 127, 128, 129, nkg4 - 1, nkg4 + 1, s_max - 1] + ragged
    B = len(poses)
    slots = B + 3
    slot_ids = torch.randperm(slots, generator=torch.Generator().manual_seed(seed + 1))[:B]
    kc = torch.randn(slots, NKV, s_max, d, device="cuda", generator=g).to(dtype)
    vc = torch.randn(slots, NKV, s_max, d, device="cuda", generator=g).to(dtype)
    qkv = torch.randn(B, (nh + 2 * NKV) * d, device="cuda", generator=g).to(dtype)
    inv = (1.0 / (10000.0 ** (torch.arange(0, d, 2, device="cuda").float() / d))).contiguous()
    slot_t = slot_ids.to(device="cuda", dtype=torch.int32)
    pos_t = torch.tensor(poses, device="cuda", dtype=torch.int32)
    out = ops.decode_attn(qkv, kc, vc, slot_t, pos_t, inv, nh, NKV, d, d ** -0.5)
    torch.cuda.synchronize()
    return {"out": out, "kcache": kc, "vcache": vc}


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    dst = Path(sys.argv[1])
    dst.mkdir(parents=True, exist_ok=True)
    n = 0
    for dtype in (torch.bfloat16, torch.float16):
        for d in (64, 80, 128):
            for G in (1, 2, 4, 8):
                for s_max in (256, 512, 1536):
                    tag = f"{str(dtype).split('.')[-1]}_d{d}_g{G}_s{s_max}"
                    arrays = run_case(dtype, d, G, s_max, seed=d * 1000 + G * 100 + s_max)
                    for name, t in arrays.items():
                        np.save(dst / f"{tag}_{name}.npy", t.view(torch.int16).cpu().numpy())
                        n += 1
    print(f"wrote {n} arrays to {dst}")


if __name__ == "__main__":
    main()
