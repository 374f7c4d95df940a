"""The plain GEMM kernel's staged-only instantiation (gemm_tn_kernel with STAGED = true: every BN = 128 launch the 16-bit
staged epilogue takes) against the plain kernel at BN = 64, which keeps the fallback epilogue, bit for bit (GPU).

Both run the same per-k-block accumulation and the same staged epilogue, so every tile width gives the same bits.  The cases
cover ragged M, N not a multiple of 128, a partial last k-block (K = 592), every staged epilogue the engines use, and a
persistent grid with more tiles than SMs."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = [torch.bfloat16, torch.float16]
CASES = [   # (M, N, K, epilogue)
    (100, 256, 128, "none"),
    (300, 1920, 256, "bias"),
    (260, 200, 592, "gelu"),
    (384, 1000, 320, "residual"),
    (640, 768, 448, "swiglu"),
    (1000, 1920, 1280, "rowscale"),
    (4096, 2048, 512, "bias"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("M,N,K,epi", CASES)
def test_staged_bn128_equals_bn64(built_lib, dtype, M, N, K, epi):
    from surya_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1 if epi in ("bias", "gelu", "swiglu") else None
    rs = torch.rand(M, device="cuda", generator=g) + 0.5 if epi == "rowscale" else None
    res = (torch.randn(M, N, device="cuda", generator=g)).to(dtype) if epi == "residual" else None

    def run(bn):
        if res is not None:                 # in place: C is the residual, as in the engines
            out = res.clone()
            return ops.gemm(a, w, residual=out, out=out, force_bn=bn)
        return ops.gemm(a, w, bias=bias, act="gelu" if epi == "gelu" else "silu" if epi == "swiglu" else "none",
                        swiglu=epi == "swiglu", rowscale=rs, force_bn=bn)

    ref = run(64)
    got = run(128)
    torch.cuda.synchronize()
    assert torch.equal(got, ref), f"BN 128 (staged variant) differs from BN 64 ({M}x{N}x{K}, {epi})"
