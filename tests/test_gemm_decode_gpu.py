"""The decode-step variant of the GEMM kernel against the plain variant (GPU).

gemm_tn_kernel<T, BN, STAGES, true> must give the bits of gemm_tn_kernel<T, BN, STAGES, false> at any tile width: every
output element is the same per-k-block partial sums added in k order.  Each case runs both instantiations on the same
operands and compares them with torch.equal, in the four configurations the recognition decode step launches (qkv with the
folded RMSNorm and a bias, o-proj with an in-place residual, gate/up with SwiGLU and the folded norm, lm_head with row scales
and the argmax partials), at row counts on both sides of the 128-row tile, at every tile width the decode variant takes and
at its own table's choice, with k-block counts of 1, 2, odd, even and with a partial last block, and with more tiles than SMs
(each CTA runs several).
Operands are windows of NaN-filled buffers and outputs windows of sentinel-filled ones, as in test_gemm_contract_gpu.py."""
import pytest
import torch

from surya_b200 import ops
from surya_b200._lib import SuryaB200Error

pytestmark = pytest.mark.gpu

DT = [torch.bfloat16, torch.float16]
SENTINEL = -7.0
EPS = 1e-6
R0, C0 = 3, 8
MS = [17, 64, 100, 128, 129, 200, 256]


def _window(rows, cols, dtype, fill, src=None):
    ld = -(-(C0 + cols + 8) // 8) * 8
    buf = torch.full((R0 + rows + 5, ld), fill, device="cuda", dtype=dtype)
    view = buf[R0:R0 + rows, C0:C0 + cols]
    if src is not None:
        view.copy_(src)
    return buf, view


def _outside(buf, rows, cols):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[R0:R0 + rows, C0:C0 + cols] = False
    return buf[keep]


def _rand(shape, dtype, g, scale):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


# (name, N, K, bn): the decode step's shapes at the tile widths the kernel takes
CONFIGS = [
    ("qkv", 1920, 1280, 32),
    ("qkv", 1920, 1280, 64),
    ("oproj", 1280, 1280, 32),
    ("oproj", 1280, 1280, 64),
    ("gateup", 6848, 1280, 128),
    ("gateup", 6848, 1280, 64),
    ("lmhead", 4104, 1280, 128),
    ("lmhead", 65792, 1280, 0),      # the real vocabulary: 514 n-tiles per m-block, several tiles per CTA
    ("qkv", 1920, 1280, 0),          # the kernel's own table
    ("gateup", 6848, 1280, 0),
]


def _run(kind, a, w, bias, res_src, dtype, M, N, bn, decode, rs):
    """One launch of configuration `kind` with A a window of a NaN buffer and C a window of a sentinel buffer.  Returns the
    output buffer (whole) and the argmax partials (or None)."""
    n_out = N // 2 if kind == "gateup" else N
    a_buf, a_w = _window(M, a.shape[1], dtype, float("nan"), a)
    c_buf, c_w = _window(M, n_out, dtype, SENTINEL, res_src if kind == "oproj" else None)
    am = None
    if kind == "qkv":
        ops.gemm(a_w, w, bias=bias, out=c_w, rms_eps=EPS, force_bn=bn, decode=decode)
    elif kind == "oproj":
        ops.gemm(a_w, w, residual=c_w, out=c_w, force_bn=bn, decode=decode)
    elif kind == "gateup":
        ops.gemm(a_w, w, act="silu", swiglu=True, out=c_w, rms_eps=EPS, force_bn=bn, decode=decode)
    else:
        am = {}
        ops.gemm(a_w, w, bias=bias, out=c_w, rowscale=rs, argmax=am, force_bn=bn, decode=decode)
    return c_buf, am


def _compare(kind, dtype, M, N, K, bn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = _rand((M, K), dtype, g, 1.0)
    w = _rand((N, K), dtype, g, K ** -0.5)
    bias = torch.randn(N, device="cuda", generator=g) * 0.1
    res = _rand((M, N), dtype, g, 1.0) if kind == "oproj" else None
    rs = ops.row_rstd(a, EPS) if kind == "lmhead" else None
    want, am_want = _run(kind, a, w, bias, res, dtype, M, N, bn, 0, rs)
    got, am_got = _run(kind, a, w, bias, res, dtype, M, N, bn, 1, rs)
    torch.cuda.synchronize()
    what = f"{kind} {M}x{N}x{K} bn={bn}"
    n_out = N // 2 if kind == "gateup" else N
    assert (_outside(got, M, n_out) == SENTINEL).all(), f"{what}: elements outside the output window were written"
    assert torch.equal(got, want), f"{what}: output differs from the plain kernel"
    if am_want is not None:
        for k in ("val", "idx", "sum"):
            assert torch.equal(am_got[k], am_want[k]), f"{what}: argmax partial '{k}' differs from the plain kernel"


@pytest.mark.parametrize("dtype", DT, ids=["bf16", "fp16"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("kind,N,K,bn", CONFIGS)
def test_decode_gemm_equals_plain(built_lib, dtype, kind, N, K, bn, M):
    _compare(kind, dtype, M, N, K, bn, seed=M * 7 + N + bn)


@pytest.mark.parametrize("dtype", DT, ids=["bf16", "fp16"])
@pytest.mark.parametrize("K", [64, 128, 1216, 1256, 3424])   # k-blocks: 1, 2, 19 (odd), 20 with a partial last one, 54
@pytest.mark.parametrize("M,bn", [(17, 32), (129, 64), (256, 64), (256, 128)])
def test_decode_gemm_k_blocks(built_lib, dtype, K, M, bn):
    _compare("qkv", dtype, M, 1920, K, bn, seed=K + M + bn)
    _compare("oproj", dtype, M, 1280, K, bn, seed=K + M + bn + 1)


@pytest.mark.parametrize("dtype", DT, ids=["bf16", "fp16"])
@pytest.mark.parametrize("operand", ["a", "residual"])
@pytest.mark.parametrize("bn", [32, 128])
def test_decode_gemm_dependent_launch(built_lib, dtype, operand, bn):
    """A or the residual is written by the previous library kernel and read with no synchronise in between."""
    M, N, K = 256, 1280, 1280
    g = torch.Generator(device="cuda").manual_seed(len(operand) + bn)
    pa = _rand((M, 512), dtype, g, 1.0)
    pw = _rand((K, 512), dtype, g, 512 ** -0.5)
    w = _rand((N, K), dtype, g, K ** -0.5)
    other = _rand((M, K), dtype, g, 1.0)

    def chain(dec):
        produced = torch.empty((M, K), device="cuda", dtype=dtype)
        ops.gemm(pa, pw, out=produced, force_bn=256)     # the producer: a long plain launch
        if operand == "a":
            return ops.gemm(produced, w, bias=None, rms_eps=EPS, decode=dec, force_bn=bn)
        out = produced[:, :N]
        return ops.gemm(other, w, residual=out, out=out, decode=dec, force_bn=bn)

    want = chain(0).clone()
    torch.cuda.synchronize()
    got = chain(1)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


REFUSED = [
    pytest.param(dict(M=257), id="M>256"),
    pytest.param(dict(out_f32=True), id="out_f32"),
    pytest.param(dict(force_bn=1064), id="forced_splitk"),
    pytest.param(dict(force_bn=96), id="bn96"),
    pytest.param(dict(force_bn=256), id="bn256"),
    pytest.param(dict(decode=2), id="decode2"),
    pytest.param(dict(decode=-1), id="decode-1"),
    pytest.param(dict(N=1924), id="N%8"),
    pytest.param(dict(N=1928, swiglu=True), id="swiglu_N%16"),
    pytest.param(dict(swiglu=True, act="relu"), id="swiglu_relu"),
]


@pytest.mark.parametrize("kw", REFUSED)
def test_decode_gemm_refused(built_lib, kw):
    kw = dict(kw)
    M, N = kw.pop("M", 64), kw.pop("N", 1920)
    kw.setdefault("decode", 1)
    if kw.get("swiglu"):
        kw.setdefault("act", "silu")
    a = torch.randn(M, 1280, device="cuda").to(torch.bfloat16)
    w = torch.randn(N, 1280, device="cuda").to(torch.bfloat16)
    with pytest.raises(SuryaB200Error, match="decode"):
        ops.gemm(a, w, **kw)
    torch.cuda.synchronize()
