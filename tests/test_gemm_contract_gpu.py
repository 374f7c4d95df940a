"""The GEMM contract the engines rely on (GPU), through ops.gemm / sb_gemm:

(a) operands and outputs that are windows of wider buffers (ld > width).  Every input element outside its window is NaN and
    every output element outside its window a finite sentinel, so a read past K, M or N or a store outside the output shows.
    Window offsets and pitches are multiples of 8 elements, so a window takes the same kernel path as a contiguous operand and
    must give the same bits;
(b) C == residual: every O and down projection of the engines adds its residual in place;
(c) launches that depend on the previous library kernel with no synchronise in between: every kernel is launched with
    programmatic dependent launch and lets its successor start before it finishes.

Bit equality is asserted only between two calls that take the same kernel path.  The fp32 restatement rounds at the same op
boundaries as tests/test_ops_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = [torch.bfloat16, torch.float16]
SENTINEL = -7.0


def _ulp(dtype):
    return 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11


def _close(got, ref, dtype, ulps=2.0, what="", scale=None):
    """|got - ref| <= ulps * ulp(max(|ref|, |scale|, 1)) elementwise (the rule of test_ops_gpu._close; a NaN counts as a
    miss)."""
    got = got.float()
    ref = ref.float()
    mag = ref.abs().clamp(min=1.0)
    if scale is not None:
        mag = torch.maximum(mag, scale.float().abs())
    tol = ulps * 2.0 * _ulp(dtype) * torch.exp2(torch.floor(torch.log2(mag)))
    bad = ~((got - ref).abs() <= tol)
    assert not bad.any(), f"{what}: {bad.sum().item()} / {bad.numel()} beyond {ulps} ulp, max abs err {(got - ref).abs().max().item():.4g}"


def _act_ref(x, act):
    if act == "none":
        return x
    if act == "gelu":
        return torch.nn.functional.gelu(x)
    if act == "silu":
        return torch.nn.functional.silu(x)
    if act == "gelu_tanh":
        return torch.nn.functional.gelu(x, approximate="tanh")
    raise ValueError(act)


def _reference(a, w, dtype, bias=None, res=None, act="none", swiglu=False, rs=None):
    """fp32 restatement: acc (* rs) (+ bias) -> round -> act -> round (+ residual) -> round, or the SwiGLU product of the
    rounded (gate, up) column pairs.  Returns (ref, scale) for _close."""
    acc = a.float() @ w.float().t()
    if rs is not None:
        acc = acc * rs[:, None]
    if bias is not None:
        acc = acc + bias
    lin = acc.to(dtype).float()
    if swiglu:
        gate, up = lin[:, 0::2], lin[:, 1::2]
        return (_act_ref(gate, act).to(dtype).float() * up).to(dtype), None
    y = _act_ref(lin, act).to(dtype).float() if act != "none" else lin
    if res is None:
        return y.to(dtype), None
    return (y + res.float()).to(dtype), torch.maximum(lin.abs(), res.float().abs())


def _rand(shape, dtype, g, scale):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


R0, C0 = 3, 8     # window origin inside its buffer: any row, a column offset of 8 elements (16 bytes)


def _window(rows, cols, dtype, fill, src=None):
    """(buffer, view): a [rows, cols] view at (R0, C0) of a buffer filled with `fill` that has at least 8 more columns to
    the right and 5 more rows below; the buffer's row pitch is a multiple of 8 elements.  `src` is copied into the view."""
    ld = -(-(C0 + cols + 8) // 8) * 8
    buf = torch.full((R0 + rows + 5, ld), fill, device="cuda", dtype=dtype)
    view = buf[R0:R0 + rows, C0:C0 + cols]
    if src is not None:
        view.copy_(src)
    return buf, view


def _bias_window(b):
    """fp32 bias of length N as a view into a NaN-filled buffer (elements past N are NaN)."""
    buf = torch.full((b.numel() + 24,), float("nan"), device="cuda", dtype=torch.float32)
    view = buf[8:8 + b.numel()]
    view.copy_(b)
    return view


def _assert_outside_unchanged(buf, rows, cols, what):
    keep = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    keep[R0:R0 + rows, C0:C0 + cols] = False
    assert (buf[keep] == SENTINEL).all(), f"{what}: elements outside the output window were written"


# ------------------------------------------------------------------------------------------------ (a) strided windows
# K = 328 / 648 / 2568 end in a partly filled 64-wide k-block, so the NaN columns past K sit inside the last k-block.
WINDOW_CASES = [
    pytest.param(8, 196, 288, 0, id="skinny"),
    pytest.param(200, 392, 328, 32, id="bn32"),
    pytest.param(200, 392, 328, 64, id="bn64"),
    pytest.param(200, 392, 328, 96, id="bn96"),
    pytest.param(200, 392, 328, 128, id="bn128"),
    pytest.param(200, 392, 328, 256, id="bn256"),
    pytest.param(200, 392, 328, 0, id="heuristic"),
    pytest.param(200, 1280, 648, 3064, id="splitk_forced"),
    pytest.param(130, 512, 2568, -1, id="splitk_auto"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("M,N,K,force_bn", WINDOW_CASES)
def test_gemm_strided_windows(built_lib, dtype, M, N, K, force_bn):
    """A, W, bias and the residual are windows into NaN-filled buffers and C a window into a sentinel-filled one: the result
    must equal the contiguous call's bit for bit, nothing outside C's window may change, and it must match the fp32
    restatement."""
    from surya_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(M * 5 + N + K)
    a = _rand((M, K), dtype, g, 0.5)
    w = _rand((N, K), dtype, g, 0.05)
    bias = torch.randn(N, device="cuda", generator=g).to(dtype).float()
    res = _rand((M, N), dtype, g, 1.0)
    nan = float("nan")
    _, a_w = _window(M, K, dtype, nan, a)
    _, w_w = _window(N, K, dtype, nan, w)
    _, r_w = _window(M, N, dtype, nan, res)
    obuf, o_w = _window(M, N, dtype, SENTINEL)
    want = ops.gemm(a, w, bias=bias, residual=res, act="gelu", force_bn=force_bn)
    got = ops.gemm(a_w, w_w, bias=_bias_window(bias), residual=r_w, act="gelu", out=o_w, force_bn=force_bn)
    torch.cuda.synchronize()
    what = f"windows {M}x{N}x{K} force_bn={force_bn}"
    assert got.data_ptr() == o_w.data_ptr()
    assert torch.equal(o_w, want), f"{what}: differs from the contiguous call"
    _assert_outside_unchanged(obuf, M, N, what)
    ref, scale = _reference(a, w, dtype, bias=bias, res=res, act="gelu")
    _close(o_w, ref, dtype, ulps=3.0, what=what, scale=scale)


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("mode", ["rowscale", "inline"])
def test_gemm_folded_rmsnorm_windows(built_lib, dtype, mode):
    """The folded RMSNorm with strided, NaN-surrounded operands: its per-row scale (given, or summed in the kernel from the A
    tiles) must not see the NaN columns past K."""
    from surya_b200 import ops

    M, N, K, eps = 200, 384, 328, 1e-6
    g = torch.Generator(device="cuda").manual_seed(17)
    a = _rand((M, K), dtype, g, 1.5)
    w = _rand((N, K), dtype, g, 0.03)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).to(dtype).float()
    res = _rand((M, N), dtype, g, 0.5)
    nan = float("nan")
    _, a_w = _window(M, K, dtype, nan, a)
    _, w_w = _window(N, K, dtype, nan, w)
    _, r_w = _window(M, N, dtype, nan, res)
    obuf, o_w = _window(M, N, dtype, SENTINEL)
    rs = ops.row_rstd(a, eps)
    assert torch.equal(ops.row_rstd(a_w, eps), rs), "row_rstd of a strided window differs"
    norm = dict(rowscale=rs) if mode == "rowscale" else dict(rms_eps=eps)
    want = ops.gemm(a, w, bias=bias, residual=res, **norm)
    ops.gemm(a_w, w_w, bias=_bias_window(bias), residual=r_w, out=o_w, **norm)
    torch.cuda.synchronize()
    what = f"folded rmsnorm ({mode}) windows"
    assert torch.equal(o_w, want), f"{what}: differs from the contiguous call"
    _assert_outside_unchanged(obuf, M, N, what)
    ref, scale = _reference(a, w, dtype, bias=bias, res=res, rs=rs)
    _close(o_w, ref, dtype, ulps=2.0, what=what, scale=scale)


@pytest.mark.parametrize("dtype", DT)
def test_gemm_argmax_windows(built_lib, dtype):
    """The online argmax epilogue with strided operands: partials equal to the contiguous run's, logits written only inside
    the output window, and with argmax_only not at all."""
    from surya_b200 import ops

    M, N, K, eps = 37, 1000, 328, 1e-6
    g = torch.Generator(device="cuda").manual_seed(23)
    a = _rand((M, K), dtype, g, 1.0)
    w = _rand((N, K), dtype, g, 0.02)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.02).to(dtype).float()
    nan = float("nan")
    _, a_w = _window(M, K, dtype, nan, a)
    _, w_w = _window(N, K, dtype, nan, w)
    bias_w = _bias_window(bias)
    am, am_w, am_only = {}, {}, {}
    want = ops.gemm(a, w, bias=bias, rms_eps=eps, argmax=am)
    obuf, o_w = _window(M, N, dtype, SENTINEL)
    ops.gemm(a_w, w_w, bias=bias_w, rms_eps=eps, argmax=am_w, out=o_w)
    cbuf, c_w = _window(M, N, dtype, SENTINEL)
    ops.gemm(a_w, w_w, bias=bias_w, rms_eps=eps, argmax=am_only, argmax_only=True, out=c_w)
    torch.cuda.synchronize()
    assert torch.equal(o_w, want), "argmax epilogue logits: window differs from the contiguous call"
    _assert_outside_unchanged(obuf, M, N, "argmax epilogue logits")
    assert (cbuf == SENTINEL).all(), "argmax_only wrote the logits"
    for k in ("val", "idx", "sum"):
        assert torch.equal(am_w[k], am[k]), f"argmax partial '{k}' differs between the window and the contiguous call"
        assert torch.equal(am_only[k], am[k]), f"argmax_only partial '{k}' differs from the contiguous call"
    ref, _ = _reference(a, w, dtype, bias=bias, rs=ops.row_rstd(a, eps))
    _close(o_w, ref, dtype, ulps=2.0, what="argmax epilogue logits")


# ------------------------------------------------------------------------------------------------ (b) C is the residual
INPLACE_CASES = [
    pytest.param(300, 392, 328, 0, "gelu", None, id="staged"),
    pytest.param(300, 392, 328, 256, "none", None, id="staged_bn256"),
    pytest.param(200, 100, 256, 64, "gelu", None, id="chunk_n100"),
    pytest.param(8, 196, 288, 0, "none", None, id="skinny"),
    pytest.param(200, 1280, 648, 3064, "none", None, id="splitk_forced"),
    pytest.param(130, 512, 2568, -1, "none", None, id="splitk_auto"),
    pytest.param(200, 384, 328, 0, "none", "rowscale", id="norm_rowscale"),
    pytest.param(200, 384, 328, 0, "none", "inline", id="norm_inline"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("M,N,K,force_bn,act,norm", INPLACE_CASES)
def test_gemm_inplace_residual(built_lib, dtype, M, N, K, force_bn, act, norm):
    """out=residual (C == residual) gives the out-of-place result bit for bit on every epilogue path."""
    from surya_b200 import ops

    eps = 1e-6
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + K)
    a = _rand((M, K), dtype, g, 0.5)
    w = _rand((N, K), dtype, g, 0.05)
    bias = torch.randn(N, device="cuda", generator=g).to(dtype).float()
    res = _rand((M, N), dtype, g, 1.0)
    kw = dict(bias=bias, act=act, force_bn=force_bn)
    rs = None
    if norm == "rowscale":
        rs = ops.row_rstd(a, eps)
        kw["rowscale"] = rs
    elif norm == "inline":
        rs = ops.row_rstd(a, eps)
        kw["rms_eps"] = eps
    want = ops.gemm(a, w, residual=res, **kw)
    c = res.clone()
    got = ops.gemm(a, w, residual=c, out=c, **kw)
    torch.cuda.synchronize()
    what = f"in-place residual {M}x{N}x{K} force_bn={force_bn} {act} norm={norm}"
    assert got.data_ptr() == c.data_ptr()
    assert torch.equal(c, want), f"{what}: differs from the out-of-place call"
    ref, scale = _reference(a, w, dtype, bias=bias, res=res, act=act, rs=rs)
    _close(c, ref, dtype, ulps=3.0, what=what, scale=scale)


# ------------------------------------------------------------------------------------------------ (c) dependent launches
# The producer runs one long CTA (one 128 x 256 tile, K = 32768) and lets its successor launch at once, so the consumer's CTAs
# start on idle SMs while the producer is still writing the consumer's operand.
DEP_CASES = [
    pytest.param("w", 8, 0, id="w-skinny"),
    pytest.param("w", 64, 0, id="w-wgmma"),
    pytest.param("w", 64, 2064, id="w-splitk"),
    pytest.param("a", 8, 0, id="a-skinny"),
    pytest.param("res", 64, 0, id="res-wgmma"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("operand,M,force_bn", DEP_CASES)
def test_gemm_dependent_launch(built_lib, dtype, operand, M, force_bn):
    """A GEMM that reads the previous GEMM's output (as W, A or residual) with no synchronise in between equals the same
    GEMM run after a synchronise, bit for bit."""
    from surya_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(M + force_bn + len(operand))
    pa = _rand((128, 32768), dtype, g, 0.1)
    pw = _rand((256, 32768), dtype, g, 0.01)
    other_w = _rand((256, 256), dtype, g, 0.05)
    a = _rand((M, 256), dtype, g, 0.5)
    produced = torch.empty(128, 256, device="cuda", dtype=dtype)
    torch.cuda.synchronize()

    def consumer():
        if operand == "w":          # produced = W [N = 128, K = 256]
            return ops.gemm(a, produced, force_bn=force_bn)
        if operand == "a":          # produced[:M] = A [M, K = 256]
            return ops.gemm(produced[:M], other_w, force_bn=force_bn)
        return ops.gemm(a, other_w, residual=produced[:M], force_bn=force_bn)   # produced[:M] = residual [M, 256]

    produced.zero_()                # a torch kernel: the producer starts after it has finished
    ops.gemm(pa, pw, out=produced, force_bn=256)
    early = consumer()
    torch.cuda.synchronize()
    late = consumer()
    torch.cuda.synchronize()
    assert torch.equal(early, late), f"consumer of the previous GEMM's {operand} read it before it was complete"
