"""Detection kernels one at a time (GPU): each is called through its own C ABI entry point and compared with a plain
high-precision restatement of the same operation that rounds to the storage type at the same points as the kernel.

Tolerances are in ulps of the storage type.  Where a rounded intermediate feeds a long sum (the expand map of the fused
MBConv, the up-sampled and fused maps of the decode head), the bound is derived from the worst case of one-ulp flips in that
intermediate, and a second comparison against the op sequence the fused kernel replaces checks the tight claim: same
rounding points, same (or only a different fp32) summation order.  Every output goes into a window of a NaN-filled buffer;
nothing outside the window may change and nothing inside may stay NaN."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DT = [torch.bfloat16, torch.float16]
PAD = 64          # elements of NaN before and after every output window (128 bytes: the window stays 16-byte aligned)


def _ulp(dtype):
    return 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11


def _close(got, ref, dtype, ulps=2.0, what="", scale=None, slack=None):
    """|got - ref| <= ulps * ulp(max(|ref|, |scale|, 1)) (+ slack) elementwise; `scale` = magnitude of the largest rounded
    intermediate (a 1-ulp flip of an intermediate survives a cancelling residual add); `slack` = a derived absolute bound for
    flips carried through a sum.  NaN in `got` fails."""
    got = got.float()
    ref = ref.float()
    mag = ref.abs().clamp(min=1.0)
    if scale is not None:
        mag = torch.maximum(mag, scale.float().abs())
    tol = ulps * 2.0 * _ulp(dtype) * torch.exp2(torch.floor(torch.log2(mag)))
    if slack is not None:
        tol = tol + slack
    bad = ~((got - ref).abs() <= tol)
    frac = bad.float().mean().item()
    assert frac == 0.0, f"{what}: {bad.sum().item()} / {bad.numel()} beyond {ulps} ulp, max abs err {(got - ref).abs().max().item():.4g}"


def _within(got, ref, dtype, ulps, what, slack=None):
    """|got - ref| <= ulps ulps of max(|got|, |ref|) (+ slack) elementwise (no floor at 1: for maps whose values sit well
    below 1, such as sigmoid outputs)."""
    got, ref = got.double(), ref.double()
    tol = ulps * _spacing(torch.maximum(got.abs(), ref.abs()), dtype)
    if slack is not None:
        tol = tol + slack
    bad = ~((got - ref).abs() <= tol)
    assert not bool(bad.any()), f"{what}: {bad.sum().item()} / {bad.numel()} beyond {ulps} ulp, max abs err {(got - ref).abs().max().item():.4g}"


def _spacing(x, dtype):
    """Distance between adjacent storage-type values at |x| (normal range; 16-bit subnormals are not reached here)."""
    tiny = 2.0 ** -14
    return 2.0 * _ulp(dtype) * torch.exp2(torch.floor(torch.log2(x.double().abs().clamp(min=tiny))))


def _sigmoid_flip(logit, dtype):
    """How far sigmoid's output moves when its rounded logit flips to a neighbouring value: the spacing u at the logit times
    the largest slope over that step, sigmoid'(max(|logit| - u, 0)).  Below 1/4 of an ulp of the logit, but not below an ulp
    of the output, whose spacing shrinks with it."""
    u = _spacing(logit, dtype)
    s = torch.sigmoid((logit.double().abs() - u).clamp(min=0.0))
    return s * (1.0 - s) * u


def _window(shape, dtype):
    """(buffer, view): a dense `shape` window in the middle of a NaN-filled buffer."""
    n = math.prod(shape)
    buf = torch.full((PAD + n + PAD,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[PAD:PAD + n].view(shape)


def _untouched(buf, what):
    bits = buf.view(torch.int16)
    nan = torch.full((1,), float("nan"), dtype=buf.dtype).view(torch.int16).item()
    assert bool((bits[:PAD] == nan).all()) and bool((bits[-PAD:] == nan).all()), f"{what}: wrote outside its output"


def _t(x, dtype):
    """Round to the storage type and back to float64 (an op boundary of the kernels)."""
    return x.to(dtype).double()


def _hardswish(x):
    """x * min(max(x + 3, 0), 6) * (1/6) in fp32, left to right: the kernels' expression."""
    x = x.float()
    return x * torch.clamp(x + 3.0, 0.0, 6.0) * (1.0 / 6.0)


def _conv(x_nhwc, w_k, stride):
    """3x3 pad-1 conv in float64: x NHWC, w [Cout, 9*Cin] with K ordered (r, s, c) -> NHWC."""
    cout, cin = w_k.shape[0], x_nhwc.shape[3]
    w = w_k.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    return F.conv2d(x_nhwc.double().permute(0, 3, 1, 2), w, stride=stride, padding=1).permute(0, 2, 3, 1)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ stem conv
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("in_f32", [True, False], ids=["in_f32", "in_16"])
@pytest.mark.parametrize("B,H,W", [(1, 2, 260), (3, 6, 514), (3, 2, 514), (1, 6, 260)])
def test_stem_conv(built_lib, dtype, in_f32, B, H, W):
    """W/2 = 130 and 257 leave a partial 128-thread block; H = 2 and 6 put every output row next to a padded border."""
    from surya_b200 import ops

    g = _gen(B * 1000 + H * 10 + W)
    x = torch.randn(B, 3, H, W, device="cuda", generator=g) * 1.5
    w = torch.randn(32, 27, device="cuda", generator=g) * 0.3        # [cout][r][s][c], fp32 as the engine packs it
    b = torch.randn(32, device="cuda", generator=g) * 0.5
    xin = x if in_f32 else x.to(dtype)
    buf, out = _window((B, H // 2, W // 2, 32), dtype)
    ops.det_stem_conv(xin, w, b, dtype=dtype, out=out)
    torch.cuda.synchronize()
    _untouched(buf, "stem")
    # the kernel rounds fp32 pixels to the model dtype first; then fp32 taps + bias -> T -> Hardswish (fp32) -> T
    xs = x.to(dtype).double()
    wt = w.double().reshape(32, 3, 3, 3).permute(0, 3, 1, 2)
    pre = _t(F.conv2d(xs, wt, b.double(), stride=2, padding=1).float(), dtype).permute(0, 2, 3, 1)
    ref = _hardswish(pre).to(dtype)
    # Only the fp32 summation order differs, so the pre-activation flips by at most one ulp u of its binade.  Hardswish's
    # slope is at most 1.5 and both sides round once more: |diff| <= 1.5 u + 1 ulp(out), and as a difference of two values on
    # the grid of |pre|'s binade (or finer) that is at most 2 u.  scale=pre makes the bound 2 ulps of max(|out|, |pre|, 1).
    _close(out, ref, dtype, ulps=2, what="stem", scale=pre)
    # flips are rare (fp32 error against half an ulp of the storage type): almost every value must be bit-equal
    same = (out.float() == ref.float()).float().mean().item()
    assert same >= 0.99, f"stem: only {100 * same:.2f} % bit-equal to the float64 restatement"


# ------------------------------------------------------------------------------------------------ fused MBConv
FMB_CASES = [
    # Cin, Cmid, Cout, stride, residual, B, H, W
    pytest.param(64, 256, 128, 1, True, 3, 72, 112, id="wrap-189tiles"),       # more tiles than SMs: the persistent loop wraps
    pytest.param(64, 256, 128, 2, False, 2, 37, 45, id="s2-odd-partial"),       # Ho 19, Wo 23: partial tiles, odd H and W
    pytest.param(128, 512, 64, 2, True, 2, 37, 45, id="s2-res-partial"),
    pytest.param(128, 1024, 128, 1, True, 1, 21, 37, id="b1-9tiles"),           # B = 1, fewer tiles than SMs, partial both ways
    pytest.param(64, 1024, 64, 1, False, 1, 20, 40, id="b1-6tiles"),
    pytest.param(64, 512, 128, 1, False, 2, 21, 37, id="s1-partial"),
    pytest.param(128, 256, 64, 1, True, 2, 24, 40, id="s1-res-wpartial"),
    pytest.param(128, 128, 128, 2, False, 3, 63, 95, id="s2-cmid128"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("cin,cmid,cout,stride,res,B,H,W", FMB_CASES)
def test_fmb_fused(built_lib, dtype, cin, cmid, cout, stride, res, B, H, W):
    from surya_b200 import ops

    g = _gen(cin + cmid + cout + stride + B + H)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g).to(dtype)
    w1 = (torch.randn(cmid, 9 * cin, device="cuda", generator=g) * 1.5 * (9 * cin) ** -0.5).to(dtype)
    b1 = torch.randn(cmid, device="cuda", generator=g) * 0.3
    w2 = (torch.randn(cout, cmid, device="cuda", generator=g) * cmid ** -0.5).to(dtype)
    b2 = torch.randn(cout, device="cuda", generator=g) * 0.3
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    r = torch.randn(B, Ho, Wo, cout, device="cuda", generator=g).to(dtype) if res else None
    buf, out = _window((B, Ho, Wo, cout), dtype)
    ops.det_fmb_fused(x, w1, b1, w2, b2, residual=r, stride=stride, out=out)
    # the op pair the fused kernel replaces.  M = B*Ho*Wo >= 777 keeps the GEMM off the skinny (M <= 16) kernel, and split-K
    # is not requested, so this is the tiled wgmma GEMM that sums the mid channels in 64-wide k-blocks like the fused kernel
    mid = ops.conv2d_nhwc(x, w1, b1, None, 3, stride, 1, "hardswish")
    unf = ops.gemm(mid.reshape(-1, cmid), w2, bias=b2, residual=r.reshape(-1, cout) if res else None).reshape(B, Ho, Wo, cout)
    torch.cuda.synchronize()
    _untouched(buf, "fmb_fused")
    what = f"fmb_fused {cin}->{cmid}->{cout} s{stride} res={res} {B}x{H}x{W}"
    assert torch.equal(out.view(torch.int16), unf.view(torch.int16)), f"{what}: differs from conv_igemm -> gemm"
    pre1 = _t(_conv(x, w1, stride) + b1.double(), dtype)
    e = _t(_hardswish(pre1), dtype)
    proj = e.reshape(-1, cmid) @ w2.double().t() + b2.double()
    proj_t = _t(proj, dtype).reshape(B, Ho, Wo, cout)
    ref = _t(proj_t + r.double(), dtype) if res else proj_t
    # Bound: every expand value may flip by one ulp u_k of its pre-activation's binade, which moves its Hardswish output by at
    # most 2 u_k (see test_stem_conv).  Each flip enters the projection through one product, so the projection moves by at
    # most sum_k |w2[o, k]| * 2 u_k; its own rounding (and the residual add's) flips by one more ulp each (ulps=2, scale).
    flips = (w2.double().abs() @ (2 * _spacing(pre1, dtype)).reshape(-1, cmid).t()).t().reshape(B, Ho, Wo, cout)
    _close(out, ref, dtype, ulps=2, what=what, scale=torch.maximum(proj_t.abs(), r.double().abs()) if res else proj_t,
           slack=flips)


# ------------------------------------------------------------------------------------------------ decode head
def _bilinear_pinned(src, HO, WO):
    """The fused head's builder blend (and upsample_cat's) for 16-bit src NHWC [B, hs, ws, C] at integer ratios, fp32 fma
    emulated exactly: float64 products of fp32 / 16-bit operands rounded once to fp32.
      p = fma(lx, b, hx * a);  q = fma(lx, d, hx * c);  v = fma(ly, q, hy * p)."""
    B, hs, ws, C = src.shape
    dev = src.device

    def coords(n_out, n_in):
        o = torch.arange(n_out, device=dev, dtype=torch.float32)
        s = torch.clamp((o + 0.5) * (float(n_in) / n_out) - 0.5, min=0.0)       # exact for the ratios 2, 4, 8
        i0 = s.long()
        i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
        lam = (s - i0.float()).double()
        return i0, i1, lam, (1.0 - lam.float()).double()

    y0, y1, ly, hy = coords(HO, hs)
    x0, x1, lx, hx = coords(WO, ws)
    s = src.double()
    a, b_ = s[:, y0][:, :, x0], s[:, y0][:, :, x1]
    c, d = s[:, y1][:, :, x0], s[:, y1][:, :, x1]
    lx, hx = lx.view(1, 1, -1, 1), hx.view(1, 1, -1, 1)
    ly, hy = ly.view(1, -1, 1, 1), hy.view(1, -1, 1, 1)
    f32 = lambda t: t.float().double()                                          # noqa: E731
    p = f32(lx * b_ + f32(hx * a))
    q = f32(lx * d + f32(hx * c))
    return f32(ly * q + f32(hy * p))


def _bilinear_ref(src, HO, WO, dtype):
    """F.interpolate(bilinear, align_corners=False) in fp32 on the 16-bit values, rounded to the storage type (NHWC)."""
    return F.interpolate(src.permute(0, 3, 1, 2).float(), size=(HO, WO), mode="bilinear",
                         align_corners=False).to(dtype).permute(0, 2, 3, 1)


HEAD_CASES = [
    # B, HO, WO, (fy, fx) of the three low-resolution sources, channel offset of the identity source
    pytest.param(1, 40, 24, [(2, 2), (4, 4), (8, 8)], 384, id="40x24-engine-order"),      # WO % 16 = 8: partial tiles in x
    pytest.param(3, 80, 112, [(2, 8), (8, 4), (4, 2)], 0, id="80x112-b3-mixed"),         # 210 tiles: more than SMs
    pytest.param(2, 44, 40, [(2, 8), (4, 2), (4, 4)], 384, id="44x40-partial-xy"),       # HO % 8 = 4 and WO % 16 = 8
    pytest.param(1, 80, 112, [(2, 2), (4, 4), (8, 8)], 0, id="80x112-b1"),
]


def _head_inputs(B, HO, WO, ratios, id_off, dtype, seed):
    g = _gen(seed)
    shapes = [(HO, WO)] + [(HO // fy, WO // fx) for fy, fx in ratios]
    srcs = [torch.randn(B, h, w, 128, device="cuda", generator=g).to(dtype) for h, w in shapes]
    # the identity source at channel 0 (offsets 0, 128, 256, 384) or at 384 (the engine's reversed concat order)
    offs = [0, 128, 256, 384] if id_off == 0 else [384, 256, 128, 0]
    fw = (torch.randn(512, 512, device="cuda", generator=g) * 512 ** -0.5).to(dtype)
    fb = torch.randn(512, device="cuda", generator=g) * 0.2
    cw = (torch.randn(2, 512, device="cuda", generator=g) * 0.1).to(dtype)
    cb = (torch.randn(2, device="cuda", generator=g) * 0.5).to(dtype)
    return srcs, offs, fw, fb, cw, cb


def _classify(fmap, cw, cb, dtype):
    """fmap NHWC [B, H, W, C] (16-bit values) -> T(sigmoid(T(fp32(dot) + b))) NCHW, the dot in float64."""
    B, H, W, C = fmap.shape
    dot = (fmap.reshape(-1, C).double() @ cw.double().t()).float()
    logit = (dot + cb.float()).to(dtype).float()
    return torch.sigmoid(logit).to(dtype).reshape(B, H, W, -1).permute(0, 3, 1, 2), logit.reshape(B, H, W, -1)


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("B,HO,WO,ratios,id_off", HEAD_CASES)
def test_head_fused(built_lib, dtype, B, HO, WO, ratios, id_off):
    from surya_b200 import ops

    srcs, offs, fw, fb, cw, cb = _head_inputs(B, HO, WO, ratios, id_off, dtype, seed=B * 7 + HO + WO + id_off)
    buf, out = _window((B, 2, HO, WO), dtype)
    ops.det_head_fused(srcs, offs, fw, fb, cw, cb, HO, WO, out=out)
    # the unfused chain: upsample_cat -> gemm(relu) -> classifier
    cat = ops.det_upsample_cat(srcs, offs, HO, WO)
    fz = ops.gemm(cat.reshape(-1, 512), fw, bias=fb, act="relu").reshape(B, HO, WO, 512)
    unf = ops.det_classifier(fz.reshape(-1, 512), cw, cb, HO * WO).reshape(B, 2, HO, WO)
    torch.cuda.synchronize()
    _untouched(buf, "head_fused")
    what = f"head_fused {B}x{HO}x{WO} {ratios} id@{id_off}"
    # reference: bilinear (fp32 on T values) -> T -> concat -> fuse GEMM + bias -> T -> ReLU -> classifier + T(b) -> T -> sigmoid
    up = torch.zeros(B, HO, WO, 512, device="cuda", dtype=torch.float64)
    dup = torch.zeros_like(up)
    for s, o in zip(srcs, offs):
        if s.shape[1] == HO:
            up[..., o:o + 128] = s.double()
        else:
            u = _bilinear_ref(s, HO, WO, dtype).double()
            up[..., o:o + 128] = u
            dup[..., o:o + 128] = _spacing(u, dtype)          # the blend may round to the neighbouring value
    fpre = up.reshape(-1, 512) @ fw.double().t() + fb.double()
    f = torch.relu(_t(fpre, dtype))
    ref, logit = _classify(f.reshape(B, HO, WO, 512), cw, cb, dtype)
    # Bound, worst case of every rounded intermediate flipping by one ulp: up-sampled values (dup) move the fuse output by
    # |fw| @ dup, plus its own rounding (one ulp); that moves the logit by |cw| @ df, plus one ulp of the logit; the sigmoid's
    # slope is at most 1/4, and its rounding adds one ulp of the output (ulps=1).
    df = dup.reshape(-1, 512) @ fw.double().abs().t() + _spacing(fpre, dtype)
    dlogit = (df @ cw.double().abs().t()).reshape(B, HO, WO, 2) + _spacing(logit, dtype)
    _close(out, ref, dtype, ulps=1, what=what, slack=(dlogit / 4).permute(0, 3, 1, 2))
    # tight: the reference's classifier stage on the unfused fuse map.  Only the fp32 order of the 512-long dot differs, so the
    # rounded logit flips by at most one ulp, which sigmoid carries as _sigmoid_flip; the output rounds once more (1 ulp)
    tight, tlogit = _classify(fz, cw, cb, dtype)
    _within(out, tight, dtype, 1, what + " vs classifier(unfused fuse map)", slack=_sigmoid_flip(tlogit, dtype).permute(0, 3, 1, 2))
    same = (out.float() == tight.float()).float().mean().item()
    same_unf = (out.view(torch.int16) == unf.view(torch.int16)).float().mean().item()
    print(f"{what} {dtype}: bit-equal {100 * same:.3f} % to the float64 classifier on the unfused map, "
          f"{100 * same_unf:.3f} % to the unfused chain")
    assert same >= 0.99 and same_unf >= 0.99, (same, same_unf)


# ------------------------------------------------------------------------------------------------ upsample_cat
UPCAT_CASES = [
    # B, (HO, WO), source sizes, CS
    pytest.param(2, (50, 24), [(13, 7)], 8, id="n1-nonint-cs8"),
    pytest.param(3, (50, 24), [(50, 24), (13, 7)], 64, id="n2-nonint-cs64"),
    pytest.param(2, (42, 56), [(21, 28), (21, 7), (42, 56)], 128, id="n3-int-cs128"),     # HO % 4 = 2
    pytest.param(2, (40, 24), [(40, 24), (20, 12), (10, 6), (5, 3)], 128, id="n4-int-engine"),
    pytest.param(3, (41, 33), [(13, 7), (7, 24), (41, 33), (20, 16)], 8, id="n4-nonint-cs8"),  # HO % 4 = 1
    pytest.param(2, (24, 48), [(12, 6), (3, 24), (6, 12), (24, 48)], 64, id="n4-int-mixed-cs64"),
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("B,size,shapes,CS", UPCAT_CASES)
def test_upsample_cat(built_lib, dtype, B, size, shapes, CS):
    from surya_b200 import ops

    HO, WO = size
    g = _gen(B + HO + WO + CS + len(shapes))
    srcs = [torch.randn(B, h, w, CS, device="cuda", generator=g).to(dtype) for h, w in shapes]
    n = len(srcs)
    offs = [(n - 1 - i) * CS for i in range(n)]              # reversed order, as the engine concatenates
    buf, out = _window((B, HO, WO, n * CS), dtype)
    ops.det_upsample_cat(srcs, offs, HO, WO, out=out)
    torch.cuda.synchronize()
    _untouched(buf, "upsample_cat")
    for i, (s, o) in enumerate(zip(srcs, offs)):
        got = out[..., o:o + CS]
        what = f"upsample_cat source {i} {tuple(s.shape[1:3])} -> {size}"
        if s.shape[1:3] == (HO, WO):
            assert torch.equal(got, s), what
            continue
        _within(got, _bilinear_ref(s, HO, WO, dtype), dtype, 1, what)
        if HO % s.shape[1] == 0 and WO % s.shape[2] == 0 and (HO // s.shape[1]) in (2, 4, 8) and (WO // s.shape[2]) in (2, 4, 8):
            # the fused head's ratios: the same bits as its builders' pinned blend
            pinned = _bilinear_pinned(s, HO, WO).to(dtype)
            assert torch.equal(got.view(torch.int16), pinned.view(torch.int16)), f"{what}: not the fused head's blend"


# ------------------------------------------------------------------------------------------------ classifier
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C", [8, 24, 512, 520])
@pytest.mark.parametrize("B,HW", [(1, 301), (3, 45)])
def test_classifier(built_lib, dtype, C, B, HW):
    """C = 520 leaves a ragged last pass of the 256-wide lane loop; P = B*HW is not a multiple of the 8 pixels per block."""
    from surya_b200 import ops

    g = _gen(C + B + HW)
    x = torch.relu(torch.randn(B * HW, C, device="cuda", generator=g)).to(dtype)
    w = (torch.randn(2, C, device="cuda", generator=g) * 3.0 * C ** -0.5).to(dtype)
    b = (torch.randn(2, device="cuda", generator=g) * 0.5).to(dtype)
    buf, out = _window((B, 2, HW), dtype)
    ops.det_classifier(x, w, b, HW, out=out)
    torch.cuda.synchronize()
    _untouched(buf, "classifier")
    ref, logit = _classify(x.reshape(B, HW, 1, C), w, b, dtype)
    ref = ref.reshape(B, 2, HW)
    # only the fp32 order of the dot differs: the rounded logit flips by at most one ulp (carried as _sigmoid_flip), and the
    # output rounds once more
    _within(out, ref, dtype, 1, f"classifier C={C} B={B} HW={HW}", slack=_sigmoid_flip(logit, dtype).reshape(B, HW, 2).transpose(1, 2))
    same = (out.float() == ref.float()).float().mean().item()
    assert same >= 0.99, f"classifier: only {100 * same:.2f} % bit-equal"


# ------------------------------------------------------------------------------------------------ conv_igemm / conv_halo
CONV_CASES = [
    # Cin, Cout, stride, act, residual, B, H, W          conv_typed instance (channel chunk BKC, tile width BN)
    pytest.param(64, 256, 1, "hardswish", False, 2, 21, 37, id="bkc64-bn128"),
    pytest.param(128, 64, 2, "none", True, 2, 37, 45, id="bkc64-bn64"),
    pytest.param(64, 96, 1, "relu", True, 1, 17, 23, id="bkc64-bn64-ragged"),      # Cout 96: a partial 64-wide n-tile
    pytest.param(64, 32, 2, "hardswish", False, 3, 40, 56, id="bkc64-bn32"),
    pytest.param(96, 128, 1, "hardswish", True, 2, 20, 40, id="bkc32-bn128"),
    pytest.param(32, 64, 2, "none", False, 2, 33, 47, id="bkc32-bn64"),
    pytest.param(96, 32, 1, "hardswish", False, 2, 21, 37, id="bkc32-bn32-cin96"),
    pytest.param(32, 32, 2, "relu", True, 3, 40, 60, id="bkc32-bn32-s2"),          # Cin = Cout = 32 at stride 2: not the halo kernel
    # the halo kernel (Cin = Cout = 32, stride 1): 8 x 16 output tiles
    pytest.param(32, 32, 1, "hardswish", False, 2, 21, 37, id="halo-partial"),
    pytest.param(32, 32, 1, "none", True, 1, 19, 13, id="halo-res-partial"),
    pytest.param(32, 32, 1, "hardswish", True, 3, 100, 88, id="halo-res-231tiles"),   # more tiles than SMs
]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("cin,cout,stride,act,res,B,H,W", CONV_CASES)
def test_conv_igemm_ulps(built_lib, dtype, cin, cout, stride, act, res, B, H, W):
    from surya_b200 import ops

    g = _gen(cin * 3 + cout + stride + H + W)
    x = torch.randn(B, H, W, cin, device="cuda", generator=g).to(dtype)
    w = (torch.randn(cout, 9 * cin, device="cuda", generator=g) * 1.5 * (9 * cin) ** -0.5).to(dtype)
    b = torch.randn(cout, device="cuda", generator=g) * 0.3
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    r = torch.randn(B, Ho, Wo, cout, device="cuda", generator=g).to(dtype) if res else None
    buf, out = _window((B, Ho, Wo, cout), dtype)
    ops.conv2d_nhwc(x, w, b, r, 3, stride, 1, act, out=out)
    torch.cuda.synchronize()
    _untouched(buf, "conv")
    pre = _t(_conv(x, w, stride) + b.double(), dtype)
    y = pre if act == "none" else _t(_hardswish(pre) if act == "hardswish" else torch.relu(pre), dtype)
    ref = _t(y + r.double(), dtype) if res else y
    # The fp32 sum flips the pre-activation by at most one ulp; Hardswish carries that as at most 2 ulps of max(|pre|, |out|)
    # (test_stem_conv), ReLU and identity as 1; a residual add rounds once more.
    ulps = (2 if act == "hardswish" else 1) + (1 if res else 0)
    scale = torch.maximum(pre.abs(), r.double().abs()) if res else pre
    _close(out, ref, dtype, ulps=ulps, what=f"conv {cin}->{cout} s{stride} {act} res={res} {B}x{H}x{W}", scale=scale)


# ------------------------------------------------------------------------------------------------ bf16 engine
def test_engine_bf16_vs_oracle(built_lib):
    """The bf16 engine end to end (every detection kernel's bf16 instance) against the fp32 oracle at 384 x 512, with the
    fp16 engine's tiny-config bound (test_engine_vs_oracle) scaled by the bf16 / fp16 ulp ratio (8)."""
    from oracle import det_oracle as D
    from surya_b200.config import det_tiny
    from surya_b200.detection import DetEngine
    from surya_b200.synth import det_normalize, det_state_dict, det_synthetic_pages

    cfg = det_tiny()
    sd = det_state_dict(cfg, seed=0)
    size = (384, 512)
    pages = det_synthetic_pages(2, max(size), seed=3)[:, : size[0], : size[1]]
    x = det_normalize(pages)
    eng = DetEngine(cfg, sd, torch.bfloat16, max_batch=2, max_hw=size)
    got = eng.forward(x.cuda())
    up = eng.upsample(got, size)
    torch.cuda.synchronize()
    assert got.dtype == torch.bfloat16
    ref = D.forward(sd, cfg, x)
    err = (got.float().cpu() - ref).abs().max().item()
    err_up = (up.cpu() - D.upsample_to_input(ref, size)).abs().max().item()
    print(f"bf16 engine 384x512: max |err| {err:.3g}, upsampled {err_up:.3g}")
    tol = 8 * 1e-3
    assert err < tol and err_up < tol, (err, err_up)
    eng.close()
