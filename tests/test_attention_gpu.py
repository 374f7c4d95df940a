"""Attention kernels one at a time (GPU): attn_varlen, decode_attn (with its RoPE and KV append), rope_kv_append and
attn_single_query, each in fp16 and bf16, against float64 restatements.  u is the unit roundoff of the storage type T
(2^-8 for bf16, 2^-11 for fp16).

Every output is checked twice:
(a) against plain float64 attention O* = softmax(scale q k^T + mask) v of the exact 16-bit values the kernel read, with the
    worst-case bound |got - O*| <= u|O*| + (u + eps) A + eps |O*| + tiny, A = sum_j p*_j |v_j|.  u|O*| is the final rounding,
    u A the one rounding of each P entry to T, eps the fp32 score / exp / sum errors (derived in `_eps`) and `tiny` the
    absolute error of P entries that round into T's subnormal range.  This catches semantic errors: masks, GQA head mapping,
    tile edges, missing keys, a dropped rescale.
(b) against a float64 restatement of the kernel's own rounding points: within 1 ulp of T plus the shift of up to two P
    entries that round to the neighbouring T value (the fp32 scores differ from the float64 ones in their last bits), and
    at least BIT_EQUAL of the values bit-equal.  This catches a moved or removed rounding.
Exact checks need no bound: a decode row at pos = 0 returns its own v (p = 1, l = 1), and a row with q = 0 weights its
visible keys uniformly (2^0 and e^0 are exact), so it is within 1 ulp of the float64 mean of exactly those keys.

Outputs go into column windows of NaN-filled buffers; nothing outside a window (and no packed row outside every sequence)
may change.  The references also run on CPU tensors; test_references_match_sdpa rehearses them against
F.scaled_dot_product_attention in float64 without a GPU."""
import math

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu

DT = [torch.bfloat16, torch.float16]
# check (b): least fraction of bit-equal outputs, for outputs of at least BIT_EQUAL_MIN values.  Calibrated on an H100 (the
# lowest case measured 0.995 in bf16 and 0.951 in fp16): what is not bit-equal is the final rounding of a P V sum whose
# fp32 accumulation order differs from the float64 one, which matters more where fp16's finer spacing meets cancellation.
BIT_EQUAL = {torch.bfloat16: 0.99, torch.float16: 0.94}
BIT_EQUAL_MIN = 4096
LOG2E_F32 = 1.4426950408889634


def _u(dtype):
    return 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11


def _half_min_sub(dtype):
    """Largest rounding error of a value in T's subnormal range (half the least subnormal)."""
    return 2.0 ** -134 if dtype == torch.bfloat16 else 2.0 ** -25


def _spacing(x, dtype):
    """Distance between adjacent T values at |x|, subnormals included."""
    min_norm = 2.0 ** -126 if dtype == torch.bfloat16 else 2.0 ** -14
    e = torch.exp2(torch.floor(torch.log2(x.double().abs().clamp(min=min_norm))))
    return 2.0 * _u(dtype) * e


def _rnd(x, dtype):
    return x.to(dtype).double()


def _nan_bits(dtype):
    return torch.full((1,), float("nan"), dtype=dtype).view(torch.int16).item()


# ------------------------------------------------------------------------------------------------ float64 references
def _exact(q, k, v, scale, vis):
    """Plain float64 attention of q [n, d] over k, v [m, d] with visibility vis [n, m] (every row sees >= 1 key).
    Returns O*, A = sum_j p*_j |v_j| (per element), and per row: l = sum_j exp(s_j - max s), the score range R, the
    largest |scale q| . |k_j| (bound for the fp32 dot products) and the number of visible keys."""
    s = (q @ k.T) * scale
    s = s.masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    w = torch.exp(s - m)
    l = w.sum(-1, keepdim=True)
    p = w / l
    R = (m - s).masked_fill(~vis, 0.0).amax(-1, keepdim=True)
    dot = ((q.abs() @ k.abs().T) * scale).masked_fill(~vis, 0.0).amax(-1, keepdim=True)
    n = vis.sum(-1, keepdim=True).double()
    return p @ v, p @ v.abs(), dict(l=l, R=R, dot=dot, n=n, vsum=(vis.double() @ v.abs()))


def _eps(info, d):
    """Relative error of the fp32 softmax weights, l and P V sums, per row.
    - score: d exact 16-bit products summed in fp32 (tensor-core accumulation may truncate: 2^-23 per add) and one multiply
      by the scale: |ds| <= 2^-23 (d + 2) max_j |q| . |k_j|.  A weight exp(s_j - m) carries the error of s_j and of m: 2 |ds|.
    - exp / exp2: the approximation (< 2^-21 relative) plus the rounded argument, 2^-23 |s - m| <= 2^-23 R (natural log
      units; R is capped at 64: a weight below e^-64 contributes nothing T can hold next to the largest weight, 1).
    - l and the P V accumulation: n fp32 additions, n 2^-23 relative in the worst case, the rescales of the online softmax
      included (both O and l are multiplied by the same rounded factor).
    eps = 2 (2 |ds| + exp error) + n 2^-23: the weights enter numerator and denominator of O = sum p v / l."""
    ds = 2.0 ** -23 * (d + 2) * info["dot"]
    e_exp = 2.0 ** -21 + 2.0 ** -23 * info["R"].clamp(max=64.0)
    return 2.0 * (2.0 * ds + e_exp) + info["n"] * 2.0 ** -23


def _check_a(got, O, A, info, d, dtype, what):
    u = _u(dtype)
    eps = _eps(info, d)
    tiny = _half_min_sub(dtype) * info["vsum"] / info["l"]
    bound = (u * O.abs() + (u + eps) * A + eps * O.abs() + tiny) * (1.0 + 4.0 * u)
    g = got.double()
    bad = ~((g - O).abs() <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} / {bad.numel()} beyond the float64 bound, "
                                 f"max err {(g - O).abs().max().item():.3g}, max bound {bound.max().item():.3g}")


class BitStats:
    """Collects check (b)'s bit-equal counts of one test case."""

    def __init__(self, dtype):
        self.dtype = dtype
        self.eq = 0
        self.n = 0

    def add(self, got, ref, dtype):
        self.eq += int((got.to(dtype).view(torch.int16) == ref.to(dtype).view(torch.int16)).sum())
        self.n += got.numel()

    def check(self, what, record=None):
        frac = self.eq / max(self.n, 1)
        if record is not None:
            record("bit_equal", f"{frac:.5f} of {self.n}")
        if self.n >= BIT_EQUAL_MIN:
            assert frac >= BIT_EQUAL[self.dtype], f"{what}: {frac:.4%} of {self.n} outputs bit-equal to the rounding restatement"


def _check_b(got, y, flips, A, info, d, dtype, stats, what):
    """got within 1 ulp of rnd_T(y), plus the P entries whose rounding the fp32 / float64 difference can flip (`flips`,
    from the restatement), plus 2^-20 A for the remaining differences of the unrounded quantities (exp approximation,
    fp32 sums)."""
    ref = _rnd(y, dtype)
    g = got.double()
    bound = _spacing(torch.maximum(g.abs(), ref.abs()), dtype) + flips + (2.0 ** -20 + info["n"] * 2.0 ** -24) * A
    bad = ~((g - ref).abs() <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} / {bad.numel()} beyond 1 ulp + P flips of the rounding "
                                 f"restatement, max err {(g - ref).abs().max().item():.3g}")
    stats.add(got, ref, dtype)


def _f32_scores(q, k, scale):
    """Scores with the kernels' fp32 rounding points: the dot product rounded to fp32, times the fp32 scale in fp32.
    Returns (scores, per-key bound of the fp32 accumulation-order difference).  That difference is modelled as a random
    walk of d roundings of the partial sums, d 2^-24 sqrt(sum_i (q_i k_i)^2) (the worst case, d 2^-24 sum_i |q_i k_i|,
    would make almost every P entry ambiguous at head_dim 128), plus 2^-20 sum_i |q_i k_i| for the tensor cores' truncating
    accumulation and the rounding of large scores."""
    s = (q @ k.T).float() * torch.tensor(scale, dtype=torch.float32)
    ds = scale * (2.0 ** -24 * q.shape[-1] * ((q * q) @ (k * k).T).sqrt() + 2.0 ** -20 * (q.abs() @ k.abs().T))
    return s, ds


def _flip_allowance(w, e, v, dtype, resc=1.0):
    """Sum of spacing_T(w_j) |v_j| over the P entries w [n, m] (in output units) whose rounding to T can change when w moves
    by the relative error e [n, m] between the kernel's fp32 weight and the restatement's: the entries within e of a T
    rounding boundary.  Each such flip moves the output by one T spacing of the entry times |v_j| (times the online-softmax
    rescale `resc` of the entry's tile)."""
    amb = _rnd(w * (1.0 + e), dtype) != _rnd(w * (1.0 - e), dtype)
    return (amb.double() * _spacing(w, dtype) * resc) @ v.abs()


def _weight_err(ds, x):
    """Relative error window of a kernel weight exp(x) (x = s - m <= 0, natural log units): the score and the max each off
    by ds, the exp approximation (< 2^-21) and the fp32 argument, 2^-23 |x|."""
    return 2.0 * ds + 2.0 ** -21 + 2.0 ** -23 * x.abs()


def varlen_rounding_ref(q, k, v, scale, causal, dtype):
    """attn_varlen's rounding points for one sequence and head: fp32 scores times fp32(scale * log2 e); keys in 64-key
    tiles, in order; per query row the running max m_t over tiles 0..t; p = rnd_T(2^(s - m_t)) (fp32 argument); O and l
    rescaled by 2^(m_{t-1} - m_t) (so a key of tile t enters the final sums with 2^(m_t - m_last)); l sums the unrounded
    weights; out = rnd_T(O / l).  Returns (O / l before the final rounding, flip allowance per element)."""
    L = q.shape[0]
    sl2 = float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E_F32, dtype=torch.float32))
    s, ds = _f32_scores(q, k, sl2)
    if causal:
        s = s.masked_fill(~torch.ones(L, L, dtype=torch.bool, device=q.device).tril(), -math.inf)
    nt = (L + 63) // 64
    sp = F.pad(s, (0, nt * 64 - L), value=-math.inf)
    mt = sp.view(L, nt, 64).amax(-1).cummax(-1).values              # [L, nt] running max after tile t
    m_key = mt.repeat_interleave(64, dim=1)[:, :L]
    m_last = mt[:, -1:]
    x = (s - m_key).double()
    w_t = torch.exp2(x)
    resc = torch.exp2((m_key - m_last).double())
    w = _rnd(w_t, dtype) * resc
    l = torch.exp2((s - m_last).double()).sum(-1, keepdim=True)
    e = _weight_err(ds / LOG2E_F32, x.abs() / LOG2E_F32)
    return (w @ v) / l, _flip_allowance(w_t, e, v, dtype, resc) / l


def decode_rounding_ref(q, k, v, scale, dtype):
    """decode_attn's rounding points for one (row, kv head): fp32 scores, m their global max, p = rnd_T(exp(s - m)),
    l = sum exp(s - m) unrounded, out = rnd_T(sum p v / l)."""
    s, ds = _f32_scores(q, k, scale)
    x = (s - s.amax(-1, keepdim=True)).double()
    w = torch.exp(x)
    l = w.sum(-1, keepdim=True)
    return (_rnd(w, dtype) @ v) / l, _flip_allowance(w, _weight_err(ds, x), v, dtype) / l


def single_query_rounding_ref(q, k, v, scale, dtype):
    """attn_single_query's rounding points: fp32 scores, p = rnd_T(exp(s - m) / l) (normalised in fp32, then rounded),
    out = rnd_T(sum p v)."""
    s, ds = _f32_scores(q, k, scale)
    x = (s - s.amax(-1, keepdim=True)).double()
    w = torch.exp(x)
    l = w.sum(-1, keepdim=True)
    pn = (w.float() / l.float()).double()
    # the normalisation adds the error of l (n fp32 additions, n 2^-24) to each entry's window
    e = _weight_err(ds, x) + w.shape[-1] * 2.0 ** -24
    return _rnd(pn, dtype) @ v, _flip_allowance(pn, e, v, dtype)


def rope_ref(x, pos, inv_freq, dtype):
    """RoPE of x [n, heads, d] (exact T values, float64): cos / sin in float64 of the fp32 product float(pos) * inv_freq,
    rounded to T; o1 = rnd(rnd(x1 c) + rnd(-x2 s)), o2 = rnd(rnd(x2 c) + rnd(x1 s)).  Returns (out, flip allowance): the
    change of the output if c or s rounded to the neighbouring T value (fp32 cosf / sinf are not correctly rounded)."""
    f = (pos.float()[:, None] * inv_freq.float()[None, :]).double()
    c, s = _rnd(torch.cos(f), dtype)[:, None, :], _rnd(torch.sin(f), dtype)[:, None, :]
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    a1, b1 = _rnd(x1 * c, dtype), _rnd(-x2 * s, dtype)
    a2, b2 = _rnd(x2 * c, dtype), _rnd(x1 * s, dtype)
    o = torch.cat([_rnd(a1 + b1, dtype), _rnd(a2 + b2, dtype)], -1)
    sc, ss = _spacing(c, dtype), _spacing(s, dtype)
    fl1 = x1.abs() * sc + _spacing(a1.abs() + x1.abs() * sc, dtype) + x2.abs() * ss + _spacing(b1.abs() + x2.abs() * ss, dtype)
    fl2 = x2.abs() * sc + _spacing(a2.abs() + x2.abs() * sc, dtype) + x1.abs() * ss + _spacing(b2.abs() + x1.abs() * ss, dtype)
    return o, torch.cat([fl1, fl2], -1)


def _check_rope(got, x, pos, inv_freq, dtype, what):
    ref, flip = rope_ref(x, pos, inv_freq, dtype)
    g = got.double()
    bad = ~((g - ref).abs() <= flip + _spacing(torch.maximum(g.abs(), ref.abs()), dtype))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} / {bad.numel()} beyond a cos / sin flip of the RoPE restatement"
    eq = (got.view(torch.int16) == ref.to(dtype).view(torch.int16)).double().mean().item()
    assert eq >= 0.999, f"{what}: only {eq:.4%} of RoPE outputs bit-equal"


# ------------------------------------------------------------------------------------------------ CPU rehearsal
@pytest.mark.parametrize("dtype", DT)
def test_references_match_sdpa(dtype):
    """The float64 references (and the rounding restatements, within bound (a)) agree with F.scaled_dot_product_attention
    in float64, at tiny shapes, with GQA and causal masks.  Runs on CPU."""
    g = torch.Generator().manual_seed(3)
    L, d, nh, nkv = 150, 32, 4, 2
    scale = d ** -0.5
    q = _rnd(torch.randn(nh, L, d, generator=g, dtype=torch.float64), dtype)
    k = _rnd(torch.randn(nkv, L, d, generator=g, dtype=torch.float64), dtype)
    v = _rnd(torch.randn(nkv, L, d, generator=g, dtype=torch.float64), dtype)
    for causal in (False, True):
        sd = F.scaled_dot_product_attention(q[None], k.repeat_interleave(nh // nkv, 0)[None],
                                            v.repeat_interleave(nh // nkv, 0)[None], is_causal=causal, scale=scale)[0]
        vis = torch.ones(L, L, dtype=torch.bool)
        if causal:
            vis = vis.tril()
        for h in range(nh):
            kv = h // (nh // nkv)
            O, A, info = _exact(q[h], k[kv], v[kv], scale, vis)
            torch.testing.assert_close(O, sd[h], rtol=1e-12, atol=1e-12)
            y, _ = varlen_rounding_ref(q[h], k[kv], v[kv], scale, causal, dtype)
            _check_a(_rnd(y, dtype), O, A, info, d, dtype, "varlen restatement")
            yd, _ = decode_rounding_ref(q[h, -1:], k[kv], v[kv], scale, dtype)
            _check_a(_rnd(yd, dtype), O[-1:], A[-1:], {x: t[-1:] for x, t in info.items()}, d, dtype, "decode restatement")
            ys, _ = single_query_rounding_ref(q[h, -1:], k[kv], v[kv], scale, dtype)
            _check_a(_rnd(ys, dtype), O[-1:], A[-1:], {x: t[-1:] for x, t in info.items()}, d, dtype, "single-query restatement")
    # zero q: uniform weights over exactly the visible keys
    O, _, _ = _exact(torch.zeros(L, d, dtype=torch.float64), k[0], v[0], scale, torch.ones(L, L, dtype=torch.bool).tril())
    torch.testing.assert_close(O, v[0].cumsum(0) / torch.arange(1, L + 1, dtype=torch.float64)[:, None])
    # RoPE restatement at position 0 is the identity
    x = _rnd(torch.randn(3, 2, d, generator=g, dtype=torch.float64), dtype)
    inv = 1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float) / d))
    assert torch.equal(rope_ref(x, torch.zeros(3, dtype=torch.int32), inv, dtype)[0], x)


# ------------------------------------------------------------------------------------------------ input families
def _fill(family, q, k, v, scale, g):
    """Overwrite q [L, nh, d], k / v [L, nkv, d] (float64, one sequence) for an input family; values are rounded to T later.
    moving   : scores rise by ~3 per 64-key tile (q[..., 0] = 4, k[j, :, 0] a ramp), the running max moves in every tile.
    peak_diag: key j dominates query j by ~100 (k_j = 100 q_j / (scale |q_j|^2), q shared across a GQA group).
    peak_last: the sequence's last key dominates every query by ~100 (put it alone in a partial tile).
    zero_q   : q = 0, v > 0: uniform weights, checked against the mean of the visible keys.
    large    : q, k scaled by 10: almost every weight underflows to 0."""
    L, nh, d = q.shape
    nkv = k.shape[1]
    G = nh // nkv
    if family == "moving":
        q[..., 0] = 4.0
        k[:, :, 0] = (0.75 / scale) * torch.arange(L, dtype=torch.float64, device=k.device)[:, None] / 64.0
    elif family == "peak_diag":
        q[:] = q[:, ::G].repeat_interleave(G, 1)
        qk = q[:, ::G]
        k[:] = 100.0 * qk / (scale * (qk * qk).sum(-1, keepdim=True))
    elif family == "peak_last":
        w = torch.randn(1, nkv, d, generator=g, device=q.device, dtype=torch.float64)
        q[:] = w.repeat_interleave(G, 1) + 0.3 * q
        k[-1] = 100.0 * w[0] / (scale * (w[0] * w[0]).sum(-1, keepdim=True))
    elif family == "zero_q":
        q.zero_()
        v.abs_().add_(0.5)
    elif family == "large":
        q.mul_(10.0)
        k.mul_(10.0)


# ------------------------------------------------------------------------------------------------ attn_varlen
VARLEN_CASES = [
    # head_dim, nh, nkv, causal, sequence lengths (0 = empty sequence), family
    (32, 4, 4, False, [1, 63, 0, 64, 65], "randn"),
    (32, 4, 2, True, [128, 129, 63], "zero_q"),
    (64, 8, 1, True, [127, 128, 0, 129], "randn"),
    (64, 4, 1, True, [1024, 127], "moving"),
    (64, 4, 4, False, [129, 65, 1], "peak_last"),
    (64, 8, 8, True, [200, 64], "large"),
    (80, 16, 16, False, [1030, 65], "randn"),        # recognition vision tower
    (80, 16, 4, True, [1100, 0, 129], "randn"),      # recognition prefill (GQA 16:4)
    (80, 4, 2, False, [700, 129], "moving"),
    (80, 8, 4, True, [200, 65], "peak_diag"),
    (80, 4, 4, False, [300, 65], "large"),
    (96, 4, 2, True, [200, 63], "randn"),
    (96, 4, 4, False, [129, 64], "peak_diag"),
    (128, 8, 2, True, [300, 65], "randn"),
    (128, 4, 4, False, [256, 97], "zero_q"),
    (128, 16, 2, False, [129, 1], "moving"),
]


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("d,nh,nkv,causal,lens,family", VARLEN_CASES)
def test_attn_varlen(built_lib, record_property, dtype, d, nh, nkv, causal, lens, family):
    """Packed sequences with 3-row gaps that belong to no sequence, max_len above every length, q / k / v as column
    windows of a wider qkv buffer, and out as a window of a NaN-filled buffer with ldo > nh * d."""
    from surya_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(d * 131 + nh * 7 + sum(lens))
    GAP = 3
    starts, s = [], GAP
    for L in lens:
        starts.append(s)
        s += L + GAP
    T = s
    scale = d ** -0.5
    q = torch.randn(T, nh, d, device="cuda", generator=g, dtype=torch.float64)
    k = torch.randn(T, nkv, d, device="cuda", generator=g, dtype=torch.float64)
    v = torch.randn(T, nkv, d, device="cuda", generator=g, dtype=torch.float64)
    for st, L in zip(starts, lens):
        if L:
            _fill(family, q[st:st + L], k[st:st + L], v[st:st + L], scale, g)
    width = (nh + 2 * nkv) * d
    qkv = torch.empty(T, width + 8, device="cuda", dtype=dtype)
    qkv[:, :nh * d] = q.reshape(T, -1).to(dtype)
    qkv[:, nh * d:(nh + nkv) * d] = k.reshape(T, -1).to(dtype)
    qkv[:, (nh + nkv) * d:width] = v.reshape(T, -1).to(dtype)
    qw, kw, vw = qkv[:, :nh * d], qkv[:, nh * d:(nh + nkv) * d], qkv[:, (nh + nkv) * d:width]
    buf = torch.full((T, nh * d + 16), float("nan"), device="cuda", dtype=dtype)
    out = buf[:, 8:8 + nh * d]
    st_t = torch.tensor(starts, device="cuda", dtype=torch.int32)
    len_t = torch.tensor(lens, device="cuda", dtype=torch.int32)
    ops.attn_varlen(qw, kw, vw, st_t, len_t, max(lens) + 37, nh, nkv, d, causal, scale, out=out)
    torch.cuda.synchronize()

    nan = _nan_bits(dtype)
    bits = buf.view(torch.int16)
    inside = torch.zeros(T, dtype=torch.bool, device="cuda")
    for st, L in zip(starts, lens):
        inside[st:st + L] = True
    assert bool((bits[:, :8] == nan).all()) and bool((bits[:, 8 + nh * d:] == nan).all()), "wrote outside the output window"
    assert bool((bits[~inside] == nan).all()), "wrote a packed row that belongs to no sequence"
    assert not bool(out[inside].isnan().any()), "left an output of a sequence unwritten"

    qd = qw.double().reshape(T, nh, d)
    kd, vd = kw.double().reshape(T, nkv, d), vw.double().reshape(T, nkv, d)
    stats = BitStats(dtype)
    G = nh // nkv
    for st, L in zip(starts, lens):
        if L == 0:
            continue
        vis = torch.ones(L, L, dtype=torch.bool, device="cuda")
        if causal:
            vis = vis.tril()
        for h in range(nh):
            qq, kk, vv = qd[st:st + L, h], kd[st:st + L, h // G], vd[st:st + L, h // G]
            got = out[st:st + L, h * d:(h + 1) * d]
            what = f"attn_varlen seq@{st} len {L} head {h}"
            O, A, info = _exact(qq, kk, vv, scale, vis)
            _check_a(got, O, A, info, d, dtype, what)
            y, flips = varlen_rounding_ref(qq, kk, vv, scale, causal, dtype)
            _check_b(got, y, flips, A, info, d, dtype, stats, what)
            if family == "zero_q":
                mean = (vis.double() @ vv) / vis.sum(-1, keepdim=True)
                assert bool(((got.double() - mean).abs() <= _spacing(mean, dtype)).all()), f"{what}: not the mean of the visible keys"
    stats.check(f"attn_varlen {family}", record_property)


# ------------------------------------------------------------------------------------------------ decode_attn + RoPE
def _inv_freq(d):
    return (1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float) / d))).cuda()


DECODE_CASES = [(d, G, 2, 320, "randn") for d in (64, 80, 128) for G in (1, 2, 4, 8)] + [
    (80, 4, 4, 1536, "randn"),       # recognition decoder
    (80, 4, 4, 1536, "peak_new"),
    (64, 4, 4, 512, "zero_q"),       # layout decoder
    (64, 2, 4, 512, "large"),        # table decoder
    (128, 8, 2, 1536, "randn"),      # 86 KB of shared memory: the > 48 KB opt-in
]


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("d,G,nkv,s_max,family", DECODE_CASES)
def test_decode_attn(built_lib, record_property, dtype, d, G, nkv, s_max, family):
    """Rows at pos 0, 127 / 128 / 129, both sides of the PV batching stride (NKG * 4), s_max - 1 and two random positions,
    in non-contiguous slots, with qkv's pitch above its width and out in a window of a NaN-filled buffer; plus rows with
    pos = s_max and pos = -1, which must output zeros and leave the cache unchanged.  The appended K row must equal the row
    rope_kv_append writes for the same qkv row and position, bit for bit."""
    from surya_b200 import ops

    nh = G * nkv
    g = torch.Generator(device="cuda").manual_seed(d * 17 + G * 5 + s_max + len(family))
    nkg4 = 4 * (128 // (d // 8))
    poses = [0, 127, 128, 129, nkg4 - 1, nkg4, s_max - 1, 37, s_max // 2 + 11]
    valid = len(poses)
    poses += [s_max, -1]
    B = len(poses)
    slots = 2 * B + 1
    slot_ids = torch.randperm(slots, generator=torch.Generator().manual_seed(s_max))[:B]
    slot_ids[valid] = slot_ids[0]        # an out-of-range row shares a slot with a valid row: its writes would be visible
    kc = torch.randn(slots, nkv, s_max, d, device="cuda", generator=g).to(dtype)
    vc = torch.randn(slots, nkv, s_max, d, device="cuda", generator=g).to(dtype)
    width = (nh + 2 * nkv) * d
    q = torch.randn(B, nh, d, device="cuda", generator=g, dtype=torch.float64)
    kn = torch.randn(B, nkv, d, device="cuda", generator=g, dtype=torch.float64)
    vn = torch.randn(B, nkv, d, device="cuda", generator=g, dtype=torch.float64)
    scale = d ** -0.5
    if family == "zero_q":
        q.zero_()
        vn.abs_().add_(0.5)
        vc.abs_().add_(0.5)
    elif family == "large":
        q.mul_(10.0)
        kn.mul_(10.0)
        kc.mul_(10.0)
    elif family == "peak_new":     # the appended key dominates by ~60: k = lambda q before RoPE keeps q . k after it
        q[:] = q[:, ::G].repeat_interleave(G, 1)
        kn[:] = 60.0 * q[:, ::G] / (scale * (q[:, ::G] ** 2).sum(-1, keepdim=True))
    qkv = torch.zeros(B, width + 24, device="cuda", dtype=dtype)
    qkv[:, :nh * d] = q.reshape(B, -1).to(dtype)
    qkv[:, nh * d:(nh + nkv) * d] = kn.reshape(B, -1).to(dtype)
    qkv[:, (nh + nkv) * d:width] = vn.reshape(B, -1).to(dtype)
    qkv_in = qkv[:, :width]
    raw = qkv_in.clone()
    kc0, vc0 = kc.clone(), vc.clone()
    inv = _inv_freq(d)
    slot_t = slot_ids.to(device="cuda", dtype=torch.int32)
    pos_t = torch.tensor(poses, device="cuda", dtype=torch.int32)
    buf = torch.full((B, nh * d + 16), float("nan"), device="cuda", dtype=dtype)
    out = buf[:, 8:8 + nh * d]
    ops.decode_attn(qkv_in, kc, vc, slot_t, pos_t, inv, nh, nkv, d, scale, out=out)
    # the rotated q / k the kernel used: rope_kv_append on the same rows (its own cache copies)
    rot = raw.clone()
    kc_r, vc_r = kc0.clone(), vc0.clone()
    ops.rope_kv_append_(rot[:valid], pos_t[:valid], slot_t[:valid], inv, kc_r, vc_r, nh, nkv, d)
    torch.cuda.synchronize()

    assert torch.equal(qkv_in, raw), "decode_attn changed its qkv input"
    nan = _nan_bits(dtype)
    bits = buf.view(torch.int16)
    assert bool((bits[:, :8] == nan).all()) and bool((bits[:, 8 + nh * d:] == nan).all()), "wrote outside the output window"
    assert bool((out[valid:] == 0).all()), "rows with pos outside [0, s_max) must output zeros"
    # the cache: bit-identical except the appended rows of the valid rows
    kc_exp, vc_exp = kc0.clone(), vc0.clone()
    for b in range(valid):
        s_, p_ = int(slot_ids[b]), poses[b]
        assert torch.equal(kc[s_, :, p_], kc_r[s_, :, p_]), f"row {b}: appended K differs from rope_kv_append's"
        kc_exp[s_, :, p_] = kc[s_, :, p_]
        vc_exp[s_, :, p_] = raw[b, (nh + nkv) * d:].reshape(nkv, d)
    assert torch.equal(kc, kc_exp), "decode_attn changed K cache rows other than the appended ones"
    assert torch.equal(vc, vc_exp), "decode_attn changed V cache rows other than the appended ones (or appended a wrong v)"
    _check_rope(rot[:valid, :(nh + nkv) * d].reshape(valid, nh + nkv, d), raw[:valid, :(nh + nkv) * d].double().reshape(valid, nh + nkv, d),
                pos_t[:valid], inv, dtype, "decode RoPE")

    stats = BitStats(dtype)
    qr = rot[:, :nh * d].double().reshape(B, nh, d)
    for b in range(valid):
        s_, p_ = int(slot_ids[b]), poses[b]
        for kvh in range(nkv):
            qq = qr[b, kvh * G:(kvh + 1) * G]
            kk, vv = kc[s_, kvh, :p_ + 1].double(), vc[s_, kvh, :p_ + 1].double()
            got = out[b, kvh * G * d:(kvh + 1) * G * d].reshape(G, d)
            what = f"decode_attn row {b} (pos {p_}) kv head {kvh}"
            if p_ == 0:
                assert torch.equal(got, vc[s_, kvh, 0].expand(G, d)), f"{what}: pos 0 must return its own v"
            vis = torch.ones(G, p_ + 1, dtype=torch.bool, device="cuda")
            O, A, info = _exact(qq, kk, vv, scale, vis)
            _check_a(got, O, A, info, d, dtype, what)
            y, flips = decode_rounding_ref(qq, kk, vv, scale, dtype)
            _check_b(got, y, flips, A, info, d, dtype, stats, what)
            if family == "zero_q":
                mean = vv.mean(0, keepdim=True)
                assert bool(((got.double() - mean).abs() <= _spacing(mean, dtype)).all()), f"{what}: not the mean of the keys"
    stats.check(f"decode_attn {family}", record_property)


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("d,nh,nkv", [(80, 16, 4), (64, 8, 2), (128, 4, 4)])
def test_rope_kv_append(built_lib, dtype, d, nh, nkv):
    """Positions up to 1535 against the float64 RoPE restatement; k and v land in cache[slot][kv head][pos].  Tokens with
    pos = s_max or s_max + 5 (in slot 0) and pos = -1 (in slot 1) are rotated but leave the cache untouched; the slots are
    chosen so that a stray write would land inside the cache buffer."""
    from surya_b200 import ops

    s_max, slots = 1536, 3
    g = torch.Generator(device="cuda").manual_seed(d + nh)
    poses = list(range(0, 1536, 7)) + [1535, 1534]
    slot_l = [1 + (i % 2) for i in range(len(poses))]
    bad = [s_max, s_max + 5, -1]
    poses += bad
    slot_l += [0, 0, 1]
    n = len(poses)
    width = (nh + 2 * nkv) * d
    qkv_buf = torch.randn(n, width + 8, device="cuda", generator=g).to(dtype)
    qkv = qkv_buf[:, :width]
    raw = qkv.clone()
    kc = torch.randn(slots, nkv, s_max, d, device="cuda", generator=g).to(dtype)
    vc = torch.randn_like(kc)
    kc0, vc0 = kc.clone(), vc.clone()
    inv = _inv_freq(d)
    pos_t = torch.tensor(poses, device="cuda", dtype=torch.int32)
    slot_t = torch.tensor(slot_l, device="cuda", dtype=torch.int32)
    ops.rope_kv_append_(qkv, pos_t, slot_t, inv, kc, vc, nh, nkv, d)
    torch.cuda.synchronize()
    assert torch.equal(qkv[:, (nh + nkv) * d:], raw[:, (nh + nkv) * d:]), "v columns changed"
    _check_rope(qkv[:, :(nh + nkv) * d].reshape(n, nh + nkv, d), raw[:, :(nh + nkv) * d].double().reshape(n, nh + nkv, d),
                pos_t, inv, dtype, "rope_kv_append")
    kc_exp, vc_exp = kc0.clone(), vc0.clone()
    for i in range(n - len(bad)):
        kc_exp[slot_l[i], :, poses[i]] = qkv[i, nh * d:(nh + nkv) * d].reshape(nkv, d)
        vc_exp[slot_l[i], :, poses[i]] = raw[i, (nh + nkv) * d:].reshape(nkv, d)
    assert torch.equal(kc[0], kc0[0]) and torch.equal(vc[0], vc0[0]), "a token with pos outside [0, s_max) wrote the cache"
    assert torch.equal(kc, kc_exp) and torch.equal(vc, vc_exp), "cache rows differ from the rotated k / raw v"


# ------------------------------------------------------------------------------------------------ attn_single_query
SQ_CASES = [(1, 1), (2, 95), (4, 96), (1, 97), (2, 255), (4, 256), (1, 257), (4, 576), (2, 576), (4, 2500)]


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("G,n_keys", SQ_CASES)
def test_attn_single_query(built_lib, record_property, dtype, G, n_keys):
    """K / V as the strided halves of the fused cross K/V rows (as layout.py passes them), out into a window of a
    NaN-filled buffer; n_keys = 2500 with G = 4 needs the shared-memory opt-in.  Row 1 has a dominant key."""
    from surya_b200 import ops

    B, nkv, hd = 3, 2, 64
    nh = G * nkv
    scale = hd ** -0.5
    g = torch.Generator(device="cuda").manual_seed(G * 1000 + n_keys)
    q = torch.randn(B, nh * hd, device="cuda", generator=g).to(dtype)
    kv = torch.randn(B * n_keys, 2 * nkv * hd, device="cuda", generator=g, dtype=torch.float64)
    kv3 = kv.view(B, n_keys, 2, nkv, hd)
    q1 = q[1].double().view(nkv, G, hd)[:, 0]
    kv3[1, n_keys // 2, 0] = 60.0 * q1 / (scale * (q1 * q1).sum(-1, keepdim=True))      # peaked row (head 0 of each group)
    kv = kv.to(dtype)
    buf = torch.full((B, nh * hd + 16), float("nan"), device="cuda", dtype=dtype)
    out = buf[:, 8:8 + nh * hd]
    ops.attn_single_query(q, kv, n_keys, nh, nkv, hd, scale, out=out)
    torch.cuda.synchronize()
    nan = _nan_bits(dtype)
    bits = buf.view(torch.int16)
    assert bool((bits[:, :8] == nan).all()) and bool((bits[:, 8 + nh * hd:] == nan).all()), "wrote outside the output window"
    kvd = kv.double().view(B, n_keys, 2, nkv, hd)
    stats = BitStats(dtype)
    for b in range(B):
        for kvh in range(nkv):
            qq = q[b].double().view(nh, hd)[kvh * G:(kvh + 1) * G]
            kk, vv = kvd[b, :, 0, kvh], kvd[b, :, 1, kvh]
            got = out[b, kvh * G * hd:(kvh + 1) * G * hd].reshape(G, hd)
            what = f"attn_single_query row {b} kv head {kvh}"
            O, A, info = _exact(qq, kk, vv, scale, torch.ones(G, n_keys, dtype=torch.bool, device="cuda"))
            _check_a(got, O, A, info, hd, dtype, what)
            y, flips = single_query_rounding_ref(qq, kk, vv, scale, dtype)
            _check_b(got, y, flips, A, info, hd, dtype, stats, what)
    stats.check("attn_single_query", record_property)


# ------------------------------------------------------------------------------------------------ dependent launch
@gpu
@pytest.mark.parametrize("dtype", DT)
def test_decode_dependent_launch(built_lib, dtype):
    """qkv GEMM -> decode_attn -> o-projection GEMM with the residual, with no synchronise in between (as a decode step
    runs them), equals the same chain with a synchronise after each call, bit for bit: outputs and caches."""
    from surya_b200 import ops

    B, nh, nkv, d, H, K, s_max = 8, 16, 4, 80, 1280, 16384, 1536
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn(B, K, device="cuda", generator=g) * 0.1).to(dtype)
    w_qkv = (torch.randn((nh + 2 * nkv) * d, K, device="cuda", generator=g) * 0.01).to(dtype)
    w_o = (torch.randn(H, nh * d, device="cuda", generator=g) * 0.05).to(dtype)
    res = torch.randn(B, H, device="cuda", generator=g).to(dtype)
    kc0 = torch.randn(B + 2, nkv, s_max, d, device="cuda", generator=g).to(dtype)
    vc0 = torch.randn_like(kc0)
    slot = torch.arange(2, B + 2, device="cuda", dtype=torch.int32)
    pos = torch.randint(900, s_max, (B,), device="cuda", generator=g, dtype=torch.int32)
    inv = _inv_freq(d)

    def chain(sync):
        kc, vc = kc0.clone(), vc0.clone()
        qkv = torch.empty(B, (nh + 2 * nkv) * d, device="cuda", dtype=dtype)
        attn = torch.empty(B, nh * d, device="cuda", dtype=dtype)
        torch.cuda.synchronize()
        qkv.zero_()
        attn.zero_()
        ops.gemm(x, w_qkv, out=qkv)
        if sync:
            torch.cuda.synchronize()
        ops.decode_attn(qkv, kc, vc, slot, pos, inv, nh, nkv, d, d ** -0.5, out=attn)
        if sync:
            torch.cuda.synchronize()
        o = ops.gemm(attn, w_o, residual=res)
        torch.cuda.synchronize()
        return o, attn, kc, vc

    early, late = chain(False), chain(True)
    for a, b, what in zip(early, late, ("o-projection", "attention", "K cache", "V cache")):
        assert torch.equal(a, b), f"{what} differs when the chain runs without synchronises"


# ------------------------------------------------------------------------------------------------ errors
ERROR_CASES = ["decode_smem", "decode_nkv0", "sq_group", "sq_no_keys", "sq_nkv0", "varlen_q_align", "varlen_k_align",
               "varlen_v_align", "varlen_out_align", "varlen_nkv0"]


@gpu
@pytest.mark.parametrize("case", ERROR_CASES)
def test_errors_are_loud(built_lib, case):
    """A bad call raises SuryaB200Error with a message, and an ordinary call of the same kernel right after it succeeds
    (no stale CUDA error is left for the next call's launch check).  Only host-side validation runs for the bad calls."""
    from surya_b200 import _lib, ops

    dt = torch.float16
    if case.startswith("decode"):
        d, nh, nkv, B = 64, 4, 1, 2
        qkv = torch.randn(B, (nh + 2 * nkv) * d, device="cuda").to(dt)
        kc = torch.randn(B, nkv, 64, d, device="cuda").to(dt)
        vc = torch.randn_like(kc)
        slot = torch.arange(B, device="cuda", dtype=torch.int32)
        pos = torch.tensor([0, 5], device="cuda", dtype=torch.int32)
        inv = _inv_freq(d)
        out = torch.empty(B, nh * d, device="cuda", dtype=dt)
        torch.cuda.synchronize()
        if case == "decode_smem":        # 266 KB of scores: beyond the device's shared memory
            huge = torch.empty(1, nkv, 65536, d, device="cuda", dtype=dt)
            zero_slot = torch.zeros(B, device="cuda", dtype=torch.int32)
            torch.cuda.synchronize()
            with pytest.raises(_lib.SuryaB200Error, match="shared memory"):
                ops.decode_attn(qkv, huge, huge, zero_slot, pos, inv, nh, nkv, d, 1.0, out=out)
        else:
            with pytest.raises(_lib.SuryaB200Error, match="n_kv_heads"):
                ops.decode_attn(qkv, kc, vc, slot, pos, inv, nh, 0, d, 1.0, out=out)
        ops.decode_attn(qkv, kc, vc, slot, pos, inv, nh, nkv, d, 1.0, out=out)
        torch.cuda.synchronize()
        assert torch.equal(out[0], vc[0, 0, 0].repeat(nh)), "decode_attn after an error: pos 0 must return its v"
    elif case.startswith("sq"):
        B, hd, n_keys = 2, 64, 16
        q = torch.randn(B, 4 * hd, device="cuda").to(dt)
        kv = torch.randn(B * n_keys, 2 * 2 * hd, device="cuda").to(dt)
        out = torch.empty(B, 4 * hd, device="cuda", dtype=dt)
        if case == "sq_group":           # nh = 6, nkv = 4: a group of 1.5 heads
            q6 = torch.randn(B, 6 * hd, device="cuda").to(dt)
            kv4 = torch.randn(B * n_keys, 2 * 4 * hd, device="cuda").to(dt)
            with pytest.raises(_lib.SuryaB200Error, match="multiple of nkv"):
                ops.attn_single_query(q6, kv4, n_keys, 6, 4, hd, hd ** -0.5)
        elif case == "sq_no_keys":
            with pytest.raises(_lib.SuryaB200Error, match="n_keys"):
                ops.attn_single_query(q, kv, 0, 4, 2, hd, hd ** -0.5)
        else:
            with pytest.raises(_lib.SuryaB200Error, match="multiple of nkv"):
                ops.attn_single_query(q, kv, n_keys, 4, 0, hd, hd ** -0.5)
        ops.attn_single_query(q, kv, n_keys, 4, 2, hd, hd ** -0.5, out=out)
        torch.cuda.synchronize()
        assert not bool(out.isnan().any()), "attn_single_query after an error"
    else:
        T, nh, d = 70, 2, 64
        wide = torch.randn(T, 3 * nh * d + 16, device="cuda").to(dt)
        qw, kw, vw = wide[:, :nh * d], wide[:, nh * d:2 * nh * d], wide[:, 2 * nh * d:3 * nh * d]
        shift = wide[:, 4:4 + nh * d]    # 8 bytes into each row: the pitch is fine, the base is not 16-byte aligned
        starts = torch.tensor([0], device="cuda", dtype=torch.int32)
        lens = torch.tensor([T], device="cuda", dtype=torch.int32)
        obuf = torch.empty(T, nh * d + 8, device="cuda", dtype=dt)
        args = dict(varlen_q_align=(shift, kw, vw, obuf[:, :nh * d], nh), varlen_k_align=(qw, shift, vw, obuf[:, :nh * d], nh),
                    varlen_v_align=(qw, kw, shift, obuf[:, :nh * d], nh),
                    varlen_out_align=(qw, kw, vw, obuf[:, 1:1 + nh * d], nh),   # 2 bytes into each row
                    varlen_nkv0=(qw, kw, vw, obuf[:, :nh * d], 0))[case]
        with pytest.raises(_lib.SuryaB200Error, match="n_kv_heads" if case == "varlen_nkv0" else "aligned"):
            ops.attn_varlen(*args[:3], starts, lens, T, nh, args[4], d, True, d ** -0.5, out=args[3])
        o = ops.attn_varlen(qw, kw, vw, starts, lens, T, nh, nh, d, True, d ** -0.5, out=obuf[:, :nh * d])
        torch.cuda.synchronize()
        assert torch.equal(o[0], vw[0]), "attn_varlen after an error: causal row 0 must return its v"
