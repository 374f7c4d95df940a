"""decode_attn (GPU): properties of the output bits that a streamed, chunked kernel could break and the tolerance checks of
test_attention_gpu.py would not catch, all compared with torch.equal:
- identical (q, k, v, pos) give identical bits in any row, slot and KV head, in a ragged batch and alone;
- the same cache contents under s_max = 256 and s_max = 1536 give identical outputs;
- a CUDA graph replay gives the bits of an eager launch;
and the recognition benchmark's shape (B = 256, 4 KV heads of 4 query heads, head_dim 80, s_max = 256, ragged positions
46 .. 172) passes the float64 checks (a) and (b) of test_attention_gpu.py."""
import pytest
import torch

from test_attention_gpu import DT, BitStats, _check_a, _check_b, _exact, decode_rounding_ref, gpu


def _inv_freq(d):
    return (1.0 / (10000.0 ** (torch.arange(0, d, 2, dtype=torch.float) / d))).cuda()


def _qkv_width(nh, nkv, d):
    return (nh + 2 * nkv) * d


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("d,G,nkv", [(80, 4, 4), (128, 8, 2), (64, 1, 4)])
@pytest.mark.parametrize("P", [0, 31, 32, 33, 95, 96, 129, 173, 255])
def test_same_inputs_same_bits(built_lib, dtype, d, G, nkv, P):
    """Rows 1, 4, 6 and 9 of a ragged batch carry the same (q, k, v, pos = P) in every KV head, in different slots whose
    cache rows 0 .. P-1 are equal; every (row, KV head) of them, and the same inputs launched alone, give the same output
    bits and append the same cache rows."""
    from surya_b200 import ops

    s_max, nh, B = 256, G * nkv, 11
    gen = torch.Generator(device="cuda").manual_seed(P * 7 + d + G)
    copies = [1, 4, 6, 9]
    poses = torch.randint(0, s_max, (B,), generator=torch.Generator().manual_seed(P + 1))
    poses[copies] = P
    slot_ids = torch.randperm(B + 5, generator=torch.Generator().manual_seed(P + 2))[:B]
    kc = torch.randn(B + 5, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    vc = torch.randn(B + 5, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    bk = torch.randn(s_max, d, device="cuda", generator=gen).to(dtype)
    bv = torch.randn(s_max, d, device="cuda", generator=gen).to(dtype)
    qkv = torch.randn(B, _qkv_width(nh, nkv, d), device="cuda", generator=gen).to(dtype)
    bq = torch.randn(G * d, device="cuda", generator=gen).to(dtype)
    bkn = torch.randn(d, device="cuda", generator=gen).to(dtype)
    bvn = torch.randn(d, device="cuda", generator=gen).to(dtype)
    for r in copies:
        s_ = int(slot_ids[r])
        kc[s_, :, :P] = bk[:P]
        vc[s_, :, :P] = bv[:P]
        qkv[r, :nh * d] = bq.repeat(nkv)
        qkv[r, nh * d:(nh + nkv) * d] = bkn.repeat(nkv)
        qkv[r, (nh + nkv) * d:] = bvn.repeat(nkv)
    inv = _inv_freq(d)
    slot_t = slot_ids.to(device="cuda", dtype=torch.int32)
    pos_t = poses.to(device="cuda", dtype=torch.int32)
    out = ops.decode_attn(qkv, kc, vc, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5)

    # alone: one row, one slot, the same cache rows 0 .. P-1
    kc1 = torch.randn(1, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    vc1 = torch.randn(1, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    kc1[0, :, :P] = bk[:P]
    vc1[0, :, :P] = bv[:P]
    zero = torch.zeros(1, dtype=torch.int32, device="cuda")
    out1 = ops.decode_attn(qkv[copies[0]:copies[0] + 1].clone(), kc1, vc1, zero, zero + P, inv, nh, nkv, d, d ** -0.5)
    torch.cuda.synchronize()

    ref = out1[0, :G * d]
    for r in copies:
        s_ = int(slot_ids[r])
        for kvh in range(nkv):
            where = f"row {r} kv head {kvh} (pos {P})"
            assert torch.equal(out[r, kvh * G * d:(kvh + 1) * G * d], ref), f"{where}: output bits differ"
            assert torch.equal(kc[s_, kvh, :P + 1], kc1[0, 0, :P + 1]), f"{where}: K cache differs"
            assert torch.equal(vc[s_, kvh, :P + 1], vc1[0, 0, :P + 1]), f"{where}: V cache differs"


@gpu
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("d,G", [(80, 4), (64, 2), (128, 8)])
def test_s_max_does_not_change_bits(built_lib, dtype, d, G):
    """The same cache rows held in a 256-row and in a 1536-row cache (the rest filled with other values) give the same
    outputs and appended rows."""
    from surya_b200 import ops

    nkv, B = 2, 10
    nh = G * nkv
    gen = torch.Generator(device="cuda").manual_seed(d + G)
    poses = [0, 1, 31, 32, 33, 127, 128, 129, 200, 255]
    slot_ids = torch.randperm(B, generator=torch.Generator().manual_seed(5))
    kc = torch.randn(B, nkv, 256, d, device="cuda", generator=gen).to(dtype)
    vc = torch.randn(B, nkv, 256, d, device="cuda", generator=gen).to(dtype)
    kl = torch.randn(B, nkv, 1536, d, device="cuda", generator=gen).to(dtype)
    vl = torch.randn(B, nkv, 1536, d, device="cuda", generator=gen).to(dtype)
    kl[:, :, :256] = kc
    vl[:, :, :256] = vc
    qkv = torch.randn(B, _qkv_width(nh, nkv, d), device="cuda", generator=gen).to(dtype)
    inv = _inv_freq(d)
    slot_t = slot_ids.to(device="cuda", dtype=torch.int32)
    pos_t = torch.tensor(poses, device="cuda", dtype=torch.int32)
    out = ops.decode_attn(qkv, kc, vc, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5)
    outl = ops.decode_attn(qkv, kl, vl, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5)
    torch.cuda.synchronize()
    assert torch.equal(out, outl), "s_max changed the output bits"
    assert torch.equal(kc, kl[:, :, :256]) and torch.equal(vc, vl[:, :, :256]), "s_max changed the appended rows"


@gpu
@pytest.mark.parametrize("dtype", DT)
def test_graph_replay_matches_eager(built_lib, dtype):
    """decode_attn captured in a CUDA graph and replayed gives the output and cache bits of an eager launch."""
    from surya_b200 import ops

    d, G, nkv, s_max, B = 80, 4, 4, 256, 64
    nh = G * nkv
    gen = torch.Generator(device="cuda").manual_seed(11)
    kc = torch.randn(B, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    vc = torch.randn(B, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    qkv = torch.randn(B, _qkv_width(nh, nkv, d), device="cuda", generator=gen).to(dtype)
    inv = _inv_freq(d)
    slot_t = torch.randperm(B, generator=torch.Generator().manual_seed(3)).to(device="cuda", dtype=torch.int32)
    pos_t = torch.randint(0, s_max, (B,), generator=torch.Generator().manual_seed(4)).to(device="cuda", dtype=torch.int32)
    kg_, vg_ = kc.clone(), vc.clone()
    out = ops.decode_attn(qkv, kc, vc, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5)
    outg = torch.full_like(out, float("nan"))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.decode_attn(qkv, kg_, vg_, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5, out=outg)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, outg), "graph replay output differs from the eager launch"
    assert torch.equal(kc, kg_) and torch.equal(vc, vg_), "graph replay cache differs from the eager launch"


@gpu
@pytest.mark.parametrize("dtype", DT)
def test_bench_shape_float64(built_lib, record_property, dtype):
    """B = 256 rows at ragged positions 46 .. 172 with head_dim 80, 16 query heads over 4 KV heads and s_max = 256 (the
    recognition benchmark's decode step): every (row, KV head) passes checks (a) and (b)."""
    from surya_b200 import ops

    d, G, nkv, s_max, B = 80, 4, 4, 256, 256
    nh = G * nkv
    gen = torch.Generator(device="cuda").manual_seed(17)
    kc = torch.randn(B, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    vc = torch.randn(B, nkv, s_max, d, device="cuda", generator=gen).to(dtype)
    qkv = torch.randn(B, _qkv_width(nh, nkv, d), device="cuda", generator=gen).to(dtype)
    inv = _inv_freq(d)
    slot_ids = torch.randperm(B, generator=torch.Generator().manual_seed(18))
    poses = torch.randint(46, 173, (B,), generator=torch.Generator().manual_seed(19))
    slot_t = slot_ids.to(device="cuda", dtype=torch.int32)
    pos_t = poses.to(device="cuda", dtype=torch.int32)
    raw = qkv.clone()
    out = ops.decode_attn(qkv, kc, vc, slot_t, pos_t, inv, nh, nkv, d, d ** -0.5)
    # the rotated q the kernel used: rope_kv_append on the same rows (its own cache copies)
    rot = raw.clone()
    ops.rope_kv_append_(rot, pos_t, slot_t, inv, kc.clone(), vc.clone(), nh, nkv, d)
    torch.cuda.synchronize()

    stats = BitStats(dtype)
    qr = rot[:, :nh * d].double().reshape(B, nh, d).cpu()
    kcc, vcc, outc = kc.cpu(), vc.cpu(), out.cpu()
    for b in range(B):
        s_, p_ = int(slot_ids[b]), int(poses[b])
        for kvh in range(nkv):
            qq = qr[b, kvh * G:(kvh + 1) * G]
            kk, vv = kcc[s_, kvh, :p_ + 1].double(), vcc[s_, kvh, :p_ + 1].double()
            got = outc[b, kvh * G * d:(kvh + 1) * G * d].reshape(G, d)
            what = f"decode_attn row {b} (pos {p_}) kv head {kvh}"
            O, A, info = _exact(qq, kk, vv, d ** -0.5, torch.ones(G, p_ + 1, dtype=torch.bool))
            _check_a(got, O, A, info, d, dtype, what)
            y, flips = decode_rounding_ref(qq, kk, vv, d ** -0.5, dtype)
            _check_b(got, y, flips, A, info, d, dtype, stats, what)
    stats.check("decode_attn bench shape", record_property)
