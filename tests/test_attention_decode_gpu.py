"""BlocksparseTransformer.attention_decode (csrc/tc_bst_decode.cuh) on the GPU: elementwise against the float64 decode
reference, the valid-key rule with NaN / Inf in the cache, bad positions, determinism across n and batch, a generation
loop against attention(), CUDA graph / stream / thread / second-GPU replays, and a cache past 2^31 elements."""
import collections
import threading

import numpy as np
import pytest
import torch

from tests._util import EPS32, MMA_C, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, assert_within
from tests._decode_oracle import oracle_decode, oracle_rows
from tests.golden.make_golden import causal_callback
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

BF16, F16 = torch.bfloat16, torch.float16
_NAME = {BF16: "bfloat16", F16: "float16"}
SPLIT = 4


def _tril(n):
    return np.tril(np.ones((n, n), np.int32))


def _per_head(lay, heads):
    return np.stack([np.roll(lay, h, axis=0) for h in range(heads)])


def _per_head_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    q, k = np.indices(blk_shape)
    m = ((q + 2 * k + head_idx) % 3) != 0
    if head_idx == 1 and qry_idx == 0:
        m[5, :] = False
    return m


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks; row 3 of query block 1 sees no key at all"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


def _ones_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    return np.ones(blk_shape, dtype=bool)


def _rect():
    lay = np.zeros((6, 9), np.int32)
    for q in range(6):
        lay[q, q % 3::1 + q % 2] = 1
        lay[q, 8] = 1
    return lay


def _hole(lay, q):
    lay = lay.copy()
    lay[..., q, :] = 0
    return lay


def _future_first(n):
    lay = _tril(n)
    lay[0, 0], lay[0, 1] = 0, 1
    return lay


Case = collections.namedtuple("Case", "name lay bs cb ak hs scale n positions")
CASES = [
    Case("tril12-bs16-hs16-n1", _tril(12), 16, causal_callback, None, 16, 0.25, 1, [5, 100, 191]),
    Case("tril10-bs32-hs64-nbs", _tril(10), 32, causal_callback, None, 64, 0.125, 32, [0, 288, 64]),
    Case("cfg3-bs64-hs128-straddle", local_strided_layout(16), 64, causal_callback, None, 128, 0.125, 16, [56, 1000, 500]),
    Case("cfg3-bs64-hs64-ak", local_strided_layout(16), 64, causal_callback, 300, 64, 0.125, 3, [280, 1021, 62]),
    Case("tril24-bs16-hs256-long", _tril(24), 16, causal_callback, None, 256, 0.0625, 16, [360, 300, 8]),
    Case("perhead-bs64-hs48-ak", _per_head(_tril(7), 3), 64, _per_head_cb, 130, 48, -0.125, 8, [100, 440, 0]),
    Case("rect-bs32-hs96-nomask", _rect(), 32, None, None, 96, 0.125, 5, [10, 187, 95]),
    Case("hole-bs64-hs64-hiderow", _hole(_tril(6), 2), 64, _hide_row_cb, None, 64, 0.125, 64, [64, 128, 0]),
    Case("future-bs64-hs32-ak0", _future_first(5), 64, _ones_cb, 0, 32, 0.125, 4, [0, 200, 60]),
    Case("tril8-bs32-hs208-perhead", _per_head(_tril(8), 3), 32, causal_callback, None, 208, 0.125, 20, [30, 236, 100]),
]
HEADS = 3


def _setup(case, dtype, seed=0, batch=None):
    bst = BlocksparseTransformer(case.lay, case.bs, heads=HEADS, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, case.bs, heads=HEADS, mask_callback=case.cb)
    batch = batch or len(case.positions)
    rng = np.random.default_rng(seed)
    S = HEADS * case.hs
    ctx_k = bst.ctx_blks_k * case.bs
    q = rng.normal(0, 1, (batch, case.n, S))
    k, v = (rng.normal(0, 1, (batch, ctx_k, S)) for _ in range(2))
    q, k, v = (torch.as_tensor(a.astype(np.float32)).to(dtype).cuda() for a in (q, k, v))
    return bst, orc, q, k, v


def decode_bound(ref, A, qk, nent, scale, hs, bs, dtype, vmax):
    """Largest |got - ref| of the decode kernels, elementwise, built like test_bst_attention_gpu.attention_bound with
    A = P |V|, qk the largest |q|.|k| of the row's valid keys and nent its LUT entries:
      * one output rounding u_out |ref|; the probabilities enter P V rounded to the input dtype: u_in A;
      * S = Q K^T accumulates hs products per score (mma.sync, MMA_C eps32 each), which moves the exponent by that much
        times |scale| qk and O by twice it: 2 MMA_C eps32 hs |scale| qk A;
      * exponent arithmetic in the kernel (scale, running max, log2 e) and in the combine (m_s - M): 24 eps32 amax A;
      * P V accumulates bs products per entry: MMA_C eps32 bs nent A; rescales, sums of l, exp2f, reciprocal and
        multiply: eps32 (16 nent + 64) A;
      * the combine of ceil(nent / 4) partials: one exp2f (2 ulp), one product and one sum each for O and l:
        eps32 (8 ns + 8) A;
      * subnormal floors: per key of the probabilities, and the output's."""
    u_in = U_OUT[_NAME[dtype]]
    amax = abs(scale) * qk
    ns = np.ceil(nent / SPLIT)
    rel = u_in + EPS32 * (2 * MMA_C * hs * abs(scale) * qk + 24 * amax + MMA_C * bs * nent + 16 * nent + 64
                          + 8 * ns + 8)
    floor = SUBNORMAL_FLOOR[_NAME[dtype]]
    return u_in * np.abs(ref) + rel * A + floor * bs * nent * vmax + floor


def _decode(bst, q, k, v, positions, case):
    pos = torch.tensor(positions, dtype=torch.int32, device=q.device)
    return _on_poisoned_output(lambda: bst.attention_decode(q, k, v, pos, scale=case.scale, autoregress_at_key=case.ak))


def _check(bst, orc, case, q, k, v, positions, dtype, out):
    rows_of, visible = oracle_rows(orc)
    npf = lambda t: t.float().cpu().numpy()
    ref, A, qk, nent = oracle_decode(rows_of, visible, case.bs, HEADS, bst.ctx_blks_q * case.bs, npf(q), npf(k),
                                     npf(v), positions, case.scale, case.ak)
    bound = decode_bound(ref, A, qk, nent, case.scale, case.hs, case.bs, dtype, float(v.float().abs().max()))
    assert_within(out, ref, bound, "%s %s" % (case.name, dtype))


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c.name for c in CASES])
def test_decode_matches_oracle(idx, dtype):
    case = CASES[idx]
    bst, orc, q, k, v = _setup(case, dtype, seed=idx)
    out = _decode(bst, q, k, v, case.positions, case)
    assert _lib.last_kernel() == "bst_attention_decode_combine"
    assert out.dtype == dtype and tuple(out.shape) == tuple(q.shape) and not out.requires_grad
    _check(bst, orc, case, q, k, v, case.positions, dtype, out)
    # q with other strides: the same rows
    qt = q.transpose(0, 1).contiguous().transpose(0, 1)
    assert torch.equal(_decode(bst, qt, k, v, case.positions, case), out)
    assert _lib.device_error() == 0


def _poison_invalid(k, positions, n, fill):
    k = k.clone()
    for b, p in enumerate(positions):
        k[b, max(p + n, 0):] = fill
    return k


@pytest.mark.parametrize("idx", [2, 6, 7], ids=[CASES[i].name for i in (2, 6, 7)])
def test_invalid_cache_rows_never_reach_the_output(idx):
    case = CASES[idx]
    bst, _, q, k, v = _setup(case, F16, seed=100 + idx)
    garbage = _decode(bst, q, _poison_invalid(k, case.positions, case.n, 7.0),
                      _poison_invalid(v, case.positions, case.n, -3.0), case.positions, case)
    for fill in (float("nan"), float("inf"), float("-inf")):
        got = _decode(bst, q, _poison_invalid(k, case.positions, case.n, fill),
                      _poison_invalid(v, case.positions, case.n, fill), case.positions, case)
        assert torch.equal(got, garbage), fill
    assert not torch.isnan(garbage).any()


def test_bad_positions_give_nan_rows_of_that_entry_only():
    case = CASES[2]
    bst, _, q, k, v = _setup(case, BF16, seed=7)
    ctx_q = bst.ctx_blks_q * case.bs
    good = [56, 1000, 500]
    ref = _decode(bst, q, k, v, good, case)
    for bad in ([-1, 1000, 500], [56, ctx_q - case.n + 1, 500], [56, 1000, 2 ** 31 - 1], [-2 ** 31, 1000, 500]):
        got = _decode(bst, q, k, v, bad, case)
        for b in range(3):
            if bad[b] == good[b]:
                assert torch.equal(got[b], ref[b]), (bad, b)
            else:
                assert torch.isnan(got[b]).all(), (bad, b)
        assert _lib.device_error() == 0


@pytest.mark.parametrize("bs", [16, 32, 64])
def test_row_bits_do_not_depend_on_n_batch_or_other_rows(bs):
    case = Case("det", local_strided_layout(24), bs, causal_callback, None, 64, 0.125, bs, None)
    bst, _, q, k, v = _setup(case._replace(positions=[0, 0, 0, 0]), F16, seed=bs)
    ctx = bst.ctx_blks_q * bs
    positions = [ctx - bs, 3 * bs - 5, 7, ctx - 2 * bs + 3]
    a = _decode(bst, q, k, v, positions, case)
    assert torch.equal(a, _decode(bst, q, k, v, positions, case))
    for b in (0, 3):
        for i in (0, bs // 2, bs - 1):
            row = _decode(bst, q[b:b + 1, i:i + 1], k[b:b + 1], v[b:b + 1], [positions[b] + i], case)
            assert torch.equal(row[0, 0], a[b, i]), (b, i)
            chunk = _decode(bst, q[b:b + 1, i:], k[b:b + 1], v[b:b + 1], [positions[b] + i], case)
            assert torch.equal(chunk[0], a[b, i:]), (b, i)


@pytest.mark.parametrize("bs", [32, 64])
def test_generation_loop_follows_attention(bs):
    """Prefill the cache, then decode token by token, writing each step's key and value first; every row stays within
    the bounds of attention()'s row over the full context."""
    heads, hs, batch, dtype = 2, 64, 2, F16
    lay = local_strided_layout(8)
    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal_callback)
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    ctx, S = 8 * bs, heads * hs
    rng = np.random.default_rng(bs)
    q, k, v = (torch.as_tensor(rng.normal(0, 1, (batch, ctx, S)).astype(np.float32)).to(dtype).cuda() for _ in range(3))
    full = bst.attention(q, k, v, scale=0.125)
    kc, vc = torch.zeros_like(k), torch.zeros_like(v)
    prefill = 3 * bs - 5
    kc[:, :prefill], vc[:, :prefill] = k[:, :prefill], v[:, :prefill]
    pos = torch.full((batch,), prefill, dtype=torch.int32, device="cuda")
    outs = []
    for t in range(prefill, ctx):
        kc[:, t], vc[:, t] = k[:, t], v[:, t]
        outs.append(bst.attention_decode(q[:, t:t + 1], kc, vc, pos, scale=0.125))
        pos.add_(1)
    got = torch.cat(outs, dim=1)
    npf = lambda t: t.float().cpu().numpy()
    rows_of, visible = oracle_rows(orc)
    Q = npf(q[:, prefill:])
    ref = np.zeros(Q.shape)
    A, qk, nent = np.zeros(Q.shape), np.zeros(Q.shape), np.zeros(Q.shape)
    for j in range(Q.shape[1]):
        r, a_, m_, e_ = oracle_decode(rows_of, visible, bs, heads, ctx, Q[:, j:j + 1], npf(k), npf(v),
                                      [prefill + j] * batch, 0.125)
        ref[:, j:j + 1], A[:, j:j + 1], qk[:, j:j + 1], nent[:, j:j + 1] = r, a_, m_, e_
    bound = decode_bound(ref, A, qk, nent, 0.125, hs, bs, dtype, float(v.float().abs().max()))
    assert_within(got, ref, bound, "decode loop bs %d" % bs)
    # attention() at bs 64 is the fused kernel; below it the three-op chain, whose scores are rounded to bfloat16
    # (relative 2^-9 of up to amax, doubled through P and its normalisation) and probabilities to fp16
    chain = 0.0 if bs == 64 else (2.0 ** -8 * 0.125 * qk + 2.0 ** -10) * A
    assert_within(got, npf(full[:, prefill:]), 2 * bound + chain, "decode loop vs attention() bs %d" % bs)


def _step_fn(bst, q_all, kc, vc, k_all, v_all, pos, out, steps):
    """One decode step with the cache write inside: row positions[b] of every entry is written, decoded, stored."""
    bidx = torch.arange(q_all.shape[0], device=q_all.device)

    def step(j):
        p = pos.long()
        kc.index_put_((bidx, p), k_all[bidx, p])
        vc.index_put_((bidx, p), v_all[bidx, p])
        qrow = q_all[bidx, p].unsqueeze(1)
        out[:, j:j + 1].copy_(bst.attention_decode(qrow, kc, vc, pos, scale=0.125))
        pos.add_(1)
    return step


def _run_loop(device, graph=False, stream=None):
    torch.manual_seed(0)
    heads, hs, batch, bs, steps = 4, 64, 3, 64, 12
    bst = BlocksparseTransformer(local_strided_layout(8), bs, heads=heads, mask_callback=causal_callback)
    ctx, S = 8 * bs, heads * hs
    with torch.cuda.device(device):
        g = torch.Generator(device="cpu").manual_seed(1)
        q, k, v = (torch.randn(batch, ctx, S, generator=g).half().to(device) for _ in range(3))
        start = torch.tensor([100, 250, 300], dtype=torch.int32, device=device)
        kc, vc = torch.zeros_like(k), torch.zeros_like(v)
        kc[:, :100], vc[:, :100] = k[:, :100], v[:, :100]
        kc0, vc0 = kc.clone(), vc.clone()
        pos = start.clone()
        out = torch.empty(batch, steps, S, dtype=torch.float16, device=device)
        step = _step_fn(bst, q, kc, vc, k, v, pos, out, steps)
        s = stream or torch.cuda.current_stream(device)
        with torch.cuda.stream(s):
            if not graph:
                for j in range(steps):
                    step(j)
            else:
                step(0)                                   # warm-up: module load and kernel attributes
                kc.copy_(kc0); vc.copy_(vc0); pos.copy_(start)
                gr = torch.cuda.CUDAGraph()
                side = torch.cuda.Stream(device)
                side.wait_stream(s)
                with torch.cuda.stream(side):
                    with torch.cuda.graph(gr, stream=side):
                        step(0)
                s.wait_stream(side)
                kc.copy_(kc0); vc.copy_(vc0); pos.copy_(start)
                outs = []
                for j in range(steps):
                    gr.replay()
                    outs.append(out[:, :1].clone())
                out = torch.cat(outs, dim=1)
        torch.cuda.synchronize(device)
        return out.cpu()


def test_graph_stream_thread_and_second_gpu_replays_are_bit_identical():
    eager = _run_loop("cuda:0")
    assert not torch.isnan(eager).any()
    assert torch.equal(_run_loop("cuda:0", graph=True), eager)
    assert torch.equal(_run_loop("cuda:0", stream=torch.cuda.Stream("cuda:0")), eager)
    box = {}
    t = threading.Thread(target=lambda: box.setdefault("out", _run_loop("cuda:0")))
    t.start()
    t.join()
    assert torch.equal(box["out"], eager)
    assert _lib.device_error() == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_second_gpu_is_bit_identical():
    assert torch.equal(_run_loop("cuda:1"), _run_loop("cuda:0"))


def test_cache_past_2_31_elements():
    """batch 2 x 4097 blocks of 64 rows x 4096 columns: 2^31 + 2^19 elements per cache. Rows of the last entry read
    keys at element offsets past 2^31."""
    heads, hs, bs, batch, nb = 16, 256, 64, 2, 4097
    S, ctx = heads * hs, nb * bs
    free, _ = torch.cuda.mem_get_info()
    need = 2 * batch * ctx * S * 2 + (1 << 30)
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, free / 2 ** 30))
    assert batch * ctx * S > 2 ** 31
    lay = np.eye(nb, dtype=np.int32)
    lay[:, 0] = 1                                         # rows of two entries: block 0 and the diagonal
    bst = BlocksparseTransformer(lay, bs, heads=heads)
    g = torch.Generator(device="cuda").manual_seed(3)
    k = torch.empty(batch, ctx, S, dtype=BF16, device="cuda").normal_(generator=g)
    v = torch.empty(batch, ctx, S, dtype=BF16, device="cuda").normal_(generator=g)
    n = 4
    positions = [ctx // 2, ctx - n]
    q = torch.randn(batch, n, S, generator=torch.Generator().manual_seed(4)).to(BF16).cuda()
    out = _decode(bst, q, k, v, positions, Case("big", lay, bs, None, None, hs, 0.0625, n, positions))
    b, pos = 1, positions[1]
    L = pos + n
    keys = np.concatenate([np.arange(0, bs), np.arange((L - 1) // bs * bs, L)])
    Kb = k[b, keys].double().cpu().numpy()
    Vb = v[b, keys].double().cpu().numpy()
    Q = q[b].double().cpu().numpy()
    ref, A, qk = (np.zeros((n, S)) for _ in range(3))
    for h in range(heads):
        c = slice(h * hs, (h + 1) * hs)
        s = Q[:, c] @ Kb[:, c].T * 0.0625
        p = np.exp(s - s.max(axis=1, keepdims=True))
        p /= p.sum(axis=1, keepdims=True)
        ref[:, c], A[:, c] = p @ Vb[:, c], p @ np.abs(Vb[:, c])
        qk[:, c] = (np.abs(Q[:, c]) @ np.abs(Kb[:, c]).T).max(axis=1, keepdims=True)
    bound = decode_bound(ref, A, qk, np.full(ref.shape, 2.0), 0.0625, hs, bs, BF16, float(np.abs(Vb).max()))
    assert_within(out[b], ref, bound, "cache past 2^31 elements")
    assert _lib.device_error() == 0
