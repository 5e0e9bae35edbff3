"""BlocksparseTransformer.attention and attention_decode with kv_heads < heads (grouped-query attention): the fused
forward and dq bit for bit against the same op on k and v expanded to heads heads, the grouped dk and dv elementwise
against float64, the default backward and the fallback bit for bit against the chain on expanded k and v, what
autograd keeps, zero gradients of key blocks no head of a group sees, and the decode bit for bit against
attention_decode on expanded caches, in CUDA graphs, on side streams and past 2^31 cache elements."""
import collections

import numpy as np
import pytest
import torch

from tests._util import _on_poisoned_output, assert_within
from tests.golden.make_golden import causal_callback
from tests.test_bst_attention_bwd_gpu import _key_hole, grad_bound
from tests.test_bst_attention_dropout_gpu import dropout_grad_bound
from tests.test_bst_attention_gpu import _per_head, _per_head_cb, _tril
from tests._attention_dropout_oracle import attention_keep
from tests._gqa_oracle import sum_groups
from blocksparse_b200 import BlocksparseTransformer, _lib, ewops
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
BS = 64
HEADS, BATCH = 8, 2
SEED, CALL = 0x0F1E_2D3C_4B5A_6978, 17


def _state():
    return torch.tensor([SEED, CALL], dtype=torch.int64, device="cuda")


def _expand(x, kv, heads=HEADS):
    """k or v of kv heads -> heads heads, query head h reading kv head h // (heads // kv) (repeat_interleave)"""
    B, C, S = x.shape
    hs = S // kv
    return x.reshape(B, C, kv, 1, hs).expand(B, C, kv, heads // kv, hs).reshape(B, C, heads * hs)


Case = collections.namedtuple("Case", "name lay cb ak hs scale")
CASES = [
    Case("strided8-causal", local_strided_layout(8), causal_callback, None, 64, 0.125),
    Case("tril6-causal-ak", _tril(6), causal_callback, 130, 128, 0.125),
    Case("perhead-mask", _per_head(_tril(6), HEADS), _per_head_cb, None, 128, -0.25),
    Case("perhead-keyhole-ak", _per_head(_key_hole(_tril(6), 2), HEADS), causal_callback, 200, 64, 0.125),
]


def _inputs(lay, hs, dtype, seed, kv, heads=HEADS, batch=BATCH):
    lay3 = lay if lay.ndim == 3 else lay[None]
    cq, ck = lay3.shape[1:]
    rng = np.random.default_rng(seed)
    q, dy = (rng.normal(0, 1, (batch, cq * BS, heads * hs)) for _ in range(2))
    k, v = (rng.normal(0, 1, (batch, ck * BS, kv * hs)) for _ in range(2))
    return [torch.as_tensor(a.astype(np.float32)).to(dtype).cuda() for a in (q, k, v, dy)]


def _run(bst, q, k, v, dy, scale, ak, fused_backward, kp, kv):
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    y = bst.attention(*ins, scale=scale, autoregress_at_key=ak, fused_backward=fused_backward, keep_prob=kp,
                      dropout_state=_state() if kp < 1 else None, kv_heads=kv)
    y.backward(dy)
    return y, [t.grad for t in ins]


class _GroupRows:
    """A TransformerOracle whose tn_lut rows count every entry of a group of g heads: the grouped dk / dv accumulate
    that many entries (the bounds read the longest row)."""

    def __init__(self, orc, g):
        self._orc, self.tn_list = orc, [[r * g for r in rows] for rows in orc.tn_list]

    def __getattr__(self, name):
        return getattr(self._orc, name)


# ---- fused forward and backward ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv", [4, 2, 1])
@pytest.mark.parametrize("kp", [1.0, 0.9])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c.name for c in CASES])
def test_fused_matches_expanded_and_float64(idx, dtype, kp, kv):
    case = CASES[idx]
    g = HEADS // kv
    bst = BlocksparseTransformer(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    q, k, v, dy = _inputs(case.lay, case.hs, dtype, 100 + idx, kv)
    y, (dq, dk, dv) = _run(bst, q, k, v, dy, case.scale, case.ak, True, kp, kv)
    assert _lib.device_error() == 0, _lib.device_error_text()
    kx, vx = _expand(k, kv), _expand(v, kv)
    y_x, (dq_x, _, _) = _run(bst, q, kx, vx, dy, case.scale, case.ak, True, kp, None)
    assert torch.equal(y, y_x), "forward differs from attention on expanded k, v"
    assert torch.equal(dq, dq_x), "dq differs from the fused backward on expanded k, v"
    assert dk.shape == k.shape and dv.shape == v.shape
    orc = _GroupRows(TransformerOracle(case.lay, BS, heads=HEADS, mask_callback=case.cb), g)
    Q, Kx, Vx, dY = (t.double().cpu().numpy() for t in (q, kx, vx, dy))
    if kp == 1.0:
        refs, bounds = grad_bound(orc, Q, Kx, Vx, dY, case.scale, case.ak, case.hs, dtype)
    else:
        Z = attention_keep(orc, BATCH, SEED, CALL, kp)
        refs, bounds = dropout_grad_bound(orc, Q, Kx, Vx, dY, Z, kp, case.scale, case.ak, case.hs, dtype)
    for name, got, ref, bound in (("dk", dk, refs[1], bounds[1]), ("dv", dv, refs[2], bounds[2])):
        assert not bool(torch.isnan(got).any()), name
        assert_within(got, sum_groups(ref, HEADS, kv), sum_groups(bound, HEADS, kv),
                      "%s %s kv %d kp %g" % (name, case.name, kv, kp))
    # deterministic: a second backward gives the same bits
    _, again = _run(bst, q, k, v, dy, case.scale, case.ak, True, kp, kv)
    for a, b in zip((dq, dk, dv), again):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kp", [1.0, 0.9])
@pytest.mark.parametrize("hs,dtype", [(64, F16), (128, BF16)], ids=["hs64-fp16", "hs128-bf16"])
def test_entries_at_group_one_are_the_multi_head_kernels(hs, dtype, kp):
    """kv_heads == heads through the GQA entries gives the multi-head entries' bits."""
    case = CASES[2]
    bst = BlocksparseTransformer(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    q, k, v, dy = _inputs(case.lay, hs, dtype, 7, HEADS)
    st = _state() if kp < 1 else None
    a = bst._attention_train(q, k, v, 0.125, None, kp, st, HEADS)
    b = bst._attention_train(q, k, v, 0.125, None, kp, st)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    o, m, l = b
    ga = bst._attention_grad(q, k, v, o, dy, m, l, 0.125, None, kp, st, HEADS)
    gb = bst._attention_grad(q, k, v, o, dy, m, l, 0.125, None, kp, st)
    for x, y in zip(ga, gb):
        assert torch.equal(x, y)
    assert torch.equal(bst._attention(q, k, v, 0.125, None, kp, st, HEADS), bst._attention(q, k, v, 0.125, None, kp, st))


def _chain(bst, q, k, v, scale, ak, kp):
    p = bst.masked_softmax(bst.query_key_op(q, k), scale, ak)
    if kp < 1:
        p, _ = ewops.dropout(p, kp, mask=ewops._mask_at(p, p.numel(), kp, _state()))
    return bst.weight_value_op(p, v)


def _chain_grads(bst, q, k, v, dy, scale, ak, kp, kv):
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    y = _chain(bst, ins[0], _expand(ins[1], kv), _expand(ins[2], kv), scale, ak, kp)
    y.backward(dy)
    return y, [t.grad for t in ins]


@pytest.mark.parametrize("kv", [4, 1])
@pytest.mark.parametrize("kp", [1.0, 0.9])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", [1, 2], ids=[CASES[1].name, CASES[2].name])
def test_default_backward_is_the_chain_on_expanded_kv(idx, dtype, kp, kv):
    case = CASES[idx]
    bst = BlocksparseTransformer(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    q, k, v, dy = _inputs(case.lay, case.hs, dtype, 30 + idx, kv)
    _, got = _run(bst, q, k, v, dy, case.scale, case.ak, False, kp, kv)
    _, want = _chain_grads(bst, q, k, v, dy, case.scale, case.ak, kp, kv)
    assert _lib.device_error() == 0, _lib.device_error_text()
    for name, a, b in zip("qkv", got, want):
        assert a.shape == b.shape and torch.equal(a, b), "d%s differs from the chain on expanded k, v" % name


@pytest.mark.parametrize("fused_backward", [False, True])
@pytest.mark.parametrize("kp", [1.0, 0.9])
@pytest.mark.parametrize("dtype,bs,hs", [(F32, 64, 64), (F16, 32, 64), (BF16, 64, 32)], ids=["fp32", "bs32", "hs32"])
def test_fallback_is_the_chain_on_expanded_kv(dtype, bs, hs, kp, fused_backward):
    lay = _tril(4)
    bst = BlocksparseTransformer(lay, bs, heads=4, mask_callback=causal_callback)
    rng = np.random.default_rng(5)
    q, dy = (torch.as_tensor(rng.normal(0, 1, (2, 4 * bs, 4 * hs)).astype(np.float32)).to(dtype).cuda() for _ in range(2))
    k, v = (torch.as_tensor(rng.normal(0, 1, (2, 4 * bs, 2 * hs)).astype(np.float32)).to(dtype).cuda() for _ in range(2))
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    y = bst.attention(*ins, scale=0.25, autoregress_at_key=70, fused_backward=fused_backward, keep_prob=kp,
                      dropout_state=_state() if kp < 1 else None, kv_heads=2)
    y.backward(dy)
    ref = [t.clone().requires_grad_() for t in (q, k, v)]
    want = _chain(bst, ref[0], _expand(ref[1], 2, 4), _expand(ref[2], 2, 4), 0.25, 70, kp)
    want.backward(dy)
    assert torch.equal(y, want)
    for a, b in zip(ins, ref):
        assert torch.equal(a.grad, b.grad)


@pytest.mark.parametrize("fused_backward", [False, True])
def test_autograd_saves_kv_at_kv_head_size(fused_backward):
    case = CASES[0]
    bst = BlocksparseTransformer(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    q, k, v, dy = _inputs(case.lay, case.hs, F16, 11, 2)
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    shapes = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: shapes.append(tuple(t.shape)) or t, lambda t: t):
        y = bst.attention(qq, kk, vv, scale=0.125, fused_backward=fused_backward, kv_heads=2)
    sparse = (BATCH, HEADS, bst.blocks, BS, BS)
    assert sparse not in shapes, shapes
    assert shapes.count(tuple(k.shape)) == 2, shapes           # k and v, at kv-head size; nothing expanded
    assert len(shapes) == (6 if fused_backward else 3), shapes
    y.backward(dy)
    assert kk.grad.shape == k.shape and vv.grad.shape == v.shape


def test_key_blocks_no_head_of_a_group_sees_are_zero_on_poisoned_memory():
    """Key block 2 is seen by no head; key block 4 by heads 1.. of each group only (per-head layouts): every element is
    written, and the unseen block is exactly zero."""
    head0 = _key_hole(_key_hole(_tril(6), 2), 5)
    head0[5, 0] = 0                                            # 15 blocks in every head, as per-head layouts need
    lay = np.stack([head0] + [_key_hole(_key_hole(_tril(6), 2), 4)] * (HEADS - 1))
    assert len({int(x.sum()) for x in lay}) == 1
    bst = BlocksparseTransformer(lay, BS, heads=HEADS, mask_callback=causal_callback)
    q, k, v, dy = _inputs(lay, 64, BF16, 5, 2)

    def run():
        o, m, l = bst._attention_train(q, k, v, 0.125, None, 1.0, None, 2)
        return bst._attention_grad(q, k, v, o, dy, m, l, 0.125, None, 1.0, None, 2)
    dq, dk, dv = _on_poisoned_output(run)
    assert _lib.device_error() == 0, _lib.device_error_text()
    for t in (dq, dk, dv):
        assert not bool(torch.isnan(t).any())
    assert bool((dk[:, 2 * BS:3 * BS] == 0).all()) and bool((dv[:, 2 * BS:3 * BS] == 0).all())
    assert bool((dk[:, 4 * BS:5 * BS, :64] != 0).any())        # kv head 0's group: only head 0 sees block 4
    assert bool((dk[:, 4 * BS:5 * BS, 64:] == 0).all()) and bool((dv[:, 4 * BS:5 * BS, 64:] == 0).all())


# ---- decode -------------------------------------------------------------------------------------------------------
DCase = collections.namedtuple("DCase", "name lay cb ak hs")
DCASES = [
    DCase("strided8-causal", local_strided_layout(8), causal_callback, None, 64),
    DCase("tril8-causal-ak-hs128", _tril(8), causal_callback, 300, 128),
    DCase("perhead-mask", _per_head(_tril(8), HEADS), _per_head_cb, None, 64),
]


def _decode_inputs(bst, bs, hs, n, kv, dtype, seed, batch=3):
    rng = np.random.default_rng(seed)
    ctx = bst.ctx_blks_k * bs
    q = rng.normal(0, 1, (batch, n, HEADS * hs))
    k, v = (rng.normal(0, 1, (batch, ctx, kv * hs)) for _ in range(2))
    return [torch.as_tensor(a.astype(np.float32)).to(dtype).cuda() for a in (q, k, v)]


@pytest.mark.parametrize("kv", [4, 2, 1])
@pytest.mark.parametrize("n", ["1", "5", "bs"])
@pytest.mark.parametrize("bs", [16, 32, 64])
@pytest.mark.parametrize("idx", range(len(DCASES)), ids=[c.name for c in DCASES])
def test_decode_is_attention_decode_on_expanded_caches(idx, bs, n, kv):
    case = DCASES[idx]
    n = bs if n == "bs" else int(n)
    dtype = BF16 if bs == 32 else F16
    bst = BlocksparseTransformer(case.lay, bs, heads=HEADS, mask_callback=case.cb)
    ctx_q = bst.ctx_blks_q * bs
    q, k, v = _decode_inputs(bst, bs, case.hs, n, kv, dtype, bs + n + kv)
    positions = [0, ctx_q - n, (ctx_q // 2 - n // 2) | 3]          # ragged
    positions = [min(max(p, 0), ctx_q - n) for p in positions]
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    # garbage in every cache row past L_b: it must never reach the output
    for b, p in enumerate(positions):
        k[b, p + n:] = float("nan")
        v[b, p + n:] = float("inf")
    got = _on_poisoned_output(lambda: bst.attention_decode(q, k, v, pos, scale=0.125, autoregress_at_key=case.ak,
                                                          kv_heads=kv))
    assert _lib.device_error() == 0, _lib.device_error_text()
    want = bst.attention_decode(q, _expand(k, kv), _expand(v, kv), pos, scale=0.125, autoregress_at_key=case.ak)
    assert not bool(torch.isnan(got).any()) and not bool(torch.isinf(got).any())
    assert torch.equal(got, want)


def test_decode_graph_and_side_stream_are_bit_identical():
    case = DCASES[0]
    bs, n, kv = 64, 1, 2
    bst = BlocksparseTransformer(case.lay, bs, heads=HEADS, mask_callback=case.cb)
    q, k, v = _decode_inputs(bst, bs, case.hs, n, kv, BF16, 9)
    pos = torch.tensor([3, 200, 511], dtype=torch.int32, device="cuda")
    eager = bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv)        # warm-up off the capture
        on_side = bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(on_side, eager)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv)
    for p in ([3, 200, 511], [100, 7, 300]):
        pos.copy_(torch.tensor(p, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv))
    assert _lib.device_error() == 0


def test_decode_cache_past_2_31_elements():
    """batch 8 x 4097 blocks of 64 rows x kv_heads 4 x head_state 256: 2^31 + 2^19 elements per cache. The last entry's
    rows read keys past element 2^31; they equal attention_decode on that entry's expanded cache."""
    heads, kv, hs, bs, batch, nb = 16, 4, 256, 64, 8, 4097
    Skv, ctx = kv * hs, nb * bs
    free, _ = torch.cuda.mem_get_info()
    need = 2 * batch * ctx * Skv * 2 + 2 * ctx * heads * hs * 2 + (1 << 30)
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, free / 2 ** 30))
    assert batch * ctx * Skv > 2 ** 31
    lay = np.eye(nb, dtype=np.int32)
    lay[:, 0] = 1
    bst = BlocksparseTransformer(lay, bs, heads=heads)
    gen = torch.Generator(device="cuda").manual_seed(3)
    k = torch.empty(batch, ctx, Skv, dtype=BF16, device="cuda").normal_(generator=gen)
    v = torch.empty(batch, ctx, Skv, dtype=BF16, device="cuda").normal_(generator=gen)
    n = 4
    positions = [ctx // 2] * (batch - 1) + [ctx - n]
    q = torch.randn(batch, n, heads * hs, generator=torch.Generator().manual_seed(4)).to(BF16).cuda()
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    got = bst.attention_decode(q, k, v, pos, scale=0.0625, kv_heads=kv)
    last = pos[-1:].clone()
    want = bst.attention_decode(q[-1:], _expand(k[-1:], kv, heads), _expand(v[-1:], kv, heads), last, scale=0.0625)
    assert torch.equal(got[-1:], want)
    assert _lib.device_error() == 0
