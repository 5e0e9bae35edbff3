"""Every op family outside the eager default-stream setting of the rest of the suite: on a side stream whose inputs are
still being written, in CUDA graphs replayed with new inputs, from two host threads at once and on a second GPU.

The rest of the suite ties each op's eager result on the default stream of cuda:0 to float64. Here that eager result is
the reference and every check is bit for bit: the kernels are deterministic, so a launch on the wrong stream or GPU, a
value frozen into a graph or a per-thread cache that hands out another thread's state shows up as a difference.

Each case is (the public names it covers, make(generator, device) -> inputs, run(*inputs) -> outputs). make draws the
inputs on the host from a seeded generator, so every device gets the same values; run is functional -- it clones what
an op updates in place -- and returns forward outputs and gradients.
"""
import threading
from collections import namedtuple

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import (AdamOptimizer, BlocksparseMatMul, BlocksparseTransformer, ClipGlobalNorm, Ema, SparseProj,
                              _lib, block_reduced_full_dw, blocksparse_l2_decay, blocksparse_norm, blocksparse_prune,
                              blocksparse_reduced_dw, clip_by_global_norm, global_norm, group_param_grads, layer_norm,
                              masked_softmax, masked_top_k_softmax, rectified_top_k, softmax, softmax_cross_entropy,
                              top_k, transpose_0213, transpose_2d)
from blocksparse_b200 import matmul as mm
from blocksparse_b200.layouts import bernoulli_layout

gpu = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
SLEEP_CYCLES = 1 << 22          # torch.cuda._sleep: about 2.5 ms on an H100, long enough to be still running when
                                # the inputs' copies and the op are enqueued behind it


# ---- helpers ----------------------------------------------------------------------------------------------------------
def _rn(g, dev, shape, dtype=F32, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(dev)


def _gate(g, dev, n):
    """fp32 gate with zeros and values other than 1."""
    u = torch.rand(n, generator=g)
    return torch.where(u < 0.3, torch.zeros(()), 0.5 + u).to(dev)


def _leaf(*ts):
    return [t.detach().requires_grad_() for t in ts]


def _grad(outs, ins, douts):
    return list(torch.autograd.grad(outs, ins, douts))


def _bits(t):
    t = t.detach().reshape(-1)
    if t.dtype.is_floating_point:
        t = t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t.cpu()


def _same(got, ref, what):
    """Bit for bit, NaN and signed zeros included."""
    assert len(got) == len(ref), "%s: %d outputs, expected %d" % (what, len(got), len(ref))
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape and a.dtype == b.dtype, "%s: output %d is %s %s, expected %s %s" % (
            what, i, tuple(a.shape), a.dtype, tuple(b.shape), b.dtype)
        ba, bb = _bits(a), _bits(b)
        if not torch.equal(ba, bb):
            raise AssertionError("%s: output %d differs in %d of %d elements" % (what, i, int((ba != bb).sum()), a.numel()))


def _poisoned_like(t):
    """A buffer of t's shape and dtype that no op can mistake for real data: NaN, or the dtype's largest integer."""
    return torch.full_like(t, float("nan") if t.dtype.is_floating_point else torch.iinfo(t.dtype).max)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    m = np.ones(blk_shape, dtype=bool)
    return np.tril(m) if qry_idx == key_idx else m


# ---- the ops, built once: every test reuses them, on every device --------------------------------------------------------
_LAY32 = bernoulli_layout(np.random.default_rng(1), 8, 8, 0.5)
_TRIL4 = np.tril(np.ones((4, 4), np.int32))
BSMM32 = BlocksparseMatMul(_LAY32, block_size=32, feature_axis=1)              # 256 -> 256 features
BSMM32_AX0 = BlocksparseMatMul(_LAY32, block_size=32, feature_axis=0)
BSMM8 = BlocksparseMatMul(bernoulli_layout(np.random.default_rng(2), 8, 8, 0.5), block_size=8, feature_axis=1)
BST = BlocksparseTransformer(_TRIL4, block_size=64, heads=2, mask_callback=causal)   # context 256
SPROJ = SparseProj(96, gather_lut=np.sort(np.random.default_rng(3).choice(96, 40, replace=False)))
assert BSMM8._shadow is not None                                                  # the padded 16 x 16 route

Case = namedtuple("Case", "covers make run capture")
CASES = {}


def case(name, covers, capture=True):
    def register(fns):
        make, run = fns()
        CASES[name] = Case(tuple(covers), make, run, capture)
        return fns
    return register


# ---- block-sparse matmul ------------------------------------------------------------------------------------------------
class _tile(object):
    """Forces the output blocks per CTA of the default 32 x 32 xprop launch (None: the model's choice)."""

    def __init__(self, tile):
        self.tile = tile

    def __enter__(self):
        self.old, mm._XPROP_TILE = mm._XPROP_TILE, self.tile

    def __exit__(self, *exc):
        mm._XPROP_TILE = self.old


def _bsmm_case(bsmm, dtype, N, tile=None, gated=False):
    def make(g, dev):
        ins = [_rn(g, dev, bsmm.i_shape(N), dtype), _rn(g, dev, bsmm.w_shape, dtype, 0.1), _rn(g, dev, bsmm.o_shape(N), dtype)]
        return ins + [_gate(g, dev, bsmm.blocks)] if gated else ins

    def run(x, w, dy, gate=None):
        with _tile(tile):
            if gate is None:
                x, w = _leaf(x, w)
                y = bsmm(x, w)
                return [y] + _grad(y, (x, w), dy)
            x, w, gate = _leaf(x, w, gate)
            y = bsmm(x, w, gate=gate, gate_grad=True)
            return [y] + _grad(y, (x, w, gate), dy)
    return make, run


case("bsmm_bf16_tile1", ["BlocksparseMatMul"])(lambda: _bsmm_case(BSMM32, BF16, 128, tile=1))
case("bsmm_bf16_tile4", ["BlocksparseMatMul"])(lambda: _bsmm_case(BSMM32, BF16, 128, tile=4))
case("bsmm_pad8", ["BlocksparseMatMul"])(lambda: _bsmm_case(BSMM8, BF16, 64))
case("bsmm_gated", ["BlocksparseMatMul"])(lambda: _bsmm_case(BSMM32, BF16, 128, gated=True))
case("bsmm_fp32", ["BlocksparseMatMul"])(lambda: _bsmm_case(BSMM32_AX0, F32, 64))


@case("group_param_grads", ["group_param_grads"])
def _():
    def make(g, dev):
        return [_rn(g, dev, BSMM32.i_shape(64), BF16) for _ in range(3)] + [_rn(g, dev, BSMM32.w_shape, BF16, 0.1)] + \
               [_rn(g, dev, BSMM32.o_shape(64), BF16) for _ in range(3)]

    def run(x1, x2, x3, w, d1, d2, d3):
        xs, (w,) = _leaf(x1, x2, x3), _leaf(w)
        with group_param_grads(BSMM32, w, group_size=2):        # three uses: one pair launch, then one single
            ys = [BSMM32(x, w) for x in xs]
            torch.autograd.backward(ys, [d1, d2, d3])
        return ys + [x.grad for x in xs] + [w.grad]
    return make, run


# ---- weight utilities ---------------------------------------------------------------------------------------------------
@case("l2_normalize", ["BlocksparseMatMul"])
def _():
    def make(g, dev):
        return [_rn(g, dev, BSMM32.w_shape), _rn(g, dev, (BSMM32.K,)), _rn(g, dev, BSMM32.w_shape)]

    def run(w, gain, dy):
        w, gain = _leaf(w, gain)
        y = BSMM32.l2_normalize(w, gain=gain)
        return [y] + _grad(y, (w, gain), dy)
    return make, run


@case("block_norm_decay_prune", ["blocksparse_norm", "blocksparse_l2_decay", "blocksparse_prune"])
def _():
    def make(g, dev):
        return [_rn(g, dev, BSMM32.w_shape), (torch.rand(BSMM32.blocks, generator=g) < 0.7).float().to(dev)]

    def run(w, gate):
        decayed = blocksparse_l2_decay(w.clone(), gate, rate=0.05)
        by_share = blocksparse_prune(w, gate.clone(), step=0, sparsity=0.5)
        by_threshold = blocksparse_prune(w, gate.clone(), step=0, threshold=32.0, norm="l2")
        return [blocksparse_norm(w, "max"), blocksparse_norm(w, "l2"), decayed, by_share, by_threshold]
    return make, run


@case("identity_init", ["BlocksparseMatMul"])
def _():
    def make(g, dev):
        return [torch.zeros(1, device=dev)]                    # names the device only

    def run(t):
        return [BSMM32.identity_init(scale=0.5, dtype=BF16, device=t.device)]
    return make, run


@case("reduced_dw", ["blocksparse_reduced_dw", "block_reduced_full_dw"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (64, 256), BF16) for _ in range(2)] + [_rn(g, dev, (64, 256), BF16) for _ in range(2)]

    def run(x1, x2, d1, d2):
        dw, x_red, y_red = blocksparse_reduced_dw([x1, x2], [d1, d2], 0.5, bsize=32, norm="max", axis=1)
        full = block_reduced_full_dw([(x1, d1), (x2, d2)], scale=0.5, norm="l2", group_size=1, bsize=32, axis=1)
        return [dw, x_red, y_red, full]
    return make, run


@case("sparse_proj", ["SparseProj"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (96, 24), F16), _rn(g, dev, (40, 24), F16), _rn(g, dev, (40, 24), F16)] + \
               [_rn(g, dev, (96, 24), F16) for _ in range(3)]

    def run(x, y, d1, d2, d3, d4):
        x, y = _leaf(x, y)
        outs = [SPROJ.gather(x), SPROJ.scatter(y), SPROJ.scatter_add(x, y), SPROJ.scatter_mul(x, y)]
        return outs + _grad(outs, (x, y), (d1, d2, d3, d4))
    return make, run


# ---- block-sparse transformer ------------------------------------------------------------------------------------------
@case("bst_chain", ["BlocksparseTransformer"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (2, 256, 128), BF16) for _ in range(6)]

    def run(q, k, v, u, dy, dz):
        q, k, v, u = _leaf(q, k, v, u)
        w = BST.nt_op(q, k)
        p = BST.masked_softmax(w, scale=0.125, autoregress_at_key=64)
        y, z = BST.nn_op(p, v), BST.tn_op(p, u)
        mask = BST.partial_autoregressive_mask(64, device=q.device)
        return [w, p, y, z, mask] + _grad((y, z), (q, k, v, u), (dy, dz))
    return make, run


def _attention_case(hs):
    def make(g, dev):
        return [_rn(g, dev, (2, 256, 2 * hs), BF16) for _ in range(4)]

    def run(q, k, v, dy):
        outs = []
        for fused_backward in (False, True):
            qq, kk, vv = _leaf(q, k, v)
            o = BST.attention(qq, kk, vv, scale=0.125, fused_backward=fused_backward)
            outs += [o] + _grad(o, (qq, kk, vv), dy)
        return outs
    return make, run


case("attention_hs64", ["BlocksparseTransformer"])(lambda: _attention_case(64))
case("attention_hs128", ["BlocksparseTransformer"])(lambda: _attention_case(128))


# ---- dense ops --------------------------------------------------------------------------------------------------------
@case("dense_softmax", ["softmax", "masked_softmax"])
def _():
    def make(g, dev):
        mask = (torch.rand((1, 1, 5, 40), generator=g) < 0.7).float().to(dev)
        return [_rn(g, dev, (2, 3, 5, 40), F16), mask, _rn(g, dev, (2, 3, 5, 40), F16), _rn(g, dev, (2, 3, 5, 40), F16)]

    def run(x, mask, d1, d2):
        (x,) = _leaf(x)
        outs = [masked_softmax(x, mask, scale=0.5), softmax(x, scale=2.0)]
        return outs + _grad(outs, (x,), (d1, d2))
    return make, run


@case("top_k", ["masked_top_k_softmax", "top_k", "rectified_top_k"])
def _():
    def make(g, dev):
        mask = (torch.rand((1, 50), generator=g) < 0.8).float().to(dev)
        return [_rn(g, dev, (6, 50)), mask, _rn(g, dev, (6, 50)), _rn(g, dev, (6, 5)), _rn(g, dev, (6, 50)), _rn(g, dev, (6, 50))]

    def run(x, mask, d1, d2, d3, d4):
        (x,) = _leaf(x)
        y = masked_top_k_softmax(x, 5, mask, scale=0.5)
        vals, idx = top_k(x, 5)
        r1, r2 = rectified_top_k(x, 5, rebase=True), rectified_top_k(x, 5, rebase=False)
        return [y, vals, idx, r1, r2] + _grad((y, vals, r1, r2), (x,), (d1, d2, d3, d4))
    return make, run


@case("softmax_cross_entropy", ["softmax_cross_entropy"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (16, 1000), BF16, 3.0), torch.randint(0, 1000, (16,), generator=g).to(dev), _rn(g, dev, (16,))]

    def run(x, labels, dy):
        (x,) = _leaf(x)
        loss = softmax_cross_entropy(x, labels)
        return [loss] + _grad(loss, (x,), dy)
    return make, run


@case("transposes", ["transpose_0213", "transpose_2d"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (2, 3, 5, 8), F16), _rn(g, dev, (2, 5, 3, 8), F16), _rn(g, dev, (33, 47), BF16),
                _rn(g, dev, (47, 33), BF16)]

    def run(a, da, b, db):
        a, b = _leaf(a, b)
        outs = [transpose_0213(a), transpose_2d(b)]
        return outs + _grad(outs, (a, b), (da, db))
    return make, run


@case("layer_norm", ["layer_norm"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (32, 96), BF16), _rn(g, dev, (96,)), _rn(g, dev, (96,)), _rn(g, dev, (32, 96), BF16),
                _rn(g, dev, (96, 48), F16), _rn(g, dev, (96,)), _rn(g, dev, (96,)), _rn(g, dev, (96, 48), F16)]

    def run(x1, g1, b1, d1, x0, g0, b0, d0):
        x1, g1, b1, x0, g0, b0 = _leaf(x1, g1, b1, x0, g0, b0)
        y1, y0 = layer_norm(x1, g1, b1, axis=1), layer_norm(x0, g0, b0, axis=0, relu=True)
        return [y1, y0] + _grad((y1, y0), (x1, g1, b1, x0, g0, b0), (d1, d0))
    return make, run


# ---- optimizer --------------------------------------------------------------------------------------------------------
def _adam_case(zero_init, fp16, gated):
    def make(g, dev):
        return [_rn(g, dev, (16, 32, 32)), _rn(g, dev, (1003,)), _rn(g, dev, (16, 32, 32), BF16, 0.1),
                _rn(g, dev, (1003,), F16, 0.1), _gate(g, dev, 16)]

    def run(p1, p2, g1, g2, gate):
        p1, p2 = p1.clone(), p2.clone()
        p1.gate = gate
        opt = AdamOptimizer([p1, p2], learning_rate=0.01, gated=gated, fp16=fp16, zero_init_variables=zero_init)
        norm, scale = clip_by_global_norm([g1, g2], clip_norm=1.0)
        opt.step(grads=[g1, g2], norm_scale=scale)
        opt.step(grads=[g1, g2])
        return [p1, p2, norm, scale] + [opt.state[p][k] for p in (p1, p2) for k in ("mean", "var")]
    return make, run


case("adam_fp32", ["AdamOptimizer"])(lambda: _adam_case(True, False, False))
case("adam_fp16_gated", ["AdamOptimizer"])(lambda: _adam_case(True, True, True))
# lr_t is formed on the host from beta powers that advance every step: not capturable (test_graph_refuses_adam_...)
case("adam_bias_corrected", ["AdamOptimizer"], capture=False)(lambda: _adam_case(False, False, False))


@case("clip_by_global_norm", ["clip_by_global_norm", "global_norm", "ClipGlobalNorm"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (1000,)), _rn(g, dev, (77,), F16), _rn(g, dev, (5000,), BF16), torch.zeros(0, device=dev)]

    def run(*grads):
        norm, scale = clip_by_global_norm(grads, clip_norm=2.0)
        old_norm, old_scale = ClipGlobalNorm(grads, clip_norm=30.0)
        return [norm, scale, global_norm(grads, grad_scale=0.5), old_norm, old_scale]
    return make, run


@case("ema", ["Ema"])
def _():
    def make(g, dev):
        return [_rn(g, dev, (16, 32, 32)), _rn(g, dev, (1003,)), _rn(g, dev, (16, 32, 32)), _rn(g, dev, (1003,)),
                _gate(g, dev, 16)]

    def run(p1, p2, d1, d2, gate):
        outs = []
        for fp16 in (False, True):
            a, b = p1.clone(), p2.clone()
            a.gate = gate
            ema = Ema(decay=0.9, gated=True, fp16=fp16)
            ema.apply([a, b])
            a.add_(d1)
            b.add_(d2)
            ema.apply([a, b])
            outs += [ema.average(a), ema.average(b)]
        return outs
    return make, run


EXEMPT = {"z_order_2d": "orders a layout on the host and launches nothing",
          "ClipGlobalNorm": "an alias of clip_by_global_norm"}


def test_cases_cover_every_public_name():
    """Every name the package exports has a case here, with the variants each family has to run (pure Python; guards
    later edits of the package or of this file)."""
    covered = set()
    for c in CASES.values():
        covered.update(c.covers)
    missing = [n for n in blocksparse_b200.__all__ if n not in covered and n not in EXEMPT]
    assert not missing, "exported names without a case: %s" % missing
    assert not covered - set(blocksparse_b200.__all__)
    assert {"bsmm_bf16_tile1", "bsmm_bf16_tile4", "bsmm_pad8", "bsmm_gated", "bsmm_fp32", "group_param_grads",
            "l2_normalize", "identity_init", "attention_hs64", "attention_hs128", "adam_fp32", "adam_fp16_gated"} <= set(CASES)
    assert [n for n, c in CASES.items() if not c.capture] == ["adam_bias_corrected"]


# ---- 1. side streams -----------------------------------------------------------------------------------------------------
@gpu
def test_side_streams_do_not_wait_for_the_default_stream():
    """The premise of test_side_stream: torch's side streams are non-blocking, so work issued on the default stream does
    not wait for them. A clone on the default stream, issued while the side stream sleeps before its copy, sees NaN."""
    buf = torch.full((1 << 16,), float("nan"), device="cuda")
    src = torch.ones_like(buf)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        buf.copy_(src)
    with torch.cuda.stream(torch.cuda.default_stream()):
        seen = buf.clone()
    torch.cuda.synchronize()
    assert bool(torch.isnan(seen).all()), "the default stream waited for the side stream"
    assert bool((buf == 1).all())


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_side_stream(name):
    """On a fresh stream: sleep, then copy the inputs into NaN buffers, then run the op forward and backward. A launch or
    a workspace fill on any other stream runs before the copies and reads or leaves NaN."""
    c = CASES[name]
    staging = c.make(_gen(7), "cuda")
    ref = c.run(*staging)
    bufs = [_poisoned_like(t) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = c.run(*bufs)
    s.synchronize()
    _same(out, ref, name)
    assert _lib.device_error() == 0, _lib.device_error_text()


# ---- 2. CUDA graphs ------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.capture])
def test_graph_replay(name):
    """Warm up on a side stream, capture, then replay three times, each with new values copied into the captured inputs:
    every replay equals an eager run on those values."""
    c = CASES[name]
    static = c.make(_gen(0), "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            c.run(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = c.run(*static)
    for i in range(1, 4):
        new = c.make(_gen(i), "cuda")
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        _same(out, c.run(*new), "%s replay %d" % (name, i))


def _trainer(init):
    """Params (a block-sparse weight, layer norm gain and bias), an Adam with zero_init_variables, an Ema whose averages
    start as copies of the params, and one training step over them."""
    params = [t.clone().requires_grad_() for t in init]
    w, lg, lb = params
    opt = AdamOptimizer(params, learning_rate=1e-2, zero_init_variables=True)
    ema = Ema(decay=0.9)
    ema.apply(params)                                  # ema == param: the update leaves it bit for bit

    def step(x, labels):
        h = layer_norm(x, lg, lb, axis=1)
        y = BSMM32(h, w.to(BF16)).view(1, 256, 256)
        o = BST.attention(y, y, y, scale=0.125, fused_backward=True)
        loss = softmax_cross_entropy(o.view(256, 256), labels)
        grads = torch.autograd.grad(loss.sum(), params)
        norm, scale = clip_by_global_norm(grads, clip_norm=1.0)
        opt.step(grads=grads, norm_scale=scale)
        ema.apply(params)
        return loss, norm
    return params, opt, ema, step


@gpu
def test_graph_training_step():
    """layer_norm -> bsmm -> fused attention -> cross entropy -> backward -> clip_by_global_norm -> Adam -> Ema, captured
    whole and replayed three times on new batches: loss, norm, params, moments and averages after k replays equal k
    eager steps."""
    g = _gen(50)
    init = [(torch.randn(BSMM32.w_shape, generator=g) * 0.1).cuda(), (1 + 0.1 * torch.randn(256, generator=g)).cuda(),
            (0.1 * torch.randn(256, generator=g)).cuda()]

    def batch(i):
        gb = _gen(60 + i)
        return torch.randn((256, 256), generator=gb).to(BF16).cuda(), torch.randint(0, 256, (256,), generator=gb).cuda()

    params, opt, ema, step = _trainer(init)
    sx, sl = batch(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(sx, sl)
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():                              # undo the warm-up steps; the state tensors stay where they are
        for p, t in zip(params, init):
            p.copy_(t)
            opt.state[p]["mean"].zero_()
            opt.state[p]["var"].zero_()
            ema.average(p).copy_(t)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, norm = step(sx, sl)

    ref_params, ref_opt, ref_ema, ref_step = _trainer(init)
    for i in range(1, 4):
        x, labels = batch(i)
        sx.copy_(x)
        sl.copy_(labels)
        graph.replay()
        ref_loss, ref_norm = ref_step(x, labels)
        state = lambda ps, o, e: [t for p in ps for t in (p, o.state[p]["mean"], o.state[p]["var"], e.average(p))]
        _same([loss, norm] + state(params, opt, ema), [ref_loss, ref_norm] + state(ref_params, ref_opt, ref_ema),
              "training step, replay %d" % i)
    assert opt.param_groups[0]["beta1_power"] == 0.0


@gpu
def test_graph_refuses_adam_with_bias_correction():
    """Without zero_init_variables the bias-corrected lr_t changes every step but would be replayed as captured: step()
    refuses under capture, before it launches anything, and still steps eagerly afterwards."""
    p = torch.randn(1000, device="cuda")
    g = torch.randn(1000, device="cuda")
    opt = AdamOptimizer([p], learning_rate=0.01)
    opt.step(grads=[g])                                # moments exist: nothing to allocate under capture
    before = p.clone()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError, match="zero_init_variables"):
        with torch.cuda.graph(graph):
            opt.step(grads=[g])
    assert torch.equal(p, before)
    powers = opt.param_groups[0]["beta1_power"], opt.param_groups[0]["beta2_power"]
    opt.step(grads=[g])
    assert not torch.equal(p, before) and opt.param_groups[0]["beta1_power"] < powers[0]


# ---- 3. host threads ------------------------------------------------------------------------------------------------------
def _thread_work(x, w, dy, q, k, v, do):
    """A matmul and a fused attention, forward and backward, on op objects of the calling thread's own."""
    bsmm = BlocksparseMatMul(_LAY32, block_size=32, feature_axis=1)
    bst = BlocksparseTransformer(_TRIL4, block_size=64, heads=2, mask_callback=causal)
    x, w, q, k, v = _leaf(x, w, q, k, v)
    y = bsmm(x, w)
    o = bst.attention(q, k, v, scale=0.125, fused_backward=True)
    return [y, o] + _grad(y, (x, w), dy) + _grad(o, (q, k, v), do)


def _thread_inputs(seed):
    g = _gen(seed)
    return [_rn(g, "cuda", BSMM32.i_shape(128), BF16), _rn(g, "cuda", BSMM32.w_shape, BF16, 0.1),
            _rn(g, "cuda", BSMM32.o_shape(128), BF16)] + [_rn(g, "cuda", (2, 256, 128), BF16) for _ in range(4)]


@gpu
def test_concurrent_threads():
    """Two host threads, each with its own stream and op objects, start together from a barrier; each result equals the
    single-threaded one. The thread-local tensor-map cache, error buffer and last-kernel slot are exercised."""
    inputs = [_thread_inputs(80 + i) for i in range(2)]
    refs = [_thread_work(*ins) for ins in inputs]
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    results, errors = [None, None], []

    def worker(i):
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.default_stream())
            barrier.wait()
            with torch.cuda.stream(s):
                results[i] = _thread_work(*inputs[i])
            s.synchronize()
        except BaseException as e:                      # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for i in range(2):
        _same(results[i], refs[i], "thread %d" % i)
    assert _lib.device_error() == 0, _lib.device_error_text()


# ---- 4. a second GPU -----------------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2,
                              reason="needs two visible GPUs: runs the families on cuda:1 while cuda:0 is current")


def _cuda_events(fn):
    """(fn(), [(name, device index) of every CUDA activity fn caused on any device])."""
    from torch.profiler import ProfilerActivity, profile
    for d in range(2):
        torch.cuda.synchronize(d)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        for d in range(2):
            torch.cuda.synchronize(d)
    return out, [(e.name, e.device_index) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@gpu
@two_gpus
@pytest.mark.parametrize("name", list(CASES))
def test_second_gpu(name):
    """With cuda:0 current, the case on cuda:1 tensors runs on cuda:1 only and equals cuda:0 bit for bit. The same op
    objects then alternate between the devices, so every per-device cache (LUTs, schedules, tile choices, tensor maps,
    dynamic shared memory, device properties) is used from both sides."""
    c = CASES[name]
    torch.cuda.set_device(0)
    ins0 = c.make(_gen(11), "cuda:0")
    ins1 = c.make(_gen(11), "cuda:1")
    ref = c.run(*ins0)
    out, events = _cuda_events(lambda: c.run(*ins1))
    assert torch.cuda.current_device() == 0
    assert events and all(d == 1 for _, d in events), [e for e in events if e[1] != 1][:5]
    assert all(t.device == torch.device("cuda:1") for t in out)
    _same(out, ref, name + " on cuda:1")
    _same(c.run(*ins0), ref, name + " on cuda:0 again")
    _same(c.run(*ins1), ref, name + " on cuda:1 again")
    for d in range(2):
        with torch.cuda.device(d):
            assert _lib.device_error() == 0, (d, _lib.device_error_text())


def _mixed():
    """name -> a call whose CUDA operands live on two devices."""
    g = _gen(12)
    d0, d1 = "cuda:0", "cuda:1"
    x0, dy0, w1 = _rn(g, d0, BSMM32.i_shape(64), BF16), _rn(g, d0, BSMM32.o_shape(64), BF16), _rn(g, d1, BSMM32.w_shape, BF16)
    gate1 = torch.ones(BSMM32.blocks, device=d1)
    q0, q1 = _rn(g, d0, (2, 256, 128), BF16), _rn(g, d1, (2, 256, 128), BF16)
    wf0, gain1 = _rn(g, d0, BSMM32.w_shape), _rn(g, d1, (BSMM32.K,))
    x96, y40 = _rn(g, d0, (96, 8), F16), _rn(g, d1, (40, 8), F16)
    n0, n1 = _rn(g, d0, (64, 256), BF16), _rn(g, d1, (64, 256), BF16)
    ln0, p1 = _rn(g, d0, (8, 96)), _rn(g, d1, (96,))
    return {
        "bsmm fprop": lambda: BSMM32.fprop(x0, w1),
        "bsmm updat gate": lambda: BSMM32.updat([x0], [dy0], gate=gate1, dw_gated=True),
        "bst nt_op": lambda: BST.nt_op(q0, q1),
        "attention": lambda: BST.attention(q0, q0, q1, scale=0.125),
        "l2_normalize gain": lambda: BSMM32.l2_normalize(wf0, gain=gain1),
        "blocksparse_reduced_dw": lambda: blocksparse_reduced_dw([n0], [n1], 1.0, bsize=32, axis=1),
        "SparseProj scatter_add": lambda: SPROJ.scatter_add(x96, y40),
        "blocksparse_l2_decay gate": lambda: blocksparse_l2_decay(wf0, gate1),
        "layer_norm g": lambda: layer_norm(ln0, p1, p1),
        "softmax_cross_entropy labels": lambda: softmax_cross_entropy(ln0, torch.zeros(8, dtype=torch.int64, device=d1)),
        "AdamOptimizer grad": lambda: AdamOptimizer([wf0]).step(grads=[wf0.to(d1)]),
        "clip_by_global_norm": lambda: clip_by_global_norm([wf0, gain1]),
        "global_norm": lambda: global_norm([gain1, wf0]),
    }


@gpu
@two_gpus
def test_mixed_devices_raise():
    """Operands on two devices are refused before anything launches: a kernel would get pointers of the other GPU."""
    for name, call in _mixed().items():
        with pytest.raises(ValueError):
            call()
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
    for d in range(2):
        with torch.cuda.device(d):
            assert _lib.device_error() == 0, (d, _lib.device_error_text())


def _two_device_params(g):
    """Params on cuda:0, cuda:1, cuda:0 (16-bit moments for the large one, a gate on the first) and their grads."""
    ps = [_rn(g, "cuda:0", (16, 32, 32)), _rn(g, "cuda:1", (9000,)), _rn(g, "cuda:0", (1003,))]
    ps[0].gate = _gate(g, "cuda:0", 16)
    gs = [_rn(g, p.device, p.shape, BF16, 0.1) for p in ps]
    return ps, gs


@gpu
@two_gpus
def test_optimizer_on_two_devices():
    """One AdamOptimizer / Ema over params on two GPUs equals one per device, bit for bit, with one launch per device
    and norm_scale taken from cuda:0; clip_by_global_norm refuses grads on two devices."""
    torch.cuda.set_device(0)
    ps, gs = _two_device_params(_gen(13))
    qs = [p.clone() for p in ps]
    qs[0].gate = ps[0].gate
    kw = dict(learning_rate=0.01, gated=True, fp16=True)
    opt = AdamOptimizer(ps, **kw)
    ema = Ema(decay=0.9, gated=True)
    per_dev = [(AdamOptimizer([qs[0], qs[2]], **kw), [0, 2]), (AdamOptimizer([qs[1]], **kw), [1])]
    ema_dev = [Ema(decay=0.9, gated=True), Ema(decay=0.9, gated=True)]
    scale = torch.full((), 0.75, device="cuda:0")
    with pytest.raises(ValueError):
        clip_by_global_norm(gs)
    for step in range(2):
        _, events = _cuda_events(lambda: opt.step(grads=gs, norm_scale=scale))
        launches = sorted(d for n, d in events if "mt_adam" in n)
        assert launches == [0, 1], events
        for o, idx in per_dev:
            o.step(grads=[gs[i] for i in idx], norm_scale=scale.to(ps[idx[0]].device))
        _, events = _cuda_events(lambda: ema.apply(ps))
        assert sorted(d for n, d in events if "mt_ema" in n) == [0, 1], events
        ema_dev[0].apply([qs[0], qs[2]])
        ema_dev[1].apply([qs[1]])
        for i, (p, q) in enumerate(zip(ps, qs)):
            o = per_dev[0][0] if i != 1 else per_dev[1][0]
            e = ema_dev[0] if i != 1 else ema_dev[1]
            _same([p, opt.state[p]["mean"], opt.state[p]["var"], ema.average(p)],
                  [q, o.state[q]["mean"], o.state[q]["var"], e.average(q)], "step %d param %d" % (step, i))
    assert opt.state[ps[1]]["mean"].dtype == torch.int16
