"""Dense softmax, its gradient and the top-k family on every kernel route, elementwise against the float64 oracle.

Routes (csrc/dense_softmax.cuh): softmax and gradient take dense_softmax[_grad]_warp for rows of <= 1024 entries,
_cta for <= 8192 and _long beyond; each with 16-byte accesses when every row start is 16-byte aligned (aligned tensors,
D3 a multiple of 16 / element size) and one element per access otherwise. The top-k family runs one CTA per row
(dense_topk, dense_topk_rectified, dense_topk_softmax).
"""
import collections

import numpy as np
import pytest
import torch

from tests._util import EPS32, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, dtype_name
from blocksparse_b200 import _lib, masked_softmax, masked_top_k_softmax, rectified_top_k, softmax, top_k
from blocksparse_b200 import transformer as tr
from oracle import dense_oracle as orc

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
WARP_MAX, CTA_MAX, CTA_THREADS = 1024, 8192, 256

# mask: None or the mask's shape; dead: zero whole mask rows, so that some rows see nothing
Case = collections.namedtuple("Case", "shape dtype mask scale dead")
CASES = [
    Case((5, 1), F32, None, 1.0, False),
    Case((6,), F16, (6,), 0.5, False),                                   # rank 1
    Case((3, 4, 7), F16, (1, 4, 7), 0.5, True),
    Case((2, 3, 32), BF16, (1, 1, 32), -1.25, False),
    Case((2, 3, 5, 33), F32, (1, 3, 1, 33), 0.75, True),                 # (D1, 1, D3)
    Case((2, 2, 2, 3, 1023), BF16, (1, 1, 2, 3, 1023), 1.0, True),       # rank 5, (D1, D2, D3)
    Case((3, 2, 1024), F16, (1, 2, 1024), -0.5, True),
    Case((64, 1024), F32, (64, 1024), 0.3, True),
    Case((2, 2, 1025), F32, (2, 1, 1025), 1.0, True),
    Case((4, 8191), BF16, (1, 8191), 0.125, False),
    Case((2, 3, 8192), F16, (1, 3, 8192), 1.0, True),
    Case((3, 8193), F32, None, -1.0, False),
    Case((2, 2, 20000), BF16, (2, 1, 20000), 0.25, True),                # long route, (D1, 1, D3)
    Case((2, 20001), F16, None, 2.0, False),
]


def _route(D3):
    return "warp" if D3 <= WARP_MAX else "cta" if D3 <= CTA_MAX else "long"


def _vector(case):
    return case.shape[-1] % (16 // torch.empty((), dtype=case.dtype).element_size()) == 0


def _per_thread(D3):
    """entries one thread sums in order before the reductions"""
    return -(-D3 // (32 if _route(D3) == "warp" else CTA_THREADS))


def _case_id(c):
    return "%s-%s-m%s-s%g%s" % ("x".join(map(str, c.shape)), dtype_name(c.dtype),
                                "none" if c.mask is None else "x".join(map(str, c.mask)), c.scale, "-dead" if c.dead else "")


def test_cases_cover_every_route():
    """The covering set reaches every route, both access widths and every mask shape (pure Python)."""
    d3 = {c.shape[-1] for c in CASES}
    assert {1, 7, 32, 33, WARP_MAX - 1, WARP_MAX, WARP_MAX + 1, CTA_MAX - 1, CTA_MAX, CTA_MAX + 1} <= d3
    assert max(d3) >= 20000
    assert {(_route(c.shape[-1]), _vector(c)) for c in CASES} == {(r, v) for r in ("warp", "cta", "long") for v in (True, False)}
    assert {c.dtype for c in CASES} == {F32, F16, BF16}
    assert {len(c.shape) for c in CASES} >= {1, 2, 3, 4, 5}
    kinds = set()
    for c in CASES:
        if c.mask is None:
            kinds.add("none")
            continue
        m, x = c.mask, c.shape
        d1 = len(m) >= 3 and m[-3] == x[-3] > 1
        d2 = len(m) >= 2 and m[-2] == x[-2] > 1
        kinds.add({(False, False): "row", (False, True): "d2", (True, False): "d1", (True, True): "d1d2"}[(d1, d2)])
    assert kinds == {"none", "row", "d2", "d1", "d1d2"}
    assert any(c.scale < 0 for c in CASES) and {_route(c.shape[-1]) for c in CASES if c.dead} == {"warp", "cta", "long"}


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _inputs(case, seed):
    rng = np.random.default_rng(seed)
    x = torch.as_tensor(rng.normal(0, 3.0, case.shape).astype(np.float32)).to(case.dtype).cuda()
    mask = None
    if case.mask is not None:
        m = (rng.uniform(0.5, 2.0, case.mask) * (rng.random(case.mask) >= 0.25)).astype(np.float32)
        if case.dead:
            m.reshape(-1, case.shape[-1])[0] = 0.0
        mask = torch.as_tensor(m).cuda()
    return x, mask, rng


def _values(x, mask, scale):
    """the float64 softmax arguments and which entries are visible"""
    xv = x.double().cpu().numpy()
    mn = None if mask is None else mask.double().cpu().numpy()
    v = orc.masked_values(xv, mn, scale)
    vis = np.ones(xv.shape, bool) if mn is None else np.broadcast_to(mn != 0, xv.shape)
    return xv, mn, v, vis


def softmax_bound(p, dtype, amax, per_thread, long_route=False):
    """Largest |got - p|, elementwise, for an oracle probability p (float64 on the same rounded inputs).

    In units of eps32: each softmax argument v = x * m * scale takes two fp32 roundings and v - max one more, so every
    exponent is off by <= 4 amax (|v| <= amax); the ratio of two exponentials carries twice that: 8 amax, 16 amax with
    slack. expf: 2 ulp = 4. The sum: per_thread serial additions, 5 shuffle levels, <= 7 warp partials (+16). The
    reciprocal and the final multiply: 2. The long route also rescales its running sums once per chunk at most, each
    rescale with an exponent of its own: per_thread (4 + 4 amax). Then one rounding to dtype and the subnormal floor."""
    u = EPS32 * (16 * amax + per_thread + 16 + 8)
    if long_route:
        u += EPS32 * per_thread * (4 + 4 * amax)
    return (U_OUT[dtype_name(dtype)] + u) * p + SUBNORMAL_FLOOR[dtype_name(dtype)] + 2.0 ** -100


def grad_bound(ref, dy, y, m, scale, dtype, per_thread):
    """Largest |got - ref| of dx = (dy - sum(dy y)) y m scale: the fp32 row sum (16-bit products are exact, fp32 ones
    round once) with per_thread serial additions and <= 12 reduction levels, then the subtraction and three multiplies,
    each <= eps32 (|dy| + sum|dy y|) |y m scale|; one rounding to dtype and the subnormal floor."""
    row = np.sum(np.abs(dy * y), axis=-1, keepdims=True)
    return (U_OUT[dtype_name(dtype)] * np.abs(ref)
            + EPS32 * (per_thread + 12 + 8) * (np.abs(dy) + row) * np.abs(y * m * scale) + SUBNORMAL_FLOOR[dtype_name(dtype)])


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()


def _check_softmax(y, x, mask, scale, what):
    xv, mn, v, vis = _values(x, mask, scale)
    p = orc.masked_softmax(xv, mn, scale)
    g = y.double().cpu().numpy()
    assert not np.isnan(g).any(), "%s: %d entries never written" % (what, int(np.isnan(g).sum()))
    live = vis.any(axis=-1, keepdims=True)
    hidden = ~vis & live
    assert not np.any(g[hidden] != 0), "%s: %d masked probabilities of live rows are not 0" % (what, int((g[hidden] != 0).sum()))
    dead = np.broadcast_to(~live, g.shape)
    assert np.all(p[dead] == 1.0 / xv.shape[-1])
    D3 = xv.shape[-1]
    amax = float(np.abs(np.where(vis, v, 0)).max(initial=0.0))
    bound = softmax_bound(p, y.dtype, amax, _per_thread(D3), _route(D3) == "long")
    err = np.abs(g - p)
    assert np.all(err <= bound), "%s: %d probabilities out of bound, worst excess %.3e" % (
        what, int((err > bound).sum()), float((err - bound).max()))
    return p


def _check_grad(dx, dy, y, mask, scale, what):
    dyv, yv = dy.double().cpu().numpy(), y.double().cpu().numpy()
    mn = 1.0 if mask is None else np.broadcast_to(mask.double().cpu().numpy(), yv.shape)
    ref = orc.masked_softmax_grad(dyv, yv, None if mask is None else mn, scale)
    g = dx.double().cpu().numpy()
    assert not np.isnan(g).any(), "%s: %d gradient entries never written" % (what, int(np.isnan(g).sum()))
    assert not np.any(g[yv * mn == 0] != 0), "%s: gradient nonzero where y m == 0" % what
    bound = grad_bound(ref, dyv, yv, mn, scale, dx.dtype, _per_thread(yv.shape[-1]))
    err = np.abs(g - ref)
    assert np.all(err <= bound), "%s: %d gradient entries out of bound, worst excess %.3e" % (
        what, int((err > bound).sum()), float((err - bound).max()))


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_softmax_and_grad_match_oracle(idx):
    case = CASES[idx]
    what = _case_id(case)
    route = _route(case.shape[-1])
    x, mask, rng = _inputs(case, 100 + idx)
    y = _on_poisoned_output(lambda: masked_softmax(x, mask, case.scale))
    assert _lib.last_kernel() == "dense_softmax_" + route, (what, _lib.last_kernel())
    assert y.dtype == x.dtype and y.shape == x.shape
    _check_softmax(y, x, mask, case.scale, what)
    y2 = masked_softmax(x, mask, case.scale)
    assert _bits(y2) == _bits(y), "%s: forward not bitwise reproducible" % what

    dy = torch.as_tensor(rng.normal(0, 1, case.shape).astype(np.float32)).to(case.dtype).cuda()
    m, M1, M2 = tr._dense_mask(x, mask, "test")
    dx = _on_poisoned_output(lambda: tr._dense_softmax_bwd(y, dy, m, M1, M2, case.scale))
    assert _lib.last_kernel() == "dense_softmax_grad_" + route, (what, _lib.last_kernel())
    _check_grad(dx, dy, y, mask, case.scale, what)
    assert _bits(tr._dense_softmax_bwd(y, dy, m, M1, M2, case.scale)) == _bits(dx), "%s: gradient not reproducible" % what

    # autograd: the gradient of the public op is the formula at the op's own y
    xg = x.clone().requires_grad_()
    yg = masked_softmax(xg, mask, case.scale)
    yg.backward(dy)
    assert xg.grad.dtype == x.dtype
    _check_grad(xg.grad, dy, yg.detach(), mask, case.scale, what + " autograd")


@pytest.mark.parametrize("D3,dtype,offset", [(64, F16, 1), (1024, BF16, 3), (4096, F32, 1), (9000, F16, 5)])
def test_odd_offset_and_non_contiguous_inputs(D3, dtype, offset):
    """A view at an odd element offset runs the one-element-per-access kernels and matches the oracle; a non-contiguous
    input is made contiguous by the op and gives the same bits as its contiguous copy."""
    rng = np.random.default_rng(D3 + offset)
    shape = (3, 2, D3)
    n = int(np.prod(shape))
    src = torch.as_tensor(rng.normal(0, 3, shape).astype(np.float32)).to(dtype).cuda()
    buf = torch.zeros(n + offset, dtype=dtype, device="cuda")
    x = buf[offset:].view(shape)
    x.copy_(src)
    assert x.data_ptr() % 16
    mask = torch.as_tensor((rng.random((1, 2, D3)) > 0.3).astype(np.float32)).cuda()
    y = masked_softmax(x, mask, 0.5)
    _check_softmax(y, x, mask, 0.5, "offset %d" % offset)
    dyb = torch.zeros(n + offset, dtype=dtype, device="cuda")
    dy = dyb[offset:].view(shape)
    dy.copy_(torch.as_tensor(rng.normal(0, 1, shape).astype(np.float32)).to(dtype).cuda())
    m, M1, M2 = tr._dense_mask(x, mask, "test")
    _check_grad(tr._dense_softmax_bwd(y, dy, m, M1, M2, 0.5), dy, y, mask, 0.5, "offset %d grad" % offset)
    # non-contiguous: a transposed view
    xt = src.transpose(0, 1).contiguous().transpose(0, 1)
    assert not xt.is_contiguous()
    assert _bits(masked_softmax(xt, mask, 0.5)) == _bits(masked_softmax(src, mask, 0.5))
    mt = torch.stack([mask, mask], -1)[..., 0]          # a non-contiguous mask is made contiguous too
    assert not mt.is_contiguous()
    assert _bits(masked_softmax(src, mt, 0.5)) == _bits(masked_softmax(src, mask, 0.5))


def test_softmax_without_mask_and_empty_inputs():
    x = torch.randn(4, 100, device="cuda", dtype=F16)
    assert _bits(softmax(x, 0.7)) == _bits(masked_softmax(x, None, 0.7))
    before = _lib.last_kernel()
    for fn in (lambda t: softmax(t), lambda t: masked_top_k_softmax(t, 1), lambda t: rectified_top_k(t, 2)):
        e = torch.empty(0, 3, 5, device="cuda", dtype=BF16)
        out = fn(e)
        assert out.shape == e.shape and out.dtype == e.dtype
    vals, idx = top_k(torch.empty(0, 5, device="cuda"), 3)
    assert vals.shape == (0, 3) and idx.dtype == torch.int32
    assert _lib.last_kernel() == before


def test_more_than_2_31_elements_on_sampled_rows():
    """64-bit element offsets: a (2^21 + 1, 1024) fp16 tensor, checked on sampled rows including the last."""
    rows, D3 = (1 << 21) + 1, 1024
    assert rows * D3 > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(rows, D3, device="cuda", dtype=F16, generator=g)
    y = masked_softmax(x, None, 0.5)
    assert _lib.last_kernel() == "dense_softmax_warp"
    pick = torch.tensor([0, 1, rows // 2, rows - 2, rows - 1] + list(range(rows - 1, 0, -rows // 37)), device="cuda").unique()
    xs, ys = x[pick], y[pick]
    _check_softmax(ys, xs, None, 0.5, "2^31 forward")
    dy = torch.randn(rows, D3, device="cuda", dtype=F16, generator=g)
    dx = tr._dense_softmax_bwd(y, dy, None, 0, 0, 0.5)
    _check_grad(dx[pick], dy[pick], ys, None, 0.5, "2^31 grad")
    del x, y, dy, dx
    torch.cuda.empty_cache()


# ---- top-k family ------------------------------------------------------------------------------------------------------
TOPK_SHAPES = [((4, 1), F32), ((3, 2, 7), F16), ((5, 33), BF16), ((2, 3, 256), F32), ((3, 1000), F16), ((2, 1024), BF16)]


def _topk_input(shape, dtype, ties, seed):
    rng = np.random.default_rng(seed)
    v = rng.integers(-3, 4, shape) if ties else rng.normal(0, 2, shape)
    return torch.as_tensor(v.astype(np.float32)).to(dtype).cuda(), rng


def _ks(D3):
    return sorted({1, max(1, D3 // 2), D3})


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("shape,dtype", TOPK_SHAPES, ids=["%s-%s" % ("x".join(map(str, s)), dtype_name(d)) for s, d in TOPK_SHAPES])
def test_top_k_matches_stable_sort(shape, dtype, ties):
    x, rng = _topk_input(shape, dtype, ties, shape[-1] + ties)
    xn = x.double().cpu().numpy()
    for k in _ks(shape[-1]):
        vals = _on_poisoned_output(lambda: top_k(x, k)[0])
        assert _lib.last_kernel() == "dense_topk"
        idx = top_k(x, k)[1]
        ref_v, ref_i = orc.top_k(xn, k)
        assert idx.dtype == torch.int32 and vals.dtype == dtype and vals.shape == shape[:-1] + (k,)
        np.testing.assert_array_equal(idx.cpu().numpy(), ref_i)
        # bit-exact copies of x's entries
        assert _bits(vals) == _bits(torch.gather(x, -1, idx.long()))
        np.testing.assert_array_equal(vals.double().cpu().numpy(), ref_v)
        # the gradient is exactly the scatter of dvalues
        xg = x.clone().requires_grad_()
        dv = torch.as_tensor(rng.normal(0, 1, vals.shape).astype(np.float32)).to(dtype).cuda()
        top_k(xg, k)[0].backward(dv)
        ref = np.zeros(xn.shape)
        np.put_along_axis(ref, ref_i.astype(np.int64), dv.double().cpu().numpy(), axis=-1)
        np.testing.assert_array_equal(xg.grad.double().cpu().numpy(), ref)


@pytest.mark.parametrize("rebase", [True, False])
@pytest.mark.parametrize("shape,dtype", TOPK_SHAPES, ids=["%s-%s" % ("x".join(map(str, s)), dtype_name(d)) for s, d in TOPK_SHAPES])
def test_rectified_top_k(shape, dtype, rebase):
    """Includes rows whose kth value is negative (k = D3 of normal data) and zero (integer data with ties)."""
    for ties in (False, True):
        x, rng = _topk_input(shape, dtype, ties, 7 * shape[-1] + ties)
        xn = x.double().cpu().numpy()
        for k in _ks(shape[-1]):
            y = _on_poisoned_output(lambda: rectified_top_k(x, k, rebase))
            assert _lib.last_kernel() == "dense_topk_rectified"
            ref = orc.rectified_top_k(xn, k, rebase)
            g = y.double().cpu().numpy()
            # x and base are exact in fp32; x - base rounds once in fp32, then once to dtype
            bound = (U_OUT[dtype_name(dtype)] + 2 * EPS32) * np.abs(ref)
            assert np.all(np.abs(g - ref) <= bound), (shape, dtype, rebase, ties, k)
            assert np.all((g != 0) <= (ref != 0) | (np.abs(ref) <= bound))
            xg = x.clone().requires_grad_()
            yg = rectified_top_k(xg, k, rebase)
            dz = torch.as_tensor(rng.normal(0, 1, shape).astype(np.float32)).to(dtype).cuda()
            yg.backward(dz)
            assert torch.equal(xg.grad, torch.where(yg.detach() > 0, dz, torch.zeros_like(dz)))


TKS_CASES = [((3, 2, 7), F16, (1, 2, 7)), ((5, 33), BF16, None), ((2, 3, 256), F32, (1, 3, 256)),
             ((2, 4, 1000), F16, (2, 1, 1000)), ((3, 1024), BF16, (3, 1024))]


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("shape,dtype,mshape", TKS_CASES,
                         ids=["%s-%s" % ("x".join(map(str, s)), dtype_name(d)) for s, d, _ in TKS_CASES])
def test_masked_top_k_softmax(shape, dtype, mshape, ties):
    x, rng = _topk_input(shape, dtype, ties, 11 * shape[-1] + ties)
    D3 = shape[-1]
    mask = None
    if mshape is not None:
        m = (rng.uniform(0.5, 2.0, mshape) * (rng.random(mshape) >= 0.3)).astype(np.float32)
        flat = m.reshape(-1, D3)
        flat[0] = 0.0                                    # a fully masked row
        if flat.shape[0] > 1:
            flat[1] = 0.0
            flat[1, [2 % D3, D3 - 1]] = 1.0              # a row with fewer visible entries than most k
        mask = torch.as_tensor(m).cuda()
    xn = x.double().cpu().numpy()
    mn = None if mask is None else mask.double().cpu().numpy()
    scale = -0.75 if ties else 0.5
    # the kernels rank the fp32 values x * m * scale
    v32 = orc.masked_values(x.float().cpu().numpy(), None if mask is None else mask.cpu().numpy(), scale, dtype=np.float32)
    vis = np.ones(xn.shape, bool) if mn is None else np.broadcast_to(mn != 0, xn.shape)
    for k in _ks(D3):
        y = _on_poisoned_output(lambda: masked_top_k_softmax(x, k, mask, scale))
        assert _lib.last_kernel() == "dense_topk_softmax"
        p = orc.masked_top_k_softmax(xn, k, mn, scale, order_values=v32)
        support = np.zeros(xn.shape, bool)
        np.put_along_axis(support, orc.rank(v32)[..., :k], True, axis=-1)
        g = y.double().cpu().numpy()
        assert not np.any(g[~support] != 0), (shape, k, "entries outside the support are not 0")
        amax = float(np.abs(np.where(vis, orc.masked_values(xn, mn, scale), 0)).max())
        bound = softmax_bound(p, dtype, amax, 2)
        assert np.all(np.abs(g - p) <= bound), (shape, dtype, k, float((np.abs(g - p) - bound).max()))
        if mn is not None:
            dead = ~vis.any(axis=-1)
            first = np.zeros(D3)
            first[:k] = 1.0 / k
            assert np.all(np.abs(g[dead] - first) <= bound[dead])
            few = vis.sum(axis=-1) < k
            assert (few & ~dead).any() or k == 1
        xg = x.clone().requires_grad_()
        yg = masked_top_k_softmax(xg, k, mask, scale)
        dy = torch.as_tensor(rng.normal(0, 1, shape).astype(np.float32)).to(dtype).cuda()
        yg.backward(dy)
        _check_grad(xg.grad, dy, yg.detach(), mask, scale, "top-k softmax grad")


# ---- CUDA graph ----------------------------------------------------------------------------------------------------------
def test_masked_softmax_forward_and_backward_replay_in_a_cuda_graph():
    ctx = 1024
    x = torch.randn(2, 4, ctx, ctx, device="cuda", dtype=F16)
    dy = torch.randn_like(x)
    mask = torch.tril(torch.ones(ctx, ctx, device="cuda")).view(1, 1, ctx, ctx)
    m, M1, M2 = tr._dense_mask(x, mask, "test")
    y_ref = masked_softmax(x, mask, 0.125)
    dx_ref = tr._dense_softmax_bwd(y_ref, dy, m, M1, M2, 0.125)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            tr._dense_softmax_bwd(masked_softmax(x, mask, 0.125), dy, m, M1, M2, 0.125)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = masked_softmax(x, mask, 0.125)
        dx = tr._dense_softmax_bwd(y, dy, m, M1, M2, 0.125)
    for _ in range(2):
        y.zero_(); dx.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert _bits(y) == _bits(y_ref) and _bits(dx) == _bits(dx_ref)


def test_bench_prints_one_line_per_timed_op(capsys):
    """bench= times the forward (and, in the backward, the gradient) and prints one line each with ms and GB/s; the
    result is the op's ordinary output."""
    x = torch.randn(2, 3, 256, device="cuda", dtype=F16).requires_grad_()
    mask = torch.ones(1, 3, 256, device="cuda")
    y = masked_softmax(x, mask, 0.5, bench=3)
    y.backward(torch.ones_like(y))
    lines = [l for l in capsys.readouterr().out.splitlines() if l.strip()]
    assert len(lines) == 2, lines
    assert lines[0].startswith("masked_softmax (2, 3, 256) float16 ms: ") and " GB/s: " in lines[0]
    assert lines[1].startswith("masked_softmax_grad (2, 3, 256) float16 ms: ") and " GB/s: " in lines[1]
    assert _bits(y) == _bits(masked_softmax(x.detach(), mask, 0.5))
    softmax(x.detach(), 0.5, bench=2)
    assert len([l for l in capsys.readouterr().out.splitlines() if l.strip()]) == 1
