"""layer_norm and its gradient on every kernel route, elementwise against the float64 oracle (oracle/norms_oracle.py).

Routes (csrc/layer_norm.cuh): feature axis last: layer_norm[_grad]_nc_warp for segments of <= 1024 features, _nc_cta for
<= 8192, _nc_long beyond; feature axis 0: layer_norm[_grad]_cn when the column strips fill the GPU, _cn_split when the
rows are split across CTAs. Each with 16-byte accesses where every row start is 16-byte aligned, one element otherwise.
"""
import collections

import numpy as np
import pytest
import torch

from oracle import norms_oracle as orc
from tests._util import EPS32, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, dtype_name
from blocksparse_b200 import _lib, layer_norm
from blocksparse_b200 import norms as nm

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
WARP_MAX, CTA_MAX, CN_CTAS, CN_MIN_ROWS = 1024, 8192, 264, 64

Case = collections.namedtuple("Case", "shape axis segments relu dtype offset")
CASES = [
    Case((64, 1), -1, 1, False, F32, 0),
    Case((33, 31), -1, 1, True, F16, 0),
    Case((16, 1024), -1, 1, False, BF16, 0),
    Case((20, 512), -1, 1, False, F16, 1),
    Case((2, 5, 96), -1, 1, True, BF16, 0),
    Case((5000, 64), -1, 1, False, F32, 0),
    Case((40, 4096), -1, 4, True, F16, 0),
    Case((8, 1025), -1, 1, False, F32, 0),
    Case((10, 3300), -1, 3, False, BF16, 0),
    Case((4, 8192), -1, 1, True, F16, 0),
    Case((3000, 2048), -1, 1, False, BF16, 0),
    Case((6, 1024), -1, 1, False, F32, 3),
    Case((3, 8193), -1, 1, False, BF16, 0),
    Case((2, 32767), -1, 1, True, F32, 0),
    Case((2, 16384), -1, 1, False, BF16, 0),
    Case((3, 12000), -1, 1, False, F16, 0),
    Case((6, 16400), -1, 2, False, F32, 0),
    Case((64, 9000), 0, 1, False, F32, 0),
    Case((96, 67584), 0, 1, True, BF16, 0),
    Case((31, 100), 0, 1, True, F16, 0),
    Case((4096, 256), 0, 1, False, BF16, 0),
    Case((4096, 256), 0, 1, True, F16, 1),
    Case((4097, 250), 0, 1, False, F32, 0),
    Case((200, 300), 0, 1, False, F16, 3),
    Case((48, 2, 40), 0, 1, False, F32, 0),
]


def _vec_width(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def _dims(c):
    K = c.shape[c.axis]
    return K, int(np.prod(c.shape)) // K


def _vec(c):
    K, N = _dims(c)
    n = K // c.segments if c.axis != 0 else N
    return c.offset == 0 and n % _vec_width(c.dtype) == 0


def _route(c):
    K, N = _dims(c)
    if c.axis != 0:
        L = K // c.segments
        return "nc_warp" if L <= WARP_MAX else "nc_cta" if L <= CTA_MAX else "nc_long"
    return "cn_split" if _cn_split(c)[0] > 1 else "cn"


def _case_id(c):
    return "%s-ax%d-s%d-%s%s%s" % ("x".join(map(str, c.shape)), c.axis, c.segments, dtype_name(c.dtype),
                                   "-relu" if c.relu else "", "-off%d" % c.offset if c.offset else "")


def test_cases_cover_every_route():
    ks = {_dims(c)[0] for c in CASES}
    assert {1, 31, 1024, 1025, 8192, 8193, 32767} <= ks
    routes = {(_route(c), _vec(c)) for c in CASES}
    assert routes == {(r, v) for r in ("nc_warp", "nc_cta", "nc_long", "cn", "cn_split") for v in (True, False)}
    for dt in (F32, F16, BF16):
        assert {_route(c) for c in CASES if c.dtype == dt} == {"nc_warp", "nc_cta", "nc_long", "cn", "cn_split"}
    assert any(c.axis == 0 and _dims(c)[1] <= 256 and _dims(c)[0] >= 4096 for c in CASES)     # split-K shape
    assert any(c.segments > 1 for c in CASES) and any(c.relu for c in CASES) and any(c.offset for c in CASES)


# ---- bounds ------------------------------------------------------------------------------------------------------------
def _cn_split(c):
    """(splits, rows per split) of an axis-0 case, as csrc/layer_norm.cuh:ln_cn_partition picks them."""
    K, N = _dims(c)
    w = 32 * (_vec_width(c.dtype) if _vec(c) else 1)
    strips = -(-N // w)
    sp = 1 if strips >= CN_CTAS else min(-(-CN_CTAS // strips), -(-K // CN_MIN_ROWS))
    rps = -(-K // sp)
    return -(-K // rps), rps


def _n_chain(c):
    """Longest chain of fp32 roundings that feeds one statistic of the case's route: the serial loop of one thread
    (L / 32 values on the warp route, L / 256 on the CTA routes; rows / 8 per warp on axis 0), then 5 shuffle levels
    and 8 warp partials, or on axis 0 the 8 warps' merges and one per row split. Each step of the chain loses at most
    eps32 of the running sum of absolute values; a Welford update rounds four times, hence 4 eps32 per step below."""
    K, _ = _dims(c)
    if c.axis == 0:
        splits, rps = _cn_split(c)
        return -(-rps // 8) + 8 + splits
    L = K // c.segments
    return -(-L // (32 if L <= WARP_MAX else 256)) + 5 + 8


def _stats_err(xs, c):
    """Bound of the kernel's mean error per (row, segment), and the variance."""
    k = 4 * _n_chain(c) * EPS32
    return k * np.abs(xs).mean(axis=2) + EPS32 * np.abs(xs.mean(axis=2)), xs.var(axis=2)


def _forward_bound(x, g, b, c, eps):
    ax = 0 if c.axis == 0 else -1
    xs = orc._rows(x, ax, c.segments)
    L = xs.shape[2]
    mean, rstd = orc.statistics(x, ax, c.segments, eps)
    dmu, var = _stats_err(xs, c)
    rel_var = 4 * _n_chain(c) * EPS32 + dmu ** 2 / (var + eps)
    rel_rstd = 0.5 * rel_var + 4 * EPS32                                      # rsqrtf: 2 ulp
    gs, bs = g.reshape(1, c.segments, -1), b.reshape(1, c.segments, -1)
    xhat = (xs - mean[..., None]) * rstd[..., None]
    dxh = (dmu[..., None] + EPS32 * np.abs(xs - mean[..., None])) * rstd[..., None] * (1 + rel_rstd[..., None]) \
        + np.abs(xhat) * (rel_rstd[..., None] + 2 * EPS32)
    dpre = np.abs(gs) * dxh + 2 * EPS32 * (np.abs(xhat * gs) + np.abs(bs))
    return xhat, dxh, dpre, rel_rstd, rstd, gs, bs


def _check(c, x, g, b, dy, y, dx, dg, db, eps=1e-6):
    what = _case_id(c)
    ax = 0 if c.axis == 0 else -1
    kw = dict(axis=ax, segments=c.segments, epsilon=eps, relu=c.relu)
    u = U_OUT[dtype_name(c.dtype)]
    sub = SUBNORMAL_FLOOR[dtype_name(c.dtype)]
    xhat, dxh, dpre, rel_rstd, rstd, gs, bs = _forward_bound(x, g, b, c, eps)
    ref = orc._rows(orc.layer_norm(x, g, b, **kw), ax, c.segments)
    got = orc._rows(y.double().cpu().numpy(), ax, c.segments)
    bound = u * np.abs(ref) + (1 + u) * dpre * (1 + 2.0 ** -10) + sub
    err = np.abs(got - ref)
    assert np.all(err <= bound), "%s: y: %d of %d out of bound, worst excess %.3e" % (
        what, int((err > bound).sum()), err.size, float((err - bound).max()))
    if dx is None:
        return
    # dy is zero wherever the pre-activation lies within its error bound of 0, so the relu mask cannot differ there
    dys = orc._rows(dy, ax, c.segments)
    if c.relu:
        dys = np.where(xhat * gs + bs > 0, dys, 0.0)
    rdx, rdg, rdb = orc.layer_norm_grad(dy, x, g, b, **kw)
    rdx = orc._rows(rdx, ax, c.segments)
    L = xhat.shape[2]
    cc = 4 * _n_chain(c) * EPS32
    dyg = np.abs(dys * gs)
    s1a = (dyg * np.abs(xhat)).sum(axis=2, keepdims=True)
    s2a = dyg.sum(axis=2, keepdims=True)
    ds1 = cc * s1a + (dyg * dxh).sum(axis=2, keepdims=True)
    ds2 = cc * s2a
    r = rstd[..., None]
    inner = dyg * EPS32 + (dxh * s1a + np.abs(xhat) * ds1 + ds2) / L + 4 * EPS32 * (np.abs(xhat) * s1a + s2a) / L
    bdx = u * np.abs(rdx) + (1 + u) * (r * inner + np.abs(rdx) * (rel_rstd[..., None] + 2 * EPS32)) * (1 + 2.0 ** -10) + sub
    gdx = orc._rows(dx.double().cpu().numpy(), ax, c.segments)
    err = np.abs(gdx - rdx)
    assert np.all(err <= bdx), "%s: dx: %d of %d out of bound, worst excess %.3e" % (
        what, int((err > bdx).sum()), err.size, float((err - bdx).max()))
    rows = xhat.shape[0]
    ug = U_OUT[dtype_name(g_dtype_of(c))]
    cr = (rows + 40) * EPS32
    a_dg = np.einsum("rsl,rsl->sl", np.abs(dys), np.abs(xhat)).reshape(-1)
    b_dg = ug * np.abs(rdg) + (1 + ug) * (cr * a_dg + np.einsum("rsl,rsl->sl", np.abs(dys), dxh).reshape(-1)) \
        * (1 + 2.0 ** -10) + 2.0 ** -25
    b_db = ug * np.abs(rdb) + (1 + ug) * cr * np.abs(dys).sum(axis=0).reshape(-1) + 2.0 ** -25
    for got, ref, bnd, name in ((dg, rdg, b_dg, "dg"), (db, rdb, b_db, "db")):
        e = np.abs(got.double().cpu().numpy().reshape(-1) - ref)
        assert np.all(e <= bnd), "%s: %s: %d out of bound, worst excess %.3e" % (what, name, int((e > bnd).sum()),
                                                                                 float((e - bnd).max()))


def g_dtype_of(c):
    """Gain dtype of a case: cycles through the three so each route meets a gain dtype other than x's."""
    return (F32, BF16, F16)[CASES.index(c) % 3] if c in CASES else F32


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _tensor(a, dtype, offset=0):
    t = torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dtype)
    if not offset:
        return t.cuda()
    buf = torch.zeros(t.numel() + offset, dtype=dtype, device="cuda")
    v = buf[offset:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16
    return v


def _inputs(c, rng, eps=1e-6):
    K, N = _dims(c)
    x = _tensor(rng.normal(rng.uniform(-2, 2), rng.uniform(0.5, 3), c.shape), c.dtype, c.offset)
    gd = g_dtype_of(c)
    g = torch.as_tensor(rng.uniform(0.5, 1.5, K).astype(np.float32)).to(gd).cuda()
    b = torch.as_tensor(rng.normal(0, 0.5, K).astype(np.float32)).to(gd).cuda()
    xd, gd64, bd = x.double().cpu().numpy(), g.double().cpu().numpy(), b.double().cpu().numpy()
    dy = rng.normal(0, 1, c.shape)
    if c.relu:
        xhat, _, dpre, _, _, gs, bs = _forward_bound(xd, gd64, bd, c, eps)
        near = orc._unrows(np.abs(xhat * gs + bs) <= 4 * dpre + 1e-6, c.shape, 0 if c.axis == 0 else -1)
        dy[near] = 0.0
    dyt = _tensor(dy, c.dtype)
    return x, g, b, dyt, xd, gd64, bd, dyt.double().cpu().numpy()


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy().tobytes()


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_layer_norm_matches_oracle(idx):
    c = CASES[idx]
    rng = np.random.default_rng(500 + idx)
    x, g, b, dy, xd, gd, bd, dyd = _inputs(c, rng)
    K, N = _dims(c)
    ax = 0 if c.axis == 0 else 1
    args = (ax, N, K, c.segments, 1e-6, c.relu)
    y, mean, rstd = _on_poisoned_output(lambda: nm._ln_fwd(x, g, b, *args))
    assert _lib.last_kernel() == "layer_norm_" + _route(c), (_case_id(c), _lib.last_kernel())
    dx, dg, db = _on_poisoned_output(lambda: nm._ln_bwd(x, dy, g, b, mean, rstd, *args))
    assert _lib.last_kernel() == "layer_norm_grad_" + _route(c), (_case_id(c), _lib.last_kernel())
    assert dg.dtype == g.dtype and db.dtype == b.dtype and dx.dtype == x.dtype
    _check(c, xd, gd, bd, dyd, y, dx, dg, db)
    # bitwise reproducible
    y2, m2, r2 = nm._ln_fwd(x, g, b, *args)
    assert _bits(y2) == _bits(y) and _bits(m2) == _bits(mean) and _bits(r2) == _bits(rstd)
    dx2, dg2, db2 = nm._ln_bwd(x, dy, g, b, mean, rstd, *args)
    assert _bits(dx2) == _bits(dx) and _bits(dg2) == _bits(dg) and _bits(db2) == _bits(db)
    # the public op and autograd give the bits of the raw calls on the same (here: freshly allocated, aligned) tensor
    xa = x.detach().clone()
    ya, ma, ra = nm._ln_fwd(xa, g, b, *args)
    dxa, dga, dba = nm._ln_bwd(xa, dy, g, b, ma, ra, *args)
    if not c.offset:
        assert _bits(ya) == _bits(y) and _bits(dxa) == _bits(dx)
    xg, gg, bg = xa.requires_grad_(), g.clone().requires_grad_(), b.clone().requires_grad_()
    out = layer_norm(xg, gg, bg, axis=c.axis, segments=c.segments, relu=c.relu)
    assert out.shape == x.shape and _bits(out) == _bits(ya)
    out.backward(dy)
    assert _bits(xg.grad) == _bits(dxa) and _bits(gg.grad) == _bits(dga) and _bits(bg.grad) == _bits(dba)


def test_large_mean_is_stable():
    """|mean| = 1e4 std in fp32: y, dx, dg and db stay within the bounds, which E[x^2] - E[x]^2 would not meet."""
    for c in (Case((64, 1024), -1, 1, False, F32, 0), Case((64, 4096), -1, 1, False, F32, 0),
              Case((1024, 512), 0, 1, False, F32, 0), Case((4096, 128), 0, 1, False, F32, 0)):
        rng = np.random.default_rng(9)
        K, N = _dims(c)
        x = torch.as_tensor((1e4 + rng.normal(0, 1, c.shape)).astype(np.float32)).cuda()
        g = torch.ones(K, device="cuda")
        b = torch.zeros(K, device="cuda")
        dy = torch.as_tensor(rng.normal(0, 1, c.shape).astype(np.float32)).cuda()
        ax = 0 if c.axis == 0 else 1
        y, mean, rstd = nm._ln_fwd(x, g, b, ax, N, K, 1, 1e-6, False)
        dx, dg, db = nm._ln_bwd(x, dy, g, b, mean, rstd, ax, N, K, 1, 1e-6, False)
        _check(c, x.double().cpu().numpy(), g.double().cpu().numpy(), b.double().cpu().numpy(),
               dy.double().cpu().numpy(), y, dx, dg, db)
        yd = y.double().cpu().numpy()
        ref = orc.layer_norm(x.double().cpu().numpy(), 1.0 * np.ones(K), np.zeros(K), axis=0 if ax == 0 else -1)
        assert np.abs(yd - ref).max() < 0.05


def test_cuda_graph_capture_and_replay():
    for axis, shape in ((-1, (64, 768)), (0, (4096, 256)), (0, (512, 8192))):
        x = torch.randn(shape, device="cuda", dtype=BF16, requires_grad=True)
        K = shape[axis]
        g = torch.rand(K, device="cuda", requires_grad=True)
        b = torch.randn(K, device="cuda", requires_grad=True)
        dy = torch.randn(shape, device="cuda", dtype=BF16)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                    # warm-up on the side stream, as graph capture wants
            layer_norm(x, g, b, axis=axis, relu=True).backward(dy)
        torch.cuda.current_stream().wait_stream(s)
        x.grad = g.grad = b.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = layer_norm(x, g, b, axis=axis, relu=True)
            y.backward(dy)
        x.grad.zero_(); g.grad.zero_(); b.grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        xe, ge, be = (t.detach().clone().requires_grad_() for t in (x, g, b))
        ye = layer_norm(xe, ge, be, axis=axis, relu=True)
        ye.backward(dy)
        assert _bits(y) == _bits(ye)
        assert _bits(x.grad) == _bits(xe.grad) and _bits(g.grad) == _bits(ge.grad) and _bits(b.grad) == _bits(be.grad)


def test_zero_rows_launch_nothing():
    before = _lib.last_kernel()
    for shape, axis in (((0, 64), -1), ((64, 0), 0), ((2, 0, 16), -1)):
        K = shape[axis]
        x = torch.empty(shape, device="cuda", dtype=F16, requires_grad=True)
        g = torch.ones(K, device="cuda", requires_grad=True)
        b = torch.zeros(K, device="cuda", requires_grad=True)
        y = layer_norm(x, g, b, axis=axis)
        assert y.shape == shape
        y.sum().backward()
        assert x.grad.shape == shape and bool((g.grad == 0).all()) and bool((b.grad == 0).all())
    assert _lib.last_kernel() == before


def test_more_than_2_31_elements():
    """(2^21 + 8) rows of 1024 bf16 features: 64-bit offsets; the first and last rows against the oracle."""
    K, N = 1024, 2 ** 21 + 8
    assert K * N > 2 ** 31
    torch.manual_seed(0)
    x = torch.randn(N, K, device="cuda", dtype=BF16)
    g = torch.rand(K, device="cuda") + 0.5
    b = torch.randn(K, device="cuda")
    y, mean, rstd = nm._ln_fwd(x, g, b, 1, N, K, 1, 1e-6, False)
    dy = torch.randn_like(x)
    dx, dg, db = nm._ln_bwd(x, dy, g, b, mean, rstd, 1, N, K, 1, 1e-6, False)
    c = Case((4, K), -1, 1, False, BF16, 0)
    gd, bd = g.double().cpu().numpy(), b.double().cpu().numpy()
    for sl in (slice(0, 4), slice(N - 4, N)):
        _check(c, x[sl].double().cpu().numpy(), gd, bd, None, y[sl], None, None, None)
    # dx of the last rows needs only their own statistics
    xl, dyl = x[N - 4:].double().cpu().numpy(), dy[N - 4:].double().cpu().numpy()
    rdx, _, _ = orc.layer_norm_grad(dyl, xl, gd, bd)
    assert np.abs(dx[N - 4:].double().cpu().numpy() - rdx).max() <= 2 ** -7 * max(1.0, np.abs(rdx).max())
    # db is the column sum of dy, over every row
    rdb = dy.float().sum(0).double()
    assert (db.double() - rdb).abs().max().item() <= 1e-4 * dy.float().abs().sum(0).max().item()
    del x, y, dy, dx
    torch.cuda.empty_cache()


def test_blocksparse_matmul_feature_axis_0_end_to_end():
    """layer_norm(bsmm(x, w), axis=0) with BlocksparseMatMul(feature_axis=0), forward and backward, against the float64
    composition of the matmul oracle and the layer norm oracle."""
    from blocksparse_b200 import BlocksparseMatMul
    from oracle.bsmm_oracle import MatmulOracle
    rng = np.random.default_rng(11)
    lay = (rng.random((8, 8)) < 0.4).astype(np.int32)
    np.fill_diagonal(lay, 1)
    bs, N = 32, 256
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=0)
    mo = MatmulOracle(lay, bs, 0)
    W = rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)
    X = rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)
    K = bsmm.o_shape(N)[0]
    G = rng.uniform(0.5, 1.5, K).astype(np.float32)
    B = rng.normal(0, 0.5, K).astype(np.float32)
    DY = rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)
    x, w, g, b = (torch.as_tensor(a).cuda().requires_grad_() for a in (X, W, G, B))
    y = layer_norm(bsmm(x, w), g, b, axis=0, epsilon=1e-5)
    y.backward(torch.as_tensor(DY).cuda())
    h = mo.fprop(X.astype(np.float64), W.astype(np.float64))
    ref = orc.layer_norm(h, G, B, axis=0, epsilon=1e-5)
    dh, rdg, rdb = orc.layer_norm_grad(DY.astype(np.float64), h, G, B, axis=0, epsilon=1e-5)
    rdx = mo.bprop(dh, W.astype(np.float64))
    rdw = mo.updat(X.astype(np.float64), dh)
    for got, r, name in ((y, ref, "y"), (x.grad, rdx, "dx"), (w.grad, rdw, "dw"), (g.grad, rdg, "dg"), (b.grad, rdb, "db")):
        gd = got.detach().double().cpu().numpy().reshape(np.shape(r))
        err = np.abs(gd - r).max() / max(np.abs(r).max(), 1e-30)
        assert err <= 1e-4, "%s: max err %.3e relative to its largest entry" % (name, err)
