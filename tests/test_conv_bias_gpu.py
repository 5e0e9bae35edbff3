"""ConvEdgeBias and cwise_linear on the GPU, elementwise against the float64 oracle (oracle/conv_bias_oracle.py) with
per-element bounds derived from the rounding: every edge fixture in every dtype at N = 0, 1, 3 and 32 (forward,
inference in place, dx / dg / db through autograd); cwise_linear at every combination of gain, bias, relu and
bias_first, ranks 2 to 5 and C from 1 to 1024; bitwise reproducibility (two runs, an SM margin); the kernel names; and
both ops against the reference's own kernels (oracle/ref/conv_bias.cu, oracle/ref/cwise_linear.cu)."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv_bias import ConvEdgeBias, cwise_linear
from oracle import conv_bias_oracle as cbo
from tests._util import ROOT
from tests.test_conv_bias_oracle import EDGE, edge_args
from tests._util import GOLDEN

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DTYPES = [F32, F16, BF16]
EPS = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}
TINY = {F32: 2.0 ** -150, F16: 2.0 ** -25, BF16: 2.0 ** -134}
U = 2.0 ** -24
ids = lambda d: str(d).split(".")[-1]


def rand(shape, dtype, seed, lo=-1.0):
    g = np.random.default_rng(seed)
    return torch.as_tensor(g.uniform(lo, 1, shape).astype(np.float32)).to(dtype)


def np64(t):
    return t.detach().double().cpu().numpy()


def assert_within(got, ref, lim, what):
    err = np.abs(np64(got).reshape(ref.shape) - ref)
    bad = err > lim
    assert not bad.any(), "%s: %d bad of %d, worst %.3e vs bound %.3e" % (
        what, bad.sum(), bad.size, err[bad].max(), lim[bad][np.argmax(err[bad])])


def make_edge(name):
    z = np.load(os.path.join(GOLDEN, name))
    args = edge_args(z)
    return ConvEdgeBias(*args), cbo.EdgeBias(*args), z["io_shape"].tolist()


def edge_case(name, N, dt, seed=0):
    op, orc, io = make_edge(name)
    shape = [N] + io[1:]
    x, dy = rand(shape, dt, seed).cuda(), rand(shape, dt, seed + 1).cuda()
    g, b = rand(op.shape, F32, seed + 2).cuda(), rand(op.shape, F32, seed + 3).cuda()
    return op, orc, x, dy, g, b


@pytest.mark.parametrize("name", EDGE)
@pytest.mark.parametrize("N", [0, 1, 3, 32])
@pytest.mark.parametrize("dt", DTYPES, ids=ids)
def test_edge_bias_against_oracle(name, N, dt):
    op, orc, x, dy, g, b = edge_case(name, N, dt, seed=N)
    xv, gv, bv, dv = np64(x), np64(g), np64(b), np64(dy)
    xr = x.clone().requires_grad_()
    gr, br = g.clone().requires_grad_(), b.clone().requires_grad_()
    y = op(xr, gr, br)
    assert y.dtype == dt and y.shape == x.shape
    ref = orc.edge_bias(xv, gv, bv)
    mag = orc.edge_bias(np.abs(xv), np.abs(gv), np.abs(bv))
    assert_within(y, ref, (U + EPS[dt]) * mag + TINY[dt], "y")
    y.backward(dy)
    rdx, rdg, rdb = orc.edge_bias_grad(dv, xv, gv)
    mdx, mdg, mdb = orc.edge_bias_grad(np.abs(dv), np.abs(xv), np.abs(gv))
    assert xr.grad.dtype == dt and gr.grad.dtype == F32 and tuple(gr.grad.shape) == op.shape
    assert_within(xr.grad, rdx, (U + EPS[dt]) * mdx + TINY[dt], "dx")
    L = N * op._max_count + 64
    assert_within(gr.grad, rdg, (L + 1) * U * mdg, "dg")
    assert_within(br.grad, rdb, (L + 1) * U * mdb, "db")
    # inference: in place, edge positions only
    xi = x.clone()
    with torch.no_grad():
        out = op(xi, g, b, inference=True)
    assert out is xi
    assert_within(xi, ref, (U + EPS[dt]) * mag + TINY[dt], "inference")
    off, P = torch.as_tensor(op._pos_edge < 0).cuda(), len(op._pos_edge)
    flat = (lambda t: t.reshape(N, P, op.K)[:, off]) if op.layout else (lambda t: t.reshape(N, op.K, P)[:, :, off])
    assert torch.equal(flat(xi), flat(x))


def test_edge_bias_no_edges_returns_x():
    op = ConvEdgeBias([2, 6, 6, 4], [2, 8, 8, 4], [3, 3, 4, 4], padding="VALID")
    x = rand([2, 6, 6, 4], F32, 0).cuda()
    g = torch.zeros(op.shape, device="cuda")
    assert op(x, g, g) is x


def test_edge_bias_errors():
    op, _, x, dy, g, b = edge_case("edge_bias_stride2.npz", 2, F32)
    with pytest.raises(ValueError):
        op(x, g.double(), b)
    with pytest.raises(ValueError):
        op(x, g.t().contiguous() if g.shape[0] != g.shape[1] else g[:1], b)
    with pytest.raises(ValueError):
        op(x[:, :, :, :-1], g, b)
    with pytest.raises(ValueError):
        op(x.requires_grad_(), g, b, inference=True)
    with pytest.raises(ValueError):
        op(x.detach(), g.cpu(), b)


# ---- cwise_linear -------------------------------------------------------------------------------------------------------
CW_SHAPES = [(37, 1024), (33, 5), (5, 3, 77), (4, 64, 9, 8), (2, 1, 3, 4, 5), (0, 6, 7)]
COMBOS = [(a, b, r, s) for a in (False, True) for b in (False, True) for r in (False, True) for s in (False, True)
          if a or b]


def cw_reference(x, a, b, relu, swap, dy, y_saved):
    """(y, dx, da, db) in float64 with their magnitudes, and the elements whose relu mask the fp32 forward may set
    differently (|z| within its rounding); without a gain the mask is read from the kernel's own y, as the op does."""
    A = 1.0 if a is None else cbo._bcast(x, a)
    B = 0.0 if b is None else cbo._bcast(x, b)
    z = A * (x + B) if swap else A * x + B
    zm = np.abs(A) * (np.abs(x) + np.abs(B)) + (0 if swap else np.abs(B))
    amb = np.abs(z) <= 4 * U * zm if (relu and a is not None) else np.zeros(x.shape, bool)
    y = np.maximum(z, 0) if relu else z
    if relu:
        d = dy * (z > 0) if a is not None else dy * (y_saved > 0)
    else:
        d = dy
    axes = tuple(i for i in range(x.ndim) if i != 1)
    dx = A * d
    if swap:
        ta, tb = d * (x + B), dx
        ma, mb = np.abs(dy) * (np.abs(x) + np.abs(B)), np.abs(dy) * np.abs(A)
    else:
        ta, tb = d * x, d
        ma, mb = np.abs(dy * x), np.abs(dy)
    ma_amb, mb_amb = np.where(amb, ma, 0), np.where(amb, mb, 0)
    return (y, zm, amb, dx, np.abs(A * dy), np.sum(ta, axis=axes), np.sum(ma, axis=axes), np.sum(ma_amb, axis=axes),
            np.sum(tb, axis=axes), np.sum(mb, axis=axes), np.sum(mb_amb, axis=axes))


@pytest.mark.parametrize("shape", CW_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES, ids=ids)
@pytest.mark.parametrize("gain,bias,relu,swap", COMBOS)
def test_cwise_linear_against_oracle(shape, dt, gain, bias, relu, swap):
    C = shape[1]
    x, dy = rand(shape, dt, 1).cuda(), rand(shape, dt, 2).cuda()
    a = rand([1, C] + [1] * (len(shape) - 2), F32, 3).cuda() if gain else None
    b = rand([C], F32, 4).cuda() if bias else None
    xr = x.clone().requires_grad_()
    ar = a.clone().requires_grad_() if gain else None
    br = b.clone().requires_grad_() if bias else None
    y = cwise_linear(xr, ar, br, relu=relu, bias_first=swap)
    assert y.dtype == dt and y.shape == x.shape
    y.backward(dy)
    xv, dv = np64(x), np64(dy)
    an, bn = (np64(a).ravel() if gain else None), (np64(b) if bias else None)
    (ry, zm, amb, rdx, mdx, rda, mda, mda_amb, rdb, mdb, mdb_amb) = cw_reference(xv, an, bn, relu, swap, dv, np64(y))
    assert_within(y, ry, 2 * U * zm + EPS[dt] * np.abs(ry) + TINY[dt], "y")
    dx = np64(xr.grad).reshape(shape)
    keep = ~amb
    lim = (U + EPS[dt]) * mdx + TINY[dt]
    assert (np.abs(dx - rdx)[keep] <= lim[keep]).all(), "dx: worst %.3e" % np.abs(dx - rdx)[keep].max(initial=0)
    L = int(np.prod(shape)) // max(C, 1) + 64
    if gain:
        assert ar.grad.shape == a.shape and ar.grad.dtype == F32
        assert_within(ar.grad.view(-1), rda, (L + 2) * U * mda + mda_amb, "da")
    if bias:
        assert br.grad.shape == b.shape and br.grad.dtype == F32
        assert_within(br.grad, rdb, (L + 2) * U * mdb + mdb_amb, "db")


def test_cwise_linear_saves_what_the_reference_saves():
    x = rand([4, 8, 5], BF16, 0).cuda().requires_grad_()
    a, b = rand([8], F32, 1).cuda().requires_grad_(), rand([8], F32, 2).cuda().requires_grad_()
    y = cwise_linear(x, a, b, relu=True)
    assert y.grad_fn.saved_tensors[0].data_ptr() == x.data_ptr()
    y = cwise_linear(x, None, b, relu=True)
    assert y.grad_fn.saved_tensors[0].data_ptr() == y.data_ptr()
    y = cwise_linear(x, None, b)
    assert y.grad_fn.saved_tensors[0] is None
    dy = rand([4, 8, 5], BF16, 3).cuda()
    (dx,) = torch.autograd.grad(y, x, dy)
    assert dx.data_ptr() == dy.data_ptr()                      # no gain, no relu: dx is dy


def test_cwise_linear_errors():
    x = rand([2, 4, 3], F32, 0).cuda()
    for kw in (dict(), dict(gain=torch.ones(5, device="cuda")), dict(bias=torch.ones(4, device="cuda").half()),
               dict(bias=torch.ones(4)), dict(gain=torch.ones(4, device="cuda"), use_tf=True)):
        with pytest.raises(ValueError):
            cwise_linear(x, **kw)
    with pytest.raises(ValueError):
        cwise_linear(x[0, 0], bias=torch.ones(3, device="cuda"))


# ---- reproducibility and kernel names -----------------------------------------------------------------------------------
def _bits(t):
    return t.detach().cpu().view(torch.int16 if t.element_size() == 2 else torch.int32).numpy().tobytes()


def digests():
    out = []
    for name in ("edge_bias_ref_k24_nchw.npz", "edge_bias_conv3d.npz", "edge_bias_stride2.npz"):
        op, _, x, dy, g, b = edge_case(name, 32, BF16, seed=5)
        xr, gr, br = x.requires_grad_(), g.requires_grad_(), b.requires_grad_()
        y = op(xr, gr, br)
        y.backward(dy)
        out += [_bits(t) for t in (y, xr.grad, gr.grad, br.grad)]
    for shape in ((4096, 64), (16, 64, 33, 31)):
        x, dy = rand(shape, BF16, 6).cuda().requires_grad_(), rand(shape, BF16, 7).cuda()
        a = rand([shape[1]], F32, 8).cuda().requires_grad_()
        b = rand([shape[1]], F32, 9).cuda().requires_grad_()
        y = cwise_linear(x, a, b, relu=True, bias_first=True)
        y.backward(dy)
        out += [_bits(t) for t in (y, x.grad, a.grad, b.grad)]
    return out


def margin_digest():
    h = hashlib.sha256()
    for d in digests():
        h.update(d)
    return h.hexdigest()


def test_bitwise_reproducible():
    assert digests() == digests()


def test_bitwise_under_sm_margin():
    code = ("import sys; sys.path.insert(0, %r); from tests.test_conv_bias_gpu import margin_digest; "
            "print(margin_digest())" % ROOT)
    outs = []
    for margin in ("0", "16"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, BSMM_SM_MARGIN=margin), cwd=ROOT,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(r.stdout.split()[-1])
    assert outs[0] == outs[1] == margin_digest()


def test_kernel_names():
    """The names are thread-local and autograd runs backward on its own thread: the gradients are called directly."""
    from blocksparse_b200.conv_bias import _cwise_linear_grad
    op, _, x, dy, g, b = edge_case("edge_bias_ref_k24_nhwc.npz", 2, F16)
    op(x, g, b)
    assert _lib.last_kernel() == "edge_bias"
    op._backward(dy, x, g)
    assert _lib.last_kernel() == "edge_bias_grad"
    with torch.no_grad():
        op(x, g, b, inference=True)
    assert _lib.last_kernel() == "edge_bias_inference"
    for shape, name in (((8, 16), "cwise_linear_grad_nc"), ((8, 16, 3), "cwise_linear_grad_ncdhw")):
        x = rand(shape, F16, 0).cuda()
        a = torch.ones(16, device="cuda")
        cwise_linear(x, a)
        assert _lib.last_kernel() == "cwise_linear"
        _cwise_linear_grad(x, x, a, None, False, False)
        assert _lib.last_kernel() == name


# ---- against the reference's own kernels ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", EDGE)
@pytest.mark.parametrize("dt", DTYPES, ids=ids)
def test_edge_bias_against_reference_kernels(name, dt):
    """Both round x * g + b in fp32 once to dt; the reference's kernels may or may not contract it to an FMA and add
    dg / db in another order, so they agree to the fp32 sums' rounding, not bit for bit."""
    from oracle import ref_conv_bias as rcb
    why = rcb.missing()
    if why:
        pytest.skip(why)
    op, orc, x, dy, g, b = edge_case(name, 3, dt, seed=11)
    xr, gr, br = x.clone().requires_grad_(), g.clone().requires_grad_(), b.clone().requires_grad_()
    y = op(xr, gr, br)
    y.backward(dy)
    xv, gv, bv, dv = np64(x), np64(g), np64(b), np64(dy)
    mag = orc.edge_bias(np.abs(xv), np.abs(gv), np.abs(bv))
    assert_within(y, np64(rcb.edge_bias(op, x, g, b)), 2 * (U + EPS[dt]) * mag + 2 * TINY[dt], "y")
    assert_within(y, np64(rcb.edge_bias(op, x, g, b, inference=True)), 2 * (U + EPS[dt]) * mag + 2 * TINY[dt],
                  "inference")
    rdx, rdg, rdb = rcb.edge_bias_grad(op, dy, x, g)
    mdx, mdg, mdb = orc.edge_bias_grad(np.abs(dv), np.abs(xv), np.abs(gv))
    assert_within(xr.grad, np64(rdx), 2 * (U + EPS[dt]) * mdx + 2 * TINY[dt], "dx")
    L = 2 * (3 * op._max_count + 64)
    assert_within(gr.grad, np64(rdg), L * U * mdg, "dg")
    assert_within(br.grad, np64(rdb), L * U * mdb, "db")


@pytest.mark.parametrize("shape", [(64, 64, 32), (8, 64, 16, 16), (8, 64, 8, 8, 8), (128, 96)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES, ids=ids)
@pytest.mark.parametrize("gain,bias,relu,swap", [c for c in COMBOS if not (c[2] and not c[0])] + [(False, True, True, False)])
def test_cwise_linear_against_reference_kernels(shape, dt, gain, bias, relu, swap):
    from oracle import ref_conv_bias as rcb
    why = rcb.missing()
    if why:
        pytest.skip(why)
    C = shape[1]
    x, dy = rand(shape, dt, 21).cuda(), rand(shape, dt, 22).cuda()
    a = rand([C], F32, 23).cuda() if gain else None
    b = rand([C], F32, 24).cuda() if bias else None
    xr = x.clone().requires_grad_()
    ar = a.clone().requires_grad_() if gain else None
    br = b.clone().requires_grad_() if bias else None
    y = cwise_linear(xr, ar, br, relu=relu, bias_first=swap)
    y.backward(dy)
    ry = rcb.cwise_linear(x, a, b, relu, swap)
    xv, dv = np64(x), np64(dy)
    an, bn = (np64(a) if gain else None), (np64(b) if bias else None)
    (_, zm, amb, _, mdx, _, mda, mda_amb, _, mdb, mdb_amb) = cw_reference(xv, an, bn, relu, swap, dv, np64(y))
    assert_within(y, np64(ry), 4 * U * zm + 2 * EPS[dt] * zm + 2 * TINY[dt], "y")
    rdx, rda, rdb = rcb.cwise_linear_grad(dy, x if gain else ry, a, b, relu, swap)
    keep = ~amb
    err = np.abs(np64(xr.grad) - np64(rdx))
    lim = 2 * (U + EPS[dt]) * mdx + 2 * TINY[dt]
    assert (err[keep] <= lim[keep]).all(), "dx: worst %.3e" % err[keep].max(initial=0)
    L = 2 * (int(np.prod(shape)) // C + 64)
    if gain:
        assert_within(ar.grad, np64(rda), L * U * mda + 2 * mda_amb, "da")
    if bias:
        assert_within(br.grad, np64(rdb), L * U * mdb + 2 * mdb_amb, "db")
