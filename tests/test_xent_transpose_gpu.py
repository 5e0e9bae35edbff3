"""softmax_cross_entropy and its gradient on every kernel route, elementwise against the float64 oracle
(tests/_xent_oracle.py), and transpose_0213 / transpose_2d bit for bit against torch.

Routes (csrc/dense_softmax.cuh): softmax_xent[_grad]_warp for rows of <= 1024 entries, _cta beyond; each with 16-byte
loads when the logits are 16-byte aligned and K is a multiple of 16 / element size, one element per load otherwise.
Transposes (csrc/transpose.cuh): transpose_rows for cells of D3 * element size >= 16 bytes, transpose_tile below.

With BSMM_BOUND_LOG naming a file, every bound check appends one JSON line with the largest fraction of the bound used.
"""
import collections
import json
import os
import warnings

import numpy as np
import pytest
import torch

from tests import _xent_oracle as orc
from tests._util import EPS32, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, dtype_name
from blocksparse_b200 import _lib, softmax_cross_entropy, transpose_0213, transpose_2d
from blocksparse_b200 import transformer as tr

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
U8, U16, I32, I64 = torch.uint8, torch.uint16, torch.int32, torch.int64
WARP_MAX, CTA_THREADS = 1024, 256

Case = collections.namedtuple("Case", "shape dtype ldtype")
CASES = [
    Case((5, 1), F32, U8),
    Case((7,), F16, I64),                      # rank 1
    Case((3, 4, 10), BF16, U8),
    Case((5, 8), F16, I32),
    Case((6, 256), F16, U16),
    Case((64, 1000), F32, U16),
    Case((2, 3, 1024), BF16, I32),
    Case((9, 1025), F32, I64),
    Case((2, 2, 8192), F16, I32),
    Case((2, 3, 50257), BF16, U16),
    Case((4, 50257), F16, I64),
    Case((3, 65536), F32, I32),
    Case((3, 131072), BF16, I64),
]


def _route(K):
    return "warp" if K <= WARP_MAX else "cta"


def _vec_width(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def _case_id(c):
    return "%s-%s-%s" % ("x".join(map(str, c.shape)), dtype_name(c.dtype), dtype_name(c.ldtype))


def test_cases_cover_every_route():
    ks = {c.shape[-1] for c in CASES}
    assert {1, 7, 10, 256, 1024, 1025, 8192, 50257, 65536, 131072} <= ks
    routes = {(_route(c.shape[-1]), c.shape[-1] % _vec_width(c.dtype) == 0) for c in CASES}
    assert routes == {(r, v) for r in ("warp", "cta") for v in (True, False)}
    assert {c.dtype for c in CASES} == {F32, F16, BF16} and {c.ldtype for c in CASES} == {U8, U16, I32, I64}
    assert {len(c.shape) for c in CASES} == {1, 2, 3}


# ---- bounds -------------------------------------------------------------------------------------------------------------
def _log_ratio(what, ratio):
    log = os.environ.get("BSMM_BOUND_LOG")
    if log:
        with open(log, "a") as f:
            f.write(json.dumps({"family": "softmax_xent", "what": what, "ratio": ratio}) + "\n")


def lse_bound(x, lse, K, vec):
    """Largest |got - lse| of the kernel's fp32 log-sum-exp, per row, in units of eps32:
    * each exponential expf(fl(x - m)): the subtraction rounds once (<= A, the range of the row's finite entries) and
      expf is within 2 ulp (4): A + 4, relative to each term and so to the sum;
    * the rescales s *= expf(m - m'): 5 each plus |m - m'|, whose sum over a thread telescopes to <= A; the final
      rescale to the row max another A + 5;
    * the additions: per_thread serial ones, 5 shuffle levels, 7 warp partials;
    * logf: 2 ulp of log S <= log K (4 log K), and M + log S: one rounding of |lse|.
    A relative error of S is an absolute error of log S; a 2^-10 margin covers second-order terms."""
    threads = 32 if K <= WARP_MAX else CTA_THREADS
    per_thread = -(-K // threads)
    chunks = -(-per_thread // vec)
    fin = np.where(np.isfinite(x), x, np.nan)
    with np.errstate(all="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)            # rows without a finite entry
        A = np.nan_to_num(np.nanmax(fin, axis=-1) - np.nanmin(fin, axis=-1))
    units = np.abs(lse) + 4 * np.log(K) + 3 * A + 4 + 5 * chunks + 10 + per_thread + 12
    return EPS32 * units * (1 + 2.0 ** -10)


def _check_forward(loss, lse, x, labels, vec, what):
    xd = x.double().cpu().numpy()
    lab = labels.cpu().to(torch.int64).numpy()
    ref_loss, ref_lse = orc.softmax_cross_entropy(xd, lab)
    g_loss, g_lse = loss.double().cpu().numpy(), lse.double().cpu().numpy()
    assert loss.dtype == lse.dtype == F32 and loss.shape == x.shape[:-1]
    # NaN and infinities exactly where the oracle has them
    for g, r, name in ((g_loss, ref_loss, "loss"), (g_lse, ref_lse, "lse")):
        assert np.array_equal(np.isnan(g), np.isnan(r)), "%s: %s NaN pattern differs" % (what, name)
        inf = np.isinf(r)
        assert np.array_equal(g[inf], r[inf]), "%s: %s infinities differ" % (what, name)
    ok = np.isfinite(ref_lse)
    K = xd.shape[-1]
    b_lse = lse_bound(xd, ref_lse, K, vec)
    b_loss = b_lse + EPS32 * np.abs(ref_loss)
    worst = 0.0
    for g, r, b, name in ((g_lse, ref_lse, b_lse, "lse"), (g_loss, ref_loss, b_loss, "loss")):
        fin = ok & np.isfinite(r)
        err = np.abs(g[fin] - r[fin])
        assert np.all(err <= b[fin]), "%s: %s: %d rows out of bound, worst %.3e vs %.3e" % (
            what, name, int((err > b[fin]).sum()), float((err - b[fin]).max()), float(b[fin].max()))
        if err.size:
            worst = max(worst, float((err / b[fin]).max()))
    _log_ratio(what + " forward", worst)
    return ref_lse, b_lse


def _check_grad(dx, x, labels, dy, ref_lse, b_lse, what):
    xd = x.double().cpu().numpy()
    lab = labels.cpu().to(torch.int64).numpy().reshape(-1)
    dyd = dy.double().cpu().numpy()
    ref = orc.softmax_cross_entropy_grad(xd, lab, dyd)
    g = dx.double().cpu().numpy()
    assert dx.dtype == x.dtype and dx.shape == x.shape
    assert np.array_equal(np.isnan(g), np.isnan(ref)), "%s: gradient NaN pattern differs" % what
    with np.errstate(all="ignore"):
        p = np.exp(xd - ref_lse[..., None])
        # the kernel's p carries the lse error and its own expf(fl(x - lse)); then - onehot, * dy, one rounding each
        # p = 0 at -inf entries, whose distance to the lse is infinite: no error there
        inner = (np.where(p > 0, p * (b_lse[..., None] + EPS32 * (np.abs(xd - ref_lse[..., None]) + 4)), 0.0) * (1 + 2.0 ** -10)
                 + 2 * EPS32 * np.abs(ref / np.where(dyd == 0, 1, dyd)[..., None]))
        u = U_OUT[dtype_name(x.dtype)]
        bound = u * np.abs(ref) + (1 + u) * np.abs(dyd)[..., None] * inner + SUBNORMAL_FLOOR[dtype_name(x.dtype)]
    fin = np.isfinite(ref)
    err = np.abs(g - ref)
    assert np.all(err[fin] <= bound[fin]), "%s: %d gradient entries out of bound, worst excess %.3e" % (
        what, int((err[fin] > bound[fin]).sum()), float((err[fin] - bound[fin]).max()))
    if fin.any():
        _log_ratio(what + " gradient", float((err[fin] / bound[fin]).max()))


# ---- inputs -------------------------------------------------------------------------------------------------------------
def _labels(shape, K, ldtype, rng):
    lab = rng.integers(0, K, shape)
    flat = lab.reshape(-1)
    flat[0] = 0
    if flat.size > 1:
        flat[-1] = K - 1
    return torch.as_tensor(lab.astype(np.int64)).cuda().to(ldtype)


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().numpy().tobytes()


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_cross_entropy_matches_oracle(idx):
    case = CASES[idx]
    what = _case_id(case)
    K = case.shape[-1]
    rng = np.random.default_rng(300 + idx)
    x = torch.as_tensor(rng.normal(0, 3, case.shape).astype(np.float32)).to(case.dtype).cuda()
    labels = _labels(case.shape[:-1], K, case.ldtype, rng)
    vec = K % _vec_width(case.dtype) == 0
    flat_lab = labels.reshape(-1)
    loss, lse = _on_poisoned_output(lambda: tr._xent_fwd(x.contiguous(), flat_lab))
    assert _lib.last_kernel() == "softmax_xent_" + _route(K), (what, _lib.last_kernel())
    ref_lse, b_lse = _check_forward(loss, lse, x, labels, _vec_width(case.dtype) if vec else 1, what)
    loss2, lse2 = tr._xent_fwd(x.contiguous(), flat_lab)
    assert _bits(loss2) == _bits(loss) and _bits(lse2) == _bits(lse), "%s: forward not bitwise reproducible" % what

    dy = torch.as_tensor(rng.uniform(0.25, 2.0, case.shape[:-1]).astype(np.float32)).cuda()   # non-uniform
    dx = _on_poisoned_output(lambda: tr._xent_bwd(x, flat_lab, lse, dy))
    assert _lib.last_kernel() == "softmax_xent_grad_" + _route(K), (what, _lib.last_kernel())
    _check_grad(dx, x, labels, dy, ref_lse, b_lse, what)
    assert _bits(tr._xent_bwd(x, flat_lab, lse, dy)) == _bits(dx), "%s: gradient not bitwise reproducible" % what

    # the public op and autograd
    xg = x.clone().requires_grad_()
    out = softmax_cross_entropy(logits=xg, labels=labels)
    assert out.shape == case.shape[:-1] and out.dtype == F32
    assert _bits(out) == _bits(loss.view(out.shape))
    out.backward(dy.view(out.shape))
    assert _bits(xg.grad) == _bits(dx)


@pytest.mark.parametrize("K,dtype,offset", [(4096, F16, 1), (1000, BF16, 3), (2048, F32, 1)])
def test_unaligned_view_takes_the_scalar_path(K, dtype, offset):
    """logits at an odd element offset run the one-element-per-load kernels and match the oracle and the aligned call;
    a non-contiguous input is made contiguous and gives the same bits as its contiguous copy."""
    rng = np.random.default_rng(K + offset)
    shape = (4, K)
    src = torch.as_tensor(rng.normal(0, 3, shape).astype(np.float32)).to(dtype).cuda()
    buf = torch.zeros(src.numel() + offset, dtype=dtype, device="cuda")
    x = buf[offset:].view(shape)
    x.copy_(src)
    assert x.data_ptr() % 16
    labels = _labels(shape[:-1], K, I64, rng)
    loss, lse = tr._xent_fwd(x, labels)
    _check_forward(loss, lse, x, labels, 1, "offset %d" % offset)
    dy = torch.full(shape[:-1], 0.7, device="cuda")
    dx = tr._xent_bwd(x, labels, lse, dy)
    ref_lse, b_lse = _check_forward(loss, lse, x, labels, 1, "offset %d" % offset)
    _check_grad(dx, x, labels, dy, ref_lse, b_lse, "offset %d grad" % offset)
    xt = src.t().contiguous().t()
    assert not xt.is_contiguous()
    assert _bits(softmax_cross_entropy(xt, labels)) == _bits(softmax_cross_entropy(src, labels))


def test_infinite_logits():
    """-inf filling whole threads' chunks (thread 0's included) on both routes and both access widths, a label at a
    -inf entry, and an all -inf row: loss, lse and gradient as the oracle, NaN and infinities included."""
    for K, dtype in ((2048, F16), (2049, BF16), (512, F32), (515, F16)):
        rng = np.random.default_rng(K)
        xn = rng.normal(0, 3, (6, K)).astype(np.float32)
        xn[0, : K // 2] = -np.inf                     # threads 0 .. half of the row see only -inf
        xn[1, ::2] = -np.inf
        chunk = _vec_width(dtype) if K % _vec_width(dtype) == 0 else 1
        t = 32 if K <= WARP_MAX else CTA_THREADS
        for c in range(0, K, chunk):                  # every chunk of the even threads, thread 0's included
            if (c // chunk) % t % 2 == 0:
                xn[2, c: c + chunk] = -np.inf
        xn[3] = -np.inf                               # all -inf
        xn[4, 5] = -np.inf                            # its label points at -inf: +inf
        xn[5, 1:] = -np.inf                           # one finite entry
        x = torch.as_tensor(xn).to(dtype).cuda()
        lab = torch.tensor([K - 1, 1, K - 1, 0, 5, 0], device="cuda")
        loss, lse = _on_poisoned_output(lambda: tr._xent_fwd(x, lab))
        ref_lse, b_lse = _check_forward(loss, lse, x, lab, chunk, "inf K %d" % K)
        g = loss.cpu().numpy()
        assert np.isnan(g[3]) and np.isposinf(g[4]) and g[5] == 0.0 and np.isneginf(lse[3].item())
        dy = torch.linspace(0.5, 1.5, 6, device="cuda")
        dx = _on_poisoned_output(lambda: tr._xent_bwd(x, lab, lse, dy))
        _check_grad(dx, x, lab, dy, ref_lse, b_lse, "inf K %d grad" % K)
        d = dx.float().cpu().numpy()
        assert np.all(d[0, : K // 2] == 0) and np.all(np.isnan(d[3])) and not np.isnan(np.delete(d, 3, 0)).any()


@pytest.mark.parametrize("ldtype,K,badval", [(I32, 300, 300), (I64, 1100, 1100), (U8, 100, 255), (U8, 255, 255),
                                             (I32, 50257, -1), (I64, 64, -1), (U16, 2000, 65535)])
def test_out_of_range_labels_give_nan_rows_only(ldtype, K, badval):
    rng = np.random.default_rng(K)
    x = torch.as_tensor(rng.normal(0, 2, (5, K)).astype(np.float32)).to(F16).cuda()
    lab = rng.integers(0, min(K, 255), 5)
    lab[[1, 3]] = badval
    labels = torch.as_tensor(lab).cuda().to(ldtype)
    loss, lse = tr._xent_fwd(x, labels)
    dx = tr._xent_bwd(x, labels, lse, torch.ones(5, device="cuda"))
    torch.cuda.synchronize()                          # no fault
    g, d = loss.cpu().numpy(), dx.float().cpu().numpy()
    bad = np.array([False, True, False, True, False])
    assert np.all(np.isnan(g[bad])) and np.all(np.isnan(lse.cpu().numpy()[bad])) and np.all(np.isnan(d[bad]))
    assert np.all(np.isfinite(g[~bad])) and np.all(np.isfinite(d[~bad]))
    ref_lse, b_lse = _check_forward(loss, lse, x, labels, 8 if K % 8 == 0 else 1, "bad labels")
    _check_grad(dx, x, labels, torch.ones(5, device="cuda"), ref_lse, b_lse, "bad labels grad")


def test_empty_inputs_launch_nothing():
    before = _lib.last_kernel()
    x = torch.empty(0, 7, device="cuda", dtype=F16, requires_grad=True)
    out = softmax_cross_entropy(x, torch.empty(0, device="cuda", dtype=I64))
    assert out.shape == (0,) and out.dtype == F32
    out.sum().backward()
    assert x.grad.shape == x.shape
    assert _lib.last_kernel() == before


# ---- transposes ---------------------------------------------------------------------------------------------------------
def _int_view(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _tr_route(D3, dtype):
    return "transpose_rows" if D3 * torch.empty((), dtype=dtype).element_size() >= 16 else "transpose_tile"


TR_SHAPES = [(2, 33, 31, D3) for D3 in (1, 2, 3, 8, 64, 128, 129)] + [(3, 7, 65, 5), (1, 1, 37, 4), (2, 45, 1, 6)]


@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=dtype_name)
@pytest.mark.parametrize("shape", TR_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_transpose_0213_is_a_bitwise_copy(shape, dtype):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = torch.randn(shape, device="cuda", generator=g).to(dtype)
    y = _on_poisoned_output(lambda: transpose_0213(x))
    assert _lib.last_kernel() == _tr_route(shape[3], dtype), (shape, dtype, _lib.last_kernel())
    ref = x.permute(0, 2, 1, 3).contiguous()
    assert y.shape == ref.shape and y.dtype == dtype
    assert torch.equal(_int_view(y), _int_view(ref))
    xg = x.clone().requires_grad_()
    dy = torch.randn(ref.shape, device="cuda", generator=g).to(dtype)
    transpose_0213(xg).backward(dy)
    assert torch.equal(_int_view(xg.grad), _int_view(dy.permute(0, 2, 1, 3).contiguous()))


@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=dtype_name)
@pytest.mark.parametrize("shape", [(1, 1), (33, 31), (64, 96), (1000, 3), (3, 70001), (65537, 5)], ids=lambda s: "x".join(map(str, s)))
def test_transpose_2d_is_a_bitwise_copy(shape, dtype):
    g = torch.Generator(device="cuda").manual_seed(shape[0])
    x = torch.randn(shape, device="cuda", generator=g).to(dtype)
    y = _on_poisoned_output(lambda: transpose_2d(x))
    assert _lib.last_kernel() == "transpose_tile"
    assert torch.equal(_int_view(y), _int_view(x.t().contiguous()))
    xg = x.clone().requires_grad_()
    dy = torch.randn(shape[::-1], device="cuda", generator=g).to(dtype)
    transpose_2d(xg).backward(dy)
    assert torch.equal(_int_view(xg.grad), _int_view(dy.t().contiguous()))


@pytest.mark.parametrize("shape,dtype", [((70000, 3, 2, 1), F16), ((65537, 2, 3, 8), BF16), ((1, 65537, 3, 2), F32),
                                         ((2, 70001, 2, 16), F16)], ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else dtype_name(v))
def test_transpose_0213_large_leading_dims(shape, dtype):
    """D0 or D1 >= 65536 (the reference's limit) with small other dims."""
    x = torch.randn(shape, device="cuda").to(dtype)
    y = transpose_0213(x)
    assert _lib.last_kernel() == _tr_route(shape[3], dtype)
    assert torch.equal(_int_view(y), _int_view(x.permute(0, 2, 1, 3).contiguous()))


@pytest.mark.parametrize("D3,dtype,offset", [(64, F16, 1), (12, F16, 2), (3, F32, 1), (1, BF16, 3), (129, BF16, 1), (10, F32, 2)])
def test_transpose_unaligned_views(D3, dtype, offset):
    """A view at an odd offset takes narrower words on the row route; the tile route has no alignment requirement."""
    shape = (2, 9, 17, D3)
    n = int(np.prod(shape))
    buf = torch.randn(n + offset, device="cuda").to(dtype)
    x = buf[offset:].view(shape)
    assert x.data_ptr() % 16
    y = transpose_0213(x)
    assert _lib.last_kernel() == _tr_route(D3, dtype)
    assert torch.equal(_int_view(y), _int_view(x.permute(0, 2, 1, 3).contiguous()))
    # a destination that is not 16-byte aligned, through the C entry
    ybuf = torch.zeros(n + 1, device="cuda", dtype=dtype)
    rc = _lib.load().bst_transpose_0213(_lib.dtype_code(dtype), x.data_ptr(), ybuf[1:].data_ptr(), *shape, _lib.stream_ptr())
    assert rc == 0
    assert torch.equal(_int_view(ybuf[1:].view(y.shape)), _int_view(y))


def test_transpose_empty_and_non_contiguous():
    before = _lib.last_kernel()
    for shape in [(0, 3, 4, 5), (2, 0, 4, 5), (2, 3, 0, 5), (2, 3, 4, 0)]:
        y = transpose_0213(torch.empty(shape, device="cuda", dtype=BF16))
        assert y.shape == (shape[0], shape[2], shape[1], shape[3])
    assert transpose_2d(torch.empty(0, 5, device="cuda")).shape == (5, 0)
    assert _lib.last_kernel() == before
    x = torch.randn(4, 6, 5, 8, device="cuda", dtype=F16)
    xt = x.transpose(1, 2)
    assert not xt.is_contiguous()
    assert torch.equal(_int_view(transpose_0213(xt)), _int_view(x))
    m = torch.randn(40, 30, device="cuda")
    assert torch.equal(transpose_2d(m.t()), m)
