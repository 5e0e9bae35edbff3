"""The reference's own CUDA kernels (oracle/_ref/libbsref.so, built by oracle/ref/Makefile) next to ours and next to the
float64 oracles, on the same inputs, for bias + activation, dropout apply, the grad filter, embedding and the transposes.

Each case checks (a) that the oracle describes the reference: the reference kernel against the oracle within the bound
the family's own test applies to our kernel, widened only for the reference's own arithmetic, as noted where it
happens; (b) that ours equals the reference: bit for bit where both sides are exact, else within the bounds of (a);
(c) that the reference quirks DESIGN.md states hold for the reference as built. Every reference output carries a
poisoned guard region that must come back untouched (oracle/ref_kernels.py)."""
import numpy as np
import pytest
import torch

from blocksparse_b200 import bias_relu, dropout, embedding_lookup, set_entropy, transpose_0213, transpose_2d
from oracle import ewops_oracle as eo
from oracle import optimize_oracle
from oracle import ref_kernels as rk
from tests.test_execution_context_gpu import _gen, _same

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not rk.available(), reason="oracle/_ref/libbsref.so not built (no reference checkout)")]
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DTYPES = [F32, F16, BF16]
EPS = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}      # half an ulp, relative
TINY = {F32: 2.0 ** -149, F16: 2.0 ** -24, BF16: 2.0 ** -133}
U = 2.0 ** -24
ACTS = ["none", "relu", "fast_gelu"]


def _np(t):
    return t.detach().double().cpu().numpy()


def _check(got, ref, tol, what):
    got = _np(got) if torch.is_tensor(got) else got
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN in different places" % what
    bad = ~(np.abs(got - ref) <= tol) & ~nan & ~((got == ref) & np.isinf(ref))
    assert not bad.any(), "%s: %d of %d out of bounds, worst %s vs %s (tol %s)" % (
        what, bad.sum(), bad.size, got[bad][:3], ref[bad][:3], np.broadcast_to(tol, ref.shape)[bad][:3])


def _same_up_to_nan(a, b, what):
    """Bit for bit, except that any NaN matches any NaN (payloads differ between the kernels and torch)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN in different places" % what
    _same([torch.where(na, torch.zeros_like(a), a)], [torch.where(nb, torch.zeros_like(b), b)], what)


def _same_but_bf16_ties(got, ref, exact, what):
    """got and ref are bf16 roundings of the fp32 values `exact`: equal, except that where exact lies halfway between
    two bf16 values the reference's to_bhalf rounds away from zero and round-to-nearest-even may not."""
    tie = (exact.view(torch.int32) & 0xFFFF) == 0x8000
    diff = got.view(torch.int16) != ref.view(torch.int16)
    assert not bool((diff & ~tie).any()), "%s: %d elements differ off a tie" % (what, int((diff & ~tie).sum()))
    assert _ulp_apart(got, ref, 1), what


def _ulp_apart(a, b, n):
    """|bits(a) - bits(b)| <= n for same-signed 16-bit values (NaN where both are NaN)."""
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    both_nan = torch.isnan(a) & torch.isnan(b)
    return bool((((ia - ib).abs() <= n) | both_nan).all())


# ---- bias + activation ------------------------------------------------------------------------------------------------
def _br_inputs(shape, axis, dt, g):
    K = shape[axis]
    x = torch.randn(shape, generator=g) * 2
    b = torch.randn(K, generator=g).to(dt).float()       # representable in dt, so x = -b below is exact
    bb = b.view((-1,) + (1,) * (len(shape) - 1)) if axis == 0 else b
    # x + b exactly 0 on a quarter of the elements: the relu boundary, where dx must be 0
    x = torch.where(torch.rand(shape, generator=g) < 0.25, -bb.to(dt).float().expand(shape), x)
    return x.to(dt).cuda(), b.cuda(), torch.randn(shape, generator=g).to(dt).cuda()


def _br_bounds(x, b, dy, axis, act, yr, dxr, dbr, reference):
    """Bounds of test_ewops_gpu._br_check; `reference` adds the terms of the reference's own arithmetic: its bf16
    rounding (to_bhalf, ew_op_gpu.h:238, adds half an ulp and truncates, so ties go away from zero: one ulp, not half),
    its fast_gelu (ex2.approx and rcp.approx, ew_op_gpu.h:942, relative error about 2^-22 each, the exponent's rounding
    amplified by |1.702 z|; exp(-1.702 z) overflows to inf below z = -52, giving 0 where the value is below 2^-126 |z|),
    and its db (fp32 atomics or a tree over the rows: any order, so N - 1 roundings)."""
    xn, bn, dn = _np(x), _np(b), _np(dy)
    bb = bn.reshape((-1,) + (1,) * (x.dim() - 1)) if axis == 0 else bn
    z = np.abs(xn) + np.abs(bb)
    e = EPS[x.dtype] * (2 if reference and x.dtype == BF16 else 1)
    ty = e * np.abs(yr) + 4 * U * z + TINY[x.dtype]
    dterm = np.abs(dn) * (1 + 2 * z) if act != "none" else np.abs(dn)
    tdx = e * np.abs(dxr) + 16 * U * dterm + TINY[x.dtype]
    if reference and act == "fast_gelu":
        amp = (4 + 2 * 1.702 * z) * 2.0 ** -22
        zz = xn + bb
        flush = np.where(1.702 * zz < -88.0, 1.0, 0.0)
        ty = ty + amp * np.abs(yr) + flush * np.abs(yr)
        tdx = tdx + amp * dterm + flush * np.abs(dxr)
    K = b.numel()
    N = x.numel() // K
    dsum = dterm.sum(axis=tuple(range(1, x.dim()))) if axis == 0 else dterm.reshape(-1, K).sum(axis=0)
    tdb = EPS[F32] * np.abs(dbr) + (N + 16) * U * dsum + TINY[F32]
    if reference and act == "fast_gelu":
        a = tdx - (e * np.abs(dxr) + 16 * U * dterm + TINY[x.dtype])
        tdb = tdb + (a.sum(axis=tuple(range(1, x.dim()))) if axis == 0 else a.reshape(-1, K).sum(axis=0))
    return ty, tdx, tdb


BR_SHAPES = [((37, 29), -1), ((64, 96), -1), ((1, 40), -1), ((3, 5, 24), -1), ((2000, 36), -1), ((900, 1030), -1),
             ((29, 37), 0), ((96, 64), 0), ((40,), 0), ((40, 1), 0), ((24, 3, 5), 0), ((6, 1000), 0)]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_bias_relu(dt, act):
    """Both axes; K and N multiples of 4 and not; N = 1; x + b = 0 exactly; both db paths of the last axis (atomics
    and partial sums)."""
    g = _gen(7000 + 10 * DTYPES.index(dt) + ACTS.index(act))
    relu = ACTS.index(act)
    for shape, axis in BR_SHAPES:
        what = "%s %s %s axis %d" % (dt, act, shape, axis)
        x, b, dy = _br_inputs(shape, axis, dt, g)
        kw = dict(axis=axis, relu=act == "relu", fast_gelu=act == "fast_gelu")
        xn, bn, dn = _np(x), _np(b), _np(dy)
        yr = eo.bias_relu(xn, bn, **kw)
        dxr, dbr = eo.bias_relu_grad(dn, xn, bn, **kw)
        y_ref = rk.bias_relu(x, b, axis, relu)
        ty, tdx, tdb = _br_bounds(x, b, dy, axis, act, yr, dxr, dbr, reference=True)
        _check(y_ref, yr, ty, what + " reference y")
        src = y_ref if act == "relu" else x
        # On axis 0 the reference's bias_relu_axis_0_grad zeroes its 32 shared partials with no barrier before the
        # other warps store theirs (ew_op_gpu.cu:1053-1090), so with more than one warp per block (over 128 rows, or
        # 128 vectors of 4) a warp's share of db can be lost: its db is compared only where one warp runs.
        N = x.numel() // b.numel()
        racy = axis == 0 and -(-(N // 4 if N % 4 == 0 else N) // 128) > 1
        for atomics in (True, False):
            dx_ref, db_ref = rk.bias_relu_grad(dy, src, b, axis, relu, atomics)
            if act != "none":
                _check(dx_ref, dxr, tdx, what + " reference dx")
            if not racy:
                _check(db_ref, dbr, tdb, what + " reference db atomics=%s" % atomics)
        xl, bl = x.clone().requires_grad_(), b.clone().requires_grad_()
        y = bias_relu(xl, bl, **kw)
        y.backward(dy)
        if act != "fast_gelu" and dt != BF16:
            _same([y, xl.grad], [y_ref, dx_ref], what + " ours vs reference")
        elif act != "fast_gelu":
            # y rounds the exact fp32 x + b (relu of it is exact) once; dx is dy or 0, a copy
            z32 = x.float() + (b.view(-1, *([1] * (x.dim() - 1))) if axis == 0 else b)
            _same_but_bf16_ties(y, y_ref, z32.clamp(min=0) if act == "relu" else z32, what + " ours vs reference y")
            _same([xl.grad], [dx_ref], what + " ours vs reference dx")
        else:
            ty0, tdx0, _ = _br_bounds(x, b, dy, axis, act, yr, dxr, dbr, reference=False)
            _check(y, _np(y_ref), ty + ty0, what + " ours vs reference y")
            _check(xl.grad, _np(dx_ref), tdx + tdx0, what + " ours vs reference dx")
        _check(bl.grad, dbr, tdb, what + " ours db")
        if not racy:
            _check(bl.grad, _np(db_ref), 2 * tdb, what + " ours vs reference db")
        if act == "relu":
            at0 = (_np(x) + (bn.reshape(-1, *([1] * (x.dim() - 1))) if axis == 0 else bn)) == 0
            assert at0.any() and not _np(dx_ref)[at0].any(), what + ": the reference's dx at x + b = 0 is 0"


def test_fast_gelu_extremes():
    """z = +-20, +-60, +-100 and 16-bit infinities. The reference's sigmoid is rcp.approx(1 + ex2.approx(-1.702 z)):
    below z = -52 the exponential overflows and y and dx are exactly 0; at z = +inf dx is dy + (dy inf) (1 - 1) 1.702,
    NaN, as in the float64 oracle; z = -inf gives NaN for y, as inf / inf does in the oracle."""
    zs = [20.0, -20.0, 60.0, -60.0, 100.0, -100.0, float("inf"), float("-inf")]
    for dt in DTYPES:
        x = torch.tensor(zs).to(dt).view(1, -1).repeat(3, 1).cuda()
        b = torch.zeros(len(zs), device="cuda")
        dy = torch.ones_like(x)
        y_ref = rk.bias_relu(x, b, -1, 2)
        dx_ref, _ = rk.bias_relu_grad(dy, x, b, -1, 2)
        with np.errstate(all="ignore"):
            yr = eo.bias_relu(_np(x), _np(b), fast_gelu=True)
            dxr, _ = eo.bias_relu_grad(_np(dy), _np(x), _np(b), fast_gelu=True)
        yn, dxn = _np(y_ref)[0], _np(dx_ref)[0]
        assert np.array_equal(np.isnan(yn), np.isnan(yr[0])) and np.array_equal(np.isnan(dxn), np.isnan(dxr[0])), dt
        assert yn[3] == 0 and yn[5] == 0 and dxn[3] == 0 and dxn[5] == 0, (dt, yn, dxn)
        assert np.isinf(yn[6]) and yn[6] > 0 and np.isnan(dxn[6]), (dt, yn[6], dxn[6])
        xl = x.clone().requires_grad_()
        y = bias_relu(xl, b, fast_gelu=True)
        y.backward(dy)
        fin = np.isfinite(yr[0])
        tol = (2 * EPS[dt] + (4 + 2 * 1.702 * np.abs(yr[0][fin])) * 2.0 ** -22) * np.abs(yn[fin]) + 1e-30
        _check(_np(y)[0][fin], yn[fin], tol, "%s ours vs reference at extremes" % dt)


def test_bias_relu_refuses_what_the_op_refuses():
    x = torch.zeros(4, 5, 6, device="cuda")
    with pytest.raises(ValueError):
        rk.bias_relu(x, torch.zeros(5, device="cuda"), axis=1)
    with pytest.raises(ValueError):
        rk.bias_relu(x, torch.zeros(6, device="cuda", dtype=F16))
    with pytest.raises(ValueError):
        rk.bias_relu(x, torch.zeros(7, device="cuda"))


# ---- dropout ----------------------------------------------------------------------------------------------------------
DROP_CASES = [((64, 96), None), ((37, 29), None), ((1003,), None), ((7, 9, 11), None), ((64, 96), (1, 96)),
              ((8, 33, 16), (1, 33, 1)), ((4, 6, 8, 10), (4, 1, 8, 1)), ((2, 3, 4, 5, 16), (1, 3, 1, 5, 16)),
              ((2, 3, 4, 5, 7), (2, 1, 4, 1, 1)), ((3, 5, 7, 9, 11), (3, 5, 7, 9, 11)), ((5, 1, 33), (1, 1, 33))]


@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_dropout_apply(dt):
    """Masks drawn by our dropout, applied by the reference's ApplyDropoutMask: y and dx equal ours and the oracle's
    where(bit e % 32 of word e / 32, round(fp32(x) * fp32(1 / keep_prob)), 0) bit for bit, on full and broadcast masks
    up to rank 5 and odd sizes, so the mask format carries over."""
    g = _gen(7100 + DTYPES.index(dt))
    set_entropy(4321)
    for shape, ms in DROP_CASES:
        what = "%s %s mask %s" % (dt, shape, ms)
        x = torch.randn(shape, generator=g).to(dt).cuda().requires_grad_()
        dy = torch.randn(shape, generator=g).to(dt).cuda()
        y, mask = dropout(x, 0.7, mask_shape=ms)
        y.backward(dy)
        for src, ours in ((x.detach(), y), (dy, x.grad)):
            ref = rk.apply_dropout_mask(src, mask, 0.7, ms)
            keep = torch.as_tensor(np.ascontiguousarray(eo.broadcast_keep(mask.cpu().numpy(), shape, ms))).cuda()
            scale = torch.tensor(1.0 / 0.7, dtype=F32, device="cuda")
            expect = torch.where(keep, (src.float() * scale).to(dt), torch.zeros((), dtype=dt, device="cuda"))
            if dt == BF16:
                exact = torch.where(keep, src.float() * scale, torch.zeros((), device="cuda"))
                _same_but_bf16_ties(ref, expect, exact, what + " reference vs oracle")
                _same_but_bf16_ties(ours, ref, exact, what + " ours vs reference")
            else:
                _same([ref], [expect], what + " reference vs oracle")
                _same([ours], [ref], what + " ours vs reference")


def test_dropout_keep_prob_zero():
    """DESIGN.md 7f: the reference scales by 1 / keep_prob = inf, so keep_prob = 0 gives NaN (0 * inf) where the mask
    drops, +-inf where it keeps a nonzero x; ours refuses keep_prob = 0."""
    x = torch.tensor([1.0, -2.0, 3.0, -4.0] * 8, device="cuda")
    mask = torch.tensor([0x55555555], dtype=torch.int64).to(torch.int32).cuda()     # keeps the even elements
    y = rk.apply_dropout_mask(x, mask, 0.0).cpu()
    assert torch.isnan(y[1::2]).all() and torch.equal(y[0::2], x[0::2].cpu() * float("inf"))
    with pytest.raises(ValueError):
        dropout(x, 0.0, mask=mask)


def test_dropout_refuses_what_the_op_refuses():
    x = torch.zeros(4, 6, device="cuda")
    m = torch.zeros(1, dtype=torch.int32, device="cuda")
    for ms in ((4, 3), (4,), (1, 1, 6)):
        with pytest.raises(ValueError):
            rk.apply_dropout_mask(x, m, 0.5, ms)
    with pytest.raises(ValueError):
        rk.apply_dropout_mask(x, torch.zeros(2, dtype=torch.int32, device="cuda"), 0.5)
    with pytest.raises(ValueError):
        rk.apply_dropout_mask(torch.zeros(64, device="cuda"), m, 0.5, (1,))


# ---- grad filter ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_filter_tensor(dt):
    """FilterTensor (zero_infs, then zero_nans, then scale, then the clamp to +-saturate) against
    optimize_oracle.condition, bit for bit after rounding the oracle to the dtype, with inf, NaN and values past
    saturate, on both access widths (size % 4 == 0 and not)."""
    g = _gen(7200 + DTYPES.index(dt))
    for n in (1000, 1003, 7):
        x = torch.randn(n, generator=g) * 4
        x[::11] = float("inf")
        x[5::13] = float("-inf")
        x[3::17] = float("nan")
        x = x.to(dt).cuda()
        for sat in (0.0, 3.3):
            for zi in (False, True):
                for zn in (False, True):
                    for scale in (1.0, 0.5):
                        ref = rk.filter_tensor(x, scale, sat, zi, zn)
                        # the clamp runs in fp32, so the bound is fp32(saturate), then rounded to the dtype
                        s32 = float(np.float32(sat))
                        o = optimize_oracle.condition(_np(x) * scale, s32, zi, zn)
                        expect = torch.as_tensor(o).float().to(dt).cuda()
                        _same_up_to_nan(ref, expect, "%s n %d sat %s zi %s zn %s scale %s" % (dt, n, sat, zi, zn, scale))


# ---- embedding --------------------------------------------------------------------------------------------------------
IDX = [torch.int32, torch.uint8] + ([torch.uint16] if hasattr(torch, "uint16") else [])


@pytest.mark.parametrize("idt", IDX, ids=str)
@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_embedding(dt, idt):
    """Lookups bit for bit (out-of-range indices give zero rows on both sides) and, with integer-valued dy, the sorted
    and unsorted gradients bit for bit against ours and the exact sums; C = 50257 where the index dtype reaches it; K
    not a multiple of 8."""
    g = _gen(7300 + 10 * DTYPES.index(dt) + IDX.index(idt))
    top = {torch.int32: 2 ** 31 - 1, torch.uint8: 255}.get(idt, 65535)
    cases = [(200, 20, 3001), (250, 33, 64), (37, 96, 5000)]
    if idt != torch.uint8:
        cases.append((50257, 24, 4099))
    for C, K, n in cases:
        what = "%s %s C %d K %d n %d" % (dt, idt, C, K, n)
        lo = -5 if idt == torch.int32 else 0
        v = torch.randint(lo, min(C + 5, top + 1), (n,), generator=g)
        v[: n // 3] = 7                       # a long run of one row
        idx = v.to(idt).cuda()
        emb = torch.randn(C, K, generator=g).to(dt).cuda()
        dy = torch.randint(-3, 4, (n, K), generator=g).to(dt).cuda()
        y_ref = rk.embedding_lookup(emb, idx)
        ok = ((v >= 0) & (v < C)).cuda()
        rows = emb[v.clamp(0, C - 1).cuda()]
        _same([y_ref], [torch.where(ok[:, None], rows, torch.zeros((), dtype=dt, device="cuda"))], what + " lookup")
        e = emb.clone().requires_grad_()
        y = embedding_lookup(e, idx)
        _same([y], [y_ref], what + " ours vs reference lookup")
        y.backward(dy)
        # integer dy: every fp32 partial sum is exact, so any order of adds gives the exact sums
        exact = torch.as_tensor(eo.embedding_grad(_np(dy), v.numpy(), C)).float().cuda()
        for sorted_ in (True, False):
            dw_ref = rk.embedding_grad(dy, idx, C, sorted_)
            _same([dw_ref], [exact], what + " reference dw sorted=%s" % sorted_)
        _same([e.grad], [exact.to(dt)], what + " ours vs reference dw")


# ---- transposes -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_transposes(dt):
    """Transpose_2D on multiples of 4 (the only sizes its 4 x 4 vector tiles take) and Transpose_0213 on D3 up to and
    past 64, bit for bit against ours and torch's permute."""
    g = _gen(7400 + DTYPES.index(dt))
    for shape in ((4, 8), (64, 128), (132, 68), (100, 260), (1024, 4)):
        x = torch.randn(shape, generator=g).to(dt).cuda()
        ref = rk.transpose_2d(x)
        _same([ref, transpose_2d(x)], [x.t().contiguous(), ref], "%s 2d %s" % (dt, shape))
    for shape in ((2, 5, 3, 64), (1, 7, 9, 65), (3, 2, 130, 200), (2, 3, 5, 1), (1, 1, 17, 31)):
        x = torch.randn(shape, generator=g).to(dt).cuda()
        ref = rk.transpose_0213(x)
        _same([ref, transpose_0213(x)], [x.permute(0, 2, 1, 3).contiguous(), ref], "%s 0213 %s" % (dt, shape))
    with pytest.raises(ValueError):
        rk.transpose_2d(torch.zeros(6, 8, dtype=dt, device="cuda"))
    with pytest.raises(ValueError):
        rk.transpose_0213(torch.zeros(1, 65536, 1, 1, dtype=dt, device="cuda"))


# ---- Adam with 16-bit moments -----------------------------------------------------------------------------------------
def _our_adam(grad, param, mean, var, lr_t, beta1, beta2, eps):
    """One step of our bsmm_adam on clones (the entry AdamOptimizer.step calls), with lr_t given directly."""
    from blocksparse_b200 import _lib
    from blocksparse_b200.optimize import _i32, _i64, _ptrs
    p, m, v = param.clone(), mean.clone(), var.clone()
    arrs = (_ptrs([grad]), _i32([0]), _ptrs([p]), _ptrs([m]), _ptrs([v]), _i32([int(m.dtype == torch.int16)]),
            _i64([p.numel()]), np.zeros(1, dtype=np.uint64), _i32([0]))
    rc = _lib.load().bsmm_adam(1, *[a.ctypes.data for a in arrs], None, float(lr_t), float(beta1), float(beta2),
                               float(eps), 1.0, 0.0, 0.0, 0, 0, _lib.stream_ptr())
    _lib.check(rc, "bsmm_adam")
    torch.cuda.synchronize()
    return p, m, v


def test_adam_every_16_bit_code_round_trips():
    """DESIGN.md 7e: the 16-bit moments hold the reference's codes. All 65536 mean codes and all 65536 variance codes
    through a step that leaves the moments' values unchanged (zero grad, beta1 = beta2 = 1, lr = 0): each side decodes,
    re-encodes and stores, so ours, the reference and the oracle's mean_encode(mean_decode(c)) /
    var_encode(var_decode(c)) must give the same codes bit for bit."""
    n = 65536
    codes = torch.arange(n, dtype=torch.int32).to(torch.int16).cuda()
    var = codes.flip(0).contiguous()
    grad, param = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    _, m_ref, v_ref = rk.apply_adam(grad, param, codes, var, 0.0, 1.0, 1.0, 1e-8)
    _, m_our, v_our = _our_adam(grad, param, codes, var, 0.0, 1.0, 1.0, 1e-8)
    cn, vn = codes.cpu().numpy().view(np.uint16), var.cpu().numpy().view(np.uint16)
    m_orc = optimize_oracle.mean_encode(optimize_oracle.mean_decode(cn)).astype(np.uint16)
    v_orc = optimize_oracle.var_encode(optimize_oracle.var_decode(vn)).astype(np.uint16)
    assert np.array_equal(m_ref.cpu().numpy().view(np.uint16), m_orc), "reference mean codes vs oracle"
    assert np.array_equal(v_ref.cpu().numpy().view(np.uint16), v_orc), "reference var codes vs oracle"
    _same([m_our, v_our], [m_ref, v_ref], "ours vs reference codes")


def test_adam_16_bit_steps_from_shared_state():
    """Ten Adam steps; before each, ours takes the reference's state, so each step starts from identical codes. The
    two differ in arithmetic (the reference takes rcp.approx of sigma + eps), so each new code may sit one code from
    the reference's where the value falls within rounding of a tie; the share of equal codes is printed."""
    g = _gen(7500)
    n = 1 << 16
    p = torch.randn(n, generator=g).cuda()
    m = torch.zeros(n, dtype=torch.int16, device="cuda")
    v = torch.zeros(n, dtype=torch.int16, device="cuda")
    equal = []
    for step in range(10):
        grad = (torch.randn(n, generator=g) * 0.1).cuda()
        lr_t = 1e-3 * np.sqrt(1 - 0.999 ** (step + 1)) / (1 - 0.9 ** (step + 1))
        p_ref, m_ref, v_ref = rk.apply_adam(grad, p, m, v, lr_t, 0.9, 0.999, 1e-8)
        p_our, m_our, v_our = _our_adam(grad, p, m, v, lr_t, 0.9, 0.999, 1e-8)
        gn = grad.double().cpu().numpy()
        terms = {"mean": 0.9 * np.abs(optimize_oracle.mean_decode(m.cpu().numpy().view(np.uint16))) + 0.1 * np.abs(gn),
                 "var": 0.999 * optimize_oracle.var_decode(v.cpu().numpy().view(np.uint16)) + 0.001 * gn * gn}
        for ours, ref, dec, rel, low, what in ((m_our, m_ref, optimize_oracle.mean_decode, 2.0 ** -9,
                                                optimize_oracle.MEAN_MIN, "mean"),
                                               (v_our, v_ref, optimize_oracle.var_decode, 2.0 ** -10,
                                                optimize_oracle.VAR_MIN, "var")):
            # mean codes are sign-magnitude, so closeness is judged on the decoded values: one code step, plus the
            # fp32 rounding of the moment's two terms, which cancellation can make large next to a small new mean
            da, db = dec(ours.cpu().numpy().view(np.uint16)), dec(ref.cpu().numpy().view(np.uint16))
            far = np.abs(da - db) > rel * np.maximum(np.abs(da), np.abs(db)) + 4 * U * terms[what] + low
            assert not far.any(), "step %d %s: %d codes more than one step apart, e.g. %s vs %s" % (
                step, what, far.sum(), da[far][:3], db[far][:3])
            equal.append(float((ours == ref).float().mean()))
        tol = 2.0 ** -8 * (p_ref - p).abs() + 2.0 ** -22 * p.abs()       # the update's error and two ulps of p
        assert bool(((p_our - p_ref).abs() <= tol).all()), "step %d param update" % step
        p, m, v = p_ref, m_ref, v_ref
    print("share of equal codes per step (mean, var):", ["%.5f" % e for e in equal])


def test_adam_16_bit_encoding_rounds_like_the_oracle():
    """With beta1 = 0 the new mean is the fp32 grad itself, and with beta2 = 0 the new variance is fp32(g * g), so the
    stored codes are the encodings of known values: every midpoint between neighbouring mean codes (the ties, which
    round away from zero) and log-uniform values of both signs over the whole range and past it. The reference's codes
    must equal the oracle's mean_encode / var_encode bit for bit, and ours the reference's."""
    g = _gen(7600)
    c = np.arange(1, 0x7FFF, dtype=np.int64)
    c = c[(c & 511) != 511]                                   # neighbours within one exponent
    mids = (optimize_oracle.mean_decode(c) + optimize_oracle.mean_decode(c + 1)) / 2
    mids = mids[(mids > 2.0 ** -126) & (mids < 16)]
    rnd = np.exp2(torch.empty(1 << 16).uniform_(-66, 5, generator=g).double().numpy())
    vals = np.concatenate([mids, -mids, rnd, -rnd]).astype(np.float32)
    n = vals.size
    grad = torch.as_tensor(vals).cuda()
    param = torch.zeros(n, device="cuda")
    zero = torch.zeros(n, dtype=torch.int16, device="cuda")
    for beta1, beta2 in ((0.0, 1.0), (1.0, 0.0)):
        _, m_ref, v_ref = rk.apply_adam(grad, param, zero, zero, 0.0, beta1, beta2, 1e-8)
        _, m_our, v_our = _our_adam(grad, param, zero, zero, 0.0, beta1, beta2, 1e-8)
        if beta1 == 0.0:
            got, want = m_ref, optimize_oracle.mean_encode(vals.astype(np.float64))
        else:
            got, want = v_ref, optimize_oracle.var_encode((grad * grad).double().cpu().numpy())
        assert np.array_equal(got.cpu().numpy().view(np.uint16), want.astype(np.uint16)), (beta1, beta2)
        _same([m_our, v_our], [m_ref, v_ref], "ours vs reference codes beta1 %s beta2 %s" % (beta1, beta2))
