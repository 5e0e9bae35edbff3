"""Block-sparse softmax and its gradient on every kernel route, elementwise against the oracle.

Routes (csrc/api.cu bst_softmax / bst_softmax_grad):
  * staged kernel: 16-bit in and out, block size 32 / 64, rows of at most 16 key blocks; the MAXE = 4 / 8 / 12 / 16
    instantiation is picked from the longest row (nn_max);
  * register kernel: everything else (fp32, block size 8 / 16, rows longer than 16 blocks), and every case in a
    process started with BSMM_SOFTMAX_STAGED=0. Rows longer than KEEP key blocks (4 at bs 32 / 64 and in the grad,
    8 at bs 8 / 16) take its re-read branch, rows longer than 32 blocks also reload their LUT entries from memory.

Random scores go straight into BlocksparseTransformer._softmax / _softmax_grad (no NT in front, so shapes stay cheap),
rounded to their storage dtype first; the oracle sees the same rounded values.
"""
import collections
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._util import EPS32, ROOT, U_OUT, softmax_grad_bound, softmax_row_sums
from tests.golden.make_golden import causal_callback
from blocksparse_b200 import BlocksparseTransformer, _lib
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
_NAME = {BF16: "bfloat16", F16: "float16", F32: "float32"}


# ---- layouts and masks ---------------------------------------------------------------------------------------------
def _tril(n):
    """causal block layout: query block q holds q + 1 key blocks, so the rows have every length 1..n"""
    return np.tril(np.ones((n, n), np.int32))


def _hole(lay, q):
    """query block q holds no key block: an empty softmax row"""
    lay = lay.copy()
    lay[..., q, :] = 0
    return lay


def _future_first(n):
    """tril, except that query block 0 holds only key block 1: with autoregress_at_key <= bs every key of its rows lies
    in the future, so each of those rows is hidden completely"""
    lay = _tril(n)
    lay[0, 0], lay[0, 1] = 0, 1
    return lay


def _per_head(lay, heads):
    """one layout per head, query rows rotated by the head index: equal block counts, different row lengths"""
    return np.stack([np.roll(lay, h, axis=0) for h in range(heads)])


def _ones_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    return np.ones(blk_shape, dtype=bool)


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks, and row 3 of query block 1 sees no key at all"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


def _per_head_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """a different pattern in every head; in head 1, row 5 of query block 0 sees no key at all"""
    q, k = np.indices(blk_shape)
    m = ((q + 2 * k + head_idx) % 3) != 0
    if head_idx == 1 and qry_idx == 0:
        m[5, :] = False
    return m


# ---- the covering set ----------------------------------------------------------------------------------------------
# values: "normal" = N(0, 1.5) after scaling; "big" = uniform +-300 before scaling (a missing max subtraction
# overflows); "late" = normal plus 4 on the LAST key block of every row, so the running maximum of the register
# kernel grows at the end of the row and everything before must be rescaled.
Case = collections.namedtuple("Case", "bs xdt ydt lay cb ak scale values heads batch")
Case.__new__.__defaults__ = (None, None, 1.0, "normal", 2, 2)

CASES = [
    # staged kernel, one case per MAXE bucket and dtype pair at least
    Case(64, BF16, BF16, _tril(4), causal_callback, scale=0.125),                            # MAXE 4
    Case(64, F16, F16, _tril(7), _hide_row_cb, values="late"),                               # MAXE 8, hidden row
    Case(64, BF16, F16, _tril(11), causal_callback, scale=0.125),                            # MAXE 12, the fp16 chain
    Case(64, F16, BF16, _tril(16), scale=-0.25, values="big"),                               # MAXE 16, no mask
    Case(32, BF16, BF16, _per_head(_tril(13), 3), _per_head_cb, scale=0.125, values="big", heads=3),   # per-head mask
    Case(32, F16, F16, _hole(_tril(6), 2), causal_callback, ak=80, values="late"),           # empty row, autoregress
    Case(64, BF16, BF16, _future_first(5), _ones_cb, ak=0, scale=0.125),                     # autoregress hides rows
    Case(32, BF16, F16, np.ones((3, 10), np.int32), values="late"),                          # rectangular, MAXE 12
    Case(64, F16, F16, _tril(3), causal_callback, ak=100, scale=-0.25, values="big"),
    # register kernel
    Case(64, BF16, BF16, _tril(40), causal_callback, scale=0.125, values="late", batch=1),   # > 32 blocks: LUT reload
    Case(32, F16, F16, _per_head(_tril(24), 2), _per_head_cb, scale=-0.25),                  # 17..32 blocks
    Case(64, F16, BF16, np.ones((2, 34), np.int32), values="big"),
    Case(8, BF16, BF16, _tril(12), causal_callback, values="big"),                           # bs 8, > KEEP = 8
    Case(8, F16, BF16, _per_head(_tril(9), 2), _per_head_cb, scale=0.125, values="late"),
    Case(8, F32, F32, _tril(36), values="late", batch=1),                                    # bs 8, > 32 blocks
    Case(16, F16, F16, _tril(10), _ones_cb, ak=40, scale=0.125),
    Case(16, F32, BF16, _tril(6), _hide_row_cb, scale=0.125, values="big"),
    Case(16, BF16, F16, _hole(_tril(9), 4)),
    Case(32, F32, F32, _per_head(_tril(9), 2), _per_head_cb, values="late"),
    Case(64, F32, BF16, _tril(20), causal_callback, ak=300, scale=-0.25),
    Case(64, F32, F32, _tril(5), _hide_row_cb, scale=0.125, values="big"),
]


def _nn_max(case):
    lay = case.lay if case.lay.ndim == 3 else case.lay[None]
    return int(lay.sum(axis=2).max())


def _staged(case, x_dtype=None, env_off=False):
    """whether csrc/api.cu picks the staged kernel (x_dtype: the input dtype, if not the case's scores)"""
    xd = x_dtype or case.xdt
    return not env_off and xd != F32 and case.ydt != F32 and case.bs in (32, 64) and _nn_max(case) <= 16


def _case_id(c):
    mask = "nomask" if c.cb is None else c.cb.__name__.strip("_").replace("_callback", "").replace("_cb", "")
    lh = "" if c.lay.ndim == 2 else "-perhead"
    return "bs%d-%s-%s-L%d%s-%s%s-s%g-%s" % (c.bs, _NAME[c.xdt], _NAME[c.ydt], _nn_max(c), lh, mask,
                                              "" if c.ak is None else "-ak%d" % c.ak, c.scale, c.values)


def test_cases_cover_every_route():
    """The covering set really reaches every route and bucket the header lists (pure Python; guards later edits)."""
    maxe = {min(b for b in (4, 8, 12, 16) if _nn_max(c) <= b) for c in CASES if _staged(c)}
    assert maxe == {4, 8, 12, 16}
    reg = [c for c in CASES if not _staged(c)]
    assert any(c.bs in (32, 64) and c.xdt != F32 and c.ydt != F32 for c in reg)          # 16-bit, too long to stage
    assert any(_nn_max(c) > 32 and c.bs == 64 for c in reg) and any(_nn_max(c) > 32 and c.bs == 8 for c in reg)
    assert any(c.bs in (8, 16) and _nn_max(c) > 8 for c in reg)                          # bs 8/16 re-read branch
    for route in (True, False):
        sub = [c for c in CASES if _staged(c) == route]
        assert {_per_head_cb, causal_callback, None} <= {c.cb for c in sub}
        assert any(c.ak is not None for c in sub) and any(c.values == "big" for c in sub)
        assert any(c.scale < 0 for c in sub)
    assert {(c.xdt, c.ydt) for c in CASES} >= {(BF16, BF16), (F16, F16), (BF16, F16), (F16, BF16), (F32, F32), (F32, BF16)}
    assert {c.bs for c in CASES} == {8, 16, 32, 64}


# ---- running one case ------------------------------------------------------------------------------------------------
def _ulp(a, dtype):
    """spacing of the 16-bit dtype at |a| (float64 array)"""
    mant, emin = (7, -126) if dtype == BF16 else (10, -14)
    return 2.0 ** (np.floor(np.log2(np.maximum(np.abs(a), 2.0 ** emin))) - mant)


def _visibility(orc, case):
    """vis[h, blk, r, j]: key j visible to query r; live[h, blk, r]: the row has at least one visible key"""
    nb, bs = orc.blocks, case.bs
    vis = np.ones((case.heads, nb, bs, bs), bool)
    if case.cb is not None:
        for h in range(case.heads):
            hl = orc._hl(h)
            for b, (q, k) in enumerate(orc.nt_list[hl]):
                vis[h, b] = orc._mask_bits(hl, b, k, case.ak)
    live = np.zeros((case.heads, nb, bs), bool)
    for h in range(case.heads):
        for row in orc.nn_list[orc._hl(h)]:
            if row:
                bids = [b for b, _ in row]
                live[h, bids] = vis[h, bids].any(axis=(0, 2))[None, :]
    return vis, live


def _scores(case, orc, rng):
    shape = (case.batch, case.heads, orc.blocks, case.bs, case.bs)
    if case.values == "big":
        x = rng.uniform(-300, 300, shape)
    else:
        z = rng.normal(0, 1.5, shape)
        if case.values == "late":
            for h in range(case.heads):
                for row in orc.nn_list[orc._hl(h)]:
                    if row:
                        z[:, h, row[-1][0]] += 4.0
        x = z / case.scale
    t = torch.as_tensor(x.astype(np.float32)).to(case.xdt)
    return t, t.float().numpy()


def softmax_bound(p, y_dtype, amax, longest):
    """Largest |got - p| for a probability p of the oracle (fp32 on the same rounded scores), elementwise.

    u = one output rounding (u_out) plus the fp32 error of both computations, in units of eps32 = 2^-24:
      * exponent arguments: the kernels form v = x * (scale * log2 e) (two roundings) for each entry and for the row
        maximum, the oracle x * scale - max; with |x scale| <= amax that is < 4 amax eps32 in the exponent (log2 e and
        ln 2 cancel), and the online / final rescale factors exp2((m_old - m) log2 e) add at most as much again over a
        row, because the growth of the running max telescopes to <= 2 amax: 16 amax in all, generously;
      * the sum: each thread adds <= 8 keys per block over `longest` blocks in order, rescaled once per block, then
        <= 5 shuffle levels: 16 longest;
      * exp2f (2 ulp), reciprocal and the two final multiplies, and the oracle's exp / divide: 64.
    Then 2^-20 absolute, which also covers exp2 underflow and 16-bit subnormal outputs."""
    u = U_OUT[_NAME[y_dtype]] + EPS32 * (16 * amax + 16 * longest + 64)
    return u * p + 2.0 ** -20


def _run(idx, env_off=False):
    """Softmax and softmax grad of CASES[idx] (env_off: in a BSMM_SOFTMAX_STAGED=0 process), checked against the
    oracle. Returns y and dx as CPU tensors, and the fp32 row-sum accumulation term of the grad bound."""
    case = CASES[idx]
    staged = _staged(case, env_off=env_off)
    g_staged = _staged(case, x_dtype=case.ydt, env_off=env_off)        # the grad runs at the probabilities' dtype
    bst = BlocksparseTransformer(case.lay, case.bs, heads=case.heads, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, case.bs, heads=case.heads, mask_callback=case.cb)
    rng = np.random.default_rng(4000 + idx)
    L = _nn_max(case)
    assert bst.nn_max == L
    what = _case_id(case)

    x, xn = _scores(case, orc, rng)
    y = bst._softmax(x.cuda(), case.scale, case.cb is not None, case.ak, case.ydt)
    kern = _lib.last_kernel()
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert kern == ("bst_softmax_staged" if staged else "bst_softmax"), (what, kern)
    got = y.cpu()
    g = got.double().numpy()
    p = orc.masked_softmax(xn, scale=case.scale, autoregress_at_key=case.ak).astype(np.float64)
    vis, live = _visibility(orc, case)
    # masked keys of a row that sees anything: exp2 of -FLT_MAX minus a finite maximum is exactly 0
    hidden = np.broadcast_to(~vis & live[..., None], g.shape)
    assert not np.any(g[hidden] != 0.0), "%s: %d masked probabilities are not 0" % (what, int((g[hidden] != 0).sum()))
    # a row that sees nothing is the oracle's uniform row 1 / (blocks * bs); the bound below checks it with the rest
    amax = float(np.abs(xn * case.scale).max())
    bound = softmax_bound(p, case.ydt, amax, L)
    err = np.abs(g - p)
    i = np.unravel_index(np.argmax(err - bound), err.shape)
    assert np.all(err <= bound), "%s: probs %d out of bound, worst |d| %.3e at p %.6e (bound %.3e)" % (
        what, int((err > bound).sum()), err[i], p[i], bound[i])

    # gradient at the oracle's probabilities, rounded as the op stores them, with random upstream gradients
    yin = torch.as_tensor(p.astype(np.float32)).to(case.ydt)
    dy = torch.as_tensor(rng.normal(0, 1, p.shape).astype(np.float32)).to(case.ydt)
    dx = bst._softmax_grad(dy.cuda(), yin.cuda(), case.scale)
    kern = _lib.last_kernel()
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert kern == ("bst_softmax_grad_staged" if g_staged else "bst_softmax_grad"), (what, kern)
    assert dx.dtype == case.ydt
    dxc = dx.cpu()
    gd = dxc.double().numpy()
    yv, dv = yin.double().numpy(), dy.double().numpy()
    ref = orc.masked_softmax_grad(dv, yv, scale=case.scale)                  # float64 in, float64 out
    row_dyy = softmax_row_sums(np.abs(dv * yv), orc)
    bound = softmax_grad_bound(ref, dv, yv, row_dyy, _NAME[case.ydt], case.scale, L)
    err = np.abs(gd - ref)
    i = np.unravel_index(np.argmax(err - bound), err.shape)
    assert np.all(err <= bound), "%s: grad %d out of bound, worst |d| %.3e at ref %.6e (bound %.3e)" % (
        what, int((err > bound).sum()), err[i], ref[i], bound[i])
    assert not np.any(gd[yv == 0] != 0.0), "%s: grad nonzero where y == 0" % what
    acc_term = EPS32 * (8 * L + 12) * (np.abs(dv) + row_dyy) * yv * abs(case.scale)
    return got, dxc, acc_term


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_softmax_and_grad_match_oracle(idx):
    _run(idx)


# ---- the register kernels at staged-eligible shapes ------------------------------------------------------------------
STAGED_IDX = [i for i, c in enumerate(CASES) if _staged(c)]


def child_register_outputs(path):
    """Run in a child process started with BSMM_SOFTMAX_STAGED=0 (the library reads it once per process): the
    staged-eligible cases on the register kernels, each checked against the oracle; saves the outputs to `path`."""
    assert os.environ.get("BSMM_SOFTMAX_STAGED") == "0"
    torch.cuda.set_device(0)
    out = {}
    for i in STAGED_IDX:
        y, dx, _ = _run(i, env_off=True)
        out["y%d" % i], out["dx%d" % i] = y.double().numpy(), dx.double().numpy()
    np.savez(path, **out)


def test_register_kernels_at_staged_shapes_agree(tmp_path):
    path = str(tmp_path / "register_route.npz")
    env = dict(os.environ, BSMM_SOFTMAX_STAGED="0")
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from tests.test_bst_softmax_gpu import child_register_outputs\n"
            "child_register_outputs(%r)\n" % (ROOT, path))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "register-route child failed:\n" + r.stdout[-4000:] + r.stderr[-4000:]
    reg = np.load(path)
    for i in STAGED_IDX:
        case = CASES[i]
        y, dx, acc_term = _run(i)
        ys, yr = y.double().numpy(), reg["y%d" % i]
        # same rounded scores, two fp32 computations whose difference is far below one 16-bit ulp: their roundings
        # differ by at most one ulp
        worst = float((np.abs(ys - yr) / _ulp(np.maximum(np.abs(ys), np.abs(yr)), case.ydt)).max())
        assert worst <= 1.0, "%s: staged and register softmax differ by %.2f ulp" % (_case_id(case), worst)
        # the gradient subtracts the row sum sum(dy y), accumulated in a different order by the two kernels; where
        # dy - sum cancels, that fp32 difference (twice the per-kernel accumulation term of softmax_grad_bound)
        # comes on top of the one ulp
        ds, dr = dx.double().numpy(), reg["dx%d" % i]
        ulp = _ulp(np.maximum(np.abs(ds), np.abs(dr)), case.ydt)
        over = np.abs(ds - dr) - 2 * acc_term
        assert np.all(over <= ulp), "%s: staged and register grad differ by %.2f ulp beyond the fp32 slack" % (
            _case_id(case), float((over / ulp).max()))


# ---- misaligned views ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs,dtype,offset", [(64, BF16, 1), (32, F16, 3), (16, F32, 2)])
def test_misaligned_views_through_public_softmax(bs, dtype, offset):
    """A contiguous view at an odd element offset into a flat buffer is legal torch; the kernels need 16-byte aligned
    operands, so the op hands them an aligned copy. Forward (masked_softmax) and backward both match the oracle."""
    lay = _tril(4)
    heads, batch, scale = 2, 2, 0.125
    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal_callback)
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    shape = (batch, heads, bst.blocks, bs, bs)
    n = int(np.prod(shape))
    rng = np.random.default_rng(bs + offset)
    xs = torch.as_tensor(rng.normal(0, 8, shape).astype(np.float32)).to(dtype)
    dys = torch.as_tensor(rng.normal(0, 1, shape).astype(np.float32)).to(dtype)
    x = torch.zeros(n + offset, dtype=dtype, device="cuda")[offset:].view(shape)
    dy = torch.zeros(n + offset, dtype=dtype, device="cuda")[offset:].view(shape)
    x.copy_(xs.cuda()); dy.copy_(dys.cuda())
    assert x.is_contiguous() and x.data_ptr() % 16 and dy.is_contiguous() and dy.data_ptr() % 16
    x.requires_grad_()
    y = bst.masked_softmax(x, scale=scale)
    assert _lib.last_kernel() == ("bst_softmax_staged" if dtype != F32 else "bst_softmax")
    y.backward(dy)
    assert _lib.device_error() == 0, _lib.device_error_text()
    p = orc.masked_softmax(xs.float().numpy(), scale=scale).astype(np.float64)
    err = np.abs(y.detach().double().cpu().numpy() - p)
    assert np.all(err <= softmax_bound(p, dtype, float(np.abs(xs.float().numpy() * scale).max()), 4))
    # backward at the op's own probabilities
    yv, dv = y.detach().double().cpu().numpy(), dys.double().numpy()
    ref = orc.masked_softmax_grad(dv, yv, scale=scale)
    bound = softmax_grad_bound(ref, dv, yv, softmax_row_sums(np.abs(dv * yv), orc), _NAME[dtype], scale, 4)
    assert np.all(np.abs(x.grad.double().cpu().numpy() - ref) <= bound)
    # the raw grad op with misaligned y / dy views as well
    yflat = torch.zeros(n + offset, dtype=dtype, device="cuda")
    ymis = yflat[offset:].view(shape)
    ymis.copy_(y.detach())
    assert ymis.data_ptr() % 16
    dx = bst._softmax_grad(dy, ymis, scale)
    assert torch.equal(dx, x.grad)
