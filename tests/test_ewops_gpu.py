"""bias_relu, dropout and embedding_lookup on the GPU: elementwise against float64 with bounds from fp32 arithmetic and
one final rounding, bit for bit where the op is a copy or a mask, bitwise reproducible, in the execution contexts of
test_execution_context_gpu.py (side streams, replayed CUDA graphs, two host threads, a second GPU), past 2^31 elements,
and in one enwik8-shaped training step against a float64 torch composition."""
import threading

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import (BlocksparseMatMul, BlocksparseTransformer, _lib, bias_relu, dropout, embedding_lookup,
                              get_entropy, layer_norm, set_entropy, softmax_cross_entropy)
from blocksparse_b200 import embed, ewops
from oracle import ewops_oracle as eo
from oracle.bsmm_oracle import MatmulOracle
from tests.test_execution_context_gpu import SLEEP_CYCLES, _gen, _poisoned_like, _same

pytestmark = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DTYPES = [F32, F16, BF16]
EPS = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}      # half an ulp, relative
TINY = {F32: 2.0 ** -149, F16: 2.0 ** -24, BF16: 2.0 ** -133}  # half the smallest subnormal
U = 2.0 ** -24                                                  # fp32 unit roundoff
ACTS = ["none", "relu", "fast_gelu"]


def _np(t):
    return t.detach().double().cpu().numpy()


def _offset(t, off):
    """A copy of t whose storage starts `off` elements into its buffer (misaligned for off % 8 != 0)."""
    if not off:
        return t.clone()
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    out = buf[off:].view(t.shape)
    out.copy_(t)
    return out


def _check(got, ref, tol, what):
    got = _np(got)
    bad = ~(np.abs(got - ref) <= tol)
    assert not bad.any(), "%s: %d of %d out of bounds, worst %s vs %s (tol %s)" % (
        what, bad.sum(), bad.size, got[bad][:3], ref[bad][:3], np.broadcast_to(tol, ref.shape)[bad][:3])


# ---- bias_relu ----------------------------------------------------------------------------------------------------------
def _br_run(x, b, dy, axis, act):
    x, b = x.detach().requires_grad_(), b.detach().requires_grad_()
    y = bias_relu(x, b, axis=axis, relu=act == "relu", fast_gelu=act == "fast_gelu")
    y.backward(dy)
    return y, x.grad, b.grad


def _db_depth(axis, N, K):
    """Longest chain of fp32 adds behind one db entry, from the kernels' partition (csrc/ewops.cuh): on the last axis rp
    rows per partial, on axis 0 eight elements per thread, the warp tree and eight warps per 2048-element segment; then
    ceil(partials / 32) per lane of the reduce kernel and its five-level tree."""
    if axis == 0:
        return 8 + 5 + 8 + -(-(-(-N // 2048)) // 32) + 5
    rp = max(8, -(-N * K // 2 ** 20))
    return rp + -(-(-(-N // rp)) // 32) + 5


def _br_check(x, b, dy, axis, act, what):
    y, dx, db = _br_run(x, b, dy, axis, act)
    kw = dict(axis=axis, relu=act == "relu", fast_gelu=act == "fast_gelu")
    xn, bn, dn = _np(x), _np(b), _np(dy)
    yr = eo.bias_relu(xn, bn, **kw)
    dxr, dbr = eo.bias_relu_grad(dn, xn, bn, **kw)
    bb = bn.reshape((-1,) + (1,) * (x.dim() - 1)) if axis == 0 else bn
    z = np.abs(xn) + np.abs(bb)                  # bounds |fp32(x + b) - (x + b)| / U
    e = EPS[x.dtype]
    _check(y, yr, e * np.abs(yr) + 4 * U * z + TINY[x.dtype], what + " y")
    if act == "none":
        assert dx.data_ptr() == dy.data_ptr() or torch.equal(dx, dy), what + " dx is dy"
        dterm = np.abs(dn)
    else:
        dterm = np.abs(dn) * (1 + 2 * (np.abs(xn) + np.abs(bb)))
        _check(dx, dxr, e * np.abs(dxr) + 16 * U * dterm + TINY[x.dtype], what + " dx")
    depth = _db_depth(axis, x.numel() // b.numel(), b.numel())
    dsum = dterm.sum(axis=tuple(range(1, x.dim()))) if axis == 0 else dterm.reshape(-1, b.numel()).sum(axis=0)
    _check(db, dbr, EPS[b.dtype] * np.abs(dbr) + (depth + 16) * U * dsum + TINY[b.dtype], what + " db")
    assert db.dtype == b.dtype and db.shape == b.shape
    return y, dx, db


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("axis", [-1, 0])
@pytest.mark.parametrize("bdt", DTYPES, ids=str)
@pytest.mark.parametrize("dt", DTYPES, ids=str)
def test_bias_relu_elementwise(dt, bdt, axis, act):
    """Ranks 2-4 on both access widths: K and N multiples of 8 (16-byte accesses) and not, odd storage offsets, and on
    axis 0 rows of several 2048-element segments."""
    g = _gen(100 * DTYPES.index(dt) + 10 * DTYPES.index(bdt) + ACTS.index(act) + 1000 * (axis == 0))
    for shape, off in [((64, 96), 0), ((37, 29), 0), ((3, 5, 24), 0), ((2, 3, 4, 40), 0), ((48, 64), 1), ((40, 17), 3),
                       ((24, 5000), 0), ((16, 6147), 1)]:
        K = shape[axis]
        x = _offset((torch.randn(shape, generator=g) * 2).to(dt).cuda(), off)
        b = torch.randn(K, generator=g).to(bdt).cuda()
        dy = _offset(torch.randn(shape, generator=g).to(dt).cuda(), off)
        _br_check(x, b, dy, axis, act, "%s %s axis %d %s %s off %d" % (dt, bdt, axis, act, shape, off))


@pytest.mark.parametrize("bdt", [F32, BF16], ids=str)
@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("axis", [-1, 0])
def test_bias_relu_db_over_a_million_rows(axis, act, bdt):
    """db over ~10^6 rows: 87382 partials per feature on the last axis and 513 row segments on axis 0, so the reduce
    kernel's lanes loop. Integer x and dy with b = 0.5 keep every fp32 partial exact, so y, dx and db must equal the
    exact values bit for bit (relu drops the elements with x < 0)."""
    g = _gen(5)
    shape = (1 << 20, 12) if axis == -1 else (12, (1 << 20) + 5)
    x = torch.randint(-3, 4, shape, generator=g).to(BF16).cuda()
    dy = torch.randint(-4, 5, shape, generator=g).to(BF16).cuda()
    b = torch.full((12,), 0.5).to(bdt).cuda()
    y, dx, db = _br_run(x, b, dy, axis, act)
    z = x.float() + 0.5
    dxr = torch.where(x >= 0, dy, torch.zeros((), dtype=BF16, device="cuda")) if act == "relu" else dy
    dbr = dxr.long().sum(dim=tuple(range(1, x.dim())) if axis == 0 else 0)
    assert dbr.abs().sum() > 0
    _same([y, dx, db], [(z.clamp(min=0) if act == "relu" else z).to(BF16), dxr, dbr.float().to(bdt)],
          "1M rows axis %d %s" % (axis, act))
    _same(list(_br_run(x, b, dy, axis, act)), [y, dx, db], "1M rows rerun")


def test_bias_relu_empty_and_reproducible():
    for shape, axis in [((0, 16), -1), ((16, 0), 0)]:
        x = torch.zeros(shape, device="cuda", requires_grad=True)
        b = torch.ones(16, device="cuda", requires_grad=True)
        y = bias_relu(x, b, axis=axis, relu=True)
        y.sum().backward()
        assert y.shape == shape and torch.equal(b.grad, torch.zeros(16, device="cuda"))
    g = _gen(9)
    x, dy = torch.randn(300, 520, generator=g).half().cuda(), torch.randn(300, 520, generator=g).half().cuda()
    b = torch.randn(520, generator=g).half().cuda()
    for axis, bb in ((-1, b), (0, b[:300])):
        for act in ACTS:
            _same(list(_br_run(x, bb, dy, axis, act)), list(_br_run(x, bb, dy, axis, act)), "rerun %d %s" % (axis, act))


# ---- dropout ------------------------------------------------------------------------------------------------------------
def _expected(x, mask, kp, mask_shape=None):
    keep = torch.as_tensor(np.ascontiguousarray(eo.broadcast_keep(mask.cpu().numpy(), tuple(x.shape), mask_shape)),
                           device=x.device)
    scale = torch.tensor(1.0 / kp, dtype=F32, device=x.device)
    return torch.where(keep, (x.float() * scale).to(x.dtype), torch.zeros((), dtype=x.dtype, device=x.device))


def test_dropout_mask_matches_philox():
    for M in (1003, 77, 4096 + 5):
        set_entropy(123456789012345, "cuda")
        x = torch.zeros(M, device="cuda")
        for call in range(3):
            _, mask = dropout(x, 0.6)
            assert get_entropy()[1].item() == call + 1
            assert mask.dtype == torch.int32 and mask.shape == ((M + 31) // 32,)
            np.testing.assert_array_equal(mask.cpu().numpy(), eo.dropout_mask(123456789012345, call, M, 0.6))
    set_entropy(-7)
    first = [dropout(x, 0.5)[1] for _ in range(3)]
    set_entropy(-7)
    assert all(torch.equal(a, dropout(x, 0.5)[1]) for a in first)
    torch.manual_seed(11)
    s1 = set_entropy()[0].item()
    torch.manual_seed(11)
    assert set_entropy()[0].item() == s1


@pytest.mark.parametrize("kp", [0.1, 0.5, 0.9, 1.0])
def test_dropout_keep_fraction(kp):
    M = 1 << 22
    _, mask = dropout(torch.zeros(M, device="cuda", dtype=F16), kp)
    kept = eo.unpack_mask(mask.cpu().numpy(), M).mean()
    if kp == 1.0:
        assert kept == 1.0
    else:
        assert abs(kept - kp) <= 5 * (kp * (1 - kp) / M) ** 0.5, (kept, kp)


@pytest.mark.parametrize("dt", DTYPES, ids=str)
@pytest.mark.parametrize("shape,mask_shape", [((64, 96), None), ((37, 29), None), ((64, 96), (1, 96)),
                                              ((8, 33, 16), (1, 33, 1)), ((4, 6, 8, 10), (4, 1, 8, 1)),
                                              ((2, 3, 4, 5, 16), (1, 3, 1, 5, 16)), ((2, 3, 4, 5, 7), (2, 1, 4, 1, 1))])
def test_dropout_bitwise(dt, shape, mask_shape):
    """y and dx equal where(bit, (x.float() * scale).to(dtype), 0), with and without a broadcast mask, on both access
    widths; a reused mask gives the same y."""
    g = _gen(21)
    for off in (0, 1):
        x = _offset(torch.randn(shape, generator=g).to(dt).cuda(), off).requires_grad_()
        dy = _offset(torch.randn(shape, generator=g).to(dt).cuda(), off)
        y, mask = dropout(x, 0.7, mask_shape=mask_shape)
        M = int(np.prod(mask_shape if mask_shape else shape))
        assert mask.numel() == (M + 31) // 32
        y.backward(dy)
        _same([y, x.grad], [_expected(x.detach(), mask, 0.7, mask_shape), _expected(dy, mask, 0.7, mask_shape)],
              "%s %s %s off %d" % (dt, shape, mask_shape, off))
        y2, mask2 = dropout(x.detach(), 0.7, mask=mask, mask_shape=mask_shape)
        assert mask2 is mask
        _same([y2], [y], "reused mask")


def test_dropout_second_gpu_has_its_own_state():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    torch.cuda.set_device(0)
    set_entropy(99, "cuda:0")
    set_entropy(99, "cuda:1")
    x0, x1 = torch.ones(1000, device="cuda:0"), torch.ones(1000, device="cuda:1")
    _, m1 = dropout(x1, 0.5)
    _, m1b = dropout(x1, 0.5)
    assert m1.device == torch.device("cuda:1")
    assert get_entropy("cuda:1")[1].item() == 2 and get_entropy("cuda:0")[1].item() == 0
    _, m0 = dropout(x0, 0.5)
    assert torch.equal(m0.cpu(), m1.cpu()) and not torch.equal(m1.cpu(), m1b.cpu())


# ---- embedding ----------------------------------------------------------------------------------------------------------
IDX_DTYPES = [torch.uint8, torch.int32, torch.int64] + ([torch.uint16] if hasattr(torch, "uint16") else [])


def _idx(kind, n, C, g):
    if kind == "uniform":
        v = torch.randint(0, C, (n,), generator=g)
    elif kind == "byte_skewed":                   # one token at 50 %
        v = torch.randint(0, C, (n,), generator=g)
        v[torch.rand(n, generator=g) < 0.5] = 32
    elif kind == "all_equal":
        v = torch.full((n,), C // 2)
    else:                                         # out of range entries mixed in
        v = torch.randint(-5, C + 5, (n,), generator=g)
    return v


def _emb_check(emb, idx, dy, what):
    """idx: int64 on the host; it is run in the dtype and shape of its device copy `idx.dev`."""
    e = emb.detach().requires_grad_()
    dev_idx = idx.dev if hasattr(idx, "dev") else idx.cuda()
    y = embedding_lookup(e, dev_idx)
    C, K = emb.shape
    iv = idx.numpy().astype(np.int64).reshape(dev_idx.shape)
    okn = (iv >= 0) & (iv < C)
    ok = torch.as_tensor(okn, device=emb.device)
    rows = emb[torch.as_tensor(np.where(okn, iv, 0), device=emb.device)]
    _same([y], [torch.where(ok[..., None], rows, torch.zeros((), dtype=emb.dtype, device=emb.device))], what + " y")
    y.backward(dy)
    dn = _np(dy).reshape(-1, K)
    dwr = eo.embedding_grad(dn, iv, C)
    flat = iv.reshape(-1)
    cnt = np.bincount(flat[(flat >= 0) & (flat < C)], minlength=C)[:, None]
    tol = EPS[emb.dtype] * np.abs(dwr) + (cnt + 1) * U * eo.embedding_grad(np.abs(dn), iv, C) + TINY[emb.dtype]
    _check(e.grad, dwr, tol, what + " dw")
    e2 = emb.detach().requires_grad_()
    embedding_lookup(e2, dev_idx).backward(dy)
    _same([e2.grad], [e.grad], what + " dw rerun")


@pytest.mark.parametrize("kind", ["uniform", "byte_skewed", "all_equal", "out_of_range"])
@pytest.mark.parametrize("dt", DTYPES, ids=str)
@pytest.mark.parametrize("idt", IDX_DTYPES, ids=str)
def test_embedding(idt, dt, kind):
    """Every index dtype; uniform indices, a byte vocabulary with one token at 50 %, all indices equal, and indices
    outside [0, C) (negative ones only where the dtype has them)."""
    g = _gen(31)
    top = {torch.uint8: 255, torch.int32: 2 ** 31 - 1, torch.int64: 2 ** 62}.get(idt, 65535)
    low = 0 if idt in (torch.uint8, getattr(torch, "uint16", None)) else -(2 ** 31)
    for C, K, n in [(256, 64, 5001), (200, 20, 3001), (1000, 72, 777)]:
        v = _idx(kind, n, C, g).clamp(low, top)
        shape = (n // 3, 3) if n % 3 == 0 else (n,)
        idx = v.view(shape)
        idx.dev = v.to(idt).view(shape).cuda()
        emb = torch.randn(C, K, generator=g).to(dt).cuda()
        dy = torch.randn(shape + (K,), generator=g).to(dt).cuda()
        _emb_check(emb, idx, dy, "%s %s %s C %d K %d n %d" % (idt, dt, kind, C, K, n))


def test_embedding_unaligned_and_long_runs():
    g = _gen(33)
    emb = _offset(torch.randn(50257, 96, generator=g).half().cuda(), 1)   # scalar route
    _emb_check(emb, torch.randint(0, 50257, (4, 2048), generator=g),
               _offset(torch.randn(4, 2048, 96, generator=g).half().cuda(), 3), "gpt2 vocab unaligned")
    idx = torch.full((20000,), 7, dtype=torch.int64)
    idx[::3] = 9
    _emb_check(torch.randn(16, 40, generator=g).cuda(), idx, torch.randn(20000, 40, generator=g).cuda(),
               "runs over many chunks")
    e = torch.randn(8, 16, device="cuda", requires_grad=True)
    y = embedding_lookup(e, torch.zeros(0, dtype=torch.int64, device="cuda"))
    y.sum().backward()
    assert y.shape == (0, 16) and torch.equal(e.grad, torch.zeros_like(e))


@pytest.mark.parametrize("dt", [F32, BF16], ids=str)
def test_embedding_grad_of_long_runs_is_exact(dt):
    """Two rows hit by 55999 and 14001 of 70001 indices: their runs span many aligned groups of 32 chunks, whose sums
    stand in for the chunks. Integer dy keeps every fp32 sum exact, so dw must equal the exact column sums."""
    g = _gen(34)
    n, C, K = 70001, 10, 40
    idx = torch.full((n,), 3, dtype=torch.int32)
    idx[::5] = 7
    idx[12345] = 11                                           # out of range: adds nothing
    dy = torch.randint(-2, 3, (n, K), generator=g)
    e = torch.zeros(C, K, dtype=dt, device="cuda", requires_grad=True)
    embedding_lookup(e, idx.cuda()).backward(dy.to(dt).cuda())
    ref = torch.zeros(C, K, dtype=torch.int64)
    ok = idx < C
    ref.index_add_(0, idx[ok].long(), dy[ok])
    assert ref[3].abs().sum() > 0 and ref[7].abs().sum() > 0
    _same([e.grad], [ref.float().to(dt).cuda()], "long runs")


# ---- execution contexts -------------------------------------------------------------------------------------------------
def _rn(g, dev, shape, dtype=F32):
    return torch.randn(shape, generator=g).to(dtype).to(dev)


def _leaf(*ts):
    return [t.detach().requires_grad_() for t in ts]


def _grad(outs, ins, douts):
    return list(torch.autograd.grad(outs, ins, douts))


def _br_make(g, dev):
    return [_rn(g, dev, (64, 200), BF16), _rn(g, dev, (200,)), _rn(g, dev, (64, 200), BF16),
            _rn(g, dev, (96, 37), F16), _rn(g, dev, (96,), F16), _rn(g, dev, (96, 37), F16)]


def _br_ctx(x1, b1, d1, x0, b0, d0):
    x1, b1, x0, b0 = _leaf(x1, b1, x0, b0)
    y1, y0 = bias_relu(x1, b1, fast_gelu=True), bias_relu(x0, b0, axis=0, relu=True)
    y2 = bias_relu(x1, b1)
    return [y1, y0, y2] + _grad((y1, y0, y2), (x1, b1, x0, b0), (d1, d0, d1))


def _drop_make(g, dev):
    return [_rn(g, dev, (64, 200), BF16), _rn(g, dev, (64, 200), BF16), _rn(g, dev, (4, 33, 24), F16),
            _rn(g, dev, (4, 33, 24), F16)]


def _drop_ctx(x1, d1, x2, d2):
    x1, x2 = _leaf(x1, x2)
    y1, m1 = dropout(x1, 0.8)
    y2, m2 = dropout(x2, 0.5, mask_shape=(1, 33, 1))
    y3, _ = dropout(x2, 0.5, mask=m2, mask_shape=(1, 33, 1))
    return [y1, m1, y2, m2, y3] + _grad((y1, y2), (x1, x2), (d1, d2))


def _emb_make(g, dev):
    return [_rn(g, dev, (256, 64), BF16), torch.randint(0, 256, (3, 700), generator=g).to(torch.uint8).to(dev),
            _rn(g, dev, (3, 700, 64), BF16), _rn(g, dev, (1000, 30)),
            torch.randint(-3, 1003, (900,), generator=g).to(dev), _rn(g, dev, (900, 30))]


def _emb_ctx(e1, i1, d1, e2, i2, d2):
    e1, e2 = _leaf(e1, e2)
    y1, y2 = embedding_lookup(e1, i1), embedding_lookup(e2, i2)
    return [y1, y2] + _grad((y1, y2), (e1, e2), (d1, d2))


CASES = {"bias_relu": (["bias_relu"], _br_make, _br_ctx),
         "dropout": (["dropout", "set_entropy", "get_entropy"], _drop_make, _drop_ctx),
         "embedding_lookup": (["embedding_lookup"], _emb_make, _emb_ctx)}


def _reset(dev, seed=77):
    """Put the dropout state of dev back to a fixed (seed, call)."""
    get_entropy(dev).copy_(torch.tensor([seed, 5], dtype=torch.int64))


def test_cases_cover_every_name_of_the_modules():
    covered = {n for c in CASES.values() for n in c[0]}
    assert covered == set(ewops.__all__) | set(embed.__all__)
    assert not covered & set(blocksparse_b200.__all__)
    assert all(getattr(blocksparse_b200, n) is getattr(ewops if n in ewops.__all__ else embed, n) for n in covered)


@pytest.mark.parametrize("name", list(CASES))
def test_side_stream(name):
    _, make, run = CASES[name]
    staging = make(_gen(7), "cuda")
    _reset("cuda")
    ref = run(*staging)
    bufs = [_poisoned_like(t) for t in staging]
    _reset("cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = run(*bufs)
    s.synchronize()
    _same(out, ref, name)
    assert _lib.device_error() == 0, _lib.device_error_text()


@pytest.mark.parametrize("name", list(CASES))
def test_graph_replay(name):
    """Three replays with new inputs, each equal to an eager run from the same dropout state; every replay draws a new
    mask."""
    _, make, run = CASES[name]
    get_entropy("cuda")
    static = make(_gen(0), "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run(*static)
    masks = []
    for i in range(1, 4):
        new = make(_gen(i), "cuda")
        for t, n in zip(static, new):
            t.copy_(n)
        saved = get_entropy().clone()
        graph.replay()
        after = get_entropy().clone()
        get_entropy().copy_(saved)
        _same(out, run(*new), "%s replay %d" % (name, i))
        _same([get_entropy()], [after], "%s replay %d state" % (name, i))
        masks.append(out[1].clone() if name == "dropout" else None)
    if name == "dropout":
        assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])


def test_graph_refuses_to_create_the_state():
    dev = torch.device("cuda", torch.cuda.current_device())
    saved = ewops._ENTROPY.pop(dev.index, None)
    try:
        x = torch.ones(100, device="cuda")
        graph = torch.cuda.CUDAGraph()
        with pytest.raises(ValueError):
            with torch.cuda.graph(graph):
                dropout(x, 0.5)
    finally:
        if saved is not None:
            ewops._ENTROPY[dev.index] = saved


@pytest.mark.parametrize("name", ["bias_relu", "embedding_lookup"])
def test_concurrent_threads(name):
    _, make, run = CASES[name]
    inputs = [make(_gen(80 + i), "cuda") for i in range(2)]
    refs = [run(*ins) for ins in inputs]
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    results, errors = [None, None], []

    def worker(i):
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.default_stream())
            barrier.wait()
            with torch.cuda.stream(s):
                results[i] = run(*inputs[i])
            s.synchronize()
        except BaseException as e:
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for i in range(2):
        _same(results[i], refs[i], "%s thread %d" % (name, i))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs: runs the families on cuda:1")
@pytest.mark.parametrize("name", list(CASES))
def test_second_gpu(name):
    _, make, run = CASES[name]
    torch.cuda.set_device(0)
    ins0, ins1 = make(_gen(11), "cuda:0"), make(_gen(11), "cuda:1")
    _reset("cuda:0")
    ref = run(*ins0)
    _reset("cuda:1")
    out = run(*ins1)
    assert torch.cuda.current_device() == 0
    assert all(t.device == torch.device("cuda:1") for t in out)
    _same(out, ref, name + " on cuda:1")
    for d in range(2):
        with torch.cuda.device(d):
            assert _lib.device_error() == 0, (d, _lib.device_error_text())


# ---- past 2^31 elements -------------------------------------------------------------------------------------------------
def _need(gb):
    free = torch.cuda.mem_get_info()[0]
    if free < gb * 2 ** 30:
        pytest.skip("needs %.0f GB of free device memory, %.1f GB free" % (gb, free / 2 ** 30))


def test_large_bias_relu():
    _need(30)
    N, K = (1 << 21) + 3, 1024                                # 2^31 + 3072 elements
    x = torch.empty(N, K, dtype=F16, device="cuda").uniform_(-2, 2)
    b = torch.linspace(-1, 1, K, device="cuda")
    xr = x.requires_grad_()
    y = bias_relu(xr, b, relu=True)
    tail = slice(N - 4, N)
    ref = torch.relu(x[tail].float() + b).half()
    assert torch.equal(y[tail], ref)
    dy = torch.ones_like(x)
    y.backward(dy)
    assert torch.equal(x.grad[tail], (ref > 0).half())
    del y, dy, xr
    x.grad = None
    xt = x.detach().t()                                       # axis 0: (K, N) view, contiguous copy inside
    y0 = bias_relu(xt.contiguous(), b, axis=0)
    assert torch.equal(y0[:, -4:], (xt[:, -4:].float() + b[:, None]).half())


def test_large_dropout():
    _need(20)
    n = (1 << 31) + 77
    x = torch.ones(n, dtype=F16, device="cuda")
    set_entropy(3)
    y, mask = dropout(x, 0.5)
    e0 = n - 1000
    g = np.arange(e0 // 4, (n + 3) // 4, dtype=np.uint64)
    ctr = np.stack([g & np.uint64(0xFFFFFFFF), g >> np.uint64(32), np.zeros_like(g), np.zeros_like(g)], -1)
    u = eo.philox4x32_10(ctr.astype(np.uint32), np.broadcast_to(np.array([3, 0], np.uint32), (len(g), 2)))
    bits = (u.reshape(-1)[e0 - (e0 // 4) * 4:][:n - e0].astype(np.uint64) < np.uint64(2 ** 31))
    got = eo.unpack_mask(mask[e0 // 32:].cpu().numpy(), (n + 31) // 32 * 32 - (e0 // 32) * 32)[e0 % 32:][:n - e0]
    np.testing.assert_array_equal(got, bits)
    np.testing.assert_array_equal(y[e0:].cpu().numpy(), np.where(bits, 2.0, 0.0).astype(np.float16))


def test_large_embedding():
    _need(30)
    C, K, n = 1000, 4096, (1 << 19) + 3                       # n * K = 2^31 + 12288
    emb = torch.randn(C, K, device="cuda").half().requires_grad_()
    idx = torch.randint(0, C, (n,), device="cuda")
    y = embedding_lookup(emb, idx)
    assert torch.equal(y[-3:], emb.detach()[idx[-3:]])
    y.backward(torch.ones_like(y))
    cnt = torch.bincount(idx, minlength=C).half()
    assert torch.equal(emb.grad, cnt[:, None].expand(C, K))


# ---- end to end ---------------------------------------------------------------------------------------------------------
_LAY = np.ones((4, 4), np.int32)
_LAY[0, 3] = _LAY[3, 1] = 0
E2E_BSMM = BlocksparseMatMul(_LAY, block_size=32, feature_axis=1)                      # 128 -> 128
E2E_BST = BlocksparseTransformer(np.tril(np.ones((4, 4), np.int32)), block_size=64, heads=2)   # context 256


def _e2e_params(g):
    return [(torch.randn(256, 128, generator=g) * 0.5).half().cuda(), (1 + 0.1 * torch.randn(128, generator=g)).cuda(),
            (0.1 * torch.randn(128, generator=g)).cuda(), (torch.randn(E2E_BSMM.w_shape, generator=g) * 0.1).half().cuda(),
            (0.1 * torch.randn(128, generator=g)).cuda()]


def _e2e_leaves(g):
    return [p.requires_grad_() for p in _e2e_params(g)]


def _e2e_step(params, xs, labels):
    """embedding -> dropout -> layer_norm -> attention -> bsmm + fast_gelu bias -> dropout (mask reused on a recompute)
    -> cross entropy, forward and backward."""
    emb, lg, lb, w, bias = params
    h, m1 = dropout(embedding_lookup(emb, xs), 0.9)
    a = layer_norm(h, lg, lb, axis=-1)
    o = E2E_BST.attention(a, a, a, scale=0.125)
    u = bias_relu(E2E_BSMM(o.reshape(256, 128), w), bias, fast_gelu=True)
    d, m2 = dropout(u, 0.8)
    d2, _ = dropout(u, 0.8, mask=m2)                          # the recompute of a checkpointed block
    loss = softmax_cross_entropy(logits=d2, labels=labels)
    grads = torch.autograd.grad(loss.sum(), params)
    return [loss, d, m1, m2] + list(grads)


def _e2e_ref(params, xs, labels, m1, m2):
    emb, lg, lb, w, bias = [p.detach().double().cpu().requires_grad_() for p in params]
    orc = MatmulOracle(_LAY, 32, 1)
    keep1 = torch.as_tensor(eo.unpack_mask(m1.cpu().numpy(), 256 * 128).reshape(1, 256, 128))
    keep2 = torch.as_tensor(eo.unpack_mask(m2.cpu().numpy(), 256 * 128).reshape(256, 128))
    h = torch.where(keep1, emb[xs.cpu().long()] / 0.9, 0.0)
    mu, var = h.mean(-1, keepdim=True), h.var(-1, unbiased=False, keepdim=True)
    a = (h - mu) / torch.sqrt(var + 1e-6) * lg + lb
    ah = a.view(1, 256, 2, 64).transpose(1, 2)
    vis = torch.as_tensor(np.kron(np.tril(np.ones((4, 4))), np.ones((64, 64))).astype(bool))
    s = torch.where(vis, ah @ ah.transpose(-1, -2) * 0.125, float("-inf"))
    o = (torch.softmax(s, -1) @ ah).transpose(1, 2).reshape(256, 128)
    W = torch.zeros(128, 128, dtype=torch.float64)
    for i, (c, k) in enumerate(orc.updat_list):
        W = W.index_put((torch.arange(c * 32, c * 32 + 32)[:, None], torch.arange(k * 32, k * 32 + 32)[None]), w[i])
    z = o @ W + bias
    u = z * torch.sigmoid(1.702 * z)
    d = torch.where(keep2, u / 0.8, 0.0)
    loss = torch.nn.functional.cross_entropy(d, labels.cpu(), reduction="none")
    grads = torch.autograd.grad(loss.sum(), (emb, lg, lb, w, bias))
    return [loss, d] + list(grads)


def test_enwik8_step():
    g = _gen(40)
    params = _e2e_leaves(g)
    xs = torch.randint(0, 256, (1, 256), generator=g).to(torch.uint8).cuda()
    labels = torch.randint(0, 128, (256,), generator=g).cuda()
    set_entropy(2024)
    out = _e2e_step(params, xs, labels)
    loss, d, m1, m2 = out[:4]
    ref = _e2e_ref(params, xs, labels, m1, m2)
    for got, r, what in zip([loss, d] + out[4:], ref, ["loss", "y", "demb", "dg", "db", "dw", "dbias"]):
        r = r.detach().numpy()
        err = np.abs(_np(got) - r).max() / max(np.abs(r).max(), 1e-30)
        assert err <= 2e-2, "%s: relative error %.3e" % (what, err)

    # the same step captured whole and replayed on new batches equals eager steps from the same dropout state; the
    # captured step gets leaves of its own, first used on the capture's side stream
    gparams = [p.detach().clone().requires_grad_() for p in params]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _e2e_step(gparams, xs, labels)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _e2e_step(gparams, xs, labels)
    for i in range(3):
        gb = _gen(41 + i)
        nx, nl = torch.randint(0, 256, (1, 256), generator=gb).to(torch.uint8), torch.randint(0, 128, (256,), generator=gb)
        xs.copy_(nx)
        labels.copy_(nl)
        saved = get_entropy().clone()
        graph.replay()
        get_entropy().copy_(saved)
        _same(static, _e2e_step(params, xs, labels), "enwik8 step replay %d" % i)
