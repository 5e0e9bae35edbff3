"""dw_matmul_large_n on the GPU: elementwise accuracy against float64 on both routes in every dtype, the route each call
takes, bitwise determinism across calls and SM margins, the accuracy the minibatch split buys over one long fp32 sum,
and parity with the reference's own kernel.

Accuracy bound, per element: |u - ref| <= c * 2^-23 * depth * sum_n |x_nc * e_nk|, where depth = rows per segment + S
is the number of additions into one fp32 value (the segment's sum, then the S partials).  16-bit products are exact in
fp32 and fmaf rounds fp32 products once with the addition, so only the accumulation counts.  FMA route: c = 1, twice
the textbook gamma_n = n * 2^-24 of a rounded-to-nearest sum.  wgmma route: c = 2, because the tensor core's internal
fp32 accumulation is not IEEE round-to-nearest (it may truncate, at most doubling each step's error), and its
constant has not been measured; c = 2 covers that doubling once more."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._util import ROOT, ref_errors
from tests.test_dw_matmul_abi import split
from blocksparse_b200 import _lib, dw_matmul_large_n
from oracle import ref_matmul

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
DTYPES = [F32, F16, BF16]
REF_SHAPES = [(1 << 20, 32, 32), (1 << 17, 128, 128), (1 << 15, 512, 512), (32, 1024, 1024), (64, 8, 8), (32, 4, 4)]
RAGGED = [(1000, c, k) for c, k in ((1, 1), (7, 33), (33, 129), (129, 300), (300, 7), (1, 300))]
EDGES = [(4999, 64, 192), (65, 8, 520), (5000, 136, 264), (3000, 264, 8)]
SHAPES = REF_SHAPES + RAGGED + EDGES


def make(lead_x, C, K, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(tuple(lead_x) + (C,), generator=g, device="cuda") + 0.1).to(dtype)
    e = (torch.randn(tuple(lead_x) + (K,), generator=g, device="cuda") + 0.2).to(dtype)
    return x, e


def reference(x, e):
    """float64 x^T e and |x|^T |e| over the leading dims."""
    C, K = x.shape[-1], e.shape[-1]
    xd, ed = x.reshape(-1, C).double(), e.reshape(-1, K).double()
    return (xd.t() @ ed).cpu().numpy(), (xd.abs().t() @ ed.abs()).cpu().numpy()


def tc_ok(dtype, C, K):
    return dtype != F32 and C % 8 == 0 and K % 8 == 0


def check_bound(u, ref, absref, N, C, K, tc, what):
    S, rows = split(N, C, K, tc)
    c = 2.0 if tc else 1.0
    bound = c * 2.0 ** -23 * (rows + S) * absref
    err = np.abs(u.astype(np.float64) - ref)
    bad = err > bound
    assert not bad.any(), "%s: %d of %d elements out of bound, worst err %.3e (bound %.3e there)" % (
        what, int(bad.sum()), bad.size, float(err[bad].max()), float(bound[bad][np.argmax(err[bad])]))


def run(x, e, route):
    flags = _lib.FLAG_FORCE_TC if route == "tc" else _lib.FLAG_FORCE_GENERIC
    u = dw_matmul_large_n(x, e, flags=flags)
    kernel = _lib.last_kernel()
    torch.cuda.synchronize()
    assert _lib.device_error() == 0
    return u, kernel


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("N,C,K", SHAPES, ids=lambda v: str(v))
def test_accuracy_both_routes(N, C, K, dtype):
    x, e = make((N,), C, K, dtype, seed=N + 7 * C + 13 * K)
    ref, absref = reference(x, e)
    for route in ("tc", "fma"):
        if route == "tc" and not tc_ok(dtype, C, K):
            with pytest.raises(ValueError, match="wgmma"):
                dw_matmul_large_n(x, e, flags=_lib.FLAG_FORCE_TC)
            continue
        u, kernel = run(x, e, route)
        assert kernel == ("wgmma_dense_dw" if route == "tc" else "fma_dense_dw")
        assert u.dtype == F32 and tuple(u.shape) == (C, K) and not u.requires_grad
        check_bound(u.cpu().numpy(), ref, absref, N, C, K, route == "tc", "%s %s %s" % ((N, C, K), dtype, route))


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_rank3_and_noncontiguous(dtype):
    x, e = make((3, 700), 40, 24, dtype, seed=5)
    ref, absref = reference(x, e)
    for route in ("tc", "fma") if dtype != F32 else ("fma",):
        u, _ = run(x, e, route)
        check_bound(u.cpu().numpy(), ref, absref, 2100, 40, 24, route == "tc", "rank 3 %s %s" % (dtype, route))
    xt = x.transpose(0, 1).contiguous().transpose(0, 1)          # same values, non-contiguous
    assert not xt.is_contiguous()
    assert torch.equal(dw_matmul_large_n(xt, e), dw_matmul_large_n(x, e))


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
def test_empty_sizes(dtype):
    x, e = make((0,), 64, 40, dtype, seed=1)
    for flags in (0, _lib.FLAG_FORCE_GENERIC):
        u = dw_matmul_large_n(x, e, flags=flags)
        assert tuple(u.shape) == (64, 40) and bool((u == 0).all())
    assert _lib.last_kernel() == "memset_dense_dw"
    x, e = make((2, 0), 7, 5, dtype, seed=1)
    assert bool((dw_matmul_large_n(x, e) == 0).all())
    for C, K in ((0, 16), (16, 0), (0, 0)):
        x, e = make((300,), C, K, dtype, seed=2)
        u = dw_matmul_large_n(x, e)
        assert tuple(u.shape) == (C, K) and u.dtype == F32


def test_routes():
    cases = [((4096, 64, 64), F16, 0, "wgmma_dense_dw"), ((4096, 64, 64), BF16, 0, "wgmma_dense_dw"),
             ((4096, 64, 64), F32, 0, "fma_dense_dw"), ((4096, 66, 64), F16, 0, "fma_dense_dw"),
             ((4096, 64, 36), BF16, 0, "fma_dense_dw"), ((4096, 64, 64), F16, _lib.FLAG_FORCE_GENERIC, "fma_dense_dw")]
    for (N, C, K), dtype, flags, want in cases:
        x, e = make((N,), C, K, dtype, seed=3)
        dw_matmul_large_n(x, e, flags=flags)
        assert _lib.last_kernel() == want, ((N, C, K), dtype, flags)
    # a contiguous view that starts 2 bytes past a 16-byte boundary cannot be a TMA operand: the FMA route takes it,
    # with the same values as an aligned copy (the routes differ in rounding, so compare against the forced FMA run)
    N, C, K = 2048, 64, 64
    x, e = make((N,), C, K, F16, seed=4)
    flat = torch.empty(N * C + 8, dtype=F16, device="cuda")
    xv = flat[1:1 + N * C].view(N, C)
    xv.copy_(x)
    assert xv.data_ptr() % 16 == 2 and xv.is_contiguous()
    u = dw_matmul_large_n(xv, e)
    assert _lib.last_kernel() == "fma_dense_dw"
    assert torch.equal(u, dw_matmul_large_n(x, e, flags=_lib.FLAG_FORCE_GENERIC))
    with pytest.raises(ValueError, match="aligned"):
        dw_matmul_large_n(xv, e, flags=_lib.FLAG_FORCE_TC)


DET_CASES = [((1 << 20, 32, 32), F16), ((1 << 16, 1024, 256), BF16), ((4096, 512, 512), F16), ((200000, 33, 70), F32),
             ((70000, 64, 64), F32)]


def det_outputs():
    outs = {}
    for i, ((N, C, K), dtype) in enumerate(DET_CASES):
        x, e = make((N,), C, K, dtype, seed=100 + i)
        for route in ("tc", "fma") if tc_ok(dtype, C, K) else ("fma",):
            outs["%d_%s" % (i, route)] = run(x, e, route)[0].cpu().numpy()
    return outs


def test_bitwise_reproducible_across_calls():
    a, b = det_outputs(), det_outputs()
    for key in a:
        assert np.array_equal(a[key].view(np.uint32), b[key].view(np.uint32)), key


def child_outputs(path):
    np.savez(path, **det_outputs())


def test_same_result_under_an_sm_margin(tmp_path):
    """BSMM_SM_MARGIN is read once per process: each margin runs in a child."""
    res = []
    for margin in (0, 12):
        path = str(tmp_path / ("m%d.npz" % margin))
        code = ("import sys; sys.path.insert(0, %r)\n"
                "from tests.test_dw_matmul_gpu import child_outputs\n"
                "child_outputs(%r)\n" % (ROOT, path))
        env = dict(os.environ, BSMM_SM_MARGIN=str(margin), BSMM_WAIT_TIMEOUT_MS="2000,notrap")
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
        r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, "margin %d child failed:\n%s%s" % (margin, r.stdout[-4000:], r.stderr[-4000:])
        res.append(np.load(path))
    mine = det_outputs()
    for key in mine:
        for margin, other in zip((0, 12), res):
            assert np.array_equal(mine[key].view(np.uint32), other[key].view(np.uint32)), (key, margin)


def sequential_fp32(x, e):
    """One unsplit fp32 accumulation over the minibatch, row by row (numpy's accumulate is sequential)."""
    C, K = x.shape[1], e.shape[1]
    acc = np.zeros((C, K), np.float32)
    for n0 in range(0, x.shape[0], 1 << 16):
        p = x[n0:n0 + (1 << 16), :, None] * e[n0:n0 + (1 << 16), None, :]
        p[0] += acc
        acc = np.add.accumulate(p, axis=0)[-1]
    return acc


def test_split_is_at_least_as_accurate_as_one_long_fp32_sum():
    N, C, K = 1 << 20, 32, 32
    x, e = make((N,), C, K, F16, seed=9)
    ref, _ = reference(x, e)
    u, kernel = run(x, e, "tc")
    assert kernel == "wgmma_dense_dw"
    base = sequential_fp32(x.float().cpu().numpy(), e.float().cpu().numpy())
    err_split = np.abs(u.cpu().numpy().astype(np.float64) - ref).max()
    err_seq = np.abs(base.astype(np.float64) - ref).max()
    assert err_split <= err_seq, (err_split, err_seq)


# The reference's fp16 kernel for C, K % 8 == 0 (hmma_gemm_64x64x32_TN_vec8) fills its wmma fragments through the
# element layout of Volta; built for sm_90a it returns zeros or NaN, so fp16 parity uses shapes with C or K % 8 == 4,
# which the reference runs on its CUDA-core kernel (gemm_32x32x32_TN_vec4), like all of its fp32 shapes.
PARITY = [(s, F32) for s in REF_SHAPES] + [(s, F16) for s in ((32, 4, 4), (1 << 17, 132, 132), (1 << 15, 36, 516),
                                                             (1 << 20, 12, 20))]


@pytest.mark.skipif(not ref_matmul.available(), reason=ref_matmul.missing() or "")
@pytest.mark.parametrize("shape,dtype", PARITY, ids=lambda v: str(v).split(".")[-1])
def test_reference_parity(shape, dtype):
    N, C, K = shape
    x, e = make((N,), C, K, dtype, seed=21)
    ref, _ = reference(x, e)
    mine = dw_matmul_large_n(x, e).cpu().numpy()
    theirs = ref_matmul.dw_matmul_large_n(x, e).cpu().numpy()
    m_max, m_l2 = ref_errors(mine, ref)
    t_max, t_l2 = ref_errors(theirs, ref)
    assert t_l2 <= 1e-5, "the reference kernel itself is off: %s" % ((t_max, t_l2),)
    assert m_max <= 4 * t_max + 1e-6 and m_l2 <= 4 * t_l2 + 1e-7, ((m_max, m_l2), (t_max, t_l2))
    assert ref_errors(mine, theirs.astype(np.float64))[1] <= 1e-5
