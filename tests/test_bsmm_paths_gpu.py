"""GPU checks of the block-sparse matmul paths around the wgmma kernels, elementwise against float64:

* the CUDA-core (fp32 FMA) xprop / updat kernels on 16-bit data, reached the ways users reach them: feature axis 0
  with N % 8 != 0, operands that are contiguous but not 16-byte aligned, 8 x 8 blocks with an odd number of block rows
  or with BSMM_PAD8=0, and FLAG_FORCE_GENERIC;
* the weight helpers of the gated and padded paths: bsmm_gate_weights and bsmm_pad_blocks / bsmm_unpad_blocks bit for
  bit, bsmm_gate_grad within its bound;
* 16-bit autograd: the gated op with gate_grad, and group_param_grads flushing twice into a bf16 dw.

Each case asserts which kernel ran, so a change of dispatch cannot pass silently."""
import numpy as np
import pytest
import torch

import blocksparse_b200.matmul as mm
from tests._util import (U_OUT, _on_poisoned_output, assert_within, assert_zero_filled, dtype_name, feature_terms,
                         fma_gemm_bound, mma_gemm_bound, oracle_dense, record_kernels)
from blocksparse_b200 import BlocksparseMatMul, group_param_grads, _lib
from oracle.bsmm_oracle import MatmulOracle

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def make_layout(rng, CB, KB, density=0.4, empty_col=1, empty_row=2):
    lay = (rng.random((CB, KB)) < density).astype(np.int32)
    lay[0, 0] = lay[CB - 1, KB - 1] = 1
    lay[:, empty_col] = 0
    lay[empty_row, :] = 0
    return lay


def dense_oracle(lay, bs, axis, w_shape):
    """MatmulOracle of the layout at any (block size, axis): its dense restatement does not depend on the pair."""
    orc = MatmulOracle(lay, 32, axis)
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, lay.shape[0] * bs, lay.shape[1] * bs, w_shape
    return orc


def normal(rng, shape, s, dtype):
    return torch.as_tensor(rng.normal(0, s, shape).astype(np.float32)).to(dtype)


FMA_CASES = [
    # route, bs, axis, dtype, N
    ("n_odd", 16, 0, BF16, 7),        # feature axis 0 with N % 8 != 0: no TMA descriptor for that row pitch
    ("n_odd", 32, 0, F16, 13),
    ("n_odd", 64, 0, BF16, 65),
    ("offset", 16, 1, F16, 40),       # contiguous operands 2 bytes into their buffers
    ("offset", 32, 0, BF16, 64),
    ("offset", 64, 1, BF16, 24),
    ("odd_cb", 8, 0, BF16, 40),       # 8 x 8 blocks, 7 block rows: no 2 x 2 padding
    ("odd_cb", 8, 1, F16, 33),
    ("pad8_off", 8, 1, BF16, 48),     # BSMM_PAD8=0
    ("generic", 8, 0, F16, 48),       # FLAG_FORCE_GENERIC
    ("generic", 16, 1, BF16, 40),
    ("generic", 32, 1, F16, 72),
    ("generic", 64, 0, BF16, 16),
]


@pytest.mark.parametrize("case", FMA_CASES)
def test_fma_xprop_updat_16bit(case, monkeypatch):
    """fprop / bprop (plain and gated) and updat (fp32 and 16-bit dw, beta = 1, gated dw) on the CUDA-core kernels."""
    route, bs, axis, dtype, N = case
    if route == "pad8_off":
        monkeypatch.setattr(mm, "_PAD8", 0)
    rng = np.random.default_rng(bs * 100 + N + axis)
    lay = make_layout(rng, 7, 6) if route == "odd_cb" else make_layout(rng, 6, 8)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    if bs == 8:
        assert (bsmm._shadow is None) == (route != "generic")
    orc = dense_oracle(lay, bs, axis, bsmm.w_shape)
    flags = _lib.FLAG_FORCE_GENERIC if route == "generic" else 0
    W, X, E = normal(rng, bsmm.w_shape, 0.2, dtype), normal(rng, bsmm.i_shape(N), 1, dtype), normal(rng, bsmm.o_shape(N), 1, dtype)
    gate = ((rng.random(bsmm.blocks) < 0.7) * rng.uniform(0.5, 1.5, bsmm.blocks)).astype(np.float32)
    g, gn = torch.as_tensor(gate).cuda(), gate.astype(np.float64)[:, None, None]

    def dev(t):
        if route != "offset":
            return t.cuda()
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.data_ptr() % 16 == 2
        return v

    Xd, Ed, Wd = dev(X), dev(E), dev(W)
    name = dtype_name(dtype)
    # bs >= 16 without FLAG_FORCE_GENERIC folds the gate into a rounded weight copy (bsmm_gate_weights); otherwise the
    # CUDA-core kernel scales each loaded weight, to_f32(w) * g: one more fp32 rounding per term
    folded = bs >= 16 and route != "generic"
    Wn = W.double().numpy()
    Wg = (W.float() * torch.as_tensor(gate)[:, None, None]).to(dtype).double().numpy() if folded else Wn * gn
    for bprop, inp, xd in [(False, X, Xd), (True, E, Ed)]:
        fn = bsmm.bprop if bprop else bsmm.fprop
        op = "bprop" if bprop else "fprop"
        inp_n = inp.double().numpy()
        empty = np.nonzero(lay.sum(axis=1 if bprop else 0) == 0)[0]
        for gated in (False, True):
            w_ref = Wg if gated else Wn
            ref, ref_abs = oracle_dense(orc, op, inp_n, w_ref), oracle_dense(orc, op, np.abs(inp_n), np.abs(w_ref))
            k = feature_terms(lay, bs, bprop, axis) * (1.5 if gated and not folded else 1)
            got = _on_poisoned_output(lambda: fn(xd, Wd, gate=g if gated else None, flags=flags))
            what = "%s%s %s" % ("gated " if gated else "", op, route)
            assert _lib.device_error() == 0 and _lib.last_kernel() == "fma_sdd_xn", (what, _lib.last_kernel())
            assert_zero_filled(got, empty, bs, axis, what)
            assert_within(got, ref, fma_gemm_bound(ref, ref_abs, name, k), what)

    Xn, En = X.double().numpy(), E.double().numpy()
    ref_dw, abs_dw = oracle_dense(orc, "updat", Xn, En), oracle_dense(orc, "updat", np.abs(Xn), np.abs(En))

    def check_dw(got, r, a, k, what):
        assert _lib.device_error() == 0 and _lib.last_kernel() == "fma_dds_nt", (what, _lib.last_kernel())
        assert not bool(torch.isnan(got).any()), "%s: dw elements never written" % what
        assert_within(got, r, fma_gemm_bound(r, a, dtype_name(got.dtype), k), what)

    for dw_dtype in (F32, dtype):
        what = "%s dw %s" % (dtype_name(dw_dtype), route)
        dw = _on_poisoned_output(lambda: bsmm.updat([Xd], [Ed], dw_dtype=dw_dtype, flags=flags))
        check_dw(dw, ref_dw, abs_dw, N, what)
        old = dw.double().cpu().numpy()
        bsmm.updat([Xd], [Ed], dw=dw, flags=flags)                                  # beta = 1: one more fp32 add
        check_dw(dw, old + ref_dw, np.abs(old) + abs_dw, N + 1, "accumulate into " + what)
        dwg = _on_poisoned_output(lambda: bsmm.updat([Xd], [Ed], gate=g, dw_gated=True, dw_dtype=dw_dtype, flags=flags))
        check_dw(dwg, ref_dw * gn, abs_dw * gn, N + 1, "gated " + what)


@pytest.mark.parametrize("bs,dtype", [(8, BF16), (16, F16), (32, BF16), (64, F16), (32, F32)])
def test_gate_weights_bit_exact(bs, dtype):
    """bsmm_gate_weights (the gated wgmma xprop's weight copy) == (W.float() * g).to(dtype) bit for bit; zero gates
    give exact zero blocks."""
    rng = np.random.default_rng(bs)
    blocks = 37
    W = normal(rng, (blocks, bs, bs), 1, dtype)
    gate = rng.uniform(-1.5, 1.5, blocks).astype(np.float32)
    gate[::5] = 0.0
    Wd, g = W.cuda(), torch.as_tensor(gate).cuda()

    def run():
        out = torch.empty_like(Wd)
        _lib.check(_lib.load().bsmm_gate_weights(_lib.dtype_code(dtype), bs, blocks, Wd.data_ptr(), g.data_ptr(), out.data_ptr(),
                                                 _lib.stream_ptr()), "bsmm_gate_weights")
        return out
    out = _on_poisoned_output(run)
    assert _lib.last_kernel() == "gate_weights", _lib.last_kernel()
    ref = (W.float() * torch.as_tensor(gate)[:, None, None]).to(dtype)
    assert torch.equal(out.cpu(), ref), "%d elements differ" % int((out.cpu() != ref).sum())
    assert bool((out[torch.as_tensor(gate == 0).cuda()] == 0).all())


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_pad_unpad_blocks_bit_exact(dtype):
    """bsmm_pad_blocks / bsmm_unpad_blocks (the 8 x 8 -> 16 x 16 super-block maps of the padded path) against a NumPy
    construction from the op's _sub_map / _inv_map: absent sub-blocks zero, the gate folded in, the gated dw, in-place
    accumulation, and fp32 -> 16-bit output."""
    rng = np.random.default_rng(17)
    lay = make_layout(rng, 10, 12, 0.35)
    bsmm = BlocksparseMatMul(lay, block_size=8, feature_axis=0)
    sh, sub, inv = bsmm._shadow, bsmm._sub_map, bsmm._inv_map
    W = normal(rng, bsmm.w_shape, 1, dtype)
    gate = ((rng.random(bsmm.blocks) < 0.7) * rng.uniform(0.5, 1.5, bsmm.blocks)).astype(np.float32)
    Wd, g = W.cuda(), torch.as_tensor(gate).cuda()
    Wf = W.float().numpy()
    for gt in (None, gate):
        big = np.zeros((sh.blocks * 4, 8, 8), dtype=np.float32)
        have = sub >= 0
        big[have] = Wf[sub[have]] * (1 if gt is None else gt[sub[have]][:, None, None])
        ref = torch.as_tensor(big.reshape(sh.blocks, 2, 2, 8, 8).transpose(0, 1, 3, 2, 4).reshape(sh.w_shape)).to(dtype)
        got = _on_poisoned_output(lambda: bsmm._padded_weights(Wd, None if gt is None else g))
        assert _lib.last_kernel() == "pad_blocks", _lib.last_kernel()
        assert torch.equal(got.cpu(), ref), "pad (gate %s): %d elements differ" % (gt is not None, int((got.cpu() != ref).sum()))

    dw16 = torch.as_tensor(rng.normal(0, 1, sh.w_shape).astype(np.float32)).cuda()
    _, inv_d = bsmm._pad_maps(dw16.device)
    src = dw16.cpu().numpy().reshape(sh.blocks, 2, 8, 2, 8)[inv >> 2, (inv >> 1) & 1, :, inv & 1, :]     # (blocks, 8, 8)
    # (gate, accumulate, output dtype); not gate and accumulate together: v * g + old may compile to one fused multiply-add
    for gt, acc, out_dtype in [(None, 0, F32), (gate, 0, F32), (None, 1, F32), (gate, 0, dtype), (None, 1, dtype)]:
        old = normal(rng, bsmm.w_shape, 1, out_dtype)
        out = old.cuda()
        _lib.check(_lib.load().bsmm_unpad_blocks(_lib.F32, _lib.dtype_code(out_dtype), 8, bsmm.blocks, inv_d.data_ptr(), dw16.data_ptr(),
                                                 _lib.ptr(None if gt is None else g), out.data_ptr(), acc, _lib.stream_ptr()),
                   "bsmm_unpad_blocks")
        assert _lib.last_kernel() == "unpad_blocks", _lib.last_kernel()
        v = src * (1 if gt is None else gt[:, None, None])
        if acc:
            v = v + old.float().numpy()
        ref = torch.as_tensor(v.astype(np.float32)).to(out_dtype)
        assert torch.equal(out.cpu(), ref), "unpad (gate %s, acc %d, %s): %d elements differ" % (
            gt is not None, acc, out_dtype, int((out.cpu() != ref).sum()))


@pytest.mark.parametrize("bs,dtype", [(8, F32), (16, BF16), (32, F16), (64, BF16), (64, F32)])
def test_gate_grad_matches_float64(bs, dtype):
    """bsmm_gate_grad: dg[w] = sum(dw[w] * w[w]) -- per lane bs^2 / 32 fmaf steps, then a 5-level shuffle tree."""
    rng = np.random.default_rng(bs + 3)
    lay = np.ones((3, 11), dtype=np.int32)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=0)
    dw, w = normal(rng, bsmm.w_shape, 1, dtype), normal(rng, bsmm.w_shape, 0.3, dtype)
    dg = bsmm.gate_grad(dw.cuda(), w.cuda())
    assert _lib.last_kernel() == "gate_grad", _lib.last_kernel()
    p = dw.double().numpy() * w.double().numpy()
    ref, ref_abs = p.sum(axis=(1, 2)), np.abs(p).sum(axis=(1, 2))
    assert_within(dg, ref, fma_gemm_bound(ref, ref_abs, "float32", bs * bs + 5), "gate_grad")


def test_bf16_autograd_gated_with_gate_grad(monkeypatch):
    """bsmm(x, w, gate=g, gate_grad=True, dw_gated=True) in bf16: y and x.grad on the wgmma kernels with the folded gate,
    w.grad = (raw bf16 dw) * g in bf16, gate.grad = sum(raw dw * w) -- each against float64, with the 16-bit rounding
    of the intermediate dw in the bound."""
    rng = np.random.default_rng(23)
    bs, axis, N = 32, 1, 96
    lay = make_layout(rng, 8, 10)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, bs, axis)
    W, X, E = normal(rng, bsmm.w_shape, 0.1, BF16), normal(rng, bsmm.i_shape(N), 1, BF16), normal(rng, bsmm.o_shape(N), 1, BF16)
    gate = ((rng.random(bsmm.blocks) < 0.8) * rng.uniform(0.5, 1.5, bsmm.blocks)).astype(np.float32)
    w, x = W.cuda().requires_grad_(), X.cuda().requires_grad_()
    g = torch.as_tensor(gate).cuda().requires_grad_()
    seen = []
    record_kernels(monkeypatch, bsmm, ("fprop", "bprop", "updat", "gate_grad"), seen)
    y = bsmm(x, w, gate=g, gate_grad=True, dw_gated=True)
    y.backward(E.cuda())
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert seen == [("fprop", "wgmma_xprop_bs32"), ("bprop", "wgmma_xprop_bs32"), ("updat", "wgmma_updat_bs32"),
                    ("gate_grad", "gate_grad")], seen
    u = U_OUT["bfloat16"]
    Xn, En, Wn = X.double().numpy(), E.double().numpy(), W.double().numpy()
    Wg = (W.float() * torch.as_tensor(gate)[:, None, None]).bfloat16().double().numpy()
    for got, op, a, what in [(y, "fprop", Xn, "y"), (x.grad, "bprop", En, "x.grad")]:
        ref, ref_abs = oracle_dense(orc, op, a, Wg), oracle_dense(orc, op, np.abs(a), np.abs(Wg))
        k = feature_terms(lay, bs, op == "bprop", axis)
        assert_within(got, ref, mma_gemm_bound(ref, ref_abs, "bfloat16", k), what)
    raw, raw_abs = oracle_dense(orc, "updat", Xn, En), oracle_dense(orc, "updat", np.abs(Xn), np.abs(En))
    b_raw = mma_gemm_bound(raw, raw_abs, "bfloat16", N)                 # the bf16 dw the backward computes first
    gn = gate.astype(np.float64)[:, None, None]
    g16 = torch.as_tensor(gate).bfloat16().double().numpy()[:, None, None]
    ref_w = raw * gn
    assert w.grad.dtype == BF16
    assert_within(w.grad, ref_w, u * np.abs(ref_w) + (1 + u) * (g16 * b_raw + np.abs(raw) * np.abs(g16 - gn)), "w.grad")
    ref_g = (raw * Wn).sum(axis=(1, 2))
    b_g = (b_raw * np.abs(Wn)).sum(axis=(1, 2))
    b_g += fma_gemm_bound(ref_g, ((np.abs(raw) + b_raw) * np.abs(Wn)).sum(axis=(1, 2)), "float32", bs * bs + 5)
    assert_within(g.grad, ref_g, b_g, "gate.grad")


def test_bf16_group_param_grads_eleven_uses(monkeypatch):
    """group_param_grads in bf16 over 11 uses of one weight: an 8-pair flush into a fresh bf16 dw, then a 3-pair flush
    that accumulates into it (beta = 1, 16-bit dw) on the wgmma updat kernel."""
    rng = np.random.default_rng(29)
    bs, axis, N, T = 32, 1, 64, 11
    lay = make_layout(rng, 8, 8)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, bs, axis)
    w = normal(rng, bsmm.w_shape, 0.1, BF16).cuda().requires_grad_()
    xs = [normal(rng, bsmm.i_shape(N), 1, BF16).cuda() for _ in range(T)]
    es = [normal(rng, bsmm.o_shape(N), 1, BF16).cuda() for _ in range(T)]
    flushed, seen = [], []
    record_kernels(monkeypatch, bsmm, ("updat",), seen)
    with group_param_grads(bsmm, w) as pend:
        flush = pend.flush

        def recording_flush():                       # which (x, dy) pairs went into which launch
            flushed.append([(a.double().cpu().numpy(), b.double().cpu().numpy()) for a, b in zip(pend.xs, pend.dys)])
            flush()
        pend.flush = recording_flush
        torch.autograd.backward([bsmm(x, w) for x in xs], es)
    assert pend.launches == 2 and [len(f) for f in flushed] == [8, 3]
    assert seen == [("updat", "wgmma_updat_bs32")] * 2, seen
    assert _lib.device_error() == 0, _lib.device_error_text()
    sums = [[sum(oracle_dense(orc, "updat", f(a), f(b)) for a, b in fl) for f in (lambda t: t, np.abs)] for fl in flushed]
    (r1, a1), (r2, a2) = sums
    b1 = mma_gemm_bound(r1, a1, "bfloat16", 8 * N)
    u = U_OUT["bfloat16"]
    bound = mma_gemm_bound(r1 + r2, a1 + a2 + b1, "bfloat16", 3 * N, extra=1) + (1 + u) * b1
    assert w.grad.dtype == BF16
    assert_within(w.grad, r1 + r2, bound, "grouped bf16 dw")
