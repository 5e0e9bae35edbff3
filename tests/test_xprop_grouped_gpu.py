"""The grouped tile of the default 32 x 32 wgmma xprop route (csrc/tc_xprop2.cuh: tc_xprop_grouped_kernel; selection in
lut.pick_xprop_tile): one CTA owns several consecutive output blocks, stages each activation tile once for all of them
and multiplies only the W blocks that exist. Forced through matmul._XPROP_TILE, it must give the results of one output
block per CTA bit for bit, stay within the float64 bound with the single-block k_terms (no zero blocks are added), and
keep every output block independent of input blocks its LUT row does not list."""
import numpy as np
import pytest
import torch

import blocksparse_b200.matmul as mm
from tests.test_tc_gpu import check_xprop, layout, operands
from blocksparse_b200 import BlocksparseMatMul, _lib
from blocksparse_b200.layouts import barabasi_albert_layout, bernoulli_layout
from blocksparse_b200.lut import XPROP_GROUP
from oracle.bsmm_oracle import MatmulOracle

pytestmark = pytest.mark.gpu

GROUPED = sorted(mm._GROUPED_VARIANTS)

CASES = [
    # CB, KB, kind, N
    (24, 20, 0.08, 1),
    (24, 20, 0.25, 136),
    (16, 24, 0.5, 200),
    (12, 12, "dense", 257),
    (10, 16, "checker", 640),
    (32, 32, "skewed", 200),
    (5, 37, 0.5, 257),             # block counts that are no multiple of the tile
    (33, 17, 0.3, 136),
    (24, 24, "empty_tiles", 640),  # output blocks 8..15 have no entry in either direction: whole tiles write zeros
    (140, 140, 0.6, 136),          # more merged entries per tile than the kernel keeps in shared memory at a time
]


def make_layout(rng, CB, KB, kind):
    if kind == "dense":
        return np.ones((CB, KB), dtype=np.int32)
    if kind == "checker":
        return ((np.arange(CB)[:, None] + np.arange(KB)[None, :]) % 2).astype(np.int32)
    if kind == "skewed":
        return barabasi_albert_layout(CB, 0.25, rng)
    if kind == "empty_tiles":
        lay = layout(rng, CB, KB, 0.3)
        lay[8:16, :] = 0
        lay[:, 8:16] = 0
        lay[0, 0] = 1
        return lay
    return layout(rng, CB, KB, kind, empty_col=KB // 2, empty_row=1)


def forced(monkeypatch, tile, fn):
    monkeypatch.setattr(mm, "_XPROP_TILE", tile)
    out = fn()
    assert _lib.last_kernel() == "wgmma_xprop_bs32", _lib.last_kernel()
    return out


@pytest.mark.parametrize("tile", GROUPED)
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", CASES)
def test_grouped_tile_equals_one_block_per_cta_and_the_oracle(case, dtype, axis, tile, monkeypatch):
    CB, KB, kind, N = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    lay = make_layout(rng, CB, KB, kind)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)
    W, X, E = operands(rng, bsmm, N, dtype)
    Wd = W.cuda()
    for bprop, inp in [(False, X), (True, E)]:
        fn = bsmm.bprop if bprop else bsmm.fprop
        xd = inp.cuda()
        narrow = forced(monkeypatch, 1, lambda: fn(xd, Wd, flags=_lib.FLAG_FORCE_TC))
        monkeypatch.setattr(mm, "_XPROP_TILE", tile)
        got, kern = check_xprop(orc, lay, 32, bprop, inp, W, lambda: fn(xd, Wd, flags=_lib.FLAG_FORCE_TC),
                                "%s tile %d" % ("bprop" if bprop else "fprop", tile), family="wgmma_xprop_grouped")
        assert kern == "wgmma_xprop_bs32", kern
        assert torch.equal(got, narrow), "tile %d differs from one block per CTA" % tile


@pytest.mark.parametrize("tile", GROUPED)
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("bprop", [False, True])
def test_output_blocks_ignore_input_blocks_they_do_not_consume(bprop, axis, tile, monkeypatch):
    """One input block filled with NaN and Inf: every output block whose LUT row does not list it is bit-equal to the run
    on finite input, including blocks that share a tile with a consumer of the poisoned block."""
    rng = np.random.default_rng(7 + tile)
    lay = layout(rng, 16, 16, 0.4)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    m = (lay != 0) if bprop else (lay != 0).T                       # (output block, input block)
    shared = [i for i in range(16) if any(0 < m[t:t + tile, i].sum() < min(tile, 16 - t) for t in range(0, 16, tile))]
    assert shared, "no input block is consumed by a part of a tile"
    bad = shared[0]
    N = 200
    W, X, E = operands(rng, bsmm, N, torch.bfloat16)
    inp = (E if bprop else X).cuda()
    Wd = W.cuda()
    fn = bsmm.bprop if bprop else bsmm.fprop
    clean = forced(monkeypatch, tile, lambda: fn(inp, Wd))
    poison = torch.tensor([float("nan"), float("inf"), float("-inf"), float("nan")], dtype=inp.dtype, device="cuda").repeat(8)
    dirty_in = inp.clone()
    if axis:
        dirty_in[:, bad * 32:(bad + 1) * 32] = poison[None, :]
    else:
        dirty_in[bad * 32:(bad + 1) * 32, :] = poison[:, None]
    dirty = forced(monkeypatch, tile, lambda: fn(dirty_in, Wd))
    assert _lib.device_error() == 0, _lib.device_error_text()
    for o in range(16):
        a, b = ((clean[:, o * 32:(o + 1) * 32], dirty[:, o * 32:(o + 1) * 32]) if axis
                else (clean[o * 32:(o + 1) * 32], dirty[o * 32:(o + 1) * 32]))
        if m[o, bad]:
            assert not bool(torch.isfinite(b).all()), "output block %d consumes the poisoned block" % o
        else:
            assert torch.equal(a, b), "output block %d changed with input block %d, which it does not consume" % (o, bad)


def test_default_route_selects_the_tile_from_layout_and_minibatch():
    """The benchmark's layout at N = 4096 runs grouped, a layout of 8 x 10 blocks at N = 96 one block per CTA, and the
    1024-feature layout of tests/test_large_offsets_gpu.py at N = 2^21 + 128 grouped, so that file covers its offsets."""
    assert mm._XPROP_TILE is None
    dev = torch.device("cuda", torch.cuda.current_device())
    rng = np.random.default_rng(1236)
    lay = (rng.random((128, 128)) < 0.25).astype(np.int32)
    np.fill_diagonal(lay, 1)
    big = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    small = BlocksparseMatMul(layout(np.random.default_rng(0), 8, 10, 0.4), block_size=32, feature_axis=1)
    far = BlocksparseMatMul(bernoulli_layout(np.random.default_rng(20 + 32 + 1), 32, 32, 0.25), block_size=32, feature_axis=1)
    for bprop in (False, True):
        assert big.xprop_tile(bprop, 4096, dev) == XPROP_GROUP
        assert small.xprop_tile(bprop, 96, dev) == 1
        assert far.xprop_tile(bprop, 2 ** 21 + 128, dev) == XPROP_GROUP
    W = (torch.randn(big.w_shape, device="cuda") * 0.1).bfloat16()
    X = torch.randn(big.i_shape(4096), device="cuda").bfloat16()
    y = big.fprop(X, W)
    assert _lib.last_kernel() == "wgmma_xprop_bs32" and ("wide", False, XPROP_GROUP) in big._device_luts(dev)
    mm._XPROP_TILE = 1
    try:
        assert torch.equal(y, big.fprop(X, W))
    finally:
        mm._XPROP_TILE = None


def test_grouped_tile_in_a_cuda_graph(monkeypatch):
    """The grouped launch reads its schedule from device memory and takes its tensor maps by value: captured and replayed
    it reproduces the eager result of one block per CTA."""
    rng = np.random.default_rng(21)
    lay = layout(rng, 32, 32, 0.25)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    W = (torch.randn(bsmm.w_shape, device="cuda") * 0.1).bfloat16()
    X = torch.randn(bsmm.i_shape(512), device="cuda").bfloat16()
    E = torch.randn(bsmm.o_shape(512), device="cuda").bfloat16()
    ref = forced(monkeypatch, 1, lambda: (bsmm.fprop(X, W), bsmm.bprop(E, W)))
    monkeypatch.setattr(mm, "_XPROP_TILE", XPROP_GROUP)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            bsmm.fprop(X, W); bsmm.bprop(E, W)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = bsmm.fprop(X, W)
        dx = bsmm.bprop(E, W)
    y.zero_(); dx.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, ref[0]) and torch.equal(dx, ref[1])
    assert _lib.device_error() == 0
