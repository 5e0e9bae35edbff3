"""Host logic (blocksparse_b200/lut.py) against the reference-generated fixtures and the oracle.

The product LUT builder is vectorised NumPy and shares no code with oracle/; both
must reproduce the reference's wire formats bit for bit.
"""
import os
import pickle

import numpy as np
import pytest

from tests._util import GOLDEN, golden_files
from tests.golden.make_golden import causal_callback, checker_callback
from blocksparse_b200.lut import MatmulLuts, TransformerLuts, build_tile_schedule, z_order_2d
from oracle.bsmm_oracle import MatmulOracle, z_order_2d as z_ref
from oracle.bst_oracle import TransformerOracle


def test_z_order_vectorised_matches_scalar():
    rng = np.random.default_rng(0)
    x = rng.integers(0, 70000, 200)
    y = rng.integers(0, 70000, 200)
    got = z_order_2d(x, y)
    want = [z_ref(int(a), int(b)) for a, b in zip(x, y)]
    assert got.tolist() == want
    assert z_order_2d(3, 5) == z_ref(3, 5)


@pytest.mark.parametrize("fname", golden_files("bsmm_"))
def test_matmul_luts_match_reference(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    L = MatmulLuts(g["layout"])
    np.testing.assert_array_equal(L.fprop_lut, g["fprop_lut"])
    np.testing.assert_array_equal(L.bprop_lut, g["bprop_lut"])
    np.testing.assert_array_equal(L.updat_lut, g["updat_lut"])
    meta = [L.fprop_segments, L.fprop_locks, L.fprop_shared, L.bprop_segments, L.bprop_locks, L.bprop_shared, L.blocks]
    np.testing.assert_array_equal(np.array(meta), g["meta"][:7])


def _random_layouts():
    rng = np.random.default_rng(7)
    for shape, d in [((1, 1), 1.0), ((3, 17), 0.3), ((40, 40), 0.05), ((33, 9), 0.6), ((64, 64), 0.2), ((128, 128), 0.1)]:
        lay = (rng.random(shape) < d).astype(np.int32)
        lay[rng.integers(shape[0]), rng.integers(shape[1])] = 1
        yield lay
    lay = (rng.random((48, 48)) < 0.04).astype(np.int32)
    lay[:, :3] = 1          # skewed columns -> segmentation + locks
    yield lay


@pytest.mark.parametrize("z", [True, False])
def test_matmul_luts_match_oracle_on_random_layouts(z):
    for lay in _random_layouts():
        L = MatmulLuts(lay, z_order=z)
        O = MatmulOracle(lay, 32, 1, z_order=z)
        np.testing.assert_array_equal(L.fprop_lut, O.fprop_lut)
        np.testing.assert_array_equal(L.bprop_lut, O.bprop_lut)
        np.testing.assert_array_equal(L.updat_lut, O.updat_lut)
        assert (L.fprop_segments, L.fprop_locks, L.fprop_shared) == (O.fprop_segments, O.fprop_locks, O.fprop_shared)
        assert (L.bprop_segments, L.bprop_locks, L.bprop_shared) == (O.bprop_segments, O.bprop_locks, O.bprop_shared)
        assert L.fprop_list == O.fprop_list
        assert L.bprop_list == O.bprop_list
        assert L.updat_list == O.updat_list


def _decode_rows(rows, n_out):
    out = []
    for o in range(n_out):
        first, cnt = rows[o]
        out.append([(int(rows[first + e][1]), int(rows[first + e][0])) for e in range(cnt)])   # (in, w)
    return out


def test_row_lut_matches_lists():
    for lay in _random_layouts():
        L = MatmulLuts(lay)
        for bprop in (False, True):
            rows = L.bprop_rows if bprop else L.fprop_rows
            lists = dict(L.bprop_list if bprop else L.fprop_list)
            n_out = L.CB if bprop else L.KB
            dec = _decode_rows(rows, n_out)
            for o in range(n_out):
                assert dec[o] == lists[o]


@pytest.mark.parametrize("bsize,T,wpg", [(32, 16, 8), (32, 15, 8), (32, 4, 3), (64, 8, 4)])
def test_tile_schedule_is_a_faithful_regrouping(bsize, T, wpg):
    """Simulate the device loops on the schedule: every LUT entry is issued exactly once, on the right
    accumulator, always accumulating (the kernel's epilogue leaves the accumulators zeroed)."""
    for lay in _random_layouts():
        L = MatmulLuts(lay)
        for bprop in (False, True):
            lists = dict(L.bprop_list if bprop else L.fprop_list)
            n_out = L.CB if bprop else L.KB
            s, off = L.tile_schedule(bprop, T, bsize, wpg)
            n_tiles, Tt, n_groups, n_w_total = s[:4]
            assert Tt == T and n_w_total == L.blocks and n_tiles == -(-n_out // T) and off % 32 == 0
            wbytes16 = (bsize * bsize * 2) >> 4
            seen = set()
            gi_expected = 0
            fo_expected = 0
            for t in range(n_tiles):
                fg, ng, fo, packed = s[4 + 4 * t: 8 + 4 * t]
                no, mask = packed & 0xff, packed >> 8
                assert fg == gi_expected and fo == fo_expected and 1 <= no <= T       # contiguous tiles, at most T wide
                fo_expected += no
                assert mask == sum(1 << sl for sl in range(no) if lists[fo + sl])
                gi_expected += ng
                touched = set()
                prev_in = -1
                for g in range(fg, fg + ng):
                    rec = s[off + 32 * g: off + 32 * g + 32]
                    ib, n_w, n_runs = rec[0], rec[1] & 0xff, rec[1] >> 8
                    assert 1 <= n_w <= wpg and 1 <= n_runs <= n_w and ib >= prev_in
                    prev_in = ib
                    covered = 0
                    for r in range(n_runs):
                        r0, r1 = int(rec[12 + r]), int(rec[20 + r])
                        w_slot, col = (r0 & 0xffff) // wbytes16, r0 >> 16
                        n, acc = (r1 >> 17) << 3, r1 & 1
                        assert (r0 & 0xffff) % wbytes16 == 0 and col % bsize == 0 and n % bsize == 0 and n <= 256
                        assert w_slot == covered          # runs tile the staged W blocks in order
                        for i in range(n // bsize):
                            slot = col // bsize + i
                            w = int(rec[4 + w_slot + i])
                            assert 0 <= slot < no and (int(ib), w) in lists[fo + slot]
                            assert acc == 1
                            assert w not in seen
                            seen.add(w)
                        for i in range(n // bsize):
                            touched.add(col // bsize + i)
                        covered += n // bsize
                    assert covered == n_w
            assert len(seen) == L.blocks and gi_expected == n_groups and fo_expected == n_out


def _cb(name, has_mask):
    if not has_mask:
        return None
    return checker_callback if "perhead" in name else causal_callback


@pytest.mark.parametrize("fname", golden_files("bst_"))
def test_transformer_luts_match_reference(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    lay = g["layout"]
    if lay.ndim == 2:
        lay = lay[None]
    L = TransformerLuts(lay, int(g["bs"]), _cb(fname, bool(g["has_mask"])))
    np.testing.assert_array_equal(L.nt_lut, g["nt_lut"])
    np.testing.assert_array_equal(L.nn_lut, g["nn_lut"])
    np.testing.assert_array_equal(L.tn_lut, g["tn_lut"])
    np.testing.assert_array_equal(np.array([L.blocks, L.nn_max, L.tn_max, L.ctx_blks_q, L.ctx_blks_k]), g["meta"])
    if bool(g["has_mask"]):
        np.testing.assert_array_equal(L.softmax_mask_np, g["mask_np"])
        np.testing.assert_array_equal(L.softmax_mask, g["mask_dev"])
    O = TransformerOracle(g["layout"], int(g["bs"]), heads=int(g["heads"]))
    assert L.nt_list == O.nt_list and L.nn_list == O.nn_list and L.tn_list == O.tn_list


def test_classes_construct_and_pickle_without_gpu():
    from blocksparse_b200 import BlocksparseMatMul, BlocksparseTransformer
    lay = np.eye(4, dtype=np.int32)
    lay[0, 3] = 1
    m = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    assert m.w_shape == (5, 32, 32) and m.i_shape(7) == (7, 128) and m.o_shape(7) == (7, 128)
    assert m.block_coord(0) == (0, 0) and m.flops == 5 * 32 * 32 * 2 and m.sparsity == round(5 / 16, 3)
    m2 = pickle.loads(pickle.dumps(m))
    np.testing.assert_array_equal(m2.fprop_lut, m.fprop_lut)
    with pytest.raises(ValueError):
        BlocksparseMatMul(lay, block_size=12)
    t = BlocksparseTransformer(np.tril(np.ones((3, 3), np.int32)), block_size=16, heads=2, mask_callback=causal_callback)
    assert t.blocks == 6 and t.nn_max == 3 and t.block_coord(1) == (1, 0)
    t2 = pickle.loads(pickle.dumps(t))
    np.testing.assert_array_equal(t2.softmax_mask_np, t.softmax_mask_np)


@pytest.mark.parametrize("bsize", [32, 64])
def test_updat_schedule_covers_every_block_once(bsize):
    for lay in _random_layouts():
        L = MatmulLuts(lay)
        s, off = L.updat_schedule(bsize)
        n_tiles, G, KT, stride = s[:4]
        assert G == 128 // bsize and KT == 256 // bsize and stride == 64 and off == 4
        rec = s[off:].reshape(n_tiles, 64)
        seen, gk_seen = set(), set()
        assert (np.diff(rec[:, 1]) <= 0).all()            # longest tiles first
        for t in range(n_tiles):
            c0, n_act = rec[t, 0], rec[t, 1]
            assert c0 % G == 0 and 1 <= n_act <= KT
            ks = rec[t, 8:8 + n_act]
            assert (np.diff(ks) > 0).all()                 # distinct output blocks, ascending (windows of the group's kept blocks)
            assert all((int(c0), int(k)) not in gk_seen for k in ks)     # an output block of a group lives in one tile only
            gk_seen.update((int(c0), int(k)) for k in ks)
            for sl in range(n_act):
                col_has_block = False
                for i in range(G):
                    w = rec[t, 16 + i * KT + sl]
                    if w >= 0:
                        assert tuple(L.updat_lut[w]) == (c0 + i, ks[sl]) and w not in seen
                        seen.add(int(w))
                        col_has_block = True
                assert col_has_block                       # compacted: no slot without work
            for sl in range(n_act, KT):
                assert (rec[t, [16 + i * KT + sl for i in range(G)]] == -1).all()
        assert len(seen) == L.blocks


def test_updat_schedule_balances_whole_waves():
    """With a CTA count the window split trades a few more tiles for whole waves; coverage and compaction stay intact."""
    from blocksparse_b200.lut import _updat_makespan
    rng = np.random.default_rng(5)
    lay = (rng.random((128, 128)) < 0.25).astype(np.int32)
    L = MatmulLuts(lay)
    base, _ = L.updat_schedule(32)
    bal, off = L.updat_schedule(32, n_cta=148)
    nb, nl = int(base[0]), int(bal[0])
    assert nl >= nb and nl % 148 == 0                       # 370 -> 444 tiles = three full waves
    rec = bal[off:].reshape(nl, 64)
    cost = lambda r: np.sort(4.0 + r[:, 1].astype(float))[::-1]
    def makespan(r):
        load = np.zeros(148)
        np.add.at(load, np.arange(len(r)) % 148, cost(r))
        return load.max()
    assert makespan(rec) < makespan(base[off:].reshape(nb, 64))
    seen = set()
    for t in range(nl):
        n_act = rec[t, 1]
        assert 1 <= n_act <= 8
        for sl in range(n_act):
            ws = [int(rec[t, 16 + i * 8 + sl]) for i in range(4) if rec[t, 16 + i * 8 + sl] >= 0]
            assert ws and not (set(ws) & seen)
            seen.update(ws)
    assert len(seen) == L.blocks
    # a layout that already fills its waves, or a tiny one, is left alone
    tiny = MatmulLuts(np.ones((4, 4), dtype=np.int32))
    a, _ = tiny.updat_schedule(32)
    b, _ = tiny.updat_schedule(32, n_cta=148)
    assert np.array_equal(a, b)


def test_pick_tile_count_fills_whole_waves():
    from blocksparse_b200.lut import pick_tile_count
    # BASELINE cfg 2 with 296 CTA slots: 32 minibatch tiles, 128 output blocks
    n_kt = pick_tile_count(128, 32, 296, 8)
    assert n_kt == 18 and 32 * n_kt <= 2 * 296            # 576 tiles: two full waves instead of 512 in 1.73
    assert pick_tile_count(8, 1, 296, 8) == 2             # idle slots: narrower tiles spread a small problem over more CTAs
    for n_out, n_nt in [(5, 3), (128, 1), (37, 200), (1, 1)]:
        k = pick_tile_count(n_out, n_nt, 296, 8)
        assert -(-n_out // k) <= 8 and k >= -(-n_out // 8)
    # uneven tiles cover every block exactly once
    L = MatmulLuts((np.random.default_rng(0).random((40, 37)) < 0.3).astype(np.int32) | np.eye(40, 37, dtype=np.int32))
    s, off = L.tile_schedule(False, 8, 32, 8, n_tiles=6)
    sizes = [int(s[4 + 4 * t + 3]) & 0xff for t in range(6)]
    assert sum(sizes) == 37 and max(sizes) - min(sizes) <= 1
