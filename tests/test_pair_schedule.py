"""Host-side properties of the pair schedule and the LPT tile lists (blocksparse_b200/lut.py), no GPU needed."""
import numpy as np
import pytest

from blocksparse_b200.lut import MatmulLuts, lpt_tile_lists, PAIR_MAX_RUNS


def decode(sched, goff, loff, bsize=32):
    """-> set of (out_block, in_block, w) triples the kernel would multiply, plus per-group sanity checks."""
    n_tiles, T = int(sched[0]), int(sched[1])
    th = sched[4:4 + 4 * n_tiles].reshape(n_tiles, 4)
    recs = sched[goff:loff].reshape(-1, 32)
    triples = []
    for t in range(n_tiles):
        first, n_g, out0, packed = th[t]
        n_out, touched = packed & 0xff, packed >> 8
        seen_slots = 0
        for rec in recs[first:first + n_g]:
            pair = int(rec[0])
            n_w, nr0, nr1 = rec[1] & 0xff, (rec[1] >> 8) & 0xff, (rec[1] >> 16) & 0xff
            assert nr0 <= PAIR_MAX_RUNS and nr1 <= PAIR_MAX_RUNS and 1 <= n_w <= 14
            covered = 0
            for h, nr in ((0, nr0), (1, nr1)):
                for r in range(nr):
                    pk = int(rec[16 + 8 * h + r])
                    pos = (pk & 0xfff) // ((bsize * bsize * 2) >> 4)
                    col = (pk >> 12) & 0x1ff
                    nblk = (((pk >> 21) & 0x3f) << 3) // bsize
                    assert col % bsize == 0 and 1 <= nblk <= 256 // bsize and col + nblk * bsize <= T * bsize
                    for i in range(nblk):
                        slot = col // bsize + i
                        assert slot < n_out
                        seen_slots |= 1 << slot
                        triples.append((int(out0) + slot, 2 * pair + h, int(rec[2 + pos + i])))
                    covered += nblk
            assert covered == n_w                     # every staged W block is multiplied exactly once
        assert seen_slots == touched
    return triples


@pytest.mark.parametrize("bprop", [False, True])
@pytest.mark.parametrize("T,wps", [(8, 4), (8, 8), (16, 12)])
@pytest.mark.parametrize("shape,density", [((7, 20), 1.0), ((33, 40), 0.1), ((64, 64), 0.3), ((6, 32), -1)])
def test_pair_schedule_covers_the_lut_exactly(shape, density, T, wps, bprop):
    rng = np.random.default_rng(sum(shape) + T)
    CB, KB = shape
    if density < 0:
        lay = ((np.arange(CB)[:, None] + np.arange(KB)[None, :]) % 2).astype(np.int32)
    else:
        lay = (rng.random(shape) < density).astype(np.int32)
        lay[0, 0] = 1
    luts = MatmulLuts(lay)
    n_out = CB if bprop else KB
    n_kt = -(-n_out // T)
    sched, goff, loff = luts.pair_schedule(bprop, T, wps, n_kt, 3, 10)
    got = sorted(decode(sched, goff, loff))
    outs, ins, wids = luts._b if bprop else luts._f
    want = sorted(zip(outs.tolist(), ins.tolist(), wids.tolist()))
    assert got == want
    # tile lists: every (minibatch tile, output tile) exactly once
    offs = sched[loff:loff + 11]
    ids = sched[loff + 11:]
    assert offs[0] == 0 and offs[-1] == len(ids) == 3 * n_kt
    assert sorted(ids.tolist()) == list(range(3 * n_kt))


def test_lpt_lists_balance_a_skewed_cost_vector():
    cost = np.array([100.0] + [10.0] * 30)
    lists = lpt_tile_lists(cost, n_ntiles=4, n_ctas=8)
    offs, ids = lists[:9], lists[9:]
    load = [sum(cost[t % 31] for t in ids[offs[c]:offs[c + 1]]) for c in range(8)]
    assert max(load) <= 1.05 * (cost.sum() * 4 / 8) or max(load) == 100.0 + min(load) - min(load)   # near the mean
    assert max(load) - min(load) <= 100.0
    assert sorted(ids.tolist()) == list(range(4 * 31))


@pytest.mark.parametrize("bprop", [False, True])
@pytest.mark.parametrize("shape,density,n_kt,wpg", [((33, 40), 0.1, 5, 2), ((64, 64), 0.3, 8, 4), ((7, 20), 1.0, 3, 4), ((128, 128), 0.25, 18, 4)])
def test_pair_tile_schedule_pairs_walk_one_group_list(shape, density, n_kt, wpg, bprop):
    """build_pair_tile_schedule: tiles 2P and 2P+1 have the same number of groups with the same input blocks in the same
    order, every LUT entry is multiplied exactly once, and an odd tile count is padded with an empty tile."""
    from blocksparse_b200.lut import MatmulLuts
    rng = np.random.default_rng(sum(shape) + n_kt)
    lay = (rng.random(shape) < density).astype(np.int32)
    lay[0, 0] = 1
    luts = MatmulLuts(lay)
    n_out = shape[0] if bprop else shape[1]
    n_kt = min(n_kt, n_out)
    if -(-n_out // n_kt) > 8:
        n_kt = -(-n_out // 8)
    sched, goff = luts.pair_tile_schedule(bprop, 8, 32, wpg, n_kt)
    n_tiles = int(sched[0])
    assert n_tiles % 2 == 0 and n_tiles in (n_kt, n_kt + 1)
    th = sched[4:4 + 4 * n_tiles].reshape(n_tiles, 4)
    recs = sched[goff:].reshape(-1, 32)
    triples = []
    for P in range(n_tiles // 2):
        fa, na = th[2 * P][:2]; fb, nb = th[2 * P + 1][:2]
        assert na == nb
        assert np.array_equal(recs[fa:fa + na, 0], recs[fb:fb + nb, 0])          # same input block sequence
        assert np.all(np.diff(recs[fa:fa + na, 0]) >= 0)
    for t in range(n_tiles):
        first, n_g, out0, packed = th[t]
        for rec in recs[first:first + n_g]:
            n_w, n_runs = rec[1] & 0xff, rec[1] >> 8
            assert n_w <= wpg
            covered = 0
            for r in range(n_runs):
                pos = (rec[12 + r] & 0xffff) // 128
                col = rec[12 + r] >> 16
                nblk = ((rec[20 + r] >> 17) << 3) // 32
                for i in range(nblk):
                    triples.append((int(out0) + col // 32 + i, int(rec[0]), int(rec[4 + pos + i])))
                covered += nblk
            assert covered == n_w
    outs, ins, wids = luts._b if bprop else luts._f
    assert sorted(triples) == sorted(zip(outs.tolist(), ins.tolist(), wids.tolist()))


@pytest.mark.parametrize("bprop", [0, 1])
@pytest.mark.parametrize("T", [2, 4])
def test_wide_schedule_lists_every_block_once_in_input_order(bprop, T):
    """lut.build_wide_schedule (csrc/tc_xprop2.cuh): every (output block, input block) -> W block of the layout appears in
    exactly one merged entry of its tile, entries ascend by input block, and nothing else is listed."""
    from blocksparse_b200.lut import MatmulLuts, WIDE_REC
    rng = np.random.default_rng(5 + T)
    lay = (rng.random((9, 37)) < 0.4).astype(np.int32)
    lay[2, :] = 0
    L = MatmulLuts(lay)
    sched, n_tiles, off = L.wide_schedule(bprop, T)
    outs, ins, wids = L._b if bprop else L._f
    n_out = lay.shape[0] if bprop else lay.shape[1]
    assert n_tiles == -(-n_out // T) and off % WIDE_REC == 0 and int(sched[0]) == n_tiles and int(sched[1]) == T
    got = {}
    for t in range(n_tiles):
        rows = [sched[off + WIDE_REC * e: off + WIDE_REC * (e + 1)] for e in range(sched[2 + t], sched[3 + t])]
        assert [int(r[0]) for r in rows] == sorted({int(r[0]) for r in rows})
        for r in rows:
            assert any(r[1:1 + T] >= 0) and all(r[1 + T:] == -1)
            for j in range(T):
                if r[1 + j] >= 0:
                    got[(t * T + j, int(r[0]))] = int(r[1 + j])
    assert got == {(int(o), int(i)): int(w) for o, i, w in zip(outs, ins, wids)}
