"""Host side of the grouped xprop tile (blocksparse_b200/lut.py), no GPU needed: the byte model that picks between one
output block per CTA and the grouped kernel, and the merged-entry record at eight output blocks per tile."""
import numpy as np
import pytest

from blocksparse_b200.lut import (MatmulLuts, WIDE_REC, XPROP_GROUP, XPROP_GROUP_MAX_BYTES, XPROP_GROUP_MIN_CTAS_PER_SM,
                                  pick_xprop_tile, xprop_staged_bytes)

SMS = 132


def merged_entries(lay, bprop, group=XPROP_GROUP):
    L = MatmulLuts(lay)
    sched, _, off = L.wide_schedule(bprop, group)
    return L.blocks, (len(sched) - off) // WIDE_REC


def test_byte_model_counts_tiles_and_blocks():
    # 3 minibatch tiles: one block per CTA stages 10 KB per LUT entry, grouped 8 KB per merged entry + 2 KB per LUT entry
    assert xprop_staged_bytes(100, 40, 300) == (3 * 100 * 10240, 3 * (40 * 8192 + 100 * 2048))


@pytest.mark.parametrize("bprop", [False, True])
def test_dense_and_random_quarter_layouts_run_grouped_at_the_benchmark_size(bprop):
    rng = np.random.default_rng(1236)
    for lay in (np.ones((128, 128), np.int32), (rng.random((128, 128)) < 0.25).astype(np.int32)):
        nnz, ent = merged_entries(lay, bprop)
        assert pick_xprop_tile(nnz, ent, 128, 4096, SMS) == XPROP_GROUP


@pytest.mark.parametrize("bprop", [False, True])
def test_layouts_that_share_no_activation_tile_stay_one_block_per_cta(bprop):
    lay = np.eye(128, dtype=np.int32)                     # every merged entry serves one output block: nothing to save
    nnz, ent = merged_entries(lay, bprop)
    assert ent == nnz and pick_xprop_tile(nnz, ent, 128, 4096, SMS) == 1
    rng = np.random.default_rng(0)
    lay = (rng.random((128, 128)) < 0.01).astype(np.int32)
    nnz, ent = merged_entries(lay, bprop)
    narrow, grouped = xprop_staged_bytes(nnz, ent, 4096)
    assert grouped > XPROP_GROUP_MAX_BYTES * narrow and pick_xprop_tile(nnz, ent, 128, 4096, SMS) == 1


def test_small_grids_stay_one_block_per_cta():
    lay = np.ones((128, 128), np.int32)
    nnz, ent = merged_entries(lay, False)
    n_fill = 128 * int(np.ceil(XPROP_GROUP_MIN_CTAS_PER_SM * SMS / (128 // XPROP_GROUP)))   # minibatch that fills the SMs
    assert pick_xprop_tile(nnz, ent, 128, n_fill - 128, SMS) == 1
    assert pick_xprop_tile(nnz, ent, 128, n_fill, SMS) == XPROP_GROUP
    lay = np.ones((8, 10), np.int32)
    nnz, ent = merged_entries(lay, False)
    assert pick_xprop_tile(nnz, ent, 10, 96, SMS) == 1


@pytest.mark.parametrize("bprop", [0, 1])
def test_wide_schedule_record_holds_eight_blocks(bprop):
    """lut.build_wide_schedule at 8 output blocks per tile: every (output block, input block) -> W block of the layout is
    in exactly one merged entry of its tile, entries ascend by input block, and the rest of each record is -1."""
    rng = np.random.default_rng(13)
    lay = (rng.random((19, 37)) < 0.4).astype(np.int32)
    lay[2, :] = 0
    lay[:, 8:16] = 0
    L = MatmulLuts(lay)
    sched, n_tiles, off = L.wide_schedule(bprop, 8)
    outs, ins, wids = L._b if bprop else L._f
    n_out = lay.shape[0] if bprop else lay.shape[1]
    assert n_tiles == -(-n_out // 8) and off % WIDE_REC == 0 and WIDE_REC >= 9
    got = {}
    for t in range(n_tiles):
        rows = [sched[off + WIDE_REC * e: off + WIDE_REC * (e + 1)] for e in range(sched[2 + t], sched[3 + t])]
        assert [int(r[0]) for r in rows] == sorted({int(r[0]) for r in rows})
        for r in rows:
            assert any(r[1:9] >= 0) and all(r[9:] == -1)
            for j in range(8):
                if r[1 + j] >= 0:
                    assert (t * 8 + j, int(r[0])) not in got
                    got[(t * 8 + j, int(r[0]))] = int(r[1 + j])
    assert got == {(int(o), int(i)): int(w) for o, i, w in zip(outs, ins, wids)}
