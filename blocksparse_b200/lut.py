"""Host-side lookup-table construction (vectorised NumPy, no Python loops over blocks).

Mirrors what BlocksparseMatMul.__init__ / xprop_lut (reference blocksparse/matmul.py:82-270)
and BlocksparseTransformer.__init__ / xn_lut / init_softmax_mask
(reference blocksparse/transformer.py:61-181) compute, plus the schedules our own
kernels consume.  The reference builds these with O(blocks) interpreter loops; here
everything is sorting / cumsum so a 128x128 layout takes well under a millisecond.
"""
import numpy as np

SEG_MAX = (1 << 63) - 1


def ceil_div(x, y):
    return -(-x // y)


def z_order_2d(x, y):
    """Morton code, x on even bits and y on odd bits (reference blocksparse/utils.py:95-103).

    Accepts scalars or integer arrays.
    """
    x = np.asarray(x, dtype=np.uint64)
    y = np.asarray(y, dtype=np.uint64)
    code = np.zeros(np.broadcast(x, y).shape, dtype=np.uint64)
    for bit in range(32):
        b = np.uint64(bit)
        code |= ((x >> b) & np.uint64(1)) << np.uint64(2 * bit)
        code |= ((y >> b) & np.uint64(1)) << np.uint64(2 * bit + 1)
    return code if code.shape else int(code)


def _group(outs, n_out):
    """counts[o] and starts[o] for an array already sorted by output index."""
    counts = np.bincount(outs, minlength=n_out).astype(np.int64)
    starts = np.concatenate(([0], np.cumsum(counts)[:-1]))
    return counts, starts


def row_lut(outs, ins, wids, n_out):
    """Kernel wire format ("row LUT", include/bsmm_b200.h): int32 [n_out + nnz][2].

    `outs/ins/wids` must already be sorted by output index.  Header row o holds
    (first_entry_row, n_entries); entry rows hold (w_block, in_block).
    """
    nnz = len(outs)
    counts, starts = _group(outs, n_out)
    lut = np.empty((n_out + nnz, 2), dtype=np.int32)
    lut[:n_out, 0] = n_out + starts
    lut[:n_out, 1] = counts
    lut[n_out:, 0] = wids
    lut[n_out:, 1] = ins
    return lut, int(counts.max()) if nnz else 0


def segmented_lut(outs, ins, wids, n_out, max_seg, min_seg):
    """The reference's Volta wire format (blocksparse/matmul.py:172-270), kept for API parity.

    Returns (lut, shared_bytes, n_segments, n_locks).  Segment rule (:218): a group is
    cut after every `max_seg` entries as long as at least `min_seg` entries remain.
    """
    nnz = len(outs)
    counts, starts = _group(outs, n_out)
    nonempty = np.nonzero(counts)[0]
    empty = np.nonzero(counts == 0)[0]
    n = counts[nonempty]
    if max_seg >= SEG_MAX:
        cuts = np.zeros_like(n)
    else:
        cuts = np.where(n >= min_seg, (n - min_seg) // max_seg, 0)
    segs_per = cuts + 1
    n_seg_ne = int(segs_per.sum())
    # segment -> (group, index within group)
    grp = np.repeat(np.arange(len(nonempty)), segs_per)
    first_seg = np.concatenate(([0], np.cumsum(segs_per)[:-1]))
    j = np.arange(n_seg_ne) - first_seg[grp]
    is_last = j == cuts[grp]
    seg_len = np.where(is_last, n[grp] - cuts[grp] * max_seg if max_seg < SEG_MAX else n[grp], max_seg).astype(np.int64)
    seg_start = starts[nonempty][grp] + j * (max_seg if max_seg < SEG_MAX else 0)
    # lock ids: 1-based, in order of ascending output index, only for split groups
    split = segs_per > 1
    lock_of_group = np.where(split, np.cumsum(split), 0)
    n_locks = int(split.sum())

    n_seg = n_seg_ne + len(empty)
    lut = np.empty(4 * n_seg + 2 * nnz, dtype=np.int32)
    hdr = lut[:4 * n_seg].reshape(n_seg, 4)
    hdr[:n_seg_ne, 0] = (4 * n_seg) // 2 + seg_start          # offset in int2 units
    hdr[:n_seg_ne, 1] = seg_len
    hdr[:n_seg_ne, 2] = nonempty[grp]
    hdr[:n_seg_ne, 3] = lock_of_group[grp]
    hdr[n_seg_ne:, 0] = (4 * n_seg) // 2 + nnz
    hdr[n_seg_ne:, 1] = 0
    hdr[n_seg_ne:, 2] = empty
    hdr[n_seg_ne:, 3] = 0
    ent = lut[4 * n_seg:].reshape(nnz, 2)
    ent[:, 0] = ins
    ent[:, 1] = wids
    longest = int(seg_len.max()) if n_seg_ne else 0
    return lut, longest * 8, n_seg, n_locks


def lists_from_sorted(outs, ins, wids, n_out):
    """[(out, [(in, w), ...]), ...] in the reference's order: non-empty outputs ascending, then empty ones."""
    counts, starts = _group(outs, n_out)
    ins_l, w_l = ins.tolist(), wids.tolist()
    res, tail = [], []
    for o in range(n_out):
        c, s = int(counts[o]), int(starts[o])
        if c:
            res.append((o, list(zip(ins_l[s:s + c], w_l[s:s + c]))))
        else:
            tail.append((o, []))
    return res + tail


class MatmulLuts(object):
    """Everything BlocksparseMatMul derives from a 2-D layout."""

    def __init__(self, layout, z_order=True):
        lay = np.asarray(layout) != 0
        assert lay.ndim == 2
        CB, KB = lay.shape
        self.CB, self.KB = CB, KB
        col_sizes = lay.sum(axis=0)
        if not col_sizes.any():
            raise ValueError("layout has no non-zero blocks")
        big = int(col_sizes.max())
        small = int(col_sizes[col_sizes > 0].min())
        # "assume symmetrical transpose": the same thresholds are used for bprop (matmul.py:94)
        max_seg = max(ceil_div(big, 4), small * 2) if big / small > 2.0 else SEG_MAX
        min_seg = max(ceil_div(max_seg, 4), 4)

        # discovery order = column-major (k ascending, then c) -- the order the reference's
        # comment at matmul.py:114 assumes scipy.sparse.find returns
        ks, cs = np.nonzero(lay.T)
        cs = cs.astype(np.int64)
        ks = ks.astype(np.int64)
        nnz = len(cs)
        if z_order:
            rank = np.argsort(z_order_2d(cs, ks), kind="stable")
            wid = np.empty(nnz, dtype=np.int64)
            wid[rank] = np.arange(nnz)
            upd_c, upd_k = cs[rank], ks[rank]
        else:
            wid = np.arange(nnz, dtype=np.int64)
            upd_c, upd_k = cs, ks
        self.blocks = nnz
        self.updat_lut = np.stack([upd_c, upd_k], axis=1).astype(np.int32)
        self.updat_list = [tuple(r) for r in self.updat_lut.tolist()]

        # fprop: grouped by k (already sorted); bprop: grouped by c (stable => k ascending inside)
        by_c = np.argsort(cs, kind="stable")
        f = (ks, cs, wid)
        b = (cs[by_c], ks[by_c], wid[by_c])
        self.fprop_lut, self.fprop_shared, self.fprop_segments, self.fprop_locks = \
            segmented_lut(f[0], f[1], f[2], KB, max_seg, min_seg)
        self.bprop_lut, self.bprop_shared, self.bprop_segments, self.bprop_locks = \
            segmented_lut(b[0], b[1], b[2], CB, max_seg, min_seg)
        self.fprop_list = lists_from_sorted(f[0], f[1], f[2], KB)
        self.bprop_list = lists_from_sorted(b[0], b[1], b[2], CB)
        self.fprop_rows, self.fprop_max = row_lut(f[0], f[1], f[2], KB)
        self.bprop_rows, self.bprop_max = row_lut(b[0], b[1], b[2], CB)
        self._f, self._b = f, b

    def updat_schedule(self, bsize, k_per_tile=None, n_cta=None):
        return build_updat_schedule(self.updat_lut, self.CB, self.KB, bsize, k_per_tile, n_cta)

    def wide_schedule(self, bprop, blocks_per_tile):
        outs, ins, wids = self._b if bprop else self._f
        n_out = self.CB if bprop else self.KB
        return build_wide_schedule(outs, ins, wids, n_out, blocks_per_tile)

    def pair_schedule(self, bprop, blocks_per_tile, w_per_group, n_tiles, n_ntiles, n_ctas, bsize=32):
        outs, ins, wids = self._b if bprop else self._f
        n_out = self.CB if bprop else self.KB
        return build_pair_schedule(outs, ins, wids, n_out, blocks_per_tile, w_per_group, n_tiles, n_ntiles, n_ctas, bsize)

    def pair_tile_schedule(self, bprop, blocks_per_tile, bsize, w_per_group, n_tiles):
        outs, ins, wids = self._b if bprop else self._f
        n_out = self.CB if bprop else self.KB
        return build_pair_tile_schedule(outs, ins, wids, n_out, blocks_per_tile, bsize, w_per_group, n_tiles)

    def tile_schedule(self, bprop, blocks_per_tile, bsize=32, w_per_group=8, n_tiles=None, n_ntiles=None):
        outs, ins, wids = self._b if bprop else self._f
        n_out = self.CB if bprop else self.KB
        return build_tile_schedule(outs, ins, wids, n_out, blocks_per_tile, bsize, w_per_group, n_tiles, n_ntiles)


WIDE_REC = 16            # ints per merged entry of build_wide_schedule (csrc/tc_xprop2.cuh XP2_REC)


def build_wide_schedule(outs, ins, wids, n_out, blocks_per_tile):
    """Merged LUT rows for the wide-tile xprop kernel (csrc/tc_xprop2.cuh).

    Tile t covers output blocks [t*T, (t+1)*T), T = blocks_per_tile <= 8.  Its entries are the distinct input blocks
    consumed by any of them, in ascending order, each with the W block of every output block of the tile (-1: none).

    int32 layout:
      [0] n_tiles  [1] T  [2 .. 2+n_tiles]  first entry of every tile (n_tiles + 1 offsets)
      entries from `entry_offset` (a multiple of WIDE_REC): [in_block, w_0 .. w_{T-1}, -1 ...] (WIDE_REC ints each)
    Returns (schedule, n_tiles, entry_offset).
    """
    T = int(blocks_per_tile)
    assert 1 <= T <= 8
    outs = np.asarray(outs, dtype=np.int64)
    ins = np.asarray(ins, dtype=np.int64)
    wids = np.asarray(wids, dtype=np.int64)
    n_tiles = max(1, ceil_div(n_out, T))
    n_in = int(ins.max()) + 1 if len(ins) else 1
    key = (outs // T) * n_in + ins                       # (tile, input block)
    uniq, inv = np.unique(key, return_inverse=True)
    tile_of = uniq // n_in
    offsets = np.searchsorted(tile_of, np.arange(n_tiles + 1))
    ent_off = ceil_div(3 + n_tiles, WIDE_REC) * WIDE_REC
    sched = np.full(ent_off + WIDE_REC * len(uniq), -1, dtype=np.int32)
    sched[0:2] = (n_tiles, T)
    sched[2:3 + n_tiles] = offsets
    ent = sched[ent_off:].reshape(len(uniq), WIDE_REC)
    ent[:, 0] = uniq % n_in
    ent[inv, 1 + outs % T] = wids
    return sched, n_tiles, ent_off


# Grouped-tile selection for the default 32 x 32 wgmma xprop (csrc/tc_xprop2.cuh: tc_xprop_grouped_kernel).  Both kernels
# are bound by the bytes they stage from L2 into shared memory, per 128 minibatch rows: the one-block-per-CTA kernel
# stages an 8 KB activation tile and a 2 KB W block per LUT entry, the grouped kernel an activation tile per MERGED entry
# and the same W blocks.  The grouped tile is taken when the model says it stages at most XPROP_GROUP_MAX_BYTES of the
# narrow kernel's bytes and its grid still has XPROP_GROUP_MIN_CTAS_PER_SM CTAs for every SM.  Both thresholds are read
# off scripts/xprop_tiles.py on an H100 80GB HBM3 at 700 W (DESIGN.md section 5 has the table): at 4096 x 4096 and
# N = 4096 the grouped tile is 5-6 % faster at 5 % density, where the model says 0.93 of the bytes, and gains from there
# on; at N = 2048 (3.9 CTAs per SM, three of which run at a time) it is 17-18 % slower in spite of 0.78 of the bytes, at
# N = 4096 (7.8 per SM) 20 % faster.
XPROP_GROUP = 4
XPROP_GROUP_MAX_BYTES = 0.95
XPROP_GROUP_MIN_CTAS_PER_SM = 6.0


def xprop_staged_bytes(nnz, merged_entries, N):
    """Modelled bytes a 32 x 32, 16-bit xprop call stages into shared memory: (narrow kernel, grouped kernel)."""
    n_tiles = ceil_div(N, 128)
    return nnz * 10240 * n_tiles, (merged_entries * 8192 + nnz * 2048) * n_tiles


def pick_xprop_tile(nnz, merged_entries, n_out, N, n_sm, group=XPROP_GROUP):
    """Output blocks per CTA for the default 32 x 32 xprop route: `group` (grouped kernel) or 1 (one block per CTA).
    merged_entries: entries of build_wide_schedule(..., group) for this layout and direction."""
    narrow, grouped = xprop_staged_bytes(nnz, merged_entries, N)
    ctas = ceil_div(N, 128) * ceil_div(n_out, group)
    if grouped <= XPROP_GROUP_MAX_BYTES * narrow and ctas >= XPROP_GROUP_MIN_CTAS_PER_SM * n_sm:
        return group
    return 1


GROUP_INTS = 32          # one 128-byte record per schedule group (one coalesced warp load)
GROUP_MAX_W = 8          # W blocks per group record (ints 4..11)
GROUP_MAX_RUNS = 8       # MMA runs per group record (ints 12..27, two ints each)


def pick_tile_count(n_out, n_ntiles, cta_slots, max_blocks_per_tile):
    """Number of output tiles along the feature axis for the persistent xprop kernel.

    The kernel runs `cta_slots` CTAs (SMs x CTAs per SM) over n_ntiles * n_ktiles tiles, so the tile count should
    land just under a multiple of cta_slots (512 tiles on 296 slots waste 14 % in the second wave).  Among the tile
    counts that keep tiles <= max_blocks_per_tile blocks wide we take the one with the least idle slot-time,
    preferring wider tiles (more reuse of each activation tile) on ties.
    """
    lo = ceil_div(n_out, max_blocks_per_tile)
    best = None
    for n_kt in range(lo, min(n_out, 2 * lo) + 1):
        tiles = n_ntiles * n_kt
        waves = ceil_div(tiles, cta_slots)
        # time ~ waves * (average tile width + a fixed per-tile cost worth ~1.5 blocks: narrower tiles re-stage
        # more activation tiles per output block)
        cost = waves * (n_out / float(n_kt) + 1.5)
        if best is None or cost < best[0]:
            best = (cost, n_kt)
    return best[1]


def tile_order(tile_cost, n_ntiles):
    """Order in which the persistent CTAs pull the n_ntiles x len(tile_cost) tiles from the global counter: heaviest
    output tiles first (greedy longest-processing-time, so a skewed layout's few heavy tiles do not end up as the tail),
    costs bucketed to 12.5 % so that a uniform layout keeps the natural order (all output tiles of one minibatch tile
    back to back: its activation panel stays hot).  int32 [n_ntiles * n_ktiles] of tile ids nt * n_ktiles + kt."""
    cost = np.asarray(tile_cost, dtype=np.float64)
    n_kt = len(cost)
    top = cost.max() if n_kt and cost.max() > 0 else 1.0
    bucket = np.floor(8.0 * cost / top).astype(np.int64)
    kt = np.tile(np.arange(n_kt), n_ntiles)
    nt = np.repeat(np.arange(n_ntiles), n_kt)
    order = np.lexsort((kt, nt, -bucket[kt]))
    return (nt[order] * n_kt + kt[order]).astype(np.int32)


def build_tile_schedule(outs, ins, wids, n_out, blocks_per_tile, bsize=32, w_per_group=8, n_tiles=None, n_ntiles=None):
    """Tile schedule for a tile-grouped xprop formulation (the wgmma xprop kernel of csrc/tc.cuh walks the row
    LUTs instead and does not use it).

    An output tile covers `blocks_per_tile` consecutive output blocks (their fp32 accumulators live
    side by side, block s of the tile at columns [s*bsize, (s+1)*bsize)).  For every
    tile the LUT is regrouped by INPUT block: a *group* is one activation tile plus the <= w_per_group
    W blocks of the tile that consume it (an input block with more consumers is split into several
    groups).  Everything the device loops would otherwise derive per block is precomputed here:

      * W blocks are listed in accumulator order and staged in consecutive shared-memory slots, so
        blocks whose accumulators are adjacent form a *run* that is issued as ONE wider MMA
        (N = run_len*bsize); a dense layout degenerates to ordinary wide GEMM instructions;
      * every run accumulates (bit 0 of int1 is always 1): the kernel's epilogue leaves the accumulators zeroed,
        so no first-touch bookkeeping -- and no run split at a first touch -- is needed;
      * (the A-collector hint needs no field: the first run of a group fills the collector, the rest reuse it).

    int32 layout:
      [0] n_tiles  [1] blocks_per_tile  [2] total groups  [3] total W loads
      tile header   [n_tiles][4] = (first_group_index, n_groups, first_out_block, n_out | touched_mask << 8)
      (padding to a multiple of GROUP_INTS ints)
      group records [groups][32]:
          [0] in_block   [1] n_w | n_runs << 8   [2..3] reserved
          [4..11]  W block ids, in staging-slot order
          [12..19] run r, int0 = (w_slot * bsize*bsize*2) >> 4  |  (accumulator column << 16)
          [20..27] run r, int1 = (N >> 3) << 17 | accumulate     (N pre-shifted to its instruction-descriptor field)
    Returns (schedule, groups_offset): groups_offset is the int32 index of the first group record.
    """
    T = int(blocks_per_tile)
    assert 1 <= w_per_group <= GROUP_MAX_W
    if n_tiles is None:
        n_tiles = ceil_div(n_out, T)
    n_tiles = int(n_tiles)
    assert n_tiles * T >= n_out
    # tile t covers output blocks [bounds[t], bounds[t+1]): sizes differ by at most one block
    bounds = (np.arange(n_tiles + 1, dtype=np.int64) * n_out) // n_tiles
    assert int(np.diff(bounds).max()) <= T
    outs = np.asarray(outs, dtype=np.int64)
    ins = np.asarray(ins, dtype=np.int64)
    wids = np.asarray(wids, dtype=np.int64)
    nnz = len(outs)
    tile = np.searchsorted(bounds, outs, side="right") - 1
    order = np.lexsort((outs, ins, tile))          # by tile, then input block, then slot
    tile_s, ins_s, outs_s, w_s = tile[order], ins[order], outs[order], wids[order]
    slot_s = outs_s - bounds[tile_s]

    # position of each pair inside its (tile, in_block) cluster -> chunk of w_per_group pairs = group
    new_cluster = np.ones(nnz, dtype=bool)
    if nnz:
        new_cluster[1:] = (tile_s[1:] != tile_s[:-1]) | (ins_s[1:] != ins_s[:-1])
    cluster_id = np.cumsum(new_cluster) - 1
    cluster_start = np.nonzero(new_cluster)[0]
    pos_in_cluster = np.arange(nnz) - cluster_start[cluster_id]
    new_group = new_cluster | (pos_in_cluster % w_per_group == 0)
    group_id = np.cumsum(new_group) - 1
    g_first = np.nonzero(new_group)[0]
    n_groups = len(g_first)
    g_count = np.diff(np.concatenate((g_first, [nnz])))
    pos_in_group = np.arange(nnz) - g_first[group_id]

    # accumulators start from zero (cleared by the epilogue), so every run accumulates
    accumulate = np.ones(nnz, dtype=np.int64)

    # runs: consecutive pairs of a group with consecutive slots
    new_run = np.ones(nnz, dtype=bool)
    if nnz:
        new_run[1:] = new_group[1:] | (slot_s[1:] != slot_s[:-1] + 1)
    run_first = np.nonzero(new_run)[0]
    run_len = np.diff(np.concatenate((run_first, [nnz])))
    run_group = group_id[run_first]
    runs_per_group = np.bincount(run_group, minlength=n_groups)
    run_first_of_group = np.concatenate(([0], np.cumsum(runs_per_group)[:-1]))
    run_pos = np.arange(len(run_first)) - run_first_of_group[run_group]
    assert runs_per_group.max(initial=0) <= GROUP_MAX_RUNS

    groups_per_tile = np.bincount(tile_s[g_first], minlength=n_tiles)
    tile_first_group = np.concatenate(([0], np.cumsum(groups_per_tile)[:-1]))
    touched = np.zeros(n_tiles, dtype=np.int64)
    np.bitwise_or.at(touched, tile, np.int64(1) << (outs - bounds[tile]))

    hdr_ints = 4 + 4 * n_tiles
    grp_off = ceil_div(hdr_ints, GROUP_INTS) * GROUP_INTS
    sched = np.zeros(grp_off + GROUP_INTS * n_groups, dtype=np.int32)
    sched[0:4] = (n_tiles, T, n_groups, nnz)
    th = sched[4:hdr_ints].reshape(n_tiles, 4)
    th[:, 0] = tile_first_group
    th[:, 1] = groups_per_tile
    th[:, 2] = bounds[:-1]
    th[:, 3] = np.diff(bounds) | (touched << 8)
    gr = sched[grp_off:].reshape(n_groups, GROUP_INTS)
    gr[:, 0] = ins_s[g_first]
    gr[:, 1] = g_count | (runs_per_group << 8)
    gr[group_id, 4 + pos_in_group] = w_s
    wbytes16 = (bsize * bsize * 2) >> 4
    r0 = pos_in_group[run_first] * wbytes16 | ((slot_s[run_first] * bsize) << 16)
    r1 = (((run_len * bsize) >> 3) << 17) | accumulate[run_first]
    gr[run_group, 12 + run_pos] = r0
    gr[run_group, 20 + run_pos] = r1
    if n_ntiles is not None:
        # tile order table for the dynamic tile queue (csrc/tc.cuh): cost ~ activation tiles staged + W blocks multiplied
        w_per_tile = np.bincount(tile, minlength=n_tiles) if nnz else np.zeros(n_tiles, dtype=np.int64)
        cost = 4.0 * groups_per_tile + 1.0 * w_per_tile + 4.0
        order = tile_order(cost, int(n_ntiles))
        order_off = len(sched)
        return np.concatenate((sched, order)), grp_off, order_off
    return sched, grp_off


def build_pair_tile_schedule(outs, ins, wids, n_out, blocks_per_tile, bsize, w_per_group, n_tiles):
    """build_tile_schedule for the 2-CTA cluster kernel (csrc/tc.cuh, CL = 2): output tiles 2P and 2P+1 walk ONE merged
    group list, so that the activation tile of every group can be fetched once and multicast to both CTAs.

    For every input block with a consumer in either tile of the pair both tiles get the same number of group records (the
    larger of the two tiles' needs); a tile with nothing to multiply in a group gets a record with n_w = 0.  An odd tile
    count is padded with an empty tile.  Same record / header layout as build_tile_schedule.
    Returns (schedule, groups_offset); the tile count in schedule[0] is even.
    """
    T, WPG = int(blocks_per_tile), int(w_per_group)
    assert 1 <= WPG <= GROUP_MAX_W
    n_tiles = int(n_tiles)
    assert n_tiles * T >= n_out
    bounds = (np.arange(n_tiles + 1, dtype=np.int64) * n_out) // n_tiles
    outs = np.asarray(outs, dtype=np.int64); ins = np.asarray(ins, dtype=np.int64); wids = np.asarray(wids, dtype=np.int64)
    tile = np.searchsorted(bounds, outs, side="right") - 1
    n_even = n_tiles + (n_tiles & 1)
    wbytes16 = (bsize * bsize * 2) >> 4
    max_run = 256 // bsize
    # per tile: {in_block: [(slot, w), ...] sorted by slot}
    per_tile = [dict() for _ in range(n_even)]
    order = np.lexsort((outs, ins, tile))
    for t, c, o, w in zip(tile[order].tolist(), ins[order].tolist(), outs[order].tolist(), wids[order].tolist()):
        per_tile[t].setdefault(c, []).append((o - int(bounds[t]), w))
    recs = [[] for _ in range(n_even)]

    def records(entries, in_block, n_rec):
        out = []
        for r in range(n_rec):
            chunk = entries[r * WPG:(r + 1) * WPG]
            rec = [0] * GROUP_INTS
            rec[0] = in_block
            runs = []
            for pos, (slot, w) in enumerate(chunk):
                rec[4 + pos] = w
                if runs and runs[-1][1] + runs[-1][2] == slot and runs[-1][2] < max_run:
                    runs[-1][2] += 1
                else:
                    runs.append([pos, slot, 1])
            assert len(runs) <= GROUP_MAX_RUNS
            rec[1] = len(chunk) | (len(runs) << 8)
            for i, (pos, slot, ln) in enumerate(runs):
                rec[12 + i] = (pos * wbytes16) | ((slot * bsize) << 16)
                rec[20 + i] = (((ln * bsize) >> 3) << 17) | 1
            out.append(rec)
        return out

    for P in range(n_even // 2):
        a, b = per_tile[2 * P], per_tile[2 * P + 1]
        for c in sorted(set(a) | set(b)):
            ea, eb = a.get(c, []), b.get(c, [])
            n_rec = max(ceil_div(len(ea), WPG), ceil_div(len(eb), WPG), 1)
            recs[2 * P] += records(ea, c, n_rec)
            recs[2 * P + 1] += records(eb, c, n_rec)
    groups_per_tile = np.array([len(r) for r in recs], dtype=np.int64)
    tile_first_group = np.concatenate(([0], np.cumsum(groups_per_tile)[:-1]))
    touched = np.zeros(n_even, dtype=np.int64)
    np.bitwise_or.at(touched, tile, np.int64(1) << (outs - bounds[tile]))
    hdr_ints = 4 + 4 * n_even
    grp_off = ceil_div(hdr_ints, GROUP_INTS) * GROUP_INTS
    n_groups = int(groups_per_tile.sum())
    sched = np.zeros(grp_off + GROUP_INTS * n_groups, dtype=np.int32)
    sched[0:4] = (n_even, T, n_groups, len(outs))
    th = sched[4:hdr_ints].reshape(n_even, 4)
    th[:, 0] = tile_first_group
    th[:, 1] = groups_per_tile
    th[:n_tiles, 2] = bounds[:-1]
    th[:n_tiles, 3] = np.diff(bounds) | (touched[:n_tiles] << 8)
    if n_even > n_tiles:                      # padding tile: no output blocks, only takes part in the barrier protocol
        th[n_tiles, 2] = n_out
        th[n_tiles, 3] = 0
    flat = [r for tr in recs for r in tr]
    if flat:
        sched[grp_off:] = np.asarray(flat, dtype=np.int64).astype(np.int32).reshape(-1)
    return sched, grp_off


PAIR_MAX_W = 14          # W blocks per pair-group record (ints 2..15)
PAIR_MAX_RUNS = 8        # MMA runs per half of a pair-group (ints 16..23 / 24..31)


def lpt_tile_lists(tile_cost, n_ntiles, n_ctas):
    """Static longest-processing-time assignment of the n_ntiles x len(tile_cost) tiles to n_ctas persistent CTAs.

    The persistent grids used to deal tile t to CTA t mod grid; with skewed layouts (a few output tiles hold most of
    the blocks) that leaves CTAs idle while one works through several heavy tiles.  Here tiles are sorted by
    decreasing cost and each goes to the least-loaded CTA so far (ties: lowest CTA index => deterministic).
    Returns int32 [n_ctas + 1 offsets | tile ids], tile id = n_tile * n_ktiles + k_tile.
    """
    import heapq
    n_kt = len(tile_cost)
    cost = np.asarray(tile_cost, dtype=np.float64)
    kt = np.tile(np.arange(n_kt), n_ntiles)
    nt = np.repeat(np.arange(n_ntiles), n_kt)
    order = np.lexsort((nt, kt, -cost[kt]))                 # heaviest first; stable in (kt, nt)
    heap = [(0.0, c) for c in range(n_ctas)]
    lists = [[] for _ in range(n_ctas)]
    for i in order.tolist():
        load, c = heapq.heappop(heap)
        lists[c].append(int(nt[i]) * n_kt + int(kt[i]))
        heapq.heappush(heap, (load + float(cost[kt[i]]), c))
    offs = np.concatenate(([0], np.cumsum([len(l) for l in lists]))).astype(np.int32)
    flat = np.asarray([t for l in lists for t in l], dtype=np.int32)
    return np.concatenate((offs, flat)).astype(np.int32)


def build_pair_schedule(outs, ins, wids, n_out, blocks_per_tile, w_per_group, n_tiles, n_ntiles, n_ctas, bsize=32):
    """Schedule for a wide-activation-tile xprop formulation (32 x 32 blocks; not used by the wgmma kernels).

    Same idea as build_tile_schedule, but a group is an input-block PAIR (2p, 2p+1): its activation tile is
    128 rows x 64 features = 128-byte rows, so every TMA row request moves a full 128-byte line, and ~2x the W blocks consume each staged tile.  W blocks are listed half 0
    (input block 2p) first, then half 1, each in accumulator order, so that the runs of one half are issued back to
    back against the same K slices of the tile (A-collector reuse).

    int32 layout:
      [0] n_tiles  [1] blocks_per_tile  [2] total groups  [3] total W loads
      tile header   [n_tiles][4] = (first_group_index, n_groups, first_out_block, n_out | touched_mask << 8)
      (padding to a multiple of GROUP_INTS ints)
      group records [groups][32]:
          [0] input pair p   [1] n_w | n_runs_half0 << 8 | n_runs_half1 << 16
          [2..15]   W block ids in staging-slot order
          [16..23]  runs of half 0, [24..31] runs of half 1, one packed int each:
                    (staging slot * bsize*bsize*2) >> 4  |  accumulator column << 12  |  (N >> 3) << 21
      tile lists    lpt_tile_lists(...) for n_ntiles minibatch tiles on n_ctas CTAs
    Returns (schedule, groups_offset, tile_list_offset).
    """
    T = int(blocks_per_tile)
    WPS = int(w_per_group)
    assert 1 <= WPS <= PAIR_MAX_W and T * bsize <= 512
    n_tiles = int(n_tiles)
    assert n_tiles * T >= n_out
    bounds = (np.arange(n_tiles + 1, dtype=np.int64) * n_out) // n_tiles
    assert int(np.diff(bounds).max()) <= T
    outs = np.asarray(outs, dtype=np.int64)
    ins = np.asarray(ins, dtype=np.int64)
    wids = np.asarray(wids, dtype=np.int64)
    nnz = len(outs)
    tile = np.searchsorted(bounds, outs, side="right") - 1
    pair, half = ins >> 1, ins & 1
    slot = outs - bounds[tile]
    order = np.lexsort((slot, half, pair, tile))
    tile_s, pair_s, half_s, slot_s, w_s = tile[order], pair[order], half[order], slot[order], wids[order]
    new_cluster = np.ones(nnz, dtype=bool)
    if nnz:
        new_cluster[1:] = (tile_s[1:] != tile_s[:-1]) | (pair_s[1:] != pair_s[:-1])
    c_start = np.nonzero(new_cluster)[0].tolist() + [nnz]
    max_run = 256 // bsize
    wbytes16 = (bsize * bsize * 2) >> 4
    half_l, slot_l, w_l = half_s.tolist(), slot_s.tolist(), w_s.tolist()
    recs, rec_tile = [], []
    for ci in range(len(c_start) - 1):
        a, b = c_start[ci], c_start[ci + 1]
        t, p = int(tile_s[a]), int(pair_s[a])
        i = a
        while i < b:
            rec = [0] * GROUP_INTS
            runs = ([], [])
            j, prev = i, None
            while j < b and j - i < WPS:
                h, sl = half_l[j], slot_l[j]
                cont = prev == (h, sl - 1) and runs[h][-1][2] < max_run
                if not cont:
                    if len(runs[h]) == PAIR_MAX_RUNS:
                        break
                    runs[h].append([j - i, sl, 1])
                else:
                    runs[h][-1][2] += 1
                rec[2 + j - i] = w_l[j]
                prev = (h, sl)
                j += 1
            rec[0] = p
            rec[1] = (j - i) | (len(runs[0]) << 8) | (len(runs[1]) << 16)
            for h in (0, 1):
                for r, (pos, sl, ln) in enumerate(runs[h]):
                    rec[16 + 8 * h + r] = (pos * wbytes16) | ((sl * bsize) << 12) | (((ln * bsize) >> 3) << 21)
            recs.append(rec)
            rec_tile.append(t)
            i = j
    n_groups = len(recs)
    rec_tile = np.asarray(rec_tile, dtype=np.int64)
    groups_per_tile = np.bincount(rec_tile, minlength=n_tiles) if n_groups else np.zeros(n_tiles, dtype=np.int64)
    tile_first_group = np.concatenate(([0], np.cumsum(groups_per_tile)[:-1]))
    w_per_tile = np.bincount(tile, minlength=n_tiles) if nnz else np.zeros(n_tiles, dtype=np.int64)
    touched = np.zeros(n_tiles, dtype=np.int64)
    np.bitwise_or.at(touched, tile, np.int64(1) << (outs - bounds[tile]))

    hdr_ints = 4 + 4 * n_tiles
    grp_off = ceil_div(hdr_ints, GROUP_INTS) * GROUP_INTS
    # cost model of a tile in L1->crossbar requests / tensor-pipe cycles: 128 row requests per activation tile,
    # 32 per W block (~ its 32+ MMA cycles), plus the epilogue
    cost = 128.0 * groups_per_tile + 40.0 * w_per_tile + 10.0 * T * bsize / 8 + 200.0
    lists = lpt_tile_lists(cost, int(n_ntiles), int(n_ctas))
    list_off = grp_off + GROUP_INTS * n_groups
    sched = np.zeros(list_off + len(lists), dtype=np.int32)
    sched[0:4] = (n_tiles, T, n_groups, nnz)
    th = sched[4:hdr_ints].reshape(n_tiles, 4)
    th[:, 0] = tile_first_group
    th[:, 1] = groups_per_tile
    th[:, 2] = bounds[:-1]
    th[:, 3] = np.diff(bounds) | (touched << 8)
    if n_groups:
        sched[grp_off:list_off] = np.asarray(recs, dtype=np.int64).astype(np.int32).reshape(-1)
    sched[list_off:] = lists
    return sched, grp_off, list_off


UPDAT_REC_INTS = 64      # one 256-byte record per updat tile (<= 8 slots: bs 32 / 64); bs 16 uses 192 ints (16 slots x 8 input blocks)


def updat_record_shape(bsize):
    """(ints per tile record, offset of the W-id table) -- mirrors csrc/tc_updat.cuh:updat_rec_ints / updat_tab_off."""
    return (64, 16) if bsize >= 32 else (192, 32)


def _updat_makespan(g_cnt, g_nwin, n_cta):
    """Cost model of the persistent updat grid: a tile streams (128-feature X tile + n_act DY blocks) per K step, tiles are
    dealt round-robin in decreasing-cost order; returns the busiest CTA's load."""
    sizes = []
    for c, w in zip(g_cnt.tolist(), g_nwin.tolist()):
        if c:
            q, r = divmod(c, w)
            sizes += [q + 1] * r + [q] * (w - r)
    cost = np.sort(4.0 + np.asarray(sizes, dtype=np.float64))[::-1]
    load = np.zeros(n_cta)
    np.add.at(load, np.arange(len(cost)) % n_cta, cost)
    return load.max()


def _balance_windows(g_cnt, g_nwin, KT, n_cta):
    """More (smaller) windows than the minimum when that fills whole waves of the n_cta persistent CTAs."""
    t_min = int(g_nwin[g_cnt > 0].sum())
    best, best_cost = g_nwin, _updat_makespan(g_cnt, g_nwin, n_cta)
    target = -(-t_min // n_cta) * n_cta
    while target <= 1.35 * t_min + 1 and target <= int(g_cnt.sum()):
        nw = g_nwin.copy()
        for _ in range(target - t_min):                    # split the group with the widest windows once more
            g = int(np.argmax(np.where(nw < g_cnt, g_cnt / nw, 0.0)))
            nw[g] += 1
        c = _updat_makespan(g_cnt, nw, n_cta)
        if c < best_cost - 1e-9:
            best, best_cost = nw, c
        target += n_cta
    return best


def build_updat_schedule(updat_lut, CB, KB, bsize, k_per_tile=None, n_cta=None):
    """Schedule for the wgmma updat kernel (csrc/tc_updat.cuh): a "gathered dense GEMM".

    A tile pairs a GROUP of 128/bsize consecutive input blocks (128 features = the MMA M axis) with up
    to `k_per_tile` output blocks taken from a window of consecutive output blocks, keeping only those
    that have at least one active block in the group.  The kept output blocks are compacted side by
    side (shared-memory slots and accumulator columns s = 0..n_act-1), so each K step of the reduction
    over the minibatch is ONE MMA of N = n_act*bsize columns, and output blocks with nothing to update
    are neither loaded nor multiplied.

    int32 layout:
      [0] n_tiles  [1] blocks per group  [2] k_per_tile  [3] UPDAT_REC_INTS
      tile records [n_tiles][64], sorted by decreasing n_act (longest first for load balance):
          [0] first input block of the group   [1] n_act
          [8  .. 8+k_per_tile)            output block id of compact slot s
          [16 + i*k_per_tile + s]         W block id for (input block i of the group, slot s) or -1
    Returns (schedule, first_record_offset).
    """
    G = 128 // bsize
    if k_per_tile is None:
        k_per_tile = 256 // bsize
    KT = int(k_per_tile)
    REC, TAB = updat_record_shape(bsize)
    assert KT * bsize <= 256 and 8 + KT <= TAB and TAB + G * KT <= REC
    lut = np.asarray(updat_lut, dtype=np.int64).reshape(-1, 2)
    cs, ks = lut[:, 0], lut[:, 1]
    wid = np.arange(len(cs), dtype=np.int64)
    # Windows are cut from each group's KEPT output blocks (those with at least one active block in the group), split
    # evenly into ceil(n_kept / KT) windows: tiles come out (nearly) full -- N = 256 MMAs, the activation tile
    # re-read n_kept/KT times instead of KB/KT times -- and of almost equal cost.
    grp = cs // G
    n_grp = ceil_div(CB, G)
    gk = np.unique(grp * KB + ks)                         # distinct (group, k), sorted by group then k
    g_of, k_of = gk // KB, gk % KB
    g_first = np.searchsorted(g_of, np.arange(n_grp))     # first kept entry of each group
    g_cnt = np.diff(np.concatenate((g_first, [len(gk)])))
    g_nwin = np.maximum(1, -(-g_cnt // KT))
    if n_cta:
        g_nwin = _balance_windows(g_cnt, g_nwin, KT, int(n_cta))
    pos = np.arange(len(gk)) - g_first[g_of]              # rank of k among the group's kept blocks
    win_of_gk = (pos * g_nwin[g_of]) // np.maximum(g_cnt[g_of], 1)     # even split: sizes differ by at most 1
    n_win = int(g_nwin.max()) if len(gk) else 1
    win = win_of_gk[np.searchsorted(gk, grp * KB + ks)]
    tile_key = grp * n_win + win
    # distinct (tile, k) pairs -> compact slot numbers
    tk = tile_key * KB + ks
    uniq_tk, inv = np.unique(tk, return_inverse=True)
    u_tile = uniq_tk // KB
    u_k = uniq_tk % KB
    new_tile = np.ones(len(uniq_tk), dtype=bool)
    new_tile[1:] = u_tile[1:] != u_tile[:-1]
    tile_start = np.nonzero(new_tile)[0]
    tile_idx_of_u = np.cumsum(new_tile) - 1
    slot_of_u = np.arange(len(uniq_tk)) - tile_start[tile_idx_of_u]
    n_tiles = len(tile_start)
    n_act = np.diff(np.concatenate((tile_start, [len(uniq_tk)])))
    order = np.argsort(-n_act, kind="stable")            # longest tiles first
    rank = np.empty(n_tiles, dtype=np.int64)
    rank[order] = np.arange(n_tiles)

    off = 4
    sched = np.full(off + REC * n_tiles, -1, dtype=np.int32)
    sched[0:4] = (n_tiles, G, KT, REC)
    rec = sched[off:].reshape(n_tiles, REC)
    rec[:, 0:8] = 0
    t_of_u = rank[tile_idx_of_u]
    rec[t_of_u, 0] = (u_tile // n_win) * G
    rec[rank, 1] = n_act
    rec[t_of_u, 8 + slot_of_u] = u_k
    # blocks
    t_of_blk = rank[tile_idx_of_u[inv]]
    rec[t_of_blk, TAB + (cs % G) * KT + slot_of_u[inv]] = wid
    return sched, off


# ---------------------------------------------------------------------------------------
# block-sparse transformer
# ---------------------------------------------------------------------------------------

MASK_DTYPE = {8: np.uint8, 16: np.uint16, 32: np.uint32, 64: np.uint64}


def xn_lut(outs, ins, n_out):
    """reference transformer.py:161-181 for one head; block ids are positions in (q,k)-sorted order."""
    nnz = len(outs)
    bid = np.arange(nnz, dtype=np.int64)
    order = np.argsort(outs, kind="stable")
    lut, longest = row_lut(outs[order], ins[order], bid[order], n_out)
    counts, starts = _group(outs[order], n_out)
    b_l, i_l = bid[order].tolist(), ins[order].tolist()
    rows = [list(zip(b_l[s:s + c], i_l[s:s + c])) for s, c in zip(starts.tolist(), counts.tolist())]
    return lut, rows, longest


def build_nt_items(tn_rows_per_head):
    """Pairing of the blocks that share a key block, two at a time (an NT schedule; the wgmma NT kernel of
    csrc/tc_bst.cuh takes one block per CTA from the NT LUT and does not use it).

    tn_rows_per_head[h][k] = [(block_id, q_block), ...] (the reference's tn_list).  Returns int32
    [lut_heads][n_items][8] = (k_blk, n_valid, blk0, q0, blk1, q1, 0, 0); heads with fewer pairs are padded with
    n_valid = 0 items.
    """
    per_head = []
    for rows in tn_rows_per_head:
        items = []
        for k, row in enumerate(rows):
            for i in range(0, len(row), 2):
                b0, q0 = row[i]
                if i + 1 < len(row):
                    b1, q1 = row[i + 1]
                    items.append((k, 2, b0, q0, b1, q1, 0, 0))
                else:
                    items.append((k, 1, b0, q0, 0, 0, 0, 0))
        per_head.append(items)
    n = max(len(it) for it in per_head)
    out = np.zeros((len(per_head), n, 8), dtype=np.int32)
    for h, items in enumerate(per_head):
        if items:
            out[h, :len(items)] = np.array(items, dtype=np.int32)
    return out


class TransformerLuts(object):
    """Everything BlocksparseTransformer derives from a (heads|1, q_blks, k_blks) layout."""

    def __init__(self, layout, block_size, mask_callback=None):
        lay = np.asarray(layout) != 0
        assert lay.ndim == 3
        self.lut_heads, self.ctx_blks_q, self.ctx_blks_k = lay.shape
        self.blk_size = block_size
        nt_luts, nn_luts, tn_luts = [], [], []
        self.nt_list, self.nn_list, self.tn_list = [], [], []
        self.nn_max = self.tn_max = 0
        self.blocks = None
        for h in range(self.lut_heads):
            qs, ks = np.nonzero(lay[h])                # row-major == sorted by (q, k)
            if self.blocks is None:
                self.blocks = len(qs)
            elif len(qs) != self.blocks:
                raise ValueError("number of layout blocks must be equal across heads")
            qs = qs.astype(np.int64)
            ks = ks.astype(np.int64)
            nn, nn_rows, nn_max = xn_lut(qs, ks, self.ctx_blks_q)
            tn, tn_rows, tn_max = xn_lut(ks, qs, self.ctx_blks_k)
            nt_luts.append(np.stack([qs, ks], axis=1).astype(np.int32))
            nn_luts.append(nn)
            tn_luts.append(tn)
            self.nt_list.append(list(zip(qs.tolist(), ks.tolist())))
            self.nn_list.append(nn_rows)
            self.tn_list.append(tn_rows)
            self.nn_max = max(self.nn_max, nn_max)
            self.tn_max = max(self.tn_max, tn_max)
        if not self.blocks:
            raise ValueError("layout has no non-zero blocks")
        self.nt_lut = np.stack(nt_luts)
        self.nn_lut = np.stack(nn_luts)
        self.tn_lut = np.stack(tn_luts)
        self.nt_items = build_nt_items(self.tn_list)
        # output blocks by decreasing row length (longest first) for the persistent XN kernels
        self.nn_order = np.stack([np.argsort(-np.array([len(r) for r in rows]), kind="stable") for rows in self.nn_list]).astype(np.int32)
        self.tn_order = np.stack([np.argsort(-np.array([len(r) for r in rows]), kind="stable") for rows in self.tn_list]).astype(np.int32)
        self.softmax_mask = self.softmax_mask_np = None
        if mask_callback is not None:
            self.init_softmax_mask(mask_callback)

    def init_softmax_mask(self, mask_callback):
        """Bit j of word r of block b is set iff key j is visible to query r (transformer.py:135-159)."""
        bs = self.blk_size
        dt = MASK_DTYPE[bs]
        weights = (np.uint64(1) << np.arange(bs, dtype=np.uint64))
        masks = np.empty((self.lut_heads, self.blocks, bs), dtype=dt)
        for h in range(self.lut_heads):
            for b, (q, k) in enumerate(self.nt_list[h]):
                m = np.asarray(mask_callback((bs, bs), h, q, k, b)).astype(bool)
                if m.shape != (bs, bs):
                    raise ValueError("mask_callback must return a (%d,%d) array" % (bs, bs))
                masks[h, b] = (m.astype(np.uint64) * weights[None, :]).sum(axis=1, dtype=np.uint64).astype(dt)
        self.softmax_mask_np = masks                                                     # heads, blocks, bs
        self.softmax_mask = np.ascontiguousarray(masks.transpose(0, 2, 1))              # reference device layout
