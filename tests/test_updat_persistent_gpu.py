"""The persistent wgmma updat kernel (csrc/tc_updat.cuh) where its CTAs run several tiles each, elementwise against
float64.

min(tiles, SMs) CTAs walk the schedule's tiles round-robin: CTA b runs tiles b, b + grid, ... Each tile multiplies
at the MMA width N = 64, 128, 192 or 256 that holds its kept output blocks. The ring of stages and its phase carry on
from one tile to the next, and the producer loads the next tile while the consumers still write out the previous one.
A fault there shows only in a CTA's second and later tiles, so every case here gives each CTA several tiles of mixed
widths:
  * tall_layout makes about 290 tiles, a quarter of them at each width: two or three tiles per CTA on an H100's full
    grid (test_full_grid_matches_oracle);
  * child processes started with BSMM_SM_MARGIN, which the library reads once per process, launch 1 or 7 CTAs, or
    leave the 12 SMs free that multi-GPU training leaves to NCCL (test_small_grid_matches_full_grid_and_oracle). On the
    schedule of the full grid, a smaller launch grid must give the same dW bit for bit: every dW element comes from
    one tile, with a fixed instruction sequence and no atomics.
test_cases_keep_several_tiles_per_cta_at_every_width checks on the CPU that the cases keep that coverage.
"""
import collections
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._util import (ROOT, _on_poisoned_output, assert_within, dtype_name, mma_gemm_bound, oracle_dense,
                         ref_errors)
from blocksparse_b200 import BlocksparseMatMul, _lib
from blocksparse_b200.lut import updat_record_shape
from oracle.bsmm_oracle import MatmulOracle

BF16, F16 = torch.bfloat16, torch.float16
EMPTY_GROUP = 5                 # a group of input blocks with no active block: no tile
EMPTY_COL = 3                   # an output block column with no active block


def tall_layout(bs, n_groups, seed):
    """(CB, KB = 512 / bs) layout in which group g (128 / bs consecutive input blocks) keeps exactly 1 + g % KT output
    blocks, KT = 256 / bs, each active in a random nonempty subset of the group's input blocks. The groups fit one
    window each, so the MMA widths 1..4 (x 64 columns) come in equal shares. Group EMPTY_GROUP and output block column
    EMPTY_COL hold no block, and the last group has only half its input blocks (one at bs 64)."""
    G, KT = 128 // bs, 256 // bs
    CB, KB = n_groups * G - G // 2, 2 * KT
    rng = np.random.default_rng(seed)
    lay = np.zeros((CB, KB), np.int32)
    cols = np.array([k for k in range(KB) if k != EMPTY_COL])
    for g in range(n_groups):
        if g == EMPTY_GROUP:
            continue
        rows = np.arange(g * G, min((g + 1) * G, CB))
        for k in rng.choice(cols, 1 + g % KT, replace=False):
            on = rng.random(len(rows)) < 0.5
            on[rng.integers(len(rows))] = True
            lay[rows[on], k] = 1
    return lay


Case = collections.namedtuple("Case", "bs axis dtype N pairs groups")
# stages per tile = ceil(N / 64) x pairs; axis 0 needs N % 8 == 0. 288 groups give 287 tiles: on 132 SMs that is two
# or more per CTA and too few to re-cut the windows; on 114 SMs _balance_windows re-cuts them into 342 tiles, and
# enough groups remain at N = 256 that some tiles of that width survive.
FULL_GRID_CASES = [
    Case(16, 1, BF16, 40, 1, 288),      # 1 stage: every tile starts one ring slot further on
    Case(16, 1, F16, 320, 1, 288),      # 5
    Case(16, 0, BF16, 256, 1, 288),     # 4: every tile starts on ring slot 0, one phase further on
    Case(16, 0, F16, 136, 2, 288),      # 6
    Case(32, 1, BF16, 136, 1, 288),     # 3
    Case(32, 1, F16, 64, 1, 288),       # 1
    Case(32, 0, BF16, 72, 3, 288),      # 6
    Case(32, 0, F16, 256, 1, 288),      # 4
    Case(64, 1, BF16, 256, 1, 288),     # 4
    Case(64, 1, F16, 136, 1, 288),      # 3
    Case(64, 0, BF16, 320, 1, 288),     # 5
    Case(64, 0, F16, 40, 1, 288),       # 1
]
# launch grids of 1 and 7 CTAs already run many tiles each: small layouts, long reductions
SMALL_GRID_CASES = [
    Case(16, 1, BF16, 72, 8, 24),       # 16 stages
    Case(16, 0, F16, 40, 5, 24),        # 5
    Case(32, 1, F16, 136, 3, 24),       # 9
    Case(32, 0, BF16, 64, 8, 24),       # 8
    Case(64, 1, BF16, 200, 2, 24),      # 8
    Case(64, 0, F16, 24, 7, 24),        # 7
]
# 12 SMs left free: the full-size layouts, whose own schedule is cut into more windows for the smaller grid
MARGIN_CASES = [
    Case(16, 1, F16, 64, 2, 288),       # 2
    Case(16, 0, BF16, 136, 1, 288),     # 3
    Case(32, 1, BF16, 40, 3, 288),      # 3
    Case(32, 0, F16, 200, 1, 288),      # 4
    Case(64, 1, F16, 72, 2, 288),       # 4
    Case(64, 0, BF16, 320, 1, 288),     # 5
]
# child-process launch grids: (id, fixed number of SMs or None, SM margin, cases)
CHILD_GRIDS = [("grid1", 1, None, SMALL_GRID_CASES), ("grid7", 7, None, SMALL_GRID_CASES),
               ("margin12", None, 12, MARGIN_CASES)]
CHILD_CASES = {name: cases for name, _, _, cases in CHILD_GRIDS}


def child_grid(entry, sm_count):
    _, fixed, margin, _ = entry
    return fixed if fixed else sm_count - margin


def case_id(case):
    return "bs%d-ax%d-%s-N%dx%d" % (case.bs, case.axis, dtype_name(case.dtype), case.N, case.pairs)


def stages(case):
    return -(-case.N // 64) * case.pairs


def case_seed(case):
    return case.bs * 100000 + case.axis * 10000 + case.N * 10 + case.pairs


def case_inputs(case):
    """The layout, the (x, dy) pairs on the host in the case's dtype and a gate with zeros, all from the case's seed."""
    lay = tall_layout(case.bs, case.groups, case_seed(case))
    rng = np.random.default_rng(case_seed(case) + 1)
    C, K = lay.shape[0] * case.bs, lay.shape[1] * case.bs
    shape = (lambda F: (case.N, F)) if case.axis else (lambda F: (F, case.N))
    draw = lambda F: torch.as_tensor(rng.normal(0, 1, shape(F)).astype(np.float32)).to(case.dtype)
    xs, es = zip(*[(draw(C), draw(K)) for _ in range(case.pairs)])
    blocks = int(lay.sum())
    gate = ((rng.random(blocks) < 0.7) * rng.uniform(0.5, 1.5, blocks)).astype(np.float32)
    return lay, list(xs), list(es), gate


def tile_widths(sched, bs):
    """NCH of every tile of an updat schedule: the MMA width in 64-column chunks that holds its n_act kept blocks."""
    rec = np.asarray(sched)[4:].reshape(-1, updat_record_shape(bs)[0])
    return (rec[:, 1] * bs + 63) // 64


def block_widths(sched, bs, blocks):
    """NCH of the tile that computes each W block."""
    sched = np.asarray(sched)
    REC, TAB = updat_record_shape(bs)
    rec = sched[4:].reshape(-1, REC)
    ids = rec[:, TAB:TAB + (128 // bs) * int(sched[2])]
    tile = np.broadcast_to(np.arange(len(rec))[:, None], ids.shape)
    out = np.zeros(blocks, np.int64)
    out[ids[ids >= 0]] = tile_widths(sched, bs)[tile[ids >= 0]]
    assert out.min() >= 1, "a W block is in no tile"
    return out


ALPHA = 0.75
# output dtype of each call of run_updat: "in" = the dtype of x and dy
OUT_DTYPES = {"dw32": "float32", "dw16": "in", "acc32": "float32", "acc16": "in", "gated": "float32"}


def run_updat(bsmm, xs, es, gate):
    """The updat calls every case checks: fresh fp32 and 16-bit dW (alpha != 1) on NaN-poisoned memory, beta = 1
    accumulation into a copy of each, and a fresh gated fp32 dW with alpha != 1. Returns {name: dW}."""
    F = _lib.FLAG_FORCE_TC
    out = {}

    def call(name, fn):
        out[name] = fn()
        assert _lib.device_error() == 0, "%s: a wait timed out or the kernel faulted: %s" % (name, _lib.device_error_text())
        assert _lib.last_kernel().startswith("wgmma_updat_bs%d" % bsmm.bsize), (name, _lib.last_kernel())

    call("dw32", lambda: _on_poisoned_output(lambda: bsmm.updat(xs, es, dw_dtype=torch.float32, flags=F)))
    call("dw16", lambda: _on_poisoned_output(lambda: bsmm.updat(xs, es, alpha=ALPHA, flags=F)))
    for fresh, acc in (("dw32", "acc32"), ("dw16", "acc16")):
        dw = out[fresh].clone()
        call(acc, lambda: bsmm.updat(xs, es, dw=dw, flags=F))
    call("gated", lambda: _on_poisoned_output(lambda: bsmm.updat(xs, es, alpha=ALPHA, gate=gate, dw_gated=True,
                                                                  dw_dtype=torch.float32, flags=F)))
    return out


def check_against_oracle(out, case, lay, xs, es, gate, widths, what):
    """Every element of every run_updat result (float64 arrays) lies within mma_gemm_bound of the float64 oracle. The
    blocks are checked per MMA width of the tile that computed them (widths: block_widths), so that BSMM_BOUND_LOG
    reports each width on its own."""
    bs = case.bs
    orc = MatmulOracle(lay, 32, case.axis)   # (axis 0, bs 64) is outside the reference's pairs: reuse the restatement
    orc.bsize, orc.C, orc.K = bs, lay.shape[0] * bs, lay.shape[1] * bs
    ref, ref_abs = 0.0, 0.0
    for x, e in zip(xs, es):
        xn, en = x.float().numpy(), e.float().numpy()
        ref = ref + oracle_dense(orc, "updat", xn, en)
        ref_abs = ref_abs + oracle_dense(orc, "updat", np.abs(xn), np.abs(en))
    k, gn = case.N * case.pairs, gate.astype(np.float64)[:, None, None]
    old32, old16 = out["dw32"], out["dw16"]
    expect = {                               # name: (reference, its absolute-value sum, epilogue roundings)
        "dw32": (ref, ref_abs, 0),
        "dw16": (ALPHA * ref, ALPHA * ref_abs, 1),
        "acc32": (old32 + ref, np.abs(old32) + ref_abs, 1),
        "acc16": (old16 + ref, np.abs(old16) + ref_abs, 1),
        "gated": (ALPHA * gn * ref, ALPHA * gn * ref_abs, 2),
    }
    for name, (r, a, extra) in expect.items():
        got = out[name]
        od = dtype_name(case.dtype) if OUT_DTYPES[name] == "in" else OUT_DTYPES[name]
        label = "%s, %s, %s dw" % (what, name, od)
        assert not np.isnan(got).any(), "%s: %d dw elements never written" % (label, int(np.isnan(got).sum()))
        for nch in (1, 2, 3, 4):
            sel = widths == nch
            if sel.any():
                assert_within(got[sel], r[sel], mma_gemm_bound(r[sel], a[sel], od, k, extra),
                              "%s, N=%d tiles" % (label, 64 * nch), a[sel], k, od, "wgmma_updat")
        _, l2 = ref_errors(got, r)
        assert l2 <= {"float32": 1e-5, "bfloat16": 4e-3, "float16": 1e-3}[od], "%s: l2 %.3e" % (label, l2)


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def _to_device(xs, es, gate):
    return [x.cuda() for x in xs], [e.cuda() for e in es], torch.as_tensor(gate).cuda()


# ---- coverage, on the CPU ------------------------------------------------------------------------------------------
SM_COUNTS = {"H100 SXM": 132, "H100 PCIe": 114}


def test_cases_keep_several_tiles_per_cta_at_every_width():
    """On both H100 parts, the schedules of the cases give each CTA several tiles of mixed MMA widths: in process,
    every case has every width and at least two tiles per CTA; in the child processes, on the full grid's schedule and
    on their own, some CTA's tiles have two different widths. The cases cover every kernel instantiation and the
    stage counts per tile where the ring position of a tile's first stage moves differently."""
    def widths(case, n_cta):
        lay = tall_layout(case.bs, case.groups, case_seed(case))
        return tile_widths(BlocksparseMatMul(lay, block_size=case.bs, feature_axis=case.axis)._luts.updat_schedule(
            case.bs, n_cta=n_cta)[0], case.bs)

    for part, sms in SM_COUNTS.items():
        for case in FULL_GRID_CASES:
            w = widths(case, sms)
            assert len(w) >= 2 * sms, "%s, %s: %d tiles on %d SMs" % (part, case_id(case), len(w), sms)
            assert set(w.tolist()) == {1, 2, 3, 4}, "%s, %s: widths %s" % (part, case_id(case), sorted(set(w.tolist())))
        for entry in CHILD_GRIDS:
            grid = child_grid(entry, sms)
            for case in entry[3]:
                for n_cta in (sms, grid):        # the full grid's schedule, then the child's own
                    w = widths(case, n_cta)
                    assert len(w) >= 2 * grid, "%s, %s: %d tiles" % (part, entry[0], len(w))
                    assert any(len(set(w[b::grid].tolist())) >= 2 for b in range(grid)), \
                        "%s, %s, %s: no CTA switches width" % (part, entry[0], case_id(case))
    combos = {(c.bs, c.axis, c.dtype) for c in FULL_GRID_CASES}
    assert combos == {(bs, axis, dt) for bs in (16, 32, 64) for axis in (0, 1) for dt in (BF16, F16)}
    cases = FULL_GRID_CASES + SMALL_GRID_CASES + MARGIN_CASES
    assert all(c.N % 8 == 0 for c in cases if c.axis == 0)
    st = {stages(c) for c in cases}
    assert {1, 3, 4} <= st and any(s > 4 and s % 4 for s in st), sorted(st)
    assert any(c.pairs == _lib.MAX_PAIRS for c in cases)


def test_tall_layout_holes():
    for bs in (16, 32, 64):
        G, KT = 128 // bs, 256 // bs
        lay = tall_layout(bs, 24, 1)
        assert lay.shape == (24 * G - G // 2, 2 * KT)
        assert not lay[EMPTY_GROUP * G:(EMPTY_GROUP + 1) * G].any() and not lay[:, EMPTY_COL].any()
        kept = [int(lay[g * G:(g + 1) * G].any(axis=0).sum()) for g in range(24)]
        assert kept == [0 if g == EMPTY_GROUP else 1 + g % KT for g in range(24)]


# ---- the device's full grid, in process ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", FULL_GRID_CASES, ids=case_id)
def test_full_grid_matches_oracle(case):
    dev = _device()
    lay, xs, es, gate = case_inputs(case)
    bsmm = BlocksparseMatMul(lay, block_size=case.bs, feature_axis=case.axis)
    d = bsmm._device_luts(dev)
    assert d["updat_tiles"] >= 2 * _lib.grid_sms(dev), \
        "%d tiles on %d SMs: CTAs no longer run several tiles" % (d["updat_tiles"], _lib.grid_sms(dev))
    out = run_updat(bsmm, *_to_device(xs, es, gate))
    widths = block_widths(d["updat_sched"].cpu().numpy(), case.bs, bsmm.blocks)
    check_against_oracle({k: v.double().cpu().numpy() for k, v in out.items()}, case, lay, xs, es, gate, widths,
                         case_id(case))


# ---- smaller launch grids, in child processes ------------------------------------------------------------------------
def child_outputs(path, cases, parent_grid):
    """Run in a child process started with BSMM_SM_MARGIN (the library reads it once per process): every case of
    CHILD_CASES[cases], once on the schedule built for the parent's parent_grid SMs ("same": only the launch grid
    differs) and once on the schedule built for this process's own grid ("own"). Saves the results as float32, the
    tile counts and, for "own", the MMA width of every W block to `path`."""
    dev = _device()
    grid = _lib.grid_sms(dev)
    res = {"grid": grid}
    own_grid_sms = _lib.grid_sms
    for i, case in enumerate(CHILD_CASES[cases]):
        lay, xs, es, gate = case_inputs(case)
        xs, es, gate = _to_device(xs, es, gate)
        for mode in ("same", "own"):
            if mode == "same":
                _lib.grid_sms = lambda d: parent_grid
            try:
                bsmm = BlocksparseMatMul(lay, block_size=case.bs, feature_axis=case.axis)
                d = bsmm._device_luts(dev)
            finally:
                _lib.grid_sms = own_grid_sms
            assert d["updat_tiles"] >= 2 * grid, "%s: %d tiles on %d SMs" % (case_id(case), d["updat_tiles"], grid)
            for name, dw in run_updat(bsmm, xs, es, gate).items():
                res["%d_%s_%s" % (i, mode, name)] = dw.float().cpu().numpy()
            res["%d_%s_tiles" % (i, mode)] = d["updat_tiles"]
            if mode == "own":
                res["%d_own_widths" % i] = block_widths(d["updat_sched"].cpu().numpy(), case.bs, bsmm.blocks)
    np.savez(path, **res)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", CHILD_GRIDS, ids=[e[0] for e in CHILD_GRIDS])
def test_small_grid_matches_full_grid_and_oracle(entry, tmp_path):
    """A child process launches the kernel on a smaller grid (BSMM_SM_MARGIN = SMs - grid), so that every CTA walks
    many tiles. Its bounded waits record a device error instead of trapping (BSMM_WAIT_TIMEOUT_MS=2000,notrap), so a
    protocol fault fails its device_error() check. On the schedule of this process's full grid, the results must
    equal this process's bit for bit. On the schedule balanced for the smaller grid, they must match the oracle."""
    name, _, _, cases = entry
    dev = _device()
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    grid, parent_grid = child_grid(entry, sm_count), _lib.grid_sms(dev)
    path = str(tmp_path / "child.npz")
    env = dict(os.environ, BSMM_SM_MARGIN=str(sm_count - grid), BSMM_WAIT_TIMEOUT_MS="2000,notrap")
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from tests.test_updat_persistent_gpu import child_outputs\n"
            "child_outputs(%r, %r, %d)\n" % (ROOT, path, name, parent_grid))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "%s child failed:\n%s%s" % (name, r.stdout[-4000:], r.stderr[-4000:])
    res = np.load(path)
    assert int(res["grid"]) == grid
    for i, case in enumerate(cases):
        what = "%s, %s" % (name, case_id(case))
        lay, xs, es, gate = case_inputs(case)
        bsmm = BlocksparseMatMul(lay, block_size=case.bs, feature_axis=case.axis)
        assert int(res["%d_same_tiles" % i]) == bsmm._device_luts(dev)["updat_tiles"], what
        for key, dw in run_updat(bsmm, *_to_device(xs, es, gate)).items():
            mine, theirs = dw.float().cpu().numpy(), res["%d_same_%s" % (i, key)]
            diff = mine.view(np.uint32) != theirs.view(np.uint32)
            assert not diff.any(), "%s, %s: %d of %d dw elements differ from the full grid's, worst by %.3e" % (
                what, key, int(diff.sum()), diff.size, float(np.nanmax(np.abs(mine - theirs))))
        own = {key: res["%d_own_%s" % (i, key)].astype(np.float64) for key in OUT_DTYPES}
        check_against_oracle(own, case, lay, xs, es, gate, res["%d_own_widths" % i],
                             "%s on its own schedule (%d tiles)" % (what, int(res["%d_own_tiles" % i])))
