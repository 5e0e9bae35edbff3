"""BlocksparseMatMul for H100 -- host side.

Keeps the Python op surface of the reference's blocksparse/matmul.py (class
BlocksparseMatMul :74-483, gradient wiring :485-527, group_param_grads :612-731) but
operates on torch tensors and calls the sm_90a kernels through the C ABI in
include/bsmm_b200.h.  There is no CPU path: tensors must live on a CUDA device.
"""
import ctypes
import math
import os

import numpy as np
import torch

from . import _lib
from .checkers import MatmulCheckers
from .fp8 import check_config as _fp8_check_config, quantize_fp8, quantize_fp8_t, quantize_fp8_weights, updat_fp8, xprop_fp8
from .lut import MatmulLuts, WIDE_REC, XPROP_GROUP, pick_xprop_tile

# 32 x 32 blocks and 16-bit dtypes: the default route picks, per layout, direction and minibatch, between one output block
# per CTA (csrc/tc.cuh) and the grouped kernel of csrc/tc_xprop2.cuh (lut.pick_xprop_tile); results are bit-identical.
# Opt-in variants: BSMM_XPROP2=1..3 selects a wide-tile kernel (csrc/tc_xprop2.cuh: 2 / 2 / 4 output blocks per CTA,
# 64 / 128 / 128 minibatch rows), BSMM_PAIR_TILES=1 runs csrc/tc.cuh as 2-CTA clusters that share every W block by TMA
# multicast.
_X2_VARIANTS = {1: 2, 2: 2, 3: 4}          # variant -> output blocks per tile
_X2_FORCE = int(os.environ.get("BSMM_XPROP2", "0"))
_PAIR_TILES = int(os.environ.get("BSMM_PAIR_TILES", "0"))
_GROUPED_VARIANTS = {4: 4}                 # output blocks per CTA -> bsmm_xprop variant of the grouped kernel
_XPROP_TILE = None                         # tests / scripts: 1 forces one block per CTA, 4 the grouped tile (None: the model)
# BSMM_PAD8=0: keep 8 x 8 blocks on the CUDA-core FMA kernels instead of the padded 16 x 16 wgmma path
_PAD8 = int(os.environ.get("BSMM_PAD8", "1"))


def _as_2d(t, axis, feat):
    """Flatten all non-feature dims (reference op.cc:130-139)."""
    if axis == 0:
        if t.shape[0] != feat:
            raise ValueError("expected feature dim %d on axis 0, got shape %s" % (feat, tuple(t.shape)))
        return t.reshape(feat, -1)
    if t.shape[-1] != feat:
        raise ValueError("expected feature dim %d on the last axis, got shape %s" % (feat, tuple(t.shape)))
    return t.reshape(-1, feat)


class BlocksparseMatMul(MatmulCheckers):
    """Drop-in for blocksparse.matmul.BlocksparseMatMul (reference matmul.py:74).

    layout        : 2-D 0/1 array (CB, KB) of active blocks
    block_size    : 8, 16, 32 or 64 (any feature axis; the reference restricts the pairs, :84-89)
    feature_axis  : 0 -> activations are (C, N);  1 -> activations are (N, C)
    """

    def __getstate__(self):
        return (self.layout, self.bsize, self.axis, self.z_order, self.name)

    def __setstate__(self, state):
        self.__init__(*state)

    def __init__(self, layout, block_size=32, feature_axis=0, z_order=True, name=None):
        if feature_axis not in (0, 1) or block_size not in (8, 16, 32, 64):
            raise ValueError("Unsupported block size with this feature axis")
        layout = np.asarray(layout)
        if layout.ndim != 2:
            raise ValueError("layout must be 2-D")
        self.axis, self.bsize = feature_axis, block_size
        luts = MatmulLuts(layout, z_order=z_order)
        self._luts = luts
        for k in ("updat_list", "updat_lut", "fprop_list", "bprop_list", "fprop_lut", "bprop_lut",
                  "fprop_shared", "bprop_shared", "fprop_segments", "bprop_segments",
                  "fprop_locks", "bprop_locks", "blocks", "CB", "KB"):
            setattr(self, k, getattr(luts, k))
        self.z_order = z_order
        self.name = name or "BlocksparseMatMul"
        self.flops = self.blocks * block_size * block_size * 2
        self.w_shape = (self.blocks, block_size, block_size)
        self.g_shape = (self.blocks,)
        self.count = 0
        self.C, self.K = self.CB * block_size, self.KB * block_size
        self.sparsity = round(float(self.blocks) / float(self.CB * self.KB), 3)
        self.layout = layout != 0
        self._dev = {}          # device -> dict of LUT tensors (uploaded once, matmul.py:33-53)
        # 8 x 8 blocks: the wgmma kernels need K >= 16, so 16-bit dtypes run on a SHADOW op over 16 x 16 super-blocks (2 x 2
        # neighbourhoods, absent sub-blocks zero) fed through bsmm_pad_blocks / bsmm_unpad_blocks (csrc/wutil.cuh)
        self._shadow = None
        if block_size == 8 and _PAD8 and self.CB % 2 == 0 and self.KB % 2 == 0:
            big = self.layout.reshape(self.CB // 2, 2, self.KB // 2, 2).any(axis=(1, 3))
            sh = BlocksparseMatMul(big.astype(np.int32), block_size=16, feature_axis=feature_axis, z_order=z_order, name=self.name + "/pad16")
            big_id = -np.ones(big.shape, dtype=np.int64)
            big_id[sh.updat_lut[:, 0], sh.updat_lut[:, 1]] = np.arange(sh.blocks)
            cs, ks = self.updat_lut[:, 0].astype(np.int64), self.updat_lut[:, 1].astype(np.int64)
            inv = big_id[cs // 2, ks // 2] * 4 + (cs % 2) * 2 + (ks % 2)
            sub = -np.ones(sh.blocks * 4, dtype=np.int32)
            sub[inv] = np.arange(self.blocks, dtype=np.int32)
            self._shadow, self._sub_map, self._inv_map = sh, sub, inv.astype(np.int32)

    def i_shape(self, N):
        return (N, self.C) if self.axis else (self.C, N)

    def o_shape(self, N):
        return (N, self.K) if self.axis else (self.K, N)

    def block_coord(self, block):
        return self.updat_list[block]

    # ------------------------------------------------------------------ initialisers
    def identity_init(self, scale=1.0, dtype=torch.float32, device="cuda"):
        """W such that blocks on the (wrapped) diagonal are scale*I (matmul.py:317-329, IdentityInitCK kernel)."""
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.BsmmError("identity_init runs on the GPU (no CPU path)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        W = torch.empty(self.w_shape, dtype=dtype, device=device)
        d = self._device_luts(device)
        with torch.cuda.device(device):
            rc = _lib.load().bsmm_identity_init(_lib.dtype_code(dtype), self.bsize, self.blocks, d["updat"].data_ptr(), self.CB, self.KB,
                                                W.data_ptr(), float(scale), _lib.stream_ptr())
        _lib.check(rc, "bsmm_identity_init")
        return W

    def ortho_init(self, dtype=torch.float32, device="cuda", rng=None):
        """Orthogonal columns inside every output block column (sparse layouts) or a dense orthogonal matrix cut into
        blocks (fully dense layouts) -- matmul.py:292-322; host-side SVD, one-off."""
        rng = rng or np.random
        bs = self.bsize
        W = np.empty(self.w_shape, dtype=np.float32)
        if self.sparsity < 1.0:
            for k, col in self.fprop_list:
                if not col:
                    continue
                shape = (len(col) * bs, bs)
                a = rng.normal(0.0, 1.0, shape).astype(np.float32)
                u, _, v = np.linalg.svd(a, full_matrices=False)
                if u.shape != shape:
                    u = v
                for i, (c, w) in enumerate(col):
                    W[w] = u[i * bs:(i + 1) * bs, :]
        else:
            shape = (self.C, self.K)
            a = rng.normal(0.0, 1.0, shape).astype(np.float32)
            u, _, v = np.linalg.svd(a, full_matrices=False)
            if u.shape != shape:
                u = v
            for w, (c, k) in enumerate(self.updat_list):
                W[w] = u[c * bs:(c + 1) * bs, k * bs:(k + 1) * bs]
        return torch.as_tensor(W).to(dtype).to(device)

    def l2_normalize(self, W, gain=None, epsilon=1e-12, dtype=None):
        """y = gain * W / sqrt(max(sum(W^2), eps)), the sum taken per OUTPUT feature over its whole sparse column
        (matmul.py:445-453); differentiable in W and gain.  dtype: output dtype (default W's; fp32 allowed)."""
        return _L2NormalizeFunction.apply(W, gain, self, float(epsilon), dtype or W.dtype)

    def checker_init(self, dtype=torch.float32, device="cuda"):
        """Checkerboard gate (matmul.py:331-337)."""
        cs, ks = self.updat_lut[:, 0], self.updat_lut[:, 1]
        return torch.as_tensor(((cs & 1) ^ (ks & 1) ^ 1).astype(np.float32), device=device).to(dtype)

    def prune(self, param, gate):
        """Drop blocks whose gate is zero (matmul.py:272-291).

        Like the reference, returns (new_param, new_gate) and clears the pruned blocks in `self.layout` in place; the
        LUTs of this object are NOT rebuilt -- construct a new BlocksparseMatMul from `self.layout` for the pruned op.
        """
        gate_np = gate.detach().cpu().numpy() if torch.is_tensor(gate) else np.asarray(gate)
        keep = gate_np != 0.0
        for w in np.nonzero(~keep)[0]:
            c, k = self.updat_list[w]
            self.layout[c, k] = False
        idx = torch.as_tensor(np.nonzero(keep)[0], device=param.device)
        new_gate = torch.ones(int(keep.sum()), dtype=gate.dtype if torch.is_tensor(gate) else torch.float32,
                              device=param.device)
        return param.index_select(0, idx), new_gate

    # ------------------------------------------------------------------ device state
    def _device_luts(self, device):
        key = (device.type, device.index)
        d = self._dev.get(key)
        if d is None:
            d = {
                "fprop": torch.as_tensor(self._luts.fprop_rows, device=device),
                "bprop": torch.as_tensor(self._luts.bprop_rows, device=device),
                "updat": torch.as_tensor(self.updat_lut, device=device),
            }
            if self.bsize in (16, 32, 64):
                us, uoff = self._luts.updat_schedule(self.bsize, n_cta=_lib.grid_sms(device))
                d["updat_sched"] = torch.as_tensor(us, device=device)
                d["updat_tiles"], d["updat_kt"] = int(us[0]), int(us[2])
            self._dev[key] = d
        return d

    def _wide_schedule(self, d, device, bprop, blocks_per_tile):
        key = ("wide", bool(bprop), blocks_per_tile)
        if key not in d:
            arr, n_tiles, off = self._luts.wide_schedule(bprop, blocks_per_tile)
            d[key] = (torch.as_tensor(arr, device=device), n_tiles, off, (len(arr) - off) // WIDE_REC)
        return d[key]

    def xprop_tile(self, bprop, N, device):
        """Output blocks per CTA of the default 32 x 32 / 16-bit xprop launch at minibatch N: 1 or the grouped tile."""
        if _XPROP_TILE is not None:
            return _XPROP_TILE
        d = self._device_luts(device)
        key = ("tile", bool(bprop), N)
        if key not in d:
            entries = self._wide_schedule(d, device, bprop, XPROP_GROUP)[3]
            d[key] = pick_xprop_tile(self.blocks, entries, self.CB if bprop else self.KB, N, _lib.grid_sms(device))
        return d[key]

    # ------------------------------------------------------------------ raw ops
    def fprop(self, x, w, gate=None, flags=0):
        return self._xprop(x, w, False, gate, flags)

    def bprop(self, dy, w, gate=None, flags=0):
        return self._xprop(dy, w, True, gate, flags)

    def _pad_maps(self, device):
        d = self._device_luts(device)
        if "sub_map" not in d:
            d["sub_map"] = torch.as_tensor(self._sub_map, device=device)
            d["inv_map"] = torch.as_tensor(self._inv_map, device=device)
        return d["sub_map"], d["inv_map"]

    def _padded_weights(self, w, gate):
        """(blocks, 8, 8) -> the shadow op's (blocks16, 16, 16), gate folded in."""
        sub, _ = self._pad_maps(w.device)
        sh = self._shadow
        w16 = torch.empty(sh.w_shape, dtype=w.dtype, device=w.device)
        g = None if gate is None else gate.to(torch.float32).contiguous()
        _lib.check(_lib.load().bsmm_pad_blocks(_lib.dtype_code(w.dtype), self.bsize, sh.blocks, sub.data_ptr(), w.contiguous().data_ptr(),
                                               _lib.ptr(g), w16.data_ptr(), _lib.stream_ptr()), "bsmm_pad_blocks")
        return w16

    @_lib.guarded
    def _xprop(self, x, w, bprop, gate, flags):
        lib = _lib.load()
        if not x.is_cuda:
            raise _lib.BsmmError("BlocksparseMatMul needs CUDA tensors (no CPU path)")
        if self._shadow is not None and x.dtype != torch.float32 and not (flags & _lib.FLAG_FORCE_GENERIC):
            if tuple(w.shape) != self.w_shape or w.dtype != x.dtype:
                raise ValueError("w must have shape %s and the dtype of x" % (self.w_shape,))
            return self._shadow._xprop(x, self._padded_weights(w, gate), bprop, None, flags)
        feat_in, feat_out = (self.K, self.C) if bprop else (self.C, self.K)
        x2 = x if (x.dim() == 2 and x.is_contiguous() and x.shape[self.axis] == feat_in) else _as_2d(x, self.axis, feat_in).contiguous()
        if not w.is_contiguous():
            w = w.contiguous()
        if w.shape != self.w_shape:
            raise ValueError("w must have shape %s, got %s" % (self.w_shape, tuple(w.shape)))
        if w.dtype != x.dtype:
            raise ValueError("x and w must have the same dtype")
        N = x2.shape[1] if self.axis == 0 else x2.shape[0]
        d = self._device_luts(x.device)
        lut = d["bprop" if bprop else "fprop"]
        n_in, n_out = (self.KB, self.CB) if bprop else (self.CB, self.KB)
        sched, sched_tiles, tile_arg, sched_off = None, 0, 0, 0
        if self.bsize == 32 and x.dtype != torch.float32:
            if _X2_FORCE in _X2_VARIANTS:
                sched, sched_tiles, sched_off, _ = self._wide_schedule(d, x.device, bprop, _X2_VARIANTS[_X2_FORCE])
                tile_arg = (1 << 16) | (_X2_FORCE << 8)
            elif _PAIR_TILES:
                tile_arg = 1 << 12
            else:
                tile = self.xprop_tile(bprop, N, x.device)
                if tile > 1:
                    sched, sched_tiles, sched_off, _ = self._wide_schedule(d, x.device, bprop, tile)
                    tile_arg = (1 << 16) | (_GROUPED_VARIANTS[tile] << 8)
        y2 = torch.empty((feat_out, N) if self.axis == 0 else (N, feat_out), dtype=x.dtype, device=x.device)
        if gate is not None:
            gate = gate.to(torch.float32).contiguous()
            if self.bsize in (16, 32, 64) and x.dtype != torch.float32 and not (flags & _lib.FLAG_FORCE_GENERIC):
                # gated product on the wgmma kernel: fold the gate into a scaled copy of the (small) weight tensor,
                # as the reference's gated kernels do with the loaded weights (cn_64.cu:96-98)
                wg = torch.empty_like(w)
                _lib.check(lib.bsmm_gate_weights(_lib.dtype_code(w.dtype), self.bsize, self.blocks, w.data_ptr(),
                                                 gate.data_ptr(), wg.data_ptr(), _lib.stream_ptr()), "bsmm_gate_weights")
                w, gate = wg, None
        rc = lib.bsmm_xprop(_lib.dtype_code(x.dtype), self.axis, self.bsize, int(bprop),
                            lut.data_ptr(), n_out, n_in, self.blocks,
                            x2.data_ptr(), w.data_ptr(), y2.data_ptr(), N,
                            _lib.ptr(gate),
                            _lib.ptr(sched), sched_tiles, tile_arg, sched_off, 0, 0, 0,
                            flags, _lib.stream_ptr())
        _lib.check(rc, "bsmm_xprop")
        if self.axis == 0:
            return y2.reshape((feat_out,) + tuple(x.shape[1:]))
        return y2.reshape(tuple(x.shape[:-1]) + (feat_out,))

    @_lib.guarded
    def updat(self, xs, dys, dw=None, alpha=1.0, gate=None, dw_gated=False, dw_dtype=None, flags=0):
        """DW[w] = alpha * sum_p X_p . DY_p^T (+ dw if given: in-place accumulate, DWA semantics)."""
        lib = _lib.load()
        if torch.is_tensor(xs):
            xs, dys = [xs], [dys]
        if len(xs) != len(dys) or not 1 <= len(xs) <= _lib.MAX_PAIRS:
            raise ValueError("need 1..%d (x, dy) pairs" % _lib.MAX_PAIRS)
        x0 = xs[0]
        if not x0.is_cuda:
            raise _lib.BsmmError("BlocksparseMatMul needs CUDA tensors (no CPU path)")
        ax = self.axis
        xs2 = [x if (x.dim() == 2 and x.is_contiguous() and x.shape[ax] == self.C) else _as_2d(x, ax, self.C).contiguous() for x in xs]
        dys2 = [e if (e.dim() == 2 and e.is_contiguous() and e.shape[ax] == self.K) else _as_2d(e, ax, self.K).contiguous() for e in dys]
        N = xs2[0].shape[1] if self.axis == 0 else xs2[0].shape[0]
        for a, b in zip(xs2, dys2):
            if a.dtype != x0.dtype or b.dtype != x0.dtype:
                raise ValueError("all x / dy tensors must share one dtype")
            if (a.shape[1] if self.axis == 0 else a.shape[0]) != N or (b.shape[1] if self.axis == 0 else b.shape[0]) != N:
                raise ValueError("all x / dy tensors must share the minibatch size")
        if self._shadow is not None and x0.dtype != torch.float32 and not (flags & _lib.FLAG_FORCE_GENERIC):
            # 8 x 8 blocks: the padded 16 x 16 product in fp32, then gather this layout's blocks (alpha / gate / accumulate here)
            dw16 = self._shadow.updat(xs, dys, alpha=alpha, dw_dtype=torch.float32, flags=flags)
            _, inv = self._pad_maps(x0.device)
            acc = dw is not None
            if dw is None:
                dw = torch.empty(self.w_shape, dtype=dw_dtype or x0.dtype, device=x0.device)
            elif tuple(dw.shape) != self.w_shape or not dw.is_contiguous():
                raise ValueError("dw must be a contiguous tensor of shape %s" % (self.w_shape,))
            g = gate.to(torch.float32).contiguous() if (gate is not None and dw_gated) else None
            _lib.check(lib.bsmm_unpad_blocks(_lib.F32, _lib.dtype_code(dw.dtype), self.bsize, self.blocks, inv.data_ptr(), dw16.data_ptr(),
                                             _lib.ptr(g), dw.data_ptr(), int(acc), _lib.stream_ptr()), "bsmm_unpad_blocks")
            return dw
        if dw is None:
            out_dtype = dw_dtype or x0.dtype
            dw = torch.empty(self.w_shape, dtype=out_dtype, device=x0.device)
            beta = 0.0
        else:
            if tuple(dw.shape) != self.w_shape or not dw.is_contiguous():
                raise ValueError("dw must be a contiguous tensor of shape %s" % (self.w_shape,))
            beta = 1.0
        if gate is not None:
            gate = gate.to(torch.float32).contiguous()
        xp, ep = _lib.ptr_array(xs2), _lib.ptr_array(dys2)
        d = self._device_luts(x0.device)
        rc = lib.bsmm_updat(_lib.dtype_code(x0.dtype), _lib.dtype_code(dw.dtype), self.axis, self.bsize,
                            d["updat"].data_ptr(), self.blocks, self.CB, self.KB,
                            xp, ep, len(xs2), dw.data_ptr(), N, float(alpha), beta,
                            _lib.ptr(gate), int(bool(dw_gated)),
                            _lib.ptr(d.get("updat_sched")), d.get("updat_tiles", 0), d.get("updat_kt", 0), 0,
                            flags, _lib.stream_ptr())
        _lib.check(rc, "bsmm_updat")
        return dw

    @_lib.guarded
    def gate_grad(self, dw, w):
        """dg[w] = sum(dw[w] * w[w])  (BlocksparseMatmulDG, matmul.py:519-523)."""
        lib = _lib.load()
        dg = torch.empty(self.blocks, dtype=torch.float32, device=w.device)
        dw = dw.to(w.dtype).contiguous()
        rc = lib.bsmm_gate_grad(_lib.dtype_code(w.dtype), self.bsize, self.blocks, dw.data_ptr(),
                                w.contiguous().data_ptr(), dg.data_ptr(), _lib.stream_ptr())
        _lib.check(rc, "bsmm_gate_grad")
        return dg

    # ------------------------------------------------------------------ autograd op
    def matmul(self, I, W, gate=None, gate_grad=False, dw_gated=False, name=None, bench=0):
        return self.__call__(I, W, gate=gate, gate_grad=gate_grad, dw_gated=dw_gated, name=name, bench=bench)

    def __call__(self, I, W, gate=None, gate_grad=False, dw_gated=False, name=None, bench=0):
        """y = bsmm(x, w) with gradients for x, w (and gate when gate_grad) -- matmul.py:458-527.

        bench > 0 repeats the forward launch `bench` times between two CUDA events and prints
        the reference's one-line report (op.cc:99-106, gpu_types.cc:43-87).
        """
        self.count += 1
        if bench:
            self._bench_op("fprop", lambda: self.fprop(I, W, gate), I, bench, name or self.name)
        return _BsmmFunction.apply(I, W, gate, self, bool(gate_grad), bool(dw_gated), int(bench), name or self.name)

    def matmul_fp8(self, I, W, name=None, fp8_dw=False):
        """y = bsmm(I, W) on fp8 tensor cores, with gradients for I and W (DESIGN.md 6e, 6f).

        Forward: I and W are quantised to e4m3 with one scale each (fp8.quantize_fp8 / quantize_fp8_weights) and the fp8
        fprop runs; y comes out in I's dtype. Backward: dy is quantised to e5m2 and the fp8 bprop runs against the saved
        e4m3 weights, so dx comes out in I's dtype.
        dw: with fp8_dw=False it is the 16-bit updat of the saved I and dy, exactly as in bsmm(I, W)'s backward
        (group_param_grads included), so it is bit-identical to it. With fp8_dw=True it is the fp8 updat (fp8.updat_fp8)
        of the e4m3 I and the e5m2 dy, in W's dtype: the forward keeps a transposed e4m3 copy of I (quantize_fp8_t, one
        byte per element) instead of I itself, and the backward quantises dy once for both the bprop and the updat.
        y and dx are bit-identical to fp8_dw=False's. fp8_dw is a precision choice, not a speed switch: dw then carries
        the quantisation error of both operands, and against the float64 product of the dequantised operands it is
        within (2^-11 + (stages + 3) 2^-24) sum|x^||dy^| + u_out |dw|, stages being the 128-row minibatch chunks summed
        (DESIGN.md 6f gives the bound and where the fp8 updat is faster or slower than the 16-bit one).
        I (..., C) and W (blocks, bs, bs) are float16 or bfloat16 CUDA tensors of one dtype; feature_axis 1 and block
        sizes 32 / 64 only. There is no gate argument. `name` is accepted for symmetry with __call__."""
        _fp8_check_config(self)
        for t in (I, W):
            if not torch.is_tensor(t) or t.dtype not in (torch.float16, torch.bfloat16):
                raise ValueError("matmul_fp8 takes float16 or bfloat16 tensors, got %s" % (getattr(t, "dtype", type(t)),))
        if W.dtype != I.dtype:
            raise ValueError("matmul_fp8: I is %s, W is %s" % (I.dtype, W.dtype))
        if not I.is_cuda or not W.is_cuda:
            raise _lib.BsmmError("BlocksparseMatMul needs CUDA tensors (no CPU path)")
        if tuple(W.shape) != self.w_shape:
            raise ValueError("W must have shape %s, got %s" % (self.w_shape, tuple(W.shape)))
        if I.dim() < 1 or I.shape[-1] != self.C:
            raise ValueError("expected feature dim %d on the last axis, got shape %s" % (self.C, tuple(I.shape)))
        if I.device != W.device:
            raise ValueError("matmul_fp8: I lives on %s, W on %s" % (I.device, W.device))
        self.count += 1
        if fp8_dw:
            return _Fp8DwMatmulFunction.apply(I, W, self)
        return _Fp8MatmulFunction.apply(I, W, self)

    def _bench_op(self, what, fn, I, repeat, name):
        """The reference's `bench` attribute (op.cc:99-106,181-185, gpu_types.cc:43-87): repeat the launch `repeat` times
        between two CUDA events and print one line; applies to fprop and, through the backward pass, to bprop and updat."""
        lib = _lib.load()
        timer = ctypes.c_void_p()
        _lib.check(lib.bsmm_timer_create(ctypes.byref(timer)), "timer_create")
        fn()
        _lib.check(lib.bsmm_timer_begin(timer, _lib.stream_ptr()), "timer_begin")
        for _ in range(repeat):
            fn()
        ms = ctypes.c_float()
        _lib.check(lib.bsmm_timer_end(timer, _lib.stream_ptr(), ctypes.byref(ms)), "timer_end")
        lib.bsmm_timer_destroy(timer)
        N = I.numel() // (self.K if what == "bprop" else self.C)
        ms_per = ms.value / repeat
        gflops = self.flops * N / (ms_per * 1e6)
        print("%s %s ms: %.4f gflops: %.0f" % (name, what, ms_per, gflops))
        return ms_per


class _BsmmFunction(torch.autograd.Function):
    """Mirrors blocksparse_matmul_grad (reference matmul.py:485-527)."""

    @staticmethod
    def forward(ctx, x, w, gate, bsmm, gate_grad, dw_gated, bench=0, name=None):
        ctx.bsmm, ctx.gate_grad, ctx.dw_gated, ctx.bench, ctx.name = bsmm, gate_grad, dw_gated, bench, name
        ctx.save_for_backward(x, w, gate)
        return bsmm.fprop(x, w, gate)

    @staticmethod
    def backward(ctx, dy):
        x, w, gate = ctx.saved_tensors
        bsmm = ctx.bsmm
        dy = dy.contiguous()
        if ctx.bench:
            bsmm._bench_op("bprop", lambda: bsmm.bprop(dy, w, gate), dy, ctx.bench, ctx.name)
            bsmm._bench_op("updat", lambda: bsmm.updat([x], [dy], gate=gate, dw_gated=ctx.dw_gated), x, ctx.bench, ctx.name)
        dx = bsmm.bprop(dy, w, gate) if ctx.needs_input_grad[0] else None
        dw = dg = None
        want_dg = gate is not None and ctx.gate_grad and ctx.needs_input_grad[2]
        if want_dg:
            # reference matmul.py:519-523 + cn_64.cu:1340-1412: dw is produced ungated, then
            # dg[w] = sum(dw[w] * w[w]) and dw is scaled by the gate in the same pass
            raw = bsmm.updat([x], [dy])
            dg = bsmm.gate_grad(raw, w).to(gate.dtype)
            dw = raw * gate.to(raw.dtype).view(-1, 1, 1)
        elif ctx.needs_input_grad[1]:
            dw = _weight_grad(bsmm, x, w, dy, gate, ctx.dw_gated)
        return dx, dw, dg, None, None, None, None, None


def _weight_grad(bsmm, x, w, dy, gate=None, dw_gated=False):
    """dw of one use of w: handed to the open group_param_grads block of (bsmm, w) if there is one, else one updat."""
    pending = _pending_group(bsmm, w)
    if pending is not None:
        return pending.add(x, dy, gate, dw_gated)
    return bsmm.updat([x], [dy], gate=gate, dw_gated=dw_gated)


class _Fp8MatmulFunction(torch.autograd.Function):
    """BlocksparseMatMul.matmul_fp8: e4m3 fprop, e5m2 x e4m3 bprop, 16-bit updat."""

    @staticmethod
    def forward(ctx, x, w, bsmm):
        xq, xs = quantize_fp8(x, torch.float8_e4m3fn)
        wq, wq_t, ws = quantize_fp8_weights(bsmm, w, torch.float8_e4m3fn)
        ctx.bsmm = bsmm
        ctx.save_for_backward(x, w, wq, ws)
        return xprop_fp8(bsmm, xq, wq_t, xs, ws, bprop=False, out_dtype=x.dtype)

    @staticmethod
    def backward(ctx, dy):
        x, w, wq, ws = ctx.saved_tensors
        bsmm = ctx.bsmm
        dy = dy.contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dq, ds = quantize_fp8(dy, torch.float8_e5m2)
            dx = xprop_fp8(bsmm, dq, wq, ds, ws, bprop=True, out_dtype=x.dtype)
        if ctx.needs_input_grad[1]:
            dw = _weight_grad(bsmm, x, w, dy)
        return dx, dw, None


class _Fp8DwMatmulFunction(torch.autograd.Function):
    """BlocksparseMatMul.matmul_fp8(fp8_dw=True): e4m3 fprop, e5m2 x e4m3 bprop, e4m3 x e5m2 updat. I is kept only as
    its transposed e4m3 copy."""

    @staticmethod
    def forward(ctx, x, w, bsmm):
        x2 = x.reshape(-1, bsmm.C)
        xq, xq_t, xs = quantize_fp8_t(x2, torch.float8_e4m3fn)
        wq, wq_t, ws = quantize_fp8_weights(bsmm, w, torch.float8_e4m3fn)
        ctx.bsmm, ctx.N, ctx.x_shape = bsmm, x2.shape[0], tuple(x.shape)
        ctx.save_for_backward(xq_t, xs, w, wq, ws)
        return xprop_fp8(bsmm, xq.view(x.shape), wq_t, xs, ws, bprop=False, out_dtype=x.dtype)

    @staticmethod
    def backward(ctx, dy):
        xq_t, xs, w, wq, ws = ctx.saved_tensors
        bsmm = ctx.bsmm
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dx = dw = None
        if need_dx or need_dw:
            dq, dq_t, ds = quantize_fp8_t(dy.reshape(-1, bsmm.K), torch.float8_e5m2, with_rows=need_dx)
        if need_dx:
            dx = xprop_fp8(bsmm, dq, wq, ds, ws, bprop=True, out_dtype=w.dtype).view(ctx.x_shape)
        if need_dw:
            pending = _pending_group(bsmm, w)
            if pending is not None:
                dw = pending.add_fp8(xq_t, xs, dq_t, ds, ctx.N)
            else:
                dw = updat_fp8(bsmm, xq_t, dq_t, xs, ds, ctx.N, dw_dtype=w.dtype)
        return dx, dw, None


# ---------------------------------------------------------------------------------------
# group_param_grads: fuse the dW of a weight that is reused T times into ceil(T/8) launches
# (reference matmul.py:612-731 rewrites the TF graph; with eager autograd the same effect is
# a context manager that defers the per-use updat calls and flushes them in groups).
# ---------------------------------------------------------------------------------------

_groups = {}


class _Pending(object):
    def __init__(self, bsmm, w, group_size):
        self.bsmm, self.w, self.group_size = bsmm, w, group_size
        self.xs, self.dys = [], []
        self.gate, self.dw_gated = None, False
        self.fp8 = []                    # (xt, x_scale_inv, dyt, dy_scale_inv) of matmul_fp8(fp8_dw=True) uses
        self.fp8_n = None
        self.dw = None
        self.launches = 0                # every flush, 16-bit and fp8
        self.fp8_launches = 0

    def add(self, x, dy, gate, dw_gated):
        self.xs.append(x)
        self.dys.append(dy)
        self.gate, self.dw_gated = gate, dw_gated
        if len(self.xs) == self.group_size:
            self.flush()
        # autograd accumulates whatever backward returns into w.grad; the real sum is
        # delivered once by finish(), so intermediate uses contribute nothing.
        return None

    def add_fp8(self, xt, xs, dyt, ds, N):
        if self.fp8 and (N != self.fp8_n or xt.shape[1] != self.fp8[0][0].shape[1]):
            self.flush_fp8()                     # one updat_fp8 launch takes one N and one pitch
        self.fp8.append((xt, xs, dyt, ds))
        self.fp8_n = N
        if len(self.fp8) == self.group_size:
            self.flush_fp8()
        return None

    def flush(self):
        self.flush_fp8()
        self.flush_16()

    def flush_16(self):
        if not self.xs:
            return
        self.dw = self.bsmm.updat(self.xs, self.dys, dw=self.dw, gate=self.gate, dw_gated=self.dw_gated)
        self.launches += 1
        self.xs, self.dys = [], []

    def flush_fp8(self):
        if not self.fp8:
            return
        xts, xss, dyts, dss = (list(t) for t in zip(*self.fp8))
        self.dw = updat_fp8(self.bsmm, xts, dyts, xss, dss, self.fp8_n, dw=self.dw, dw_dtype=self.w.dtype)
        self.launches += 1
        self.fp8_launches += 1
        self.fp8 = []


def _pending_group(bsmm, w):
    return _groups.get((id(bsmm), w.data_ptr()))


class group_param_grads(object):
    """with group_param_grads(bsmm, w, group_size=8): loss.backward()

    Inside the block every backward use of `w` through `bsmm` hands its (x, dy) pair to
    a pending list instead of launching its own updat; every `group_size` (<= 8) pairs
    are flushed as ONE multi-pair launch that accumulates in place (DW then DWA in the
    reference, matmul.py:681-692).  Uses through matmul_fp8(..., fp8_dw=True) hand over their
    fp8 operands instead and are flushed the same way through updat_fp8 into the same dw, so a
    weight used both ways gets the sum.  On exit the total is added to w.grad.
    """

    def __init__(self, bsmm, w, group_size=8):
        assert 1 <= group_size <= _lib.MAX_PAIRS
        if not w.is_leaf:
            # the total is written to w.grad on exit: a derived tensor (a cast, a view of a fused parameter) would
            # swallow it, and its data_ptr would not match the tensor the op sees
            raise ValueError("group_param_grads needs the leaf parameter that is passed to the op, got a derived tensor")
        self.key = (id(bsmm), w.data_ptr())
        self.pending = _Pending(bsmm, w, group_size)
        self.w = w

    def __enter__(self):
        _groups[self.key] = self.pending
        return self.pending

    def __exit__(self, *exc):
        _groups.pop(self.key, None)
        if exc[0] is None:
            self.pending.flush()
            if self.pending.launches == 0:
                raise RuntimeError("group_param_grads: no backward use of this (op, parameter) pair was seen inside the "
                                   "block -- was the op called with a cast or a view of the parameter?")
            if self.pending.dw is not None:
                g = self.pending.dw.to(self.w.dtype)
                self.w.grad = g if self.w.grad is None else self.w.grad + g
        return False


class _L2NormalizeFunction(torch.autograd.Function):
    """L2NormalizeCK / L2NormalizeGainCK and their gradients (reference matmul.py:530-551)."""

    @staticmethod
    def forward(ctx, W, gain, bsmm, epsilon, out_dtype):
        if not W.is_cuda:
            raise _lib.BsmmError("l2_normalize needs CUDA tensors (no CPU path)")
        if tuple(W.shape) != bsmm.w_shape:
            raise ValueError("W must have shape %s" % (bsmm.w_shape,))
        W = W.contiguous()
        g = None if gain is None else gain.to(torch.float32).contiguous()
        if g is not None and g.numel() != bsmm.K:
            raise ValueError("gain must have K = %d entries" % bsmm.K)
        if g is not None and g.device != W.device:
            raise ValueError("gain lives on %s, W on %s" % (g.device, W.device))
        y = torch.empty(bsmm.w_shape, dtype=out_dtype, device=W.device)
        ss = torch.empty(bsmm.K, dtype=torch.float32, device=W.device)
        d = bsmm._device_luts(W.device)
        with torch.cuda.device(W.device):
            rc = _lib.load().bsmm_l2_normalize(_lib.dtype_code(W.dtype), _lib.dtype_code(out_dtype), bsmm.bsize, d["fprop"].data_ptr(),
                                               bsmm.KB, W.data_ptr(), _lib.ptr(g), y.data_ptr(), ss.data_ptr(), epsilon, _lib.stream_ptr())
        _lib.check(rc, "bsmm_l2_normalize")
        ctx.bsmm, ctx.epsilon, ctx.has_gain, ctx.gain_dtype = bsmm, epsilon, gain is not None, None if gain is None else gain.dtype
        ctx.save_for_backward(W, g, ss)
        return y

    @staticmethod
    def backward(ctx, dy):
        W, g, ss = ctx.saved_tensors
        bsmm = ctx.bsmm
        dy = dy.contiguous()
        if dy.dtype not in (W.dtype, torch.float32):
            dy = dy.to(W.dtype)
        dx = torch.empty_like(W)
        dg = torch.empty(bsmm.K, dtype=torch.float32, device=W.device) if ctx.has_gain else None
        d = bsmm._device_luts(W.device)
        with torch.cuda.device(W.device):
            rc = _lib.load().bsmm_l2_normalize_grad(_lib.dtype_code(W.dtype), _lib.dtype_code(dy.dtype), bsmm.bsize, d["fprop"].data_ptr(),
                                                    bsmm.KB, dy.data_ptr(), W.data_ptr(), _lib.ptr(g), ss.data_ptr(), dx.data_ptr(),
                                                    _lib.ptr(dg), ctx.epsilon, _lib.stream_ptr())
        _lib.check(rc, "bsmm_l2_normalize_grad")
        return dx, (dg.to(ctx.gain_dtype).view(-1) if dg is not None else None), None, None, None


def blocksparse_reduced_dw(xs, dys, scale, dwi=None, bsize=32, norm="max", axis=0):
    """Block-reduced FULL weight gradient for network growth (BlocksparseReducedDW, reference matmul.py:556-609,
    src/blocksparse_matmul_op.cc:639-773): every activation / gradient tensor is reduced over the bsize features of each
    block (max|.| or l2 norm), then dw[bC, bK] = scale * sum over pairs and minibatch of x_red * y_red (+ dwi, in place).

    xs, dys: lists of up to 8 16-bit tensors, (C, N) for axis 0 or (N, C) for axis 1.  Returns (dw fp32, x_red, y_red).
    """
    if torch.is_tensor(xs):
        xs, dys = [xs], [dys]
    if len(xs) != len(dys) or not 1 <= len(xs) <= _lib.MAX_PAIRS:
        raise ValueError("need 1..%d (x, dy) pairs" % _lib.MAX_PAIRS)
    x0 = xs[0]
    if not x0.is_cuda:
        raise _lib.BsmmError("blocksparse_reduced_dw needs CUDA tensors (no CPU path)")
    xs = [x.reshape(x.shape[0], -1).contiguous() if axis == 0 else x.reshape(-1, x.shape[-1]).contiguous() for x in xs]
    dys = [e.reshape(e.shape[0], -1).contiguous() if axis == 0 else e.reshape(-1, e.shape[-1]).contiguous() for e in dys]
    C, K = xs[0].shape[axis], dys[0].shape[axis]
    N = xs[0].shape[1 - axis]
    if C % bsize or K % bsize:
        raise ValueError("feature dims must be multiples of the block size")
    bC, bK, P = C // bsize, K // bsize, len(xs)
    for a, b in zip(xs, dys):
        if a.dtype != x0.dtype or b.dtype != x0.dtype or a.shape[1 - axis] != N or b.shape[1 - axis] != N or a.shape[axis] != C or b.shape[axis] != K:
            raise ValueError("all pairs must share dtype, minibatch and feature sizes")
        if a.device != x0.device or b.device != x0.device:
            raise ValueError("all pairs must live on one device, got %s and %s" % (x0.device, a.device if a.device != x0.device else b.device))
    dev = x0.device
    if dwi is not None and dwi.device != dev:
        raise ValueError("dwi lives on %s, the pairs on %s" % (dwi.device, dev))
    x_red = torch.empty((bC, P, N) if axis == 0 else (P, N, bC), dtype=x0.dtype, device=dev)
    y_red = torch.empty((bK, P, N) if axis == 0 else (P, N, bK), dtype=x0.dtype, device=dev)
    if dwi is None:
        dw, acc = torch.empty((bC, bK), dtype=torch.float32, device=dev), 0
    else:
        if tuple(dwi.shape) != (bC, bK) or dwi.dtype != torch.float32 or not dwi.is_contiguous():
            raise ValueError("dwi must be a contiguous float32 (%d, %d) tensor" % (bC, bK))
        dw, acc = dwi, 1
    lib = _lib.load()
    ws = torch.empty(lib.bsmm_reduced_dw_workspace_bytes(bC, bK), dtype=torch.uint8, device=dev)
    arr_t = ctypes.c_void_p * P
    with torch.cuda.device(dev):
        rc = lib.bsmm_reduced_dw(_lib.dtype_code(x0.dtype), axis, bsize, arr_t(*[t.data_ptr() for t in xs]), arr_t(*[t.data_ptr() for t in dys]),
                                 P, bC, bK, N, float(scale), 0 if norm.lower() == "max" else 1, dw.data_ptr(), acc,
                                 x_red.data_ptr(), y_red.data_ptr(), ws.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "bsmm_reduced_dw")
    return dw, x_red, y_red


def block_reduced_full_dw(pairs, scale=1.0, norm="max", group_size=8, bsize=32, axis=0):
    """Eager counterpart of the reference's graph rewrite (matmul.py:556-609): `pairs` is the list of (x, dy) tensors of
    every use of a shared weight (what the rewrite collects from the BlocksparseMatmulDW ops); they are reduced
    `group_size` (<= 8) at a time, accumulating into one (bC, bK) fp32 tensor."""
    assert 1 <= group_size <= _lib.MAX_PAIRS
    dw = None
    for off in range(0, len(pairs), group_size):
        chunk = pairs[off:off + group_size]
        dw, _, _ = blocksparse_reduced_dw([p[0] for p in chunk], [p[1] for p in chunk], scale, dw, bsize=bsize, norm=norm, axis=axis)
    return dw


_DW_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def dw_matmul_large_n(x, e, *, flags=0):
    """U = X^T . E in fp32 over a very large effective minibatch (the reference's top-level dw_matmul_large_n,
    src/matmul_op.cc DwMatmulLargeN), e.g. the weight gradient of a dense layer summed over batch x time.

    x (..., C) and e (..., K) have the same rank and the same leading dims, whose product N is the minibatch; both are
    fp32, fp16 or bf16, of one dtype, on one CUDA device.  Returns a new fp32 (C, K) tensor.  Any C, K, N >= 0 work
    (the reference needs C, K % 4 == 0 and N % 32 == 0): N = 0 gives zeros, C = 0 or K = 0 an empty tensor.

    The minibatch is split into segments whose number depends on (N, C, K) and the route only, each reduced in fp32,
    and the segments' partials are added in a fixed order: the result is bitwise reproducible on any device, stream or
    SM margin.  fp16 / bf16 with C and K multiples of 8 run on a wgmma kernel, everything else (fp32 included) on a true
    fp32 FMA kernel.  `flags` takes _lib.FLAG_FORCE_GENERIC / FLAG_FORCE_TC, as BlocksparseMatMul.fprop does.

    The op has no gradient, as in the reference: the result never requires grad.
    """
    if not torch.is_tensor(x) or not torch.is_tensor(e):
        raise ValueError("dw_matmul_large_n takes two tensors")
    if x.dtype != e.dtype:
        raise ValueError("dw_matmul_large_n: x is %s, e is %s" % (x.dtype, e.dtype))
    if x.dtype not in _DW_DTYPES:
        raise ValueError("dw_matmul_large_n takes float32, float16 or bfloat16, got %s" % (x.dtype,))
    if x.dim() < 1 or x.dim() != e.dim() or x.shape[:-1] != e.shape[:-1]:
        raise ValueError("dw_matmul_large_n: x %s and e %s must have one rank and the same leading dims"
                         % (tuple(x.shape), tuple(e.shape)))
    if not x.is_cuda or not e.is_cuda:
        raise ValueError("dw_matmul_large_n needs CUDA tensors (no CPU path)")
    if x.device != e.device:
        raise ValueError("dw_matmul_large_n: x lives on %s, e on %s" % (x.device, e.device))
    C, K = x.shape[-1], e.shape[-1]
    N = math.prod(x.shape[:-1])
    u = torch.empty((C, K), dtype=torch.float32, device=x.device)
    if C == 0 or K == 0:
        return u
    x2 = x.detach().reshape(N, C).contiguous()
    e2 = e.detach().reshape(N, K).contiguous()
    lib = _lib.load()
    code = _lib.dtype_code(x.dtype)
    with torch.cuda.device(x.device):
        nbytes = lib.bsmm_dw_matmul_large_n_workspace_bytes(code, N, C, K)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
        rc = lib.bsmm_dw_matmul_large_n(code, x2.data_ptr(), e2.data_ptr(), u.data_ptr(), N, C, K, _lib.ptr(ws),
                                        int(flags), _lib.stream_ptr())
    _lib.check(rc, "bsmm_dw_matmul_large_n")
    return u


class _GatherRows(torch.autograd.Function):
    """GatherScatter op (reference matmul.py:895-898): out[r] = x[idx[r]] (0 where idx < 0); the gradient is the same op
    with the reverse table."""

    @staticmethod
    def forward(ctx, x, fwd_idx, bwd_idx, n_out):
        ctx.fwd_idx, ctx.bwd_idx, ctx.n_in = fwd_idx, bwd_idx, x.shape[0]
        return _gather_rows(x, None, fwd_idx, n_out, 0)

    @staticmethod
    def backward(ctx, dy):
        return _gather_rows(dy.contiguous(), None, ctx.bwd_idx, ctx.n_in, 0), None, None, None


class _ScatterAddMul(torch.autograd.Function):
    """ScatterAddMul op (reference matmul.py:900-910): z = x (+|*) scatter(y)."""

    @staticmethod
    def forward(ctx, x, y, gather_idx, scatter_idx, op):
        ctx.op, ctx.gather_idx, ctx.scatter_idx = op, gather_idx, scatter_idx
        ctx.save_for_backward(x, y)
        return _gather_rows(x, y, scatter_idx, x.shape[0], op)

    @staticmethod
    def backward(ctx, dz):
        x, y = ctx.saved_tensors
        dz = dz.contiguous()
        if ctx.op == 1:
            return dz, _gather_rows(dz, None, ctx.gather_idx, y.shape[0], 0), None, None, None
        dx = _gather_rows(dz, y, ctx.scatter_idx, x.shape[0], 2)                               # dz * scatter(y) (1 elsewhere)
        dy = _gather_rows((dz * x).contiguous(), None, ctx.gather_idx, y.shape[0], 0)          # gather(dz * x)
        return dx, dy, None, None, None


def _gather_rows(x, y, idx, n_out, op):
    if not x.is_cuda:
        raise _lib.BsmmError("SparseProj needs CUDA tensors (no CPU path)")
    if y is not None and y.device != x.device:
        raise ValueError("SparseProj: operands live on %s and %s" % (x.device, y.device))
    x2 = x.reshape(x.shape[0], -1).contiguous()
    y2 = None if y is None else y.reshape(y.shape[0], -1).contiguous()
    out = torch.empty((n_out,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        rc = _lib.load().bsmm_gather_rows(_lib.dtype_code(x.dtype), x2.data_ptr(), _lib.ptr(y2), idx.data_ptr(), out.data_ptr(),
                                          n_out, x2.shape[1], op, _lib.stream_ptr())
    _lib.check(rc, "bsmm_gather_rows")
    return out


class SparseProj(object):
    """Drop-in for blocksparse.matmul.SparseProj (reference matmul.py:835-921): a fixed sparse projection of the feature
    axis (axis 0 of (features, N) activations) by row gather / scatter, differentiable."""

    def __getstate__(self):
        return (self.nhidden, self.nproj, self.gather_lut, self.name)

    def __setstate__(self, state):
        self.__init__(state[0], nproj=state[1], gather_lut=state[2], name=state[3])

    def __init__(self, nhidden, nproj=None, proj_stride=None, block_size=32, gather_lut=None, name=None):
        if gather_lut is None:
            gather_lut = np.arange(nhidden, dtype=np.int32)
            if nproj is not None:
                assert nproj <= nhidden
                np.random.shuffle(gather_lut)
                gather_lut = np.sort(gather_lut[0:nproj])
            elif proj_stride is not None:
                assert proj_stride <= nhidden
                gather_max = ((nhidden // proj_stride) // block_size) * block_size * proj_stride
                gather_lut = gather_lut[:gather_max:proj_stride].copy()
            else:
                raise ValueError("missing nproj, proj_stride or gather_lut")
        gather_lut = np.asarray(gather_lut, dtype=np.int32)
        nproj = int(gather_lut.size)
        scatter_lut = np.full(nhidden, -1, dtype=np.int32)
        scatter_lut[gather_lut] = np.arange(nproj, dtype=np.int32)
        self.name = name or "SparseProj"
        self.gather_lut, self.scatter_lut = gather_lut, scatter_lut
        self.nhidden, self.nproj = nhidden, nproj
        self._dev = {}

    def _luts(self, device):
        key = (device.type, device.index)
        if key not in self._dev:
            self._dev[key] = (torch.as_tensor(self.gather_lut, device=device), torch.as_tensor(self.scatter_lut, device=device))
        return self._dev[key]

    def gather(self, x):
        assert x.shape[0] == self.nhidden
        g, s = self._luts(x.device)
        return _GatherRows.apply(x.contiguous(), g, s, self.nproj)

    def scatter(self, x):
        assert x.shape[0] == self.nproj
        g, s = self._luts(x.device)
        return _GatherRows.apply(x.contiguous(), s, g, self.nhidden)

    def scatter_add(self, x, y):
        assert x.shape[0] == self.nhidden and y.shape[0] == self.nproj
        g, s = self._luts(x.device)
        return _ScatterAddMul.apply(x.contiguous(), y.contiguous(), g, s, 1)

    def scatter_mul(self, x, y):
        assert x.shape[0] == self.nhidden and y.shape[0] == self.nproj
        g, s = self._luts(x.device)
        return _ScatterAddMul.apply(x.contiguous(), y.contiguous(), g, s, 2)
