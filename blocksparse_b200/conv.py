"""Block-sparse convolution -- host side of the reference's BlocksparseConv / BlocksparseDeconv (blocksparse/conv.py:
228-899), on torch tensors, calling the sm_90a kernels of csrc/conv.cuh through bsmm_conv_xprop / bsmm_conv_updat /
bsmm_conv_l2_normalize(_grad).

A layout BCK lists blocks as (C channel list, K channel list) pairs of any sizes, overlapping or not, in any order. Each
block is a dense conv from its C channels to its K channels; outputs that several blocks write are their sum. The
spatial tables (which input position each output position reads through each filter tap) and the per-block tables are
built here in NumPy, once per object, and copied to each device on first use.

The deconv is the conv with C and K, DHW and MPQ swapped, its forward the conv's bprop: the same three kernels run with
the roles swapped, as in the reference.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .checkers import ConvCheckers

__all__ = ["BlocksparseConv", "BlocksparseDeconv"]

# the reference's conv module also holds these; they live in conv_bias.py and are reachable here too
from .conv_bias import ConvEdgeBias, conv_edge_bias_init, cwise_linear, deconv_edge_bias_init  # noqa: E402,F401


# ---- spatial helpers (reference conv.py:1003-1061) ---------------------------------------------------------------------
def ceil_div(a, b):
    return -(-a // b)


def dilation_size(S, dilate):
    return S * dilate - dilate + 1


def out_dim(S, W, padding, stride, dilate):
    return ceil_div(W - dilation_size(S, dilate) + 1 + 2 * padding, stride)


def in_dim(S, W, padding, stride, dilate):
    # inverting ceil_div is ambiguous: the reference assumes the numerator was a multiple of the stride
    return W * stride + S - 2 * padding - (S & 1)


def expand_dims(dim, pad_val=1):
    return [pad_val] * (3 - len(dim)) + list(dim)


def get_padding(padding, TRS, dilates):
    if isinstance(padding, str):
        if padding.upper() == "SAME":
            return [dilation_size(*dims) // 2 for dims in zip(TRS, dilates)]
        if padding.upper() == "VALID":
            return [0, 0, 0]
        raise ValueError("padding must be 'SAME', 'VALID' or a sequence of 1 to 3 ints, got %r" % (padding,))
    return expand_dims(padding, 0)


def fprop_lut(TRS, DHW, MPQ, padding, strides, dilates):
    """int32 [M*P*Q][T*R*S]: the input position (d*H*W + h*W + w) output position (m, p, q) reads through tap (t, r, s),
    or -1 where the tap falls on padding (reference fprop_lut, conv.py:1037-1043, combined over the three dims)."""
    idx, ok = [], []
    for S, X, Q, pad, st, dl in zip(TRS, DHW, MPQ, padding, strides, dilates):
        x = np.arange(Q)[:, None] * st - pad + np.arange(S)[None, :] * dl
        idx.append(x)
        ok.append((x >= 0) & (x < X))
    return _combine(idx, ok, DHW, MPQ, TRS)


def bprop_lut(TRS, DHW, MPQ, padding, strides, dilates):
    """int32 [D*H*W][T*R*S]: the output position whose tap (t, r, s) reads input position (d, h, w), or -1 where none
    does -- past the edge or in a stride hole (reference bprop_lut, conv.py:1045-1061, which lists the taps flipped and
    marks holes -2; the kernels need neither, so the taps keep the filter's order)."""
    idx, ok = [], []
    for S, X, Q, pad, st, dl in zip(TRS, DHW, MPQ, padding, strides, dilates):
        q = np.arange(X)[:, None] + pad - np.arange(S)[None, :] * dl
        idx.append(q // st)
        ok.append((q % st == 0) & (q >= 0) & (q // st < Q))
    return _combine(idx, ok, MPQ, DHW, TRS)


def _combine(idx, ok, src, dst, TRS):
    (d, h, w), (od, oh, ow) = idx, ok
    pos = (d[:, None, None, :, None, None] * (src[1] * src[2]) + h[None, :, None, None, :, None] * src[2] +
           w[None, None, :, None, None, :])
    valid = od[:, None, None, :, None, None] & oh[None, :, None, None, :, None] & ow[None, None, :, None, None, :]
    n_dst, trs = int(np.prod(dst)), int(np.prod(TRS))
    return np.ascontiguousarray(np.where(valid, pos, -1).reshape(n_dst, trs).astype(np.int32))


def _passes(lists):
    """Block order grouped into passes in which no two blocks share a channel: block b goes one pass after the latest
    earlier block it overlaps, so every channel receives its blocks in block order. Returns (order, offsets)."""
    last, pas = {}, []
    for ch in lists:
        p = max([last[c] + 1 for c in ch if c in last], default=0)
        pas.append(p)
        for c in ch:
            last[c] = p
    order = sorted(range(len(lists)), key=lambda b: (pas[b], b))
    offsets = np.searchsorted(np.array([pas[b] for b in order]), np.arange(max(pas) + 2)).tolist()
    return order, offsets


def _int_list(v, what):
    try:
        out = [int(c) for c in v]
    except TypeError:
        raise ValueError("%s must be a sequence of channel ids, got %r" % (what, v))
    if not out or any(c < 0 for c in out) or len(set(out)) != len(out):
        raise ValueError("%s must be a non-empty list of distinct non-negative channel ids" % what)
    return out


def _dims(v, what, lo=1):
    if not isinstance(v, (list, tuple)) or not 1 <= len(v) <= 3 or any(int(x) != x or x < lo for x in v):
        raise ValueError("%s must be 1 to 3 ints >= %d, got %r" % (what, lo, v))
    return [int(x) for x in v]


class BlocksparseConv(ConvCheckers):
    """
    BCK: ((c0, c1, ...), (k0, k1, ...)) per block -- its input (C) and output (K) channels. Blocks may have any
         rectangular size, uniform or not, may overlap in C and / or K and list channels in any order; together they
         must cover 0..C-1 and 0..K-1 (ValueError otherwise: the reference assumes it, conv.py:334).
    TRS: (T,R,S) or (R,S) or (S,)          filter spatial size
    DHW: (D,H,W) or (H,W) or (W,)          input image spatial size
    MPQ: (M,P,Q) or (P,Q) or (Q,) or None  output image spatial size (default from out_dim)
    strides, dilates: 1 to 3 ints; padding: "SAME", "VALID" or 1 to 3 ints. debug is accepted and has no effect.
    """

    def __init__(self, BCK, TRS, DHW, MPQ=None, strides=(1, 1, 1), dilates=(1, 1, 1), padding="SAME", debug=False,
                 deconv=False):
        self.userTRS = _dims(TRS, "TRS")
        if len(_dims(DHW, "DHW")) != len(self.userTRS):
            raise ValueError("TRS and DHW must have the same number of dims, got %r and %r" % (TRS, DHW))
        TRS, DHW = expand_dims(self.userTRS), expand_dims(_dims(DHW, "DHW"))
        strides, dilates = expand_dims(_dims(strides, "strides")), expand_dims(_dims(dilates, "dilates"))
        if not isinstance(padding, str):
            _dims(padding, "padding", lo=0)
        padding = get_padding(padding, TRS, dilates)
        MPQ = [out_dim(*d) for d in zip(TRS, DHW, padding, strides, dilates)] if MPQ is None else \
            expand_dims(_dims(MPQ, "MPQ"))
        if min(MPQ) < 1:
            raise ValueError("the output image would be empty: MPQ = %s" % (MPQ,))
        try:
            BCK = [[_int_list(c, "a block's C list"), _int_list(k, "a block's K list")] for c, k in BCK]
        except (TypeError, ValueError) as e:
            raise ValueError("BCK must be a non-empty list of (C list, K list) pairs: %s" % e)
        if not BCK:
            raise ValueError("BCK must list at least one block")
        trs = int(np.prod(TRS))
        cs = [c for lc, _ in BCK for c in lc]
        ks = [k for _, lk in BCK for k in lk]
        cset, kset = set(cs), set(ks)
        self.C, self.K = len(cset), len(kset)
        for name, s, n in (("C", cset, self.C), ("K", kset, self.K)):
            if max(s) != n - 1:
                raise ValueError("the blocks' %s lists cover %d channels but not 0..%d (missing %s)" %
                                 (name, n, n - 1, sorted(set(range(max(s) + 1)) - s)[:8]))
        self.overlapC, self.overlapK = len(cs) != self.C, len(ks) != self.K
        sizes = [(len(lk), len(lc)) for lc, lk in BCK]
        self.fixed_block_size = len(set(sizes)) == 1
        self.sizeF = sum(k * c for k, c in sizes) * trs
        if self.sizeF >= 2 ** 31:
            raise ValueError("the filter has %d elements; at most 2^31 - 1 are supported" % self.sizeF)
        self.BCK, self.TRS, self.DHW, self.MPQ = BCK, TRS, DHW, MPQ
        self.strides, self.dilates, self.padding = strides, dilates, padding
        self.trs, self.blocks, self.debug, self.deconv = trs, len(BCK), bool(debug), bool(deconv)
        self.flops = self.sizeF * int(np.prod(MPQ)) * 2          # per image of the minibatch, as in the reference

        # spatial tables, [positions][trs]
        self._lut_f = fprop_lut(TRS, DHW, MPQ, padding, strides, dilates)
        self._lut_b = bprop_lut(TRS, DHW, MPQ, padding, strides, dilates)
        # channel lists and per-block records (csrc/conv.cuh ConvBlk)
        ch, fp, bp, f_off = [], [], [], 0
        for lc, lk in BCK:
            c_off, k_off = len(ch), len(ch) + len(lc)
            ch += lc + lk
            fp.append([len(lk), len(lc), k_off, c_off, f_off, len(lc) * trs, trs, 0])
            bp.append([len(lc), len(lk), c_off, k_off, f_off, trs, len(lc) * trs, 0])
            f_off += len(lk) * len(lc) * trs
        self._ch = np.array(ch, np.int32)
        fo, self._f_pass = _passes([lk for _, lk in BCK])
        bo, self._b_pass = _passes([lc for lc, _ in BCK])
        self._f_blk = np.array([fp[b] for b in fo], np.int32)
        self._b_blk = np.array([bp[b] for b in bo], np.int32)
        self._u_blk = np.array(fp, np.int32)
        self._maxC, self._maxK = max(c for _, c in sizes), max(k for k, _ in sizes)
        # l2 rows (base, outer, stride): KCTRS per output channel; the deconv normalises its CKTRS per input channel
        rows, f_off = [], 0
        for kb, cb in sizes:
            if deconv:
                rows += [[f_off + c * trs, kb, cb * trs, 0] for c in range(cb)]
            else:
                rows += [[f_off + k * cb * trs, cb, trs, 0] for k in range(kb)]
            f_off += kb * cb * trs
        self._norm = np.array(rows, np.int32)
        self.normSize = len(rows)
        self._dev = {}

    def __getstate__(self):
        s = dict(self.__dict__)
        s["_dev"] = {}
        return s

    # ---- shapes (conv.py:490-499) ----
    def i_shape(self, N): return [N, self.C] + self.DHW

    def o_shape(self, N): return [N, self.K] + self.MPQ

    def f_shape(self, block=None):
        if block is None:
            if self.fixed_block_size:
                lutC, lutK = self.BCK[0]
                return [self.blocks, len(lutK), len(lutC)] + self.userTRS
            return [self.sizeF]
        lutC, lutK = self.BCK[block]
        return [len(lutK), len(lutC)] + self.userTRS

    def collapse_filter(self, F, dtype=None):
        """The per-block filters F concatenated into one flat [sizeF] array (conv.py:523-529)."""
        flat = np.empty(self.sizeF, dtype=dtype)
        off = 0
        for f in F:
            f = np.asarray(f)
            flat[off:off + f.size] = f.reshape(f.size).astype(dtype)
            off += f.size
        return flat

    # ---- device tables ----
    def _tables(self, device):
        d = self._dev.get(device)
        if d is None:
            t = lambda a: torch.as_tensor(a).to(device)
            d = self._dev[device] = {"ch": t(self._ch), "lut_f": t(self._lut_f), "lut_b": t(self._lut_b),
                                     "f_blk": t(self._f_blk), "b_blk": t(self._b_blk), "u_blk": t(self._u_blk),
                                     "norm": t(self._norm),
                                     "f_pass": (ctypes.c_int * len(self._f_pass))(*self._f_pass),
                                     "b_pass": (ctypes.c_int * len(self._b_pass))(*self._b_pass)}
        return d

    # ---- raw ops, in the conv's own terms (the deconv swaps them) ----
    def _xprop(self, f, x, bprop, flags=0):
        """fprop: [N, C, DHW] -> [N, K, MPQ]; bprop: [N, K, MPQ] -> [N, C, DHW]; the output takes x's dtype."""
        N = x.shape[0]
        DHW, MPQ = int(np.prod(self.DHW)), int(np.prod(self.MPQ))
        C_in, P_in, C_out, P_out = (self.K, MPQ, self.C, DHW) if bprop else (self.C, DHW, self.K, MPQ)
        y = torch.empty((N, C_out, P_out), dtype=x.dtype, device=x.device)
        if N == 0:
            return y
        with torch.cuda.device(x.device):
            d = self._tables(x.device)
            offs = d["b_pass" if bprop else "f_pass"]
            passes = len(offs) - 1
            acc = torch.empty(N * C_out * P_out, dtype=torch.float32, device=x.device) \
                if passes > 1 and x.dtype != torch.float32 else None
            rc = _lib.load().bsmm_conv_xprop(
                _lib.dtype_code(x.dtype), _lib.dtype_code(f.dtype), d["b_blk" if bprop else "f_blk"].data_ptr(), offs,
                passes, self._maxC if bprop else self._maxK, d["ch"].data_ptr(), d["lut_b" if bprop else "lut_f"].data_ptr(),
                self.trs, x.data_ptr(), f.data_ptr(), y.data_ptr(), _lib.ptr(acc), N, C_in, P_in, C_out, P_out, flags,
                _lib.stream_ptr())
        _lib.check(rc, "bsmm_conv_xprop")
        return y

    def _updat(self, e, x, f_dtype, flags=0):
        """dF [sizeF] in f_dtype from e [N, K, MPQ] and x [N, C, DHW]."""
        N = x.shape[0]
        DHW, MPQ = int(np.prod(self.DHW)), int(np.prod(self.MPQ))
        df = torch.empty(self.sizeF, dtype=f_dtype, device=x.device)
        with torch.cuda.device(x.device):
            d = self._tables(x.device)
            lib = _lib.load()
            nbytes = lib.bsmm_conv_updat_workspace_bytes(N * MPQ, self.sizeF)
            ws = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=x.device)
            rc = lib.bsmm_conv_updat(
                _lib.dtype_code(e.dtype), _lib.dtype_code(x.dtype), _lib.dtype_code(f_dtype), d["u_blk"].data_ptr(),
                self.blocks, self._maxK, self._maxC, d["ch"].data_ptr(), d["lut_f"].data_ptr(), self.trs, e.data_ptr(),
                x.data_ptr(), df.data_ptr(), ws.data_ptr(), N, self.C, DHW, self.K, MPQ, self.sizeF, flags,
                _lib.stream_ptr())
        _lib.check(rc, "bsmm_conv_updat")
        return df

    # ---- validation ----
    def _in_dims(self):
        """(channels, spatial dims) of the op's input: the conv reads [N, C, DHW], the deconv [N, K, MPQ]."""
        return (self.K, self.MPQ) if self.deconv else (self.C, self.DHW)

    def _out_dims(self):
        return (self.C, self.DHW) if self.deconv else (self.K, self.MPQ)

    def _check(self, F, I):
        for t, what in ((F, "F"), (I, "I")):
            if not torch.is_tensor(t) or not t.is_cuda:
                raise ValueError("%s: %s must be a CUDA tensor (there is no CPU path)" % (type(self).__name__, what))
            _lib.dtype_code(t.dtype)
        if F.device != I.device:
            raise ValueError("F lives on %s, I on %s" % (F.device, I.device))
        if {F.dtype, I.dtype} == {torch.float16, torch.bfloat16}:
            raise ValueError("F and I mix fp16 with bf16")
        if list(F.shape) not in (self.f_shape(), [self.sizeF]):
            raise ValueError("F must have shape %s or [%d], got %s" % (self.f_shape(), self.sizeF, list(F.shape)))
        C, sp = self._in_dims()
        nd = len(self.userTRS)
        if I.dim() < 2 or list(I.shape[1:]) not in ([C] + sp, [C] + sp[3 - nd:]):
            raise ValueError("I must have shape %s or %s, got %s" % (["N", C] + sp, ["N", C] + sp[3 - nd:],
                                                                     list(I.shape)))

    def __call__(self, F, I):
        """O = conv(I, F): I [N, C, DHW] (or [N, C] + the user's spatial dims) and F as f_shape() or [sizeF]; O has
        o_shape(N) (or I's rank) and I's dtype. Differentiable in F and I: dI comes back in dO's dtype, dF in F's."""
        self._check(F, I)
        return _ConvFunction.apply(F, I, self)

    def l2_normalize(self, F, gain=None, epsilon=1e-12, dtype=None):
        """y = gain * F / sqrt(max(sum(F^2), epsilon)) per output channel of each block, over (C_b, TRS) (KCTRS); for
        the deconv per input channel, over (K_b, TRS) (CKTRS) (conv.py:515-521, 817-827). Differentiable in F and
        gain. gain: normSize entries, one per normalised row in block order (read as fp32); a gain where those rows
        overlap (K for the conv, C for the deconv) raises ValueError. dtype: output dtype, F's (default) or fp32."""
        if not torch.is_tensor(F) or not F.is_cuda:
            raise ValueError("l2_normalize needs a CUDA tensor F (there is no CPU path)")
        _lib.dtype_code(F.dtype)
        if list(F.shape) not in (self.f_shape(), [self.sizeF]):
            raise ValueError("F must have shape %s or [%d], got %s" % (self.f_shape(), self.sizeF, list(F.shape)))
        out_dtype = F.dtype if dtype is None else dtype
        if out_dtype not in (F.dtype, torch.float32):
            raise ValueError("l2_normalize: dtype must be F's dtype or float32, got %s" % (out_dtype,))
        if gain is not None:
            if self.overlapC if self.deconv else self.overlapK:
                raise ValueError("l2_normalize: no gain for blocks whose %s channels overlap" %
                                 ("input" if self.deconv else "output"))
            if not torch.is_tensor(gain) or not gain.is_cuda or gain.device != F.device:
                raise ValueError("l2_normalize: gain must be a CUDA tensor on F's device")
            if gain.numel() != self.normSize:
                raise ValueError("l2_normalize: gain has %d entries, needs %d" % (gain.numel(), self.normSize))
        return _ConvL2Function.apply(F, gain, self, float(epsilon), out_dtype)


class _ConvFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, F, I, conv):
        N = I.shape[0]
        C, sp = conv._in_dims()
        x = I.contiguous().view(N, C, int(np.prod(sp)))
        f = F.contiguous()
        y = conv._xprop(f, x, bprop=conv.deconv)
        ctx.conv, ctx.i_shape = conv, I.shape
        ctx.save_for_backward(f, x)
        K, osp = conv._out_dims()
        return y.view([N, K] + osp[3 - (I.dim() - 2):])

    @staticmethod
    def backward(ctx, dy):
        conv = ctx.conv
        f, x = ctx.saved_tensors
        N = x.shape[0]
        K, osp = conv._out_dims()
        e = dy.contiguous().view(N, K, int(np.prod(osp)))
        dI = dF = None
        if ctx.needs_input_grad[1]:
            dI = conv._xprop(f, e, bprop=not conv.deconv).view(ctx.i_shape)
        if ctx.needs_input_grad[0]:
            dF = (conv._updat(x, e, f.dtype) if conv.deconv else conv._updat(e, x, f.dtype)).view(f.shape)
        return dF, dI, None


class _ConvL2Function(torch.autograd.Function):
    """L2NormalizeKCTRS / L2NormalizeCKTRS, their Gain variants and gradients (reference conv.py:704-722, 870-898)."""

    @staticmethod
    def forward(ctx, F, gain, conv, epsilon, out_dtype):
        W = F.contiguous()
        g = None if gain is None else gain.to(torch.float32).contiguous()
        y = torch.empty(W.shape, dtype=out_dtype, device=W.device)
        ss = torch.empty(conv.normSize, dtype=torch.float32, device=W.device)
        with torch.cuda.device(W.device):
            d = conv._tables(W.device)
            rc = _lib.load().bsmm_conv_l2_normalize(_lib.dtype_code(W.dtype), _lib.dtype_code(out_dtype),
                                                    d["norm"].data_ptr(), conv.normSize, conv.trs, W.data_ptr(),
                                                    _lib.ptr(g), y.data_ptr(), ss.data_ptr(), epsilon, _lib.stream_ptr())
        _lib.check(rc, "bsmm_conv_l2_normalize")
        ctx.conv, ctx.epsilon, ctx.gain_dtype = conv, epsilon, None if gain is None else gain.dtype
        ctx.gain_shape = None if gain is None else gain.shape
        ctx.save_for_backward(W, g, ss)
        return y

    @staticmethod
    def backward(ctx, dy):
        W, g, ss = ctx.saved_tensors
        conv = ctx.conv
        dy = dy.contiguous()
        if dy.dtype not in (W.dtype, torch.float32):
            dy = dy.to(W.dtype)
        dx = torch.empty_like(W)
        dg = torch.empty(conv.normSize, dtype=torch.float32, device=W.device) if g is not None else None
        with torch.cuda.device(W.device):
            d = conv._tables(W.device)
            rc = _lib.load().bsmm_conv_l2_normalize_grad(_lib.dtype_code(W.dtype), _lib.dtype_code(dy.dtype),
                                                         d["norm"].data_ptr(), conv.normSize, conv.trs, dy.data_ptr(),
                                                         W.data_ptr(), _lib.ptr(g), ss.data_ptr(), dx.data_ptr(),
                                                         _lib.ptr(dg), ctx.epsilon, _lib.stream_ptr())
        _lib.check(rc, "bsmm_conv_l2_normalize_grad")
        return dx, (dg.to(ctx.gain_dtype).view(ctx.gain_shape) if dg is not None else None), None, None, None


class BlocksparseDeconv(BlocksparseConv):
    """The transposed conv of BlocksparseConv (conv.py:728-899): BCK lists (C list, K list) as for the conv; I is
    [N, C, DHW] of the user's C and DHW, and the output [N, K, MPQ] with MPQ from in_dim unless given. Internally the
    object is the conv with C <=> K and DHW <=> MPQ swapped, as in the reference, so its C, K, DHW and MPQ attributes,
    f_shape (CKTRS) and tables are the swapped conv's."""

    def __init__(self, BCK, TRS, DHW, MPQ=None, strides=(1, 1, 1), dilates=(1, 1, 1), padding="SAME", debug=False):
        try:
            BKC = [[lk, lc] for lc, lk in BCK]
        except (TypeError, ValueError):
            raise ValueError("BCK must be a non-empty list of (C list, K list) pairs")
        if MPQ is None:
            TRS3, DHW3 = expand_dims(_dims(TRS, "TRS")), expand_dims(_dims(DHW, "DHW"))
            st3, dl3 = expand_dims(_dims(strides, "strides")), expand_dims(_dims(dilates, "dilates"))
            padding = get_padding(padding, TRS3, dl3)
            MPQ = [in_dim(*d) for d in zip(TRS3, DHW3, padding, st3, dl3)][3 - len(TRS):]
            if min(MPQ) < 1:
                raise ValueError("the output image would be empty: MPQ = %s" % (MPQ,))
            padding = padding[3 - len(TRS):]
        super(BlocksparseDeconv, self).__init__(BKC, TRS, MPQ, DHW, strides, dilates, padding, debug, True)

    def i_shape(self, N): return [N, self.K] + self.MPQ

    def o_shape(self, N): return [N, self.C] + self.DHW
