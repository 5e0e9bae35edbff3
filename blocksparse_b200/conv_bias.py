"""Conv edge bias and channel-wise linear -- host side of the reference's ConvEdgeBias, conv_edge_bias_init,
deconv_edge_bias_init (blocksparse/conv.py:46-225) and cwise_linear (conv.py:900-998), on torch tensors, calling the
sm_90a kernels of csrc/conv_bias.cuh through bsmm_edge_bias(_grad) and bsmm_cwise_linear(_grad).

ConvEdgeBias gives the output positions of a conv (or deconv) whose receptive field hangs over the padding a learned
gain and bias per output channel; positions that share the same set of padded taps share one (gain, bias) pair. The
table of those patterns is built here in NumPy, once per geometry, and copied to each device on first use.

Two differences from the reference, on purpose:
  * SAME padding uses the dilated filter extent, as TensorFlow's conv does (the reference uses the undilated size,
    conv.py:87-89, so with dilations > 1 its table disagrees with the conv it accompanies). At dilation 1 they agree.
  * VALID padding (no edges) gives shape (0, K) / (K, 0) and a call that returns x; the reference's constructor raises
    AttributeError there.
"""
import numpy as np
import torch

from . import _lib
from .checkers import EdgeBiasCheckers

__all__ = ["ConvEdgeBias", "conv_edge_bias_init", "deconv_edge_bias_init", "cwise_linear"]

_FORMATS = {"NWC": 1, "NHWC": 1, "NDHWC": 1, "NCW": 0, "NCHW": 0, "NCDHW": 0}


def conv_edge_bias_init(y, x, w, strides=None, padding="SAME", data_format="NHWC", dilations=None):
    """ConvEdgeBias for y = conv(x, w): y, x and w are tensors (their .shape is read)."""
    return ConvEdgeBias(list(y.shape), list(x.shape), list(w.shape), strides, padding, data_format, dilations)


def deconv_edge_bias_init(y, x, w, strides=None, padding="SAME", data_format="NHWC", dilations=None):
    """ConvEdgeBias for y = conv_transpose(x, w): x and y swap roles, as in the reference."""
    return ConvEdgeBias(list(x.shape), list(y.shape), list(w.shape), strides, padding, data_format, dilations,
                        deconv=True)


def _expand(dims, pad_val=1):
    return [pad_val] * (3 - len(dims)) + list(dims)


def _fprop_taps(q, X, S, pad, stride, dilate):
    """Input coordinate of each tap of output coordinate q, -1 on the padding (reference fprop_lut, conv.py:1037)."""
    x = q * stride - pad + np.arange(S) * dilate
    return np.where((x >= 0) & (x < X), x, -1)


def _bprop_taps(x, Q, S, pad, stride, dilate):
    """Output coordinate each tap of the deconv's output coordinate x reads, the taps flipped, -1 past the edge and -2
    in a stride hole (reference bprop_lut, conv.py:1045)."""
    q = x - ((S - 1) * dilate - pad) + np.arange(S - 1, -1, -1) * dilate
    return np.where(q % stride != 0, -2, np.where((q >= 0) & (q // stride < Q), q // stride, -1))


def _int_dims(v, what, allow_none_first=False):
    out = []
    for i, d in enumerate(v):
        if d is None and i == 0 and allow_none_first:
            out.append(None)
            continue
        try:
            di = int(d)
        except (TypeError, ValueError):
            raise ValueError("%s must hold ints, got %r" % (what, list(v)))
        if di != d or di < 1:
            raise ValueError("%s must hold positive ints, got %r" % (what, list(v)))
        out.append(di)
    return out


class ConvEdgeBias(EdgeBiasCheckers):
    """Edge gain and bias of a conv output (reference conv.py:55-219).

    y_shape, x_shape: the conv's output and input shapes in data_format (the batch entry may be None); w_shape: the
    filter, spatial dims first then (C, K), in both data formats. strides, dilations: rank-length, in data_format order,
    as TensorFlow gives them. padding: "SAME" or "VALID". deconv: y = conv_transpose(x) with the shapes swapped, as
    deconv_edge_bias_init passes them.

    The tables are copied to a device on the op's first call there, which must not be inside CUDA graph capture (a
    warm-up call before capturing does it).

    Attributes as the reference's: layout (1 channels last, 0 channels first), shape ((edges, K) or (K, edges)),
    edgeBiasDim (edges), edgeBiasMap (the output positions of each edge, ordered by first position), edgeEntries, and
    edgeBiasLut (its int32 table: (offset, count) per edge, then the positions, padded to a multiple of 4)."""

    Cache = dict()

    def __init__(self, y_shape, x_shape, w_shape, strides=None, padding="SAME", data_format="NHWC", dilations=None,
                 deconv=False):
        if data_format not in _FORMATS:
            raise ValueError("data_format must be one of %s, got %r" % (sorted(_FORMATS), data_format))
        if not isinstance(padding, str) or padding.upper() not in ("SAME", "VALID"):
            raise ValueError("padding must be 'SAME' or 'VALID', got %r" % (padding,))
        rank = len(data_format)
        y_shape = _int_dims(y_shape, "y_shape", True)
        x_shape = _int_dims(x_shape, "x_shape", True)
        w_shape = _int_dims(w_shape, "w_shape")
        if len(y_shape) != rank or len(x_shape) != rank or len(w_shape) != rank:
            raise ValueError("%s needs y_shape, x_shape and w_shape of rank %d, got %d, %d and %d" %
                             (data_format, rank, len(y_shape), len(x_shape), len(w_shape)))
        self.layout = _FORMATS[data_format]
        sdim, cdim = (slice(1, -1), -1) if self.layout else (slice(2, None), 1)
        C, K = x_shape[cdim], y_shape[cdim]
        if w_shape[-2:] != [C, K]:
            raise ValueError("w_shape must end in (C, K) = (%d, %d) (spatial dims first), got %r" % (C, K, w_shape))
        MPQ, DHW, TRS = _expand(y_shape[sdim]), _expand(x_shape[sdim]), _expand(w_shape[:-2])
        st = [1, 1, 1] if strides is None else _expand(self._rank_list(strides, rank, "strides")[sdim])
        dl = [1, 1, 1] if dilations is None else _expand(self._rank_list(dilations, rank, "dilations")[sdim])
        if padding.upper() == "VALID":
            pad = [0, 0, 0]
        else:
            # TensorFlow's SAME: the dilated filter extent, the larger half of the padding after the image
            pad = [max((Q - 1) * s + (S - 1) * d + 1 - W, 0) // 2 for S, Q, W, s, d in zip(TRS, MPQ, DHW, st, dl)]
        if deconv:
            taps, MPQ, DHW, K = _bprop_taps, DHW, MPQ, C
        else:
            taps = _fprop_taps
        self.deconv, self.K, self.MPQ = bool(deconv), K, MPQ
        self._in_dims = list((x_shape if deconv else y_shape)[1:])

        key = (tuple(MPQ), tuple(DHW), tuple(TRS), tuple(pad), tuple(st), tuple(dl), bool(deconv))
        entry = ConvEdgeBias.Cache.get(key)
        if entry is None:
            entry = ConvEdgeBias.Cache[key] = self._build(MPQ, DHW, TRS, pad, st, dl, taps)
        self._entry = entry
        self.edgeBiasMap, self.edgeBiasLut, self.edgeEntries, self._pos_edge = \
            entry["map"], entry["lut"], entry["entries"], entry["pos_edge"]
        self.edgeBiasDim = len(self.edgeBiasMap)
        self._max_count = max([len(m) for m in self.edgeBiasMap], default=0)
        self.shape = (self.edgeBiasDim, K) if self.layout else (K, self.edgeBiasDim)

    @staticmethod
    def _rank_list(v, rank, what):
        v = _int_dims(v, what)
        if len(v) != rank:
            raise ValueError("%s must have one entry per dim of the data format (%d), got %r" % (what, rank, v))
        return v

    @staticmethod
    def _build(MPQ, DHW, TRS, pad, st, dl, taps):
        """The edge pattern of each output position: the set of its taps (t, r, s) that fall on the padding in any dim.
        Per dim the taps form few distinct patterns, so the pattern of a position is looked up by its three per-dim
        pattern ids."""
        ids, pats = [], []
        for i in range(3):
            rows = np.array([taps(m, DHW[i], TRS[i], pad[i], st[i], dl[i]) == -1 for m in range(MPQ[i])], bool)
            u, inv = np.unique(rows, axis=0, return_inverse=True)
            ids.append(inv.reshape(-1))
            pats.append(u)
        combo = (ids[0][:, None, None] * len(pats[1]) + ids[1][None, :, None]) * len(pats[2]) + ids[2][None, None, :]
        combo = combo.reshape(-1)
        used, inv = np.unique(combo, return_inverse=True)
        keys = {}
        key_of = np.empty(len(used), np.int64)
        for n, c in enumerate(used):
            a, rest = divmod(int(c), len(pats[1]) * len(pats[2]))
            b, cc = divmod(rest, len(pats[2]))
            pad_tap = pats[0][a][:, None, None] | pats[1][b][None, :, None] | pats[2][cc][None, None, :]
            k = pad_tap.tobytes() if pad_tap.any() else None
            key_of[n] = -1 if k is None else keys.setdefault(k, len(keys))
        key = key_of[inv.reshape(-1)]
        pos_edge = np.full(key.shape, -1, np.int32)
        emap = []
        if len(keys):
            first = np.full(len(keys), key.size, np.int64)
            on = np.nonzero(key >= 0)[0]
            np.minimum.at(first, key[on], on)
            order = np.argsort(first, kind="stable")            # edges ordered by their first position
            rank = np.empty_like(order)
            rank[order] = np.arange(len(order))
            pos_edge[on] = rank[key[on]]
            srt = on[np.argsort(pos_edge[on], kind="stable")]
            counts = np.bincount(pos_edge[on], minlength=len(keys))
            emap = [m.tolist() for m in np.split(srt, np.cumsum(counts)[:-1])]
        entries = sum(len(m) for m in emap)
        head, off = [], 2 * len(emap)
        for m in emap:
            head += [off, len(m)]
            off += len(m)
        data = [p for m in emap for p in m]
        lut = np.array(head + data + [0] * ((-len(data)) % 4), np.int32)
        return {"map": emap, "lut": lut, "entries": entries, "pos_edge": pos_edge, "dev": {}}

    def __getstate__(self):
        s = dict(self.__dict__)
        s["_entry"] = dict(self._entry, dev={})
        return s

    def _tables(self, device):
        """The device copies of pos_edge and the edge table, made from host memory on the first call per device: that
        first call cannot be inside CUDA graph capture (run the op once before capturing, as a warm-up does)."""
        dev = self._entry["dev"]
        d = dev.get(device)
        if d is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("ConvEdgeBias: the first call on %s copies the edge tables to the device, which "
                                 "CUDA graph capture does not allow; call the op once before capturing" % (device,))
            d = dev[device] = (torch.as_tensor(self._pos_edge).to(device), torch.as_tensor(self.edgeBiasLut).to(device))
        return d

    def _check(self, x, params):
        if not torch.is_tensor(x) or not x.is_cuda:
            raise ValueError("ConvEdgeBias: x must be a CUDA tensor (there is no CPU path)")
        _lib.dtype_code(x.dtype)
        if x.dim() != len(self._in_dims) + 1 or list(x.shape[1:]) != self._in_dims:
            raise ValueError("ConvEdgeBias: x must have shape [N] + %s, got %s" % (self._in_dims, list(x.shape)))
        for t, what in params:
            if not torch.is_tensor(t) or not t.is_cuda or t.device != x.device:
                raise ValueError("ConvEdgeBias: %s must be a CUDA tensor on x's device (%s)" % (what, x.device))
            if t.dtype != torch.float32:
                raise ValueError("ConvEdgeBias: %s must be float32, got %s" % (what, t.dtype))
            if tuple(t.shape) != tuple(self.shape):
                raise ValueError("ConvEdgeBias: %s must have shape %s, got %s" % (what, self.shape, tuple(t.shape)))

    def __call__(self, x, g, b, inference=False, bench=0, name=None):
        """y = x * g + b at the edge positions of x (the conv's output; the deconv's for deconv=True), x elsewhere.
        Differentiable in x, g and b; with no edges it returns x itself. inference=True updates x in place over the
        edge positions only (ValueError if x requires grad under grad mode). bench and name are accepted and unused."""
        self._check(x, ((g, "g"), (b, "b")))
        if not self.edgeBiasDim:
            return x
        if inference:
            if torch.is_grad_enabled() and x.requires_grad:
                raise ValueError("ConvEdgeBias: inference=True updates x in place, which needs x not to require grad")
            if not x.is_contiguous():
                raise ValueError("ConvEdgeBias: inference=True needs a contiguous x")
            self._forward(x, g.contiguous(), b.contiguous(), x, True)
            return x
        return _EdgeBiasFunction.apply(x, g, b, self)

    def _forward(self, x, g, b, y, inference):
        N = x.shape[0]
        with torch.cuda.device(x.device):
            pos, lut = self._tables(x.device)
            rc = _lib.load().bsmm_edge_bias(_lib.dtype_code(x.dtype), self.layout, pos.data_ptr(), lut.data_ptr(),
                                            self.edgeBiasDim, self.edgeEntries, x.data_ptr(), g.data_ptr(),
                                            b.data_ptr(), y.data_ptr(), N, int(np.prod(self.MPQ)), self.K,
                                            int(inference), _lib.stream_ptr())
        _lib.check(rc, "bsmm_edge_bias")
        return y

    def _backward(self, dy, x, g):
        N = x.shape[0]
        dx = torch.empty_like(x)
        dg = torch.empty(self.shape, dtype=torch.float32, device=x.device)
        db = torch.empty(self.shape, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            pos, lut = self._tables(x.device)
            lib = _lib.load()
            nbytes = lib.bsmm_edge_bias_grad_workspace_bytes(N, self.edgeBiasDim, self._max_count, self.K)
            ws = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=x.device)
            rc = lib.bsmm_edge_bias_grad(_lib.dtype_code(x.dtype), self.layout, pos.data_ptr(), lut.data_ptr(),
                                         self.edgeBiasDim, self.edgeEntries, self._max_count, dy.data_ptr(),
                                         x.data_ptr(), g.data_ptr(), dx.data_ptr(), dg.data_ptr(), db.data_ptr(),
                                         ws.data_ptr(), N, int(np.prod(self.MPQ)), self.K, _lib.stream_ptr())
        _lib.check(rc, "bsmm_edge_bias_grad")
        return dx, dg, db


class _EdgeBiasFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, g, b, op):
        x, g, b = x.contiguous(), g.contiguous(), b.contiguous()
        y = op._forward(x, g, b, torch.empty_like(x), False)
        ctx.op = op
        ctx.save_for_backward(x, g)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g = ctx.saved_tensors
        dx, dg, db = ctx.op._backward(dy.to(x.dtype).contiguous(), x, g)
        return dx, dg, db, None


def _channel_param(t, C, x, what):
    if not torch.is_tensor(t) or not t.is_cuda or t.device != x.device:
        raise ValueError("cwise_linear: %s must be a CUDA tensor on x's device (%s)" % (what, x.device))
    if t.dtype != torch.float32:
        raise ValueError("cwise_linear: %s must be float32, got %s" % (what, t.dtype))
    if t.numel() != C:
        raise ValueError("cwise_linear: %s must have C = %d elements, got shape %s" % (what, C, tuple(t.shape)))


def cwise_linear(x, gain=None, bias=None, relu=False, bias_first=False, use_tf=False):
    """y = gain * x + bias per channel, or gain * (x + bias) with bias_first (the reference's swap), then relu if
    asked (reference conv.py:906-927). x: rank >= 2, channels on axis 1 (NC, NCW, NCHW, NCDHW), fp32, fp16 or bf16.
    gain, bias: fp32 with C elements each, in any shape; either may be None, not both. Differentiable in x, gain and
    bias; their gradients come back in their shapes, fp32. use_tf=True raises ValueError."""
    if use_tf:
        raise ValueError("cwise_linear: use_tf is a TensorFlow composition; there is none here")
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("cwise_linear needs a CUDA tensor x (there is no CPU path)")
    _lib.dtype_code(x.dtype)
    if x.dim() < 2:
        raise ValueError("cwise_linear: x must have rank >= 2 (channels on axis 1), got shape %s" % (tuple(x.shape),))
    if gain is None and bias is None:
        raise ValueError("cwise_linear: give a gain, a bias or both")
    C = x.shape[1]
    for t, what in ((gain, "gain"), (bias, "bias")):
        if t is not None:
            _channel_param(t, C, x, what)
    return _CwiseLinearFunction.apply(x, gain, bias, bool(relu), bool(bias_first))


def _cw_dims(x):
    N, C = x.shape[0], x.shape[1]
    return N, C, int(np.prod(x.shape[2:])) if x.dim() > 2 else 1


class _CwiseLinearFunction(torch.autograd.Function):
    """CWiseLinear and its gradient (reference conv.py:930-958): saves x when there is a gain, y for relu without
    one, and nothing otherwise."""

    @staticmethod
    def forward(ctx, x, gain, bias, relu, swap):
        x = x.contiguous()
        a = None if gain is None else gain.contiguous()
        b = None if bias is None else bias.contiguous()
        N, C, DHW = _cw_dims(x)
        y = torch.empty_like(x)
        if C > 0 and DHW > 0:
            with torch.cuda.device(x.device):
                rc = _lib.load().bsmm_cwise_linear(_lib.dtype_code(x.dtype), x.data_ptr(), _lib.ptr(a), _lib.ptr(b),
                                                   y.data_ptr(), N, C, DHW, int(relu), int(swap), _lib.stream_ptr())
            _lib.check(rc, "bsmm_cwise_linear")
        ctx.relu, ctx.swap = relu, swap
        ctx.shapes = (None if gain is None else gain.shape, None if bias is None else bias.shape)
        ctx.has = (gain is not None, bias is not None)
        if gain is not None:
            ctx.save_for_backward(x, a, b)
        elif relu:
            ctx.save_for_backward(y, a, b)
        else:
            ctx.save_for_backward(None, a, b)
        return y

    @staticmethod
    def backward(ctx, dy):
        xy, a, b = ctx.saved_tensors
        dx, da, db = _cwise_linear_grad(dy, xy, a, b, ctx.relu, ctx.swap)
        ga, gb = ctx.shapes
        return (dx, None if da is None else da.view(ga), None if db is None else db.view(gb), None, None)


def _cwise_linear_grad(dy, xy, a, b, relu, swap):
    """(dx, da, db) of cwise_linear: xy is x with a gain, y for relu without one, else None; da / db are None where
    a / b are, and dx is dy itself without gain and relu."""
    dy = dy.contiguous()
    if xy is not None:
        dy = dy.to(xy.dtype)
    N, C, DHW = _cw_dims(dy)
    rd = a is not None or relu
    dx = torch.empty_like(dy) if rd else dy
    da = torch.empty(C, dtype=torch.float32, device=dy.device) if a is not None else None
    db = torch.empty(C, dtype=torch.float32, device=dy.device) if b is not None else None
    if C == 0 or DHW == 0:          # no element: the sums are empty, as the forward launched nothing
        for t in (da, db):
            if t is not None:
                t.zero_()
        return dx, da, db
    with torch.cuda.device(dy.device):
        lib = _lib.load()
        nbytes = lib.bsmm_cwise_linear_grad_workspace_bytes(N, C, DHW)
        ws = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=dy.device)
        rc = lib.bsmm_cwise_linear_grad(_lib.dtype_code(dy.dtype), dy.data_ptr(), _lib.ptr(xy), _lib.ptr(a),
                                        _lib.ptr(b), dx.data_ptr() if rd else None, _lib.ptr(da), _lib.ptr(db),
                                        ws.data_ptr(), N, C, DHW, int(relu), int(swap), _lib.stream_ptr())
    _lib.check(rc, "bsmm_cwise_linear_grad")
    return dx, da, db
