"""LSTM layers -- host side of the reference's FusedBasicLSTMCell and grouped_lstm (blocksparse/lstm.py:120-199), on
torch tensors. The step product [x_t, h_{t-1}] . kernel runs on this project's wgmma xprop kernel (a BlocksparseMatMul
with a dense layout, feature_axis=1); the gates run on csrc/lstm.cuh, with the layer norm fused in front of them
through bsmm_lstm_ln_gates(_grad).

grouped_lstm's backward is one sequence-level autograd function (BPTT): per step the gates gradient (layer norm
included) and the product's bprop, and after the loop one dw_matmul_large_n over every step's saved rows for the
kernel's gradient -- the work the reference's group_lstm_grads graph rewrite does with its default group_size=None.

Torch has no variable scopes, so the kernel, bias and gain are passed in: the reference's scope, reuse and lstm_id are
not carried. The kernel's gradient is formed in fp32 and returned in the kernel's dtype.
"""
import math
import numbers

import numpy as np
import torch

from . import _lib
from .elementwise import ADD_OP, _cast, _fwd
from .ewops import ACT_NONE, _br_bwd
from .lstm import fused_lstm_gates
from .matmul import BlocksparseMatMul, dw_matmul_large_n

__all__ = ["grouped_lstm", "FusedBasicLSTMCell"]

_BS = 32             # block size of the dense-layout product; operands are zero-padded to multiples of it
_LN_EPS = 1e-6       # layer_norm's default epsilon, which the reference's grouped_lstm uses
_FLOATS = (torch.float32, torch.float16, torch.bfloat16)


def _dt(t):
    return _lib.dtype_code(t.dtype)


class _StepProduct(object):
    """z (N, Kp) = [x, h] (N, Cp) . kernel for a (C, K4) kernel, C and K4 padded up to Cp, Kp, multiples of _BS, on a
    fully dense BlocksparseMatMul. One instance per (C, K4), shared by every call."""

    _cache = {}

    @classmethod
    def get(cls, C, K4):
        p = cls._cache.get((C, K4))
        if p is None:
            p = cls._cache[(C, K4)] = cls(C, K4)
        return p

    def __init__(self, C, K4):
        self.C, self.K4 = C, K4
        self.Cp, self.Kp = -(-C // _BS) * _BS, -(-K4 // _BS) * _BS
        self.bsmm = BlocksparseMatMul(np.ones((self.Cp // _BS, self.Kp // _BS), np.int32), block_size=_BS,
                                      feature_axis=1)
        self._coords = {}

    def weights(self, kernel, dtype):
        """The kernel cast to dtype (float_cast's kernel), zero-padded and cut into blocks in block_coord order."""
        key = (kernel.device.type, kernel.device.index)
        if key not in self._coords:
            lut = torch.as_tensor(self.bsmm.updat_lut.astype(np.int64), device=kernel.device)
            self._coords[key] = (lut[:, 0], lut[:, 1])
        cs, ks = self._coords[key]
        k = kernel.detach().contiguous()
        k = k if k.dtype == dtype else _cast(k, dtype)
        if (self.Cp, self.Kp) != (self.C, self.K4):
            wp = torch.zeros((self.Cp, self.Kp), dtype=dtype, device=k.device)
            wp[:self.C, :self.K4] = k
            k = wp
        return k.view(self.Cp // _BS, _BS, self.Kp // _BS, _BS).permute(0, 2, 1, 3)[cs, ks]

    def fprop(self, xh, w):
        return self.bsmm.fprop(xh, w)

    def bprop(self, dz, w):
        return self.bsmm.bprop(dz, w)

    def kernel_grad(self, xh, dz, kernel):
        """dW (C, K4) in kernel's dtype: one dw_matmul_large_n (fp32) over the rows of xh (.., Cp) and dz (.., Kp)."""
        x = xh[..., :self.C].reshape(-1, self.C)
        e = dz[..., :self.K4].reshape(-1, self.K4)
        dw = dw_matmul_large_n(x, e)
        return dw if kernel.dtype == torch.float32 else _cast(dw, kernel.dtype)


def _concat(prod, x, h):
    """[x, h] zero-padded to (N, Cp)."""
    xh = x.new_zeros((x.shape[0], prod.Cp))
    xh[:, :x.shape[1]] = x
    xh[:, x.shape[1]:prod.C] = h
    return xh


class _ProductFunction(torch.autograd.Function):
    """z (N, 4W) = [x, h] . kernel, differentiable in x, h and kernel (FusedBasicLSTMCell's product)."""

    @staticmethod
    def forward(ctx, x, h, kernel, prod):
        with torch.cuda.device(x.device):
            xh = _concat(prod, x, h)
            w = prod.weights(kernel, x.dtype)
            z = prod.fprop(xh, w)
        ctx.prod, ctx.In = prod, x.shape[1]
        ctx.save_for_backward(xh, w, kernel)
        return z if prod.Kp == prod.K4 else z[:, :prod.K4].contiguous()

    @staticmethod
    def backward(ctx, dz):
        xh, w, kernel = ctx.saved_tensors
        prod, In = ctx.prod, ctx.In
        with torch.cuda.device(xh.device):
            dz = dz.to(xh.dtype)
            if prod.Kp != prod.K4:
                dzp = dz.new_zeros((dz.shape[0], prod.Kp))
                dzp[:, :prod.K4] = dz
            else:
                dzp = dz.contiguous()
            dxh = prod.bprop(dzp, w) if ctx.needs_input_grad[0] or ctx.needs_input_grad[1] else None
            dw = prod.kernel_grad(xh, dzp, kernel) if ctx.needs_input_grad[2] else None
        dx = dxh[:, :In] if dxh is not None else None
        dh = dxh[:, In:prod.C] if dxh is not None else None
        return dx, dh, dw, None


# ---- grouped_lstm -----------------------------------------------------------------------------------------------------
def _gate_ptrs(t, W):
    p, es = t.data_ptr(), t.element_size()
    return [p + j * W * es for j in range(4)]


def _add(a, b):
    """a + b rounded once; None stands for zero."""
    if a is None:
        return b
    if b is None:
        return a
    return _fwd(a, ADD_OP, b)


class _GroupedLstmFunction(torch.autograd.Function):
    """Forward: T steps of [x_t, h_{t-1}] . kernel then the (layer norm +) gates; saves every step's product operands
    and z, c_{t-1} and, with layernorm, the fp32 statistics. Backward: BPTT, then one dw_matmul_large_n."""

    @staticmethod
    def forward(ctx, layernorm, x, c0, h0, kernel, bias, gain):
        N, T, In = x.shape
        W = c0.shape[1]
        prod = _StepProduct.get(In + W, 4 * W)
        lib = _lib.load()
        dt = _dt(x)
        out = x.new_empty((N, T, W))
        cT, hT = torch.empty_like(c0), torch.empty_like(h0)
        xs = x.new_zeros((T, N, prod.Cp))
        cs = x.new_empty((T, N, W))
        stats = torch.empty((2, T, N, 4), dtype=torch.float32, device=x.device)
        zs = []
        w = None
        if N:
            xs[:, :, :In] = x.transpose(0, 1)
            cs[0] = c0
            w = prod.weights(kernel, x.dtype)
        h = h0
        for t in range(T if N else 0):
            xs[t, :, In:prod.C] = h
            z = prod.fprop(xs[t], w)
            zs.append(z)
            c_next = cs[t + 1] if t + 1 < T else cT
            h = hT if t + 1 == T else torch.empty_like(h0)
            if layernorm:
                rc = lib.bsmm_lstm_ln_gates(dt, _dt(gain), cs[t].data_ptr(), z.data_ptr(), prod.Kp, gain.data_ptr(),
                                            bias.data_ptr(), c_next.data_ptr(), h.data_ptr(), stats[0, t].data_ptr(),
                                            stats[1, t].data_ptr(), N, W, _LN_EPS, 1.0, _lib.stream_ptr())
                _lib.check(rc, "bsmm_lstm_ln_gates")
            else:
                rc = lib.bsmm_lstm_gates(dt, _dt(bias), cs[t].data_ptr(), *_gate_ptrs(z, W), prod.Kp, bias.data_ptr(),
                                         c_next.data_ptr(), h.data_ptr(), N, W, 1.0, _lib.stream_ptr())
                _lib.check(rc, "bsmm_lstm_gates")
            out[:, t] = h
        ctx.layernorm, ctx.prod, ctx.shape, ctx.zs = layernorm, prod, (N, T, In, W), zs
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(xs, cs, stats, w, kernel, bias, gain)
        return out, cT, hT

    @staticmethod
    def backward(ctx, g_out, g_cT, g_hT):
        xs, cs, stats, w, kernel, bias, gain = ctx.saved_tensors
        prod, layernorm, zs = ctx.prod, ctx.layernorm, ctx.zs
        N, T, In, W = ctx.shape
        K4, Kp = 4 * W, prod.Kp
        dtype = xs.dtype
        need_x, need_c, need_h, need_k, need_b, need_g = ctx.needs_input_grad[1:7]
        if N == 0:
            zeros = [None, xs.new_zeros((0, T, In)), cs.new_zeros((0, W)), cs.new_zeros((0, W)),
                     torch.zeros_like(kernel), torch.zeros_like(bias), None if gain is None else torch.zeros_like(gain)]
            return tuple(zeros)
        lib = _lib.load()
        dt = _dt(xs)
        go = None if g_out is None else g_out.to(dtype).transpose(0, 1).contiguous()     # (T, N, W)
        dc = None if g_cT is None else g_cT.to(dtype).contiguous()
        dh = None if g_hT is None else g_hT.to(dtype).contiguous()
        dzs = xs.new_zeros((T, N, Kp)) if Kp != K4 else xs.new_empty((T, N, Kp))
        dx = xs.new_empty((N, T, In))
        ws = None
        if layernorm:
            ws = torch.empty(lib.bsmm_lstm_ln_gates_workspace_bytes(N, W) // 4, dtype=torch.float32, device=xs.device)
        for t in range(T - 1, -1, -1):
            eh = _add(dh, None if go is None else go[t])
            dc_prev = torch.empty((N, W), dtype=dtype, device=xs.device)
            if layernorm:
                rc = lib.bsmm_lstm_ln_gates_grad(dt, _dt(gain), cs[t].data_ptr(), zs[t].data_ptr(), Kp, gain.data_ptr(),
                                                 bias.data_ptr(), stats[0, t].data_ptr(), stats[1, t].data_ptr(),
                                                 _lib.ptr(dc), _lib.ptr(eh), dc_prev.data_ptr(), dzs[t].data_ptr(),
                                                 ws.data_ptr(), int(t != T - 1), N, W, 1.0, _lib.stream_ptr())
                _lib.check(rc, "bsmm_lstm_ln_gates_grad")
            else:
                rc = lib.bsmm_lstm_gates_grad(dt, _dt(bias), cs[t].data_ptr(), *_gate_ptrs(zs[t], W), Kp,
                                              bias.data_ptr(), _lib.ptr(dc), _lib.ptr(eh), dc_prev.data_ptr(),
                                              *_gate_ptrs(dzs[t], W), N, W, 1.0, _lib.stream_ptr())
                _lib.check(rc, "bsmm_lstm_gates_grad")
            dxh = prod.bprop(dzs[t], w)
            dx[:, t] = dxh[:, :In]
            dh = dxh[:, In:prod.C].contiguous()
            dc = dc_prev
        dk = prod.kernel_grad(xs, dzs, kernel) if need_k else None
        db = dg = None
        if layernorm and (need_b or need_g):
            dg, db = torch.empty_like(gain), torch.empty_like(bias)
            rc = lib.bsmm_lstm_ln_gates_grad_reduce(_dt(gain), ws.data_ptr(), N, W, dg.data_ptr(), db.data_ptr(),
                                                    _lib.stream_ptr())
            _lib.check(rc, "bsmm_lstm_ln_gates_grad_reduce")
        elif not layernorm and need_b:
            e = dzs[..., :K4].reshape(T * N, K4).contiguous()
            db = _br_bwd(e, None, bias, 1, T * N, K4, ACT_NONE)[1]
        return (None, dx if need_x else None, dc if need_c else None, dh if need_h else None, dk,
                db if need_b else None, dg if need_g else None)


def _check_tensor(t, what, ref=None):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (there is no CPU path)" % what)
    if t.dtype not in _FLOATS:
        raise ValueError("%s: unsupported dtype %s (float32, float16, bfloat16 only)" % (what, t.dtype))
    if ref is not None and t.device != ref.device:
        raise ValueError("%s lives on %s, the inputs on %s" % (what, t.device, ref.device))
    return t


def _check_int(v, what):
    if not isinstance(v, numbers.Integral) or isinstance(v, bool) or v < 1:
        raise ValueError("%s must be a positive integer, got %r" % (what, v))
    return int(v)


def grouped_lstm(inputs, width, timesteps, initial_state, kernel, bias, gain=None, layernorm=True):
    """An LSTM unrolled over `timesteps` steps with one shared kernel (reference lstm.py:153-199):
        z_t = [x_t, h_{t-1}] . kernel
        c_t, h_t = fused_lstm_gates(c_{t-1}, layer_norm(z_t, gain, bias, segments=4), forget_bias=1.0)   (layernorm)
        c_t, h_t = fused_lstm_gates(c_{t-1}, z_t, bias=bias, forget_bias=1.0)                             (otherwise)
    Returns (output (N, timesteps, width), [c_T, h_T]), differentiable in inputs, both initial states, kernel, bias and
    gain; output[:, -1] is h_T bit for bit.

    inputs: (N, timesteps, in), or (N, in) when timesteps == 1; CUDA, fp32 / fp16 / bf16. initial_state: [c, h], each
    (N, width) in the inputs' dtype and device. kernel: (in + width, 4 * width), any of the three dtypes, cast to the
    inputs' dtype once per call. bias and gain: 4 * width entries; gain is required with layernorm and must be None
    without it; with layernorm they share one dtype. Gradients come back in each parameter's dtype; the kernel's is
    formed in fp32.

    The product runs on the wgmma xprop kernel (fp16 / bf16) or the FMA kernel (fp32) of a dense-layout
    BlocksparseMatMul with 32 x 32 blocks, its operands zero-padded to multiples of 32. With layernorm each step is one
    bsmm_lstm_ln_gates: the normalised value stays in fp32 (the two-op composition rounds it to the dtype), epsilon is
    1e-6. The backward is BPTT over the saved steps with one dw_matmul_large_n over all T * N rows for the kernel (the
    reference's group_lstm_grads with group_size=None), and one reduce for gain and bias."""
    timesteps, width = _check_int(timesteps, "grouped_lstm: timesteps"), _check_int(width, "grouped_lstm: width")
    x = _check_tensor(inputs, "grouped_lstm: inputs")
    if x.dim() == 2 and timesteps == 1:
        x = x.reshape(x.shape[0], 1, x.shape[1])
    if x.dim() != 3 or x.shape[1] != timesteps or x.shape[2] < 1:
        raise ValueError("grouped_lstm: inputs must be (N, %d, in)%s, got %s" %
                         (timesteps, " or (N, in)" if timesteps == 1 else "", tuple(inputs.shape)))
    N, T, In = x.shape
    if not isinstance(initial_state, (list, tuple)) or len(initial_state) != 2:
        raise ValueError("grouped_lstm: initial_state must be [c, h]")
    c0, h0 = (_check_tensor(s, "grouped_lstm: initial_state", x) for s in initial_state)
    for s in (c0, h0):
        if s.dtype != x.dtype or tuple(s.shape) != (N, width):
            raise ValueError("grouped_lstm: c and h must be (%d, %d) of %s, got %s of %s" %
                             (N, width, x.dtype, tuple(s.shape), s.dtype))
    _check_tensor(kernel, "grouped_lstm: kernel", x)
    if tuple(kernel.shape) != (In + width, 4 * width):
        raise ValueError("grouped_lstm: kernel must be (%d, %d), got %s" % (In + width, 4 * width, tuple(kernel.shape)))
    _check_tensor(bias, "grouped_lstm: bias", x)
    if layernorm:
        if gain is None:
            raise ValueError("grouped_lstm: layernorm needs a gain")
        _check_tensor(gain, "grouped_lstm: gain", x)
        if gain.dtype != bias.dtype:
            raise ValueError("grouped_lstm: gain and bias must share a dtype, got %s and %s" % (gain.dtype, bias.dtype))
    elif gain is not None:
        raise ValueError("grouped_lstm: gain is only used with layernorm")
    for p, what in ((bias, "bias"), (gain, "gain")):
        if p is not None and p.numel() != 4 * width:
            raise ValueError("grouped_lstm: %s has %d entries, 4 * width is %d" % (what, p.numel(), 4 * width))
    if 4 * width >= 2 ** 31:
        raise ValueError("grouped_lstm: 4 * width must be below 2^31")
    bias = bias.contiguous().view(-1)
    gain = None if gain is None else gain.contiguous().view(-1)
    with torch.cuda.device(x.device):
        out, cT, hT = _GroupedLstmFunction.apply(bool(layernorm), x.contiguous(), c0.contiguous(), h0.contiguous(),
                                                 kernel, bias, gain)
    return out, [cT, hT]


# ---- FusedBasicLSTMCell -----------------------------------------------------------------------------------------------
class FusedBasicLSTMCell(torch.nn.Module):
    """TF's BasicLSTMCell with the gates fused (reference lstm.py:122-145): one step
        z = [inputs, h] . kernel,   (c, h) = fused_lstm_gates(c, z, bias=bias, forget_bias=forget_bias)
    with the product on the same dense-layout kernel as grouped_lstm (its kernel gradient a dw_matmul_large_n).

    kernel (input_size + num_units, 4 * num_units) is initialised glorot-uniform and bias with zeros, as TF does; both
    are built here because torch builds parameters eagerly, hence the explicit input_size. activation must be None or
    torch.tanh (the gates kernel applies tanh). cell(inputs, state) returns (h, new_state): state is (c, h), or their
    (N, 2 * num_units) concatenation when state_is_tuple=False."""

    def __init__(self, num_units, input_size, forget_bias=1.0, state_is_tuple=True, activation=None,
                 dtype=torch.float32, device=None):
        super().__init__()
        self.num_units = _check_int(num_units, "FusedBasicLSTMCell: num_units")
        self.input_size = _check_int(input_size, "FusedBasicLSTMCell: input_size")
        if not isinstance(forget_bias, numbers.Real) or isinstance(forget_bias, bool):
            raise ValueError("FusedBasicLSTMCell: forget_bias must be a Python number, got %r" % (forget_bias,))
        if activation not in (None, torch.tanh):
            raise ValueError("FusedBasicLSTMCell: activation must be None or tanh, got %r" % (activation,))
        if dtype not in _FLOATS:
            raise ValueError("FusedBasicLSTMCell: unsupported dtype %s" % (dtype,))
        self.forget_bias, self.state_is_tuple = float(forget_bias), bool(state_is_tuple)
        C, K4 = input_size + num_units, 4 * num_units
        limit = math.sqrt(6.0 / (C + K4))
        self.kernel = torch.nn.Parameter(torch.empty((C, K4), dtype=dtype, device=device).uniform_(-limit, limit))
        self.bias = torch.nn.Parameter(torch.zeros(K4, dtype=dtype, device=device))

    @property
    def state_size(self):
        return (self.num_units, self.num_units) if self.state_is_tuple else 2 * self.num_units

    @property
    def output_size(self):
        return self.num_units

    def forward(self, inputs, state):
        W = self.num_units
        x = _check_tensor(inputs, "FusedBasicLSTMCell: inputs", self.kernel)
        if x.dim() != 2 or x.shape[1] != self.input_size:
            raise ValueError("FusedBasicLSTMCell: inputs must be (N, %d), got %s" % (self.input_size, tuple(x.shape)))
        if self.state_is_tuple:
            if not isinstance(state, (list, tuple)) or len(state) != 2:
                raise ValueError("FusedBasicLSTMCell: state must be a tuple (c, h)")
            c, h = state
        else:
            _check_tensor(state, "FusedBasicLSTMCell: state", x)
            if state.dim() != 2 or state.shape[1] != 2 * W:
                raise ValueError("FusedBasicLSTMCell: state must be (N, %d), got %s" % (2 * W, tuple(state.shape)))
            c, h = state[:, :W], state[:, W:]
        for s in (c, h):
            _check_tensor(s, "FusedBasicLSTMCell: state", x)
            if s.dtype != x.dtype or tuple(s.shape) != (x.shape[0], W):
                raise ValueError("FusedBasicLSTMCell: c and h must be (%d, %d) of %s, got %s of %s" %
                                 (x.shape[0], W, x.dtype, tuple(s.shape), s.dtype))
        prod = _StepProduct.get(self.input_size + W, 4 * W)
        z = _ProductFunction.apply(x.contiguous(), h, self.kernel, prod)
        c, h = fused_lstm_gates(c, z, bias=self.bias, forget_bias=self.forget_bias)
        return h, ((c, h) if self.state_is_tuple else torch.cat([c, h], 1))
