"""ctypes binding of the conv filter normalisation entries in oracle/_ref/libbsref.so (oracle/ref/conv_l2norm.cu): the
reference's own L2NormalizeKCTRS / L2NormalizeCKTRS launchers and their gradients, built for sm_90a, fed the reference's
norm_lut layout (conv.py:317-324) rebuilt from a BlocksparseConv / BlocksparseDeconv, and the plumbing of
oracle/ref_kernels.py. Only the test suite imports this module."""
import ctypes

import numpy as np
import torch

from . import ref_kernels as rk

_i, _f, _p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p
SIGNATURES = {
    "bsref_l2_normalize_kctrs": [_i, _p, _p, _p, _p, _p, _f, _i, _p],
    "bsref_l2_normalize_cktrs": [_i, _p, _p, _p, _p, _p, _f, _i, _i, _i, _i, _p],
    "bsref_l2_normalize_grad_kctrs": [_i, _p, _p, _p, _p, _p, _p, _p, _f, _i, _p],
    "bsref_l2_normalize_grad_cktrs": [_i, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _i, _i, _p],
}

_FNS = {}


def missing():
    """Why the entries cannot be called here, or None when they can: the library may be absent (no reference checkout
    where it was built) or built by an oracle/ref without conv_l2norm.cu."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not all(hasattr(rk.load(), name) for name in SIGNATURES):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/conv_l2norm.cu; rebuild it with "
                "make -C oracle/ref REF=<reference checkout>")
    return None


def _call(name, outs, *args):
    fn = _FNS.get(name)
    if fn is None:
        fn = _FNS[name] = getattr(rk.load(), name)
        fn.argtypes, fn.restype = SIGNATURES[name], _i
    rc = fn(*args, rk._stream())
    if rc != 0:
        raise RuntimeError("%s: CUDA error %d" % (name, rc))
    torch.cuda.current_stream().synchronize()
    return [o.check(name) for o in outs]


def magic16(nmax, d):
    """(magic, shift) with (n * magic) >> shift == n // d for every 0 <= n <= nmax, magic and n within 16 bits: the
    16-bit multiply the CKTRS kernels divide with (vmad on the low halves)."""
    if nmax >= 2 ** 16:
        raise ValueError("CKTRS rows of %d elements exceed the kernels' 16-bit division" % nmax)
    n = np.arange(nmax + 1, dtype=np.int64)
    for shift in range(0, 33):
        magic = -(-(1 << shift) // d)
        if magic >= 2 ** 16:
            break
        if np.array_equal((n * magic) >> shift, n // d):
            return magic, shift
    raise ValueError("no 16-bit magic number divides by %d up to %d" % (d, nmax))


def norm_lut(op):
    """The reference's norm_lut for op: (offset, C_b trs) per output channel of each block, or for the deconv
    (c, K_b trs, C_b trs, block offset) per input channel, in the conv's internal (swapped) terms."""
    rows, off = [], 0
    for lc, lk in op.BCK:
        cb, kb = len(lc), len(lk)
        if op.deconv:
            rows += [[c, kb * op.trs, cb * op.trs, off] for c in range(cb)]
        else:
            rows += [[off + k * cb * op.trs, cb * op.trs] for k in range(kb)]
        off += kb * cb * op.trs
    return np.array(rows, np.int32)


def _cktrs_args(op):
    nmax = max(len(lk) for _, lk in op.BCK) * op.trs
    return (op.trs,) + magic16(nmax, op.trs)


def l2_normalize(op, F, gain=None, epsilon=1e-12):
    """(y, sum_sqr) of the reference's op on F (op.sizeF elements, fp32 / fp16 / bf16); y has F's dtype."""
    F, = rk._dev(F.reshape(-1))
    g = None if gain is None else rk._dev(gain.float())[0]
    lut = torch.as_tensor(norm_lut(op)).to(F.device)
    outs = [rk._Out((op.sizeF,), F.dtype, F.device), rk._Out((op.normSize,), torch.float32, F.device)]
    args = [rk._dt(F), outs[0].t.data_ptr(), outs[1].t.data_ptr(), F.data_ptr(), None if g is None else g.data_ptr(),
            lut.data_ptr(), float(epsilon), op.normSize]
    if op.deconv:
        return _call("bsref_l2_normalize_cktrs", outs, *args, *_cktrs_args(op))
    return _call("bsref_l2_normalize_kctrs", outs, *args)


def l2_normalize_grad(op, dy, F, sum_sqr, gain=None, epsilon=1e-12):
    """(dF, dgain or None) of the reference's gradient op; dy and F of one dtype, sum_sqr from l2_normalize."""
    dy, F, ss = rk._dev(dy.reshape(-1), F.reshape(-1), sum_sqr)
    g = None if gain is None else rk._dev(gain.float())[0]
    lut = torch.as_tensor(norm_lut(op)).to(F.device)
    outs = [rk._Out((op.sizeF,), F.dtype, F.device)]
    if g is not None:
        outs.append(rk._Out((op.normSize,), torch.float32, F.device))
    args = [rk._dt(F), outs[0].t.data_ptr(), None if g is None else outs[1].t.data_ptr(), dy.data_ptr(), F.data_ptr(),
            None if g is None else g.data_ptr(), ss.data_ptr(), lut.data_ptr(), float(epsilon), op.normSize]
    if op.deconv:
        res = _call("bsref_l2_normalize_grad_cktrs", outs, *args, *_cktrs_args(op))
    else:
        res = _call("bsref_l2_normalize_grad_kctrs", outs, *args)
    return res[0], (res[1] if g is not None else None)
