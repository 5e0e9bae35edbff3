"""The optimizer entries refuse bad arguments with BSMM_E_ARG before anything is launched, and launch nothing for empty
input (no GPU needed: the pointers are fake and never dereferenced). The Python layer raises ValueError before reaching
them, and keeps the reference's signatures."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from blocksparse_b200 import AdamOptimizer, ClipGlobalNorm, Ema, _lib, clip_by_global_norm, global_norm
from blocksparse_b200 import optimize as opt

E_ARG = -3
P = 0x100000                                         # fake, 16-byte aligned device addresses


def _arr(vals, dtype):
    return np.array(vals, dtype=dtype)


def _adam(n=2, grads=None, gdt=None, params=None, means=None, vars_=None, codes=None, sizes=None, gates=None, bss=None,
          null_array=None):
    grads = [P, 2 * P] if grads is None else grads
    arrs = dict(grads=_arr(grads, np.uint64), gdt=_arr(gdt or [0, 1], np.int32),
                params=_arr(params or [3 * P, 4 * P], np.uint64), means=_arr(means or [5 * P, 6 * P], np.uint64),
                vars=_arr(vars_ or [7 * P, 8 * P], np.uint64), codes=_arr(codes or [0, 1], np.int32),
                sizes=_arr(sizes or [64, 4096], np.int64), gates=_arr(gates or [0, 9 * P], np.uint64),
                bss=_arr(bss or [0, 32], np.int32))
    ptrs = {k: (None if k == null_array else a.ctypes.data) for k, a in arrs.items()}
    return _lib.load().bsmm_adam(n, ptrs["grads"], ptrs["gdt"], ptrs["params"], ptrs["means"], ptrs["vars"],
                                 ptrs["codes"], ptrs["sizes"], ptrs["gates"], ptrs["bss"], None, 1e-3, 0.9, 0.999, 1e-8,
                                 1.0, 0.0, 0.0, 0, 0, None)


def _norm(n=2, xs=None, dts=None, sizes=None, norm=10 * P, scale=11 * P, ws=12 * P, null_array=None):
    arrs = dict(xs=_arr(xs or [P, 2 * P], np.uint64), dts=_arr(dts or [0, 2], np.int32),
                sizes=_arr(sizes or [100, 3], np.int64))
    ptrs = {k: (None if k == null_array else a.ctypes.data) for k, a in arrs.items()}
    return _lib.load().bsmm_global_norm(n, ptrs["xs"], ptrs["dts"], ptrs["sizes"], 1.0, 1.0, 0.0, 0, 0, norm, scale, ws,
                                        None)


def _ema(n=2, emas=None, edt=0, params=None, sizes=None, gates=None, bss=None, null_array=None):
    arrs = dict(emas=_arr(emas or [P, 2 * P], np.uint64), params=_arr(params or [3 * P, 4 * P], np.uint64),
                sizes=_arr(sizes or [256, 5], np.int64), gates=_arr(gates or [5 * P, 0], np.uint64),
                bss=_arr(bss or [16, 0], np.int32))
    ptrs = {k: (None if k == null_array else a.ctypes.data) for k, a in arrs.items()}
    return _lib.load().bsmm_ema(n, ptrs["emas"], edt, ptrs["params"], ptrs["sizes"], ptrs["gates"], ptrs["bss"], 0.99,
                                None)


CASES = [
    (_adam, dict(n=-1)), (_adam, dict(gdt=[0, 3])), (_adam, dict(gdt=[-1, 0])), (_adam, dict(codes=[0, 2])),
    (_adam, dict(grads=[0, 2 * P])), (_adam, dict(params=[3 * P, 0])), (_adam, dict(means=[0, 6 * P])),
    (_adam, dict(vars_=[7 * P, 0])), (_adam, dict(sizes=[-1, 4096])), (_adam, dict(sizes=[64, 4097])),
    (_adam, dict(bss=[0, 12])), (_adam, dict(bss=[0, 128])), (_adam, dict(bss=[4, 32])),
    (_adam, dict(gates=[0, 0])), (_adam, dict(null_array="grads")), (_adam, dict(null_array="sizes")),
    (_adam, dict(null_array="codes")),
    (_norm, dict(n=-2)), (_norm, dict(dts=[0, 5])), (_norm, dict(xs=[P, 0])), (_norm, dict(sizes=[100, -3])),
    (_norm, dict(norm=None)), (_norm, dict(scale=None)), (_norm, dict(ws=None)), (_norm, dict(null_array="xs")),
    (_norm, dict(null_array="dts")),
    (_ema, dict(n=-1)), (_ema, dict(edt=2)), (_ema, dict(edt=7)), (_ema, dict(emas=[0, 2 * P])),
    (_ema, dict(params=[3 * P, 0])), (_ema, dict(sizes=[256, -5])), (_ema, dict(sizes=[255, 5])),
    (_ema, dict(bss=[24, 0])), (_ema, dict(gates=[0, 0])), (_ema, dict(null_array="params")),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_empty_input_launches_nothing():
    before = _lib.last_kernel()
    assert _adam(n=0) == 0
    assert _adam(sizes=[0, 0]) == 0
    assert _adam(grads=[0, 0], sizes=[0, 0]) == 0                  # empty tensors' pointers are not read
    assert _norm(n=0) == 0
    assert _norm(sizes=[0, 0], ws=None) == 0                       # no workspace needed either
    assert _ema(n=0) == 0
    assert _ema(sizes=[0, 0]) == 0
    assert _lib.last_kernel() == before


def test_global_norm_workspace_bytes():
    ws = _lib.load().bsmm_global_norm_workspace_bytes
    sizes = np.array([0, 1, 8192, 8193, 3 * 8192], np.int64)
    assert ws(5, sizes.ctypes.data) == 4 * (0 + 1 + 1 + 2 + 3)
    assert ws(0, None) == 0 and ws(-1, sizes.ctypes.data) == 0 and ws(1, None) == 0
    bad = np.array([5, -1], np.int64)
    assert ws(2, bad.ctypes.data) == 0
    big = np.array([2 ** 40], np.int64)                            # 64-bit sizes
    assert ws(1, big.ctypes.data) == 4 * (2 ** 40 // 8192)


def test_python_argument_errors_raise_value_error():
    p = torch.zeros(4)
    for kw in (dict(param_qspec=object()), dict(mean_qspec=object()), dict(var_qspec=object())):
        with pytest.raises(ValueError):
            AdamOptimizer([p], **kw)
    with pytest.raises(ValueError):
        AdamOptimizer([p])                                         # a CPU param: no CPU path
    with pytest.raises(ValueError):
        AdamOptimizer([p], norm_scale=torch.ones(()))              # norm_scale must live on the device
    for bad in ([torch.zeros(3, dtype=torch.float64)], [torch.zeros(3, dtype=torch.int32)], [torch.zeros(3)], [3.0]):
        with pytest.raises(ValueError):
            clip_by_global_norm(bad)
        with pytest.raises(ValueError):
            global_norm(bad)
    with pytest.raises(ValueError):
        Ema().apply([p], qspec=object())
    with pytest.raises(ValueError):
        Ema().apply([p])                                           # a CPU param
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    pc = torch.zeros(4, device="cuda")
    calls = [lambda: AdamOptimizer([pc.double()]),
             lambda: AdamOptimizer([pc], fp16=True).step(grads=[pc[:3]]),
             lambda: AdamOptimizer([pc]).step(grads=[pc, pc]),
             lambda: AdamOptimizer([pc]).step(grads=[pc.double()]),
             lambda: AdamOptimizer([pc]).step(grads=[pc], norm_scale=torch.ones(2, device="cuda")),
             lambda: clip_by_global_norm([pc, pc.double()]),
             lambda: Ema().apply([pc.half()])]
    for call in calls:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def test_reference_signatures():
    p = inspect.signature(AdamOptimizer.__init__).parameters
    assert list(p) == ["self", "params", "learning_rate", "beta1", "beta2", "epsilon", "clip_sigmas", "norm_scale",
                       "grad_scale", "saturate", "zero_infs", "zero_nans", "gated", "param_qspec", "mean_qspec",
                       "var_qspec", "fp16", "zero_init_variables", "name"]
    assert [p[k].default for k in list(p)[2:]] == [3e-4, 0.9, 0.999, 1e-8, 0.0, None, 1.0, 0.0, False, False, False,
                                                   None, None, None, False, False, "Adam"]
    p = inspect.signature(AdamOptimizer.step).parameters
    assert list(p) == ["self", "closure", "norm_scale", "grads"] and all(p[k].default is None for k in list(p)[1:])
    for fn in (clip_by_global_norm, ClipGlobalNorm):
        p = inspect.signature(fn).parameters
        assert list(p) == ["grads", "clip_norm", "grad_scale", "saturate", "zero_infs", "zero_nans"]
        assert [p[k].default for k in list(p)[1:]] == [1.0, 1.0, 0.0, False, False]
    p = inspect.signature(global_norm).parameters
    assert list(p) == ["grads", "grad_scale", "saturate", "zero_infs", "zero_nans"]
    assert [p[k].default for k in list(p)[1:]] == [1.0, 0.0, False, False]
    p = inspect.signature(Ema.__init__).parameters
    assert list(p) == ["self", "decay", "gated", "fp16", "name"]
    assert [p[k].default for k in list(p)[1:]] == [0.999, False, False, "Ema"]
    assert list(inspect.signature(Ema.apply).parameters) == ["self", "params", "qspec"]
    assert list(inspect.signature(Ema.average).parameters) == ["self", "param"]
    assert issubclass(AdamOptimizer, torch.optim.Optimizer)


def test_abi_table_is_bound():
    lib = _lib.load()
    for name in ("bsmm_adam", "bsmm_global_norm", "bsmm_global_norm_workspace_bytes", "bsmm_ema"):
        assert name in _lib.SIGNATURES and isinstance(getattr(lib, name), ctypes._CFuncPtr)
    assert opt._MIN_CODED == 8192
