"""AdafactorOptimizer without a GPU: the reference's signature and defaults, ValueError for every bad argument before
anything is launched, BSMM_E_ARG from the C entries (fake, never dereferenced pointers), the workspace size, and the
float64 oracle on a case with a closed form."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import AdafactorOptimizer, _lib
from blocksparse_b200 import optimize as opt
from oracle import adafactor_oracle as ao

E_ARG = -3
P = 0x100000                                         # fake, 16-byte aligned device addresses


def test_reference_signature_and_defaults():
    p = inspect.signature(AdafactorOptimizer.__init__).parameters
    assert list(p) == ["self", "params", "learning_rate", "beta2", "epsilon", "clip_thresh", "norm_scale", "grad_scale",
                       "saturate", "zero_infs", "zero_nans", "name", "zero_init_variables"]
    assert [p[k].default for k in list(p)[2:]] == [5e-4, 0.999, 1e-30, 1.0, None, 1.0, 0.0, False, False, "Adafactor",
                                                   False]
    p = inspect.signature(AdafactorOptimizer.step).parameters
    assert list(p) == ["self", "closure", "norm_scale", "grads"] and all(p[k].default is None for k in list(p)[1:])
    assert issubclass(AdafactorOptimizer, torch.optim.Optimizer)
    assert blocksparse_b200.optimize.AdafactorOptimizer is AdafactorOptimizer
    assert "AdafactorOptimizer" in blocksparse_b200.__doc__


def test_abi_table_is_bound():
    lib = _lib.load()
    for name in ("bsmm_adafactor", "bsmm_adafactor_workspace_bytes"):
        assert name in _lib.SIGNATURES and isinstance(getattr(lib, name), ctypes._CFuncPtr)


def test_cpu_and_bad_params_raise_value_error():
    for bad in ([torch.zeros(4)], [torch.zeros(4, 4)]):                          # CPU params: there is no CPU path
        with pytest.raises(ValueError):
            AdafactorOptimizer(bad)
    with pytest.raises(ValueError):
        AdafactorOptimizer([], norm_scale=torch.ones(()))                       # norm_scale on the host
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    pc = torch.zeros(6, 8, device="cuda")
    for bad in (torch.zeros((), device="cuda"), torch.zeros(2, 3, 4, device="cuda"),
                torch.zeros(3, 32, 32, device="cuda"),                         # a (blocks, bs, bs) block-sparse weight
                pc.double(), pc.half(), pc.t(), pc[:, ::2]):
        with pytest.raises(ValueError):
            AdafactorOptimizer([bad])
    assert _lib.last_kernel() == before


def test_bad_grads_and_norm_scale_raise_before_any_launch():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device to hold the params (the CPU cases are in test_cpu_and_bad_params_raise_...)")
    before = _lib.last_kernel()
    pc = torch.zeros(6, 8, device="cuda")
    o = AdafactorOptimizer([pc])
    calls = [lambda: o.step(grads=[pc[:3]]),                                     # shape
             lambda: o.step(grads=[pc.t()]),
             lambda: o.step(grads=[pc.cpu()]),                                   # device
             lambda: o.step(grads=[pc.double()]),                                # dtype
             lambda: o.step(grads=[pc.int()]),
             lambda: o.step(grads=[pc, pc]),                                     # count
             lambda: o.step(grads=[pc], norm_scale=torch.ones(2, device="cuda")),
             lambda: o.step(grads=[pc], norm_scale=torch.ones((), device="cuda", dtype=torch.float64)),
             lambda: o.step(grads=[pc], norm_scale=torch.ones(())),
             lambda: o.step(grads=[pc], norm_scale=0.5)]
    for call in calls:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before and not o.state
    assert o.param_groups[0]["decay1_power"] == pytest.approx(0.999)            # no step taken


def _af(n=2, grads=None, gdt=None, params=None, cvs=None, rvs=None, rows=None, cols=None, ws=12 * P, null_array=None):
    arrs = dict(grads=np.array(grads or [P, 2 * P], np.uint64), gdt=np.array(gdt or [0, 2], np.int32),
                params=np.array(params or [3 * P, 4 * P], np.uint64), cvs=np.array(cvs or [5 * P, 6 * P], np.uint64),
                rvs=np.array(rvs or [7 * P, 0], np.uint64), rows=np.array(rows or [64, 1], np.int64),
                cols=np.array(cols or [256, 1003], np.int64))
    ptrs = {k: (None if k == null_array else a.ctypes.data) for k, a in arrs.items()}
    return _lib.load().bsmm_adafactor(n, ptrs["grads"], ptrs["gdt"], ptrs["params"], ptrs["cvs"], ptrs["rvs"],
                                      ptrs["rows"], ptrs["cols"], None, 1e-3, 0.999, 1e-30, 1.0, 1.0, 0.0, 0, 0, ws, None)


CASES = [dict(n=-1), dict(gdt=[0, 3]), dict(gdt=[-1, 0]), dict(rows=[-1, 1]), dict(cols=[256, -2]),
         dict(rows=[1 << 40, 1], cols=[1 << 40, 1]), dict(grads=[0, 2 * P]), dict(params=[3 * P, 0]),
         dict(cvs=[5 * P, 0]), dict(rvs=[0, 0]), dict(ws=None), dict(null_array="grads"), dict(null_array="gdt"),
         dict(null_array="params"), dict(null_array="cvs"), dict(null_array="rows"), dict(null_array="cols"),
         dict(null_array="rvs")]


@pytest.mark.parametrize("kw", CASES, ids=["-".join("%s%s" % i for i in kw.items()) for kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(kw):
    before = _lib.last_kernel()
    rc = _af(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_empty_input_launches_nothing():
    before = _lib.last_kernel()
    assert _af(n=0) == 0
    assert _af(rows=[0, 1], cols=[256, 0], ws=None) == 0
    assert _af(grads=[0, 0], params=[0, 0], cvs=[0, 0], rvs=[0, 0], rows=[5, 0], cols=[0, 7], ws=None) == 0
    assert _af(rvs=[0, 0], rows=[1, 1], cols=[0, 3], ws=12 * P, n=1) == 0     # rv is not read for rows == 1
    assert _lib.last_kernel() == before


def test_workspace_bytes():
    ws = _lib.load().bsmm_adafactor_workspace_bytes

    def call(rows, cols):
        r, c = np.array(rows, np.int64), np.array(cols, np.int64)
        return ws(len(rows), r.ctypes.data, c.ctypes.data)

    # factored (C, K): 2 scalars + one sum per 64 x 128 tile + C row partials per tile column + K column partials per
    # tile row; unfactored: 2 scalars + one sum per 8192 elements; empty: nothing
    assert call([64], [128]) == 4 * (2 + 1 + 64 + 128)
    assert call([65, 3], [129, 1]) == 4 * (2 + 4 + 65 * 2 + 2 * 129 + 2 + 1 + 3 * 1 + 1 * 1)
    assert call([1], [8193]) == 4 * (2 + 2)
    assert call([0, 5], [7, 0]) == 0
    assert call([50257], [768]) == 4 * (2 + 786 * 6 + 50257 * 6 + 786 * 768)
    assert call([1 << 20], [1 << 12]) == 4 * (2 + (1 << 14) * 32 + (1 << 20) * 32 + (1 << 14) * (1 << 12))   # 64-bit
    assert ws(0, None, None) == 0 and ws(-1, None, None) == 0 and ws(1, None, None) == 0
    assert call([-1], [5]) == 0


def test_oracle_rank_one_statistics_are_exact():
    """g^2 + eps = a_c b_k: rv = (1 - decay) a_c mean(b), cv = (1 - decay) b_k mean(a) from zero state, so
    rv[c] / mean(rv) cv[k] = (1 - decay) a_c b_k mean(b) / mean(b) = (1 - decay) (g^2 + eps) and x = g / sqrt(that)."""
    rng = np.random.default_rng(0)
    a, b, eps, decay = rng.uniform(0.5, 2, 7), rng.uniform(0.5, 2, 11), 1e-3, 0.9
    g = np.sqrt(np.outer(a, b) - eps) * rng.choice([-1, 1], (7, 11))
    p = rng.normal(0, 1, (7, 11))
    for clip in (1e9, 0.5):
        p1, cv, rv = ao.adafactor(g, p, np.zeros(11), np.zeros(7), lr=0.1, decay=decay, epsilon=eps, clip_thresh=clip)
        np.testing.assert_allclose(rv, (1 - decay) * a * b.mean(), rtol=1e-12)
        np.testing.assert_allclose(cv, (1 - decay) * b * a.mean(), rtol=1e-12)
        x = g / np.sqrt((1 - decay) * np.outer(a, b))
        rms = np.mean(x * x)
        np.testing.assert_allclose(p1, p - 0.1 * x / max(1.0, np.sqrt(rms) / clip), rtol=1e-12, atol=1e-14)
    # unfactored: the same closed form per element; norm_scale 0 returns the state as given
    p1, cv, rv = ao.adafactor(g[0], p[0], np.zeros(11), None, lr=0.1, decay=decay, epsilon=eps, clip_thresh=1e9)
    assert rv is None
    np.testing.assert_allclose(p1, p[0] - 0.1 * g[0] / np.sqrt((1 - decay) * (g[0] ** 2 + eps)), rtol=1e-12)
    p1, cv, rv = ao.adafactor(g, p, np.ones(11), np.ones(7), lr=0.1, decay=decay, norm_scale=0.0)
    assert np.array_equal(p1, p) and np.array_equal(cv, np.ones(11)) and np.array_equal(rv, np.ones(7))
    assert ao.decay(0.999, 0.0, 0.0) == 0.999 and ao.decay(0.5, 0.5, 0.25) == pytest.approx(0.5 * 0.5 / 0.75)


def test_host_decay_and_powers():
    """The decay powers start at beta2 and beta2^2 (0 and 0 with zero_init_variables) and live in the param groups."""
    if not torch.cuda.is_available():
        pytest.skip("params must be CUDA tensors")
    p = torch.zeros(3, device="cuda")
    g = AdafactorOptimizer([p], beta2=0.5).param_groups[0]
    assert (g["decay1_power"], g["decay2_power"]) == (0.5, 0.25) and g["lr"] == 5e-4
    g = AdafactorOptimizer([p], zero_init_variables=True).param_groups[0]
    assert (g["decay1_power"], g["decay2_power"]) == (0.0, 0.0)
    assert opt.AdafactorOptimizer._rows(torch.zeros(1, 5)) == 1 and opt.AdafactorOptimizer._rows(torch.zeros(2, 5)) == 2
