"""The quantize entries refuse bad arguments with BSMM_E_ARG before anything is launched (no GPU needed: the pointers are
fake and never dereferenced), the Python layer raises ValueError before reaching them, and the public names keep the
reference's signatures and defaults."""
import ast
import importlib
import inspect
import os

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import AdamOptimizer, Ema, _lib
from blocksparse_b200.quantize import QuantizeSpec, log_stats, quantize

qm = importlib.import_module("blocksparse_b200.quantize")     # the package's `quantize` attribute is the function

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference"
E_ARG = -3
X, Y, EXP, ST, WS, ENT = (0x10000 * i for i in range(1, 7))


def _q(n=1, dtype=_lib.F32, xs=(X,), ys=(Y,), exps=(EXP,), sizes=(64,), ebits=4, fbits=3, denorm=1, stoch=0, ent=ENT):
    arr = lambda v, t: None if v is None else np.array(v, dtype=t)  # noqa: E731
    a = [arr(xs, np.uint64), arr(ys, np.uint64), arr(exps, np.uint64), arr(sizes, np.int64)]
    return _lib.load().bsmm_quantize(n, dtype, *[None if v is None else v.ctypes.data for v in a], ebits, fbits,
                                     denorm, stoch, ent, None)


def _s(n=1, dtype=_lib.F32, xs=(X,), sizes=(64,), exps=(EXP,), stats=ST, ebits=4, fbits=3, denorm=1, mode=0, ws=WS):
    arr = lambda v, t: None if v is None else np.array(v, dtype=t)  # noqa: E731
    a = [arr(xs, np.uint64), arr(sizes, np.int64), arr(exps, np.uint64)]
    return _lib.load().bsmm_quantize_stats(n, dtype, *[None if v is None else v.ctypes.data for v in a], stats, ebits,
                                           fbits, denorm, mode, 2, 4.0, 65504.0, 2.0 ** -24, ws, None)


CASES = [
    (_q, dict(n=-1)), (_q, dict(dtype=_lib.F16)), (_q, dict(dtype=5)), (_q, dict(ebits=0)), (_q, dict(ebits=9)),
    (_q, dict(fbits=-1)), (_q, dict(fbits=24)), (_q, dict(dtype=_lib.BF16, fbits=8)), (_q, dict(denorm=2)),
    (_q, dict(stoch=3)), (_q, dict(stoch=2, ent=None)), (_q, dict(xs=None)), (_q, dict(ys=None)),
    (_q, dict(exps=None)), (_q, dict(sizes=None)), (_q, dict(sizes=(-1,))), (_q, dict(xs=(0,))), (_q, dict(ys=(0,))),
    (_q, dict(exps=(0,))),
    (_s, dict(n=-1)), (_s, dict(dtype=4)), (_s, dict(ebits=0)), (_s, dict(fbits=24)), (_s, dict(mode=2)),
    (_s, dict(xs=None)), (_s, dict(sizes=None)), (_s, dict(sizes=(-5,))), (_s, dict(xs=(0,))), (_s, dict(exps=(0,))),
    (_s, dict(stats=None)), (_s, dict(ws=None)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_empty_tensors_launch_nothing():
    before = _lib.last_kernel()
    assert _q(sizes=(0,), xs=(0,), ys=(0,), exps=(0,)) == 0
    assert _q(n=0, xs=None, ys=None, exps=None, sizes=None) == 0
    assert _s(sizes=(0,), xs=(0,), stats=None, ws=None) == 0
    assert _lib.last_kernel() == before
    sizes = np.array([8192, 8193, 0, 1], np.int64)
    assert _lib.load().bsmm_quantize_stats_workspace_bytes(4, sizes.ctypes.data) == 4 * 40
    assert _lib.load().bsmm_quantize_stats_workspace_bytes(-1, None) == 0


def test_header_declares_and_lib_binds_the_entries():
    with open(os.path.join(ROOT, "include", "bsmm_b200.h")) as f:
        header = f.read()
    for name in ("bsmm_quantize", "bsmm_quantize_stats", "bsmm_quantize_stats_workspace_bytes"):
        assert name + "(" in header, name
        assert name in _lib.SIGNATURES, name
        assert hasattr(_lib.load(), name), name
    assert "bsmm_quantize         <- Quantize<T>" in header and "QuantizationStats<T>" in header


def test_python_argument_errors_raise_value_error():
    s = QuantizeSpec()
    x = torch.zeros(4, 8)
    bad = [lambda: quantize(x, s), lambda: quantize(x.half(), s), lambda: quantize(x.bfloat16(), QuantizeSpec(fbits=8)),
           lambda: quantize(x.bfloat16(), s, QuantizeSpec(fbits=10)), lambda: quantize(x, QuantizeSpec(ebits=0)),
           lambda: quantize(x, QuantizeSpec(ebits=9)), lambda: quantize(x, QuantizeSpec(fbits=-1)),
           lambda: quantize(x, QuantizeSpec(fbits=24)), lambda: quantize(x, object()), lambda: quantize(x, s, object()),
           lambda: quantize(x, QuantizeSpec(stochastic=3)), lambda: quantize(x, QuantizeSpec(mode=2)),
           lambda: quantize(x.double(), s), lambda: quantize(1.0, s),
           lambda: log_stats(x, 1), lambda: log_stats(x, 1, freq=3), lambda: log_stats(x, 1, bfreq=6),
           lambda: log_stats(x.int(), 1), lambda: log_stats(x, 1.5)]
    before = _lib.last_kernel()
    for call in bad:
        with pytest.raises(ValueError):
            call()
    if torch.cuda.is_available():
        c = x.cuda()
        for call in (lambda: quantize(c.half(), s), lambda: quantize(c.bfloat16(), QuantizeSpec(fbits=8)),
                     lambda: quantize(c, QuantizeSpec(ebits=9)), lambda: quantize(c, QuantizeSpec(fbits=24)),
                     lambda: log_stats(c, 1, freq=3), lambda: log_stats(c, torch.ones(2, dtype=torch.int64))):
            with pytest.raises(ValueError):
                call()
    assert _lib.last_kernel() == before


def test_optimizers_reject_what_is_not_a_spec():
    p = torch.zeros(4)
    for kw in (dict(param_qspec=object()), dict(mean_qspec=1), dict(var_qspec="e4m3"),
               dict(param_qspec=QuantizeSpec(ebits=12))):
        with pytest.raises(ValueError):
            AdamOptimizer([p], **kw)
    for kw in (dict(mean_qspec=QuantizeSpec()), dict(var_qspec=QuantizeSpec())):
        with pytest.raises(ValueError):
            AdamOptimizer([p], fp16=True, **kw)
    with pytest.raises(ValueError):
        Ema().apply([p], qspec=object())
    with pytest.raises(ValueError):
        Ema(fp16=True).apply([p], qspec=QuantizeSpec())


def test_spec_defaults_and_copy():
    s = QuantizeSpec()
    assert (s.ebits, s.fbits, s.emax, s.stoch, s.denorm, s.freq, s.mode, s.bias_pad, s.stdv_mul, s.logfile) == \
        (4, 3, 7, 0, True, 1024, 0, 2, 4.0, "")
    assert QuantizeSpec(ebits=6, fbits=7).emax == 31 and QuantizeSpec(ebits=5, emax=3).emax == 3
    a = QuantizeSpec(ebits=5, fbits=2, stochastic=2, frequency=8, mode=1, bias_pad=1, stdv_mul=3.0, logfile="a.txt")
    c = QuantizeSpec(copy=a, ebits=1, logfile="b.txt")
    assert vars(c) == vars(a)                                  # the copied spec's logfile wins when it has one
    a.logfile = ""
    c = QuantizeSpec(copy=a, logfile="b.txt")
    assert c.logfile == "b.txt" and c.ebits == 5 and c.freq == 8


def _reference_defs():
    path = os.path.join(REF, "blocksparse", "quantize.py")
    if not os.path.isfile(path):
        pytest.skip("no reference checkout")
    tree = ast.parse(open(path).read())
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef):
            a = node.args
            defaults = [None] * (len(a.args) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults]
            out[node.name] = list(zip([x.arg for x in a.args], defaults))
    return out


def _ours(fn):
    out = []
    for p in inspect.signature(fn).parameters.values():
        out.append((p.name, None if p.default is inspect.Parameter.empty else p.default))
    return out


def test_signatures_and_defaults_match_the_reference():
    ref = _reference_defs()
    for name, fn in (("quantize", quantize), ("log_stats", log_stats)):
        ours = _ours(fn)
        theirs = ref[name]
        assert [n for n, _ in ours] == [n for n, _ in theirs], name
        for (n, d), (_, rd) in zip(ours, theirs):
            assert (d is None and rd in (None, "None")) or d == eval(rd), (name, n, d, rd)
    init = ref["__init__"]
    ours = _ours(QuantizeSpec.__init__)
    assert [n for n, _ in ours] == [n for n, _ in init]
    for (n, d), (_, rd) in zip(ours[1:], init[1:]):
        assert (d is None and rd == "None") or d == eval(rd), (n, d, rd)


def test_names_are_importable_but_stay_out_of_the_package_all():
    for name in qm.__all__:
        assert getattr(blocksparse_b200, name) is getattr(qm, name)
        assert name not in blocksparse_b200.__all__
    assert set(qm.__all__) == {"QuantizeSpec", "quantize", "log_stats", "quantize_state", "reset_quantize_states"}


def test_log_stats_step_rule():
    prev = [-1]
    first = [1 << p for p in range(3)]                              # freq 8: steps 1, 2, 4
    hits = [s for s in [0, 1, 1, 2, 3, 4, 5, 8, 8, 9, 16, 24, 32] if qm._logs_at(s, 8, first, prev)]
    assert hits == [1, 2, 4, 8, 16, 24, 32]
    assert not any(qm._logs_at(s, 0, [], [-1]) for s in range(10))
