"""The LSTM gate, sparse relu and relu-mask entries refuse bad arguments with BSMM_E_ARG before anything is launched,
and launch nothing for empty input (no GPU needed: the pointers are fake and never dereferenced). The Python layer
raises ValueError before reaching them, keeps the reference's signatures, and its names stay out of the package's and
ewops' __all__. The float64 oracle agrees with torch float64 autograd on the composed formula."""
import inspect

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import _lib, concat4, ewops, fused_lstm_gates, lstm, sparse_relu, split4
from oracle import lstm_oracle

E_ARG, E_LIMIT = -3, -4
C, I, U, F, O, B, CN, HN, EC, EH, DC, DI, DU, DF, DO = (0x10000 * i for i in range(1, 16))


def _gates(dtype=_lib.F16, bdt=_lib.F32, c=C, i=I, u=U, f=F, o=O, stride=256, bias=B, cn=CN, hn=HN, N=8, K=64):
    return _lib.load().bsmm_lstm_gates(dtype, bdt, c, i, u, f, o, stride, bias, cn, hn, N, K, 1.0, None)


def _grad(dtype=_lib.BF16, bdt=_lib.BF16, c=C, i=I, u=U, f=F, o=O, stride=64, bias=None, ec=EC, eh=EH, dc=DC, di=DI,
          du=DU, df=DF, d_o=DO, N=8, K=64):
    return _lib.load().bsmm_lstm_gates_grad(dtype, bdt, c, i, u, f, o, stride, bias, ec, eh, dc, di, du, df, d_o, N, K,
                                            0.0, None)


def _srelu(dtype=_lib.F32, x=C, y=CN, N=8, K=33):
    return _lib.load().bsmm_sparse_relu(dtype, x, y, N, K, 1.0, None)


def _mask(dtype=_lib.F16, dy=EH, y=CN, dx=DC, n=100):
    return _lib.load().bsmm_relu_mask_grad(dtype, dy, y, dx, n, None)


CASES = [
    (_gates, dict(dtype=3)), (_gates, dict(bdt=-1)), (_gates, dict(bdt=3, bias=None)), (_gates, dict(c=None)),
    (_gates, dict(i=None)), (_gates, dict(u=None)), (_gates, dict(f=None)), (_gates, dict(o=None)),
    (_gates, dict(cn=None)), (_gates, dict(hn=None)), (_gates, dict(N=-1)), (_gates, dict(K=0)),
    (_gates, dict(stride=63)),
    (_grad, dict(dtype=-1)), (_grad, dict(bdt=4)), (_grad, dict(c=None)), (_grad, dict(i=None)), (_grad, dict(u=None)),
    (_grad, dict(f=None)), (_grad, dict(o=None)), (_grad, dict(dc=None)), (_grad, dict(di=None)),
    (_grad, dict(du=None)), (_grad, dict(df=None)), (_grad, dict(d_o=None)), (_grad, dict(N=-2)), (_grad, dict(K=-1)),
    (_grad, dict(stride=0)),
    (_srelu, dict(dtype=5)), (_srelu, dict(x=None)), (_srelu, dict(y=None)), (_srelu, dict(N=-1)), (_srelu, dict(K=0)),
    (_mask, dict(dtype=3)), (_mask, dict(dy=None)), (_mask, dict(y=None)), (_mask, dict(dx=None)), (_mask, dict(n=-1)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_limits():
    before = _lib.last_kernel()
    assert _gates(N=2 ** 62, stride=4 * 2 ** 20, K=2 ** 20) == E_LIMIT
    assert _srelu(N=2 ** 62, K=4) == E_LIMIT
    assert _lib.last_kernel() == before


def test_zero_sizes_launch_nothing():
    before = _lib.last_kernel()
    assert _gates(N=0) == 0
    assert _gates(N=0, bias=None, stride=64) == 0
    assert _grad(N=0) == 0
    assert _grad(N=0, ec=None, eh=None, bias=B) == 0
    assert _srelu(N=0) == 0
    assert _mask(n=0) == 0
    assert _lib.last_kernel() == before


def test_optional_pointers_are_accepted():
    """bias, ec and eh may be NULL; with N = 0 nothing is launched either way."""
    assert _gates(bias=None, N=0) == 0
    assert _grad(ec=None, N=0) == 0 and _grad(eh=None, N=0) == 0


def test_python_argument_errors_raise_value_error():
    c, h, g = torch.zeros(4, 8), torch.zeros(4, 32), torch.zeros(4, 8)
    cpu = [lambda: fused_lstm_gates(c, h),                              # CPU tensors: no CPU path
           lambda: fused_lstm_gates(c, g, g, g, g),
           lambda: fused_lstm_gates(c),                                  # argument counts
           lambda: fused_lstm_gates(c, g, g),
           lambda: fused_lstm_gates(c, g, g, g),
           lambda: fused_lstm_gates(c, g, g, g, g, g),
           lambda: fused_lstm_gates(c, g, g, g, g, bias=torch.zeros(32)),  # bias in the four-tensor form
           lambda: fused_lstm_gates(c, h, forget_bias="1"),
           lambda: split4(h),
           lambda: concat4(g, g, g, g),
           lambda: sparse_relu(c),
           lambda: sparse_relu(c, alpha="1"),
           lambda: sparse_relu(c, alpha=None),
           lambda: sparse_relu(c, alpha=True)]
    for call in cpu:
        with pytest.raises(ValueError):
            call()
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    cc, hc, gc = c.cuda(), h.cuda(), g.cuda()
    bad = [lambda: fused_lstm_gates(cc, hc[:, :31]),                    # h not 4K wide
           lambda: fused_lstm_gates(cc, hc[:3]),                         # leading dims differ
           lambda: fused_lstm_gates(cc, hc.half()),                      # dtypes differ
           lambda: fused_lstm_gates(cc.double(), hc.double()),
           lambda: fused_lstm_gates(cc, hc, bias=torch.zeros(31, device="cuda")),
           lambda: fused_lstm_gates(cc, hc, bias=torch.zeros(32)),       # bias on the CPU
           lambda: fused_lstm_gates(cc, hc, bias=torch.zeros(32, device="cuda", dtype=torch.float64)),
           lambda: fused_lstm_gates(cc, gc, gc, gc, gc[:, :7]),
           lambda: fused_lstm_gates(cc, gc, gc.half(), gc, gc),
           lambda: fused_lstm_gates(cc, gc, gc, gc, g),                  # one gate on the CPU
           lambda: fused_lstm_gates(cc, gc, gc, gc, gc, bias=torch.zeros(32, device="cuda")),
           lambda: fused_lstm_gates(cc, hc, forget_bias=None),
           lambda: split4(gc[:, :7]),
           lambda: concat4(gc, gc, gc, gc[:3]),
           lambda: concat4(gc, gc, gc, gc.half()),
           lambda: sparse_relu(cc, alpha="x"),
           lambda: sparse_relu(cc, alpha=torch.ones(())),
           lambda: sparse_relu(cc.double())]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def test_reference_signatures():
    p = inspect.signature(fused_lstm_gates).parameters
    assert list(p) == ["c", "args", "bias", "forget_bias", "name"]
    assert p["args"].kind == inspect.Parameter.VAR_POSITIONAL
    assert [(k, p[k].default, p[k].kind == inspect.Parameter.KEYWORD_ONLY) for k in ("bias", "forget_bias", "name")] == \
        [("bias", None, True), ("forget_bias", 1.0, True), ("name", None, True)]
    assert list(inspect.signature(split4).parameters) == ["x"]
    assert list(inspect.signature(concat4).parameters) == ["z0", "z1", "z2", "z3"]
    p = inspect.signature(sparse_relu).parameters
    assert list(p) == ["x", "alpha"] and p["alpha"].default == 1.0
    p = inspect.signature(lstm.sparse_relu_test).parameters
    assert list(p) == ["x", "alpha"] and p["alpha"].default == 1.0


def test_names_and_all():
    assert lstm.__all__ == ["fused_lstm_gates", "split4", "concat4", "sparse_relu"]
    for name in lstm.__all__:
        assert getattr(blocksparse_b200, name) is getattr(lstm, name)
        assert name not in blocksparse_b200.__all__
        assert name not in ewops.__all__


def _sig(z):
    return torch.sigmoid(z)


def test_oracle_against_torch_float64_autograd():
    rng = np.random.default_rng(0)
    N, K, fb = 5, 7, 0.75
    c, i, u, f, o, ec, eh = (rng.normal(0, 2, (N, K)) for _ in range(7))
    bias = rng.normal(0, 1, 4 * K)
    tc, ti, tu, tf, to = (torch.tensor(a, requires_grad=True) for a in (c, i, u, f, o))
    tb = torch.tensor(bias, requires_grad=True)
    bi, bu, bf, bo = tb.split(K)
    cn = _sig(tf + bf + fb) * tc + _sig(ti + bi) * torch.tanh(tu + bu)
    hn = _sig(to + bo) * torch.tanh(cn)
    (cn * torch.tensor(ec) + hn * torch.tensor(eh)).sum().backward()
    rc, rh = lstm_oracle.lstm_gates(c, i, u, f, o, bias=bias, forget_bias=fb)
    np.testing.assert_allclose(rc, cn.detach().numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(rh, hn.detach().numpy(), rtol=1e-13, atol=1e-13)
    grads = lstm_oracle.lstm_gates_grad(c, i, u, f, o, ec=ec, eh=eh, bias=bias, forget_bias=fb)
    for got, t in zip(grads, (tc, ti, tu, tf, to)):
        np.testing.assert_allclose(got, t.grad.numpy(), rtol=1e-12, atol=1e-13)
    h = np.concatenate([i, u, f, o], axis=-1)
    dc, dh, db = lstm_oracle.lstm_gates_fused_grad(c, h, ec=ec, eh=eh, bias=bias, forget_bias=fb)
    np.testing.assert_allclose(db, tb.grad.numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(dh, np.concatenate([t.grad.numpy() for t in (ti, tu, tf, to)], axis=-1), rtol=1e-12,
                               atol=1e-13)
    # a missing gradient is zero
    for kw in (dict(ec=ec), dict(eh=eh)):
        got = lstm_oracle.lstm_gates_grad(c, i, u, f, o, bias=bias, forget_bias=fb, **kw)
        full = lstm_oracle.lstm_gates_grad(c, i, u, f, o, ec=kw.get("ec", np.zeros_like(c)),
                                           eh=kw.get("eh", np.zeros_like(c)), bias=bias, forget_bias=fb)
        for a, b in zip(got, full):
            np.testing.assert_array_equal(a, b)


def test_sparse_relu_oracle():
    rng = np.random.default_rng(1)
    x = rng.normal(0, 1, (3, 4, 50))
    for alpha in (0.0, 0.5, 1.0, -0.3):
        m, s = x.mean(-1, keepdims=True), np.sqrt(((x - x.mean(-1, keepdims=True)) ** 2).mean(-1, keepdims=True))
        ref = np.where(x > m + alpha * s, x - (m + alpha * s), 0.0)
        np.testing.assert_allclose(lstm_oracle.sparse_relu(x, alpha), ref, rtol=1e-14, atol=1e-14)
        np.testing.assert_allclose(lstm.sparse_relu_test(x, alpha), ref, rtol=1e-14, atol=1e-14)
    y = lstm_oracle.sparse_relu(x)
    dy = rng.normal(0, 1, x.shape)
    # the gradient is relu's on the output, by definition: dy where y > 0
    g = lstm_oracle.sparse_relu_grad(dy, y)
    assert np.array_equal(g[y > 0], dy[y > 0]) and not g[y <= 0].any()
    assert not lstm_oracle.sparse_relu(np.full((2, 9), 3.25)).any()
    assert not lstm_oracle.sparse_relu(rng.normal(0, 1, (6, 1))).any()


def test_no_line_of_the_reference_lstm_source_in_oracle():
    """oracle/ref/lstm.cu reaches lstm_op_gpu.cu by #include; none of its lines is kept in the repository."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference", "src", "lstm_op_gpu.cu")
    if not os.path.isfile(src):
        pytest.skip("no reference checkout")
    with open(src, errors="replace") as fh:
        lines = {s for s in ("".join(line.split()) for line in fh) if len(s) >= 10}
    tracked = subprocess.run(["git", "ls-files", "oracle"], cwd=root, capture_output=True, text=True)
    if tracked.returncode != 0:
        pytest.skip("not a git checkout")
    for path in tracked.stdout.split():
        with open(os.path.join(root, path), errors="replace") as fh:
            for n, line in enumerate(fh, 1):
                assert "".join(line.split()) not in lines, "%s:%d repeats a line of lstm_op_gpu.cu" % (path, n)
