"""The fused layer-norm / LSTM-gate entries refuse bad arguments with BSMM_E_ARG before anything is launched, and launch
nothing for empty input (no GPU needed: the pointers are fake and never dereferenced). grouped_lstm and
FusedBasicLSTMCell raise ValueError before reaching them, keep the reference's signatures less its variable scopes,
and stay out of lstm.__all__ and the package's __all__. The float64 oracle of the layer agrees with torch float64
autograd of the same formulas."""
import inspect

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import FusedBasicLSTMCell, _lib, grouped_lstm, lstm, lstm_layer
from oracle import lstm_layer_oracle

E_ARG, E_LIMIT = -3, -4
C, Z, G, B, CN, HN, MU, RS, EC, EH, DC, DZ, WS, DG, DB = (0x10000 * i for i in range(1, 16))


def _fwd(dtype=_lib.BF16, gdt=_lib.F32, c=C, z=Z, stride=256, g=G, b=B, cn=CN, hn=HN, mean=MU, rstd=RS, N=8, K=64,
         eps=1e-6):
    return _lib.load().bsmm_lstm_ln_gates(dtype, gdt, c, z, stride, g, b, cn, hn, mean, rstd, N, K, eps, 1.0, None)


def _grad(dtype=_lib.F16, gdt=_lib.F16, c=C, z=Z, stride=288, g=G, b=B, mean=MU, rstd=RS, ec=EC, eh=EH, dc=DC, dz=DZ,
          ws=WS, N=8, K=64):
    return _lib.load().bsmm_lstm_ln_gates_grad(dtype, gdt, c, z, stride, g, b, mean, rstd, ec, eh, dc, dz, ws, 0, N, K,
                                               1.0, None)


def _reduce(gdt=_lib.BF16, ws=WS, N=8, K=64, dg=DG, db=DB):
    return _lib.load().bsmm_lstm_ln_gates_grad_reduce(gdt, ws, N, K, dg, db, None)


CASES = [
    (_fwd, dict(dtype=3)), (_fwd, dict(gdt=-1)), (_fwd, dict(c=None)), (_fwd, dict(z=None)), (_fwd, dict(g=None)),
    (_fwd, dict(b=None)), (_fwd, dict(cn=None)), (_fwd, dict(hn=None)), (_fwd, dict(mean=None)),
    (_fwd, dict(rstd=None)), (_fwd, dict(N=-1)), (_fwd, dict(K=0)), (_fwd, dict(stride=255)), (_fwd, dict(eps=-1e-3)),
    (_fwd, dict(eps=float("nan"))),
    (_grad, dict(dtype=-1)), (_grad, dict(gdt=4)), (_grad, dict(c=None)), (_grad, dict(z=None)), (_grad, dict(g=None)),
    (_grad, dict(b=None)), (_grad, dict(mean=None)), (_grad, dict(rstd=None)), (_grad, dict(dc=None)),
    (_grad, dict(dz=None)), (_grad, dict(ws=None)), (_grad, dict(N=-2)), (_grad, dict(K=-1)), (_grad, dict(stride=0)),
    (_reduce, dict(gdt=3)), (_reduce, dict(ws=None)), (_reduce, dict(dg=None)), (_reduce, dict(db=None)),
    (_reduce, dict(N=-1)), (_reduce, dict(K=0)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_limits_and_workspace_size():
    before = _lib.last_kernel()
    assert _fwd(N=2 ** 62, stride=2 ** 22, K=2 ** 20) == E_LIMIT
    assert _fwd(K=2 ** 29, stride=2 ** 31) == E_LIMIT
    assert _grad(K=2 ** 29, stride=2 ** 31) == E_LIMIT
    assert _lib.last_kernel() == before
    ws = _lib.load().bsmm_lstm_ln_gates_workspace_bytes
    assert ws(0, 64) == 0 and ws(8, 0) == 0 and ws(-1, 64) == 0
    # one owner per row up to 264 rows, then ceil(N / ceil(N / 264)) owners: [2][P][4K] fp32
    assert ws(8, 64) == 2 * 8 * 256 * 4
    assert ws(264, 10) == 2 * 264 * 40 * 4
    assert ws(265, 10) == 2 * 133 * 40 * 4
    assert ws(10 ** 9, 16) == 2 * 264 * 64 * 4


def test_zero_sizes_launch_nothing():
    before = _lib.last_kernel()
    assert _fwd(N=0) == 0
    assert _grad(N=0) == 0
    assert _grad(N=0, ec=None, eh=None) == 0
    assert _reduce(N=0) == 0
    assert _lib.last_kernel() == before


def test_new_entries_are_bound():
    for name in ("bsmm_lstm_ln_gates", "bsmm_lstm_ln_gates_grad", "bsmm_lstm_ln_gates_grad_reduce",
                 "bsmm_lstm_ln_gates_workspace_bytes"):
        assert name in _lib.SIGNATURES


def test_python_argument_errors_raise_value_error():
    x, s = torch.zeros(4, 3, 5), torch.zeros(4, 6)
    k, b = torch.zeros(11, 24), torch.zeros(24)
    cpu = [lambda: grouped_lstm(x, 6, 3, [s, s], k, b, b),             # CPU tensors: no CPU path
           lambda: grouped_lstm(x, 6, 0, [s, s], k, b, b),             # timesteps
           lambda: grouped_lstm(x, 6, 2.0, [s, s], k, b, b),
           lambda: grouped_lstm(x, True, 3, [s, s], k, b, b),          # width
           lambda: FusedBasicLSTMCell(6, 5, forget_bias="1"),
           lambda: FusedBasicLSTMCell(6, 5, forget_bias=None),
           lambda: FusedBasicLSTMCell(6, 5, activation=torch.sigmoid),
           lambda: FusedBasicLSTMCell(0, 5),
           lambda: FusedBasicLSTMCell(6, 5, dtype=torch.float64),
           lambda: FusedBasicLSTMCell(6, 5)(x[:, 0], (s, s))]
    before = _lib.last_kernel()
    for call in cpu:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def test_reference_signatures():
    p = inspect.signature(grouped_lstm).parameters
    assert list(p) == ["inputs", "width", "timesteps", "initial_state", "kernel", "bias", "gain", "layernorm"]
    assert p["gain"].default is None and p["layernorm"].default is True
    p = inspect.signature(FusedBasicLSTMCell.__init__).parameters
    assert list(p) == ["self", "num_units", "input_size", "forget_bias", "state_is_tuple", "activation", "dtype",
                       "device"]
    assert [p[k].default for k in ("forget_bias", "state_is_tuple", "activation", "dtype", "device")] == \
        [1.0, True, None, torch.float32, None]
    cell = FusedBasicLSTMCell(6, 5)
    assert tuple(cell.kernel.shape) == (11, 24) and cell.kernel.dtype == torch.float32
    limit = np.sqrt(6.0 / (11 + 24))
    assert float(cell.kernel.detach().abs().max()) <= limit and not cell.bias.any()
    assert cell.state_size == (6, 6) and cell.output_size == 6
    assert FusedBasicLSTMCell(6, 5, state_is_tuple=False).state_size == 12


def test_names_and_all():
    assert lstm.__all__ == ["fused_lstm_gates", "split4", "concat4", "sparse_relu"]
    assert lstm_layer.__all__ == ["grouped_lstm", "FusedBasicLSTMCell"]
    for name in lstm_layer.__all__:
        assert getattr(blocksparse_b200, name) is getattr(lstm_layer, name) is getattr(lstm, name)
        assert name not in blocksparse_b200.__all__


# ---- the oracle against torch float64 autograd -------------------------------------------------------------------------
def _torch_layer(x, c, h, kernel, bias, gain, layernorm, eps):
    sig = torch.sigmoid
    outs = []
    for t in range(x.shape[1]):
        z = torch.cat([x[:, t], h], 1) @ kernel
        if layernorm:
            zs = z.reshape(z.shape[0], 4, -1)
            mu = zs.mean(2, keepdim=True)
            var = ((zs - mu) ** 2).mean(2, keepdim=True)
            z = ((zs - mu) / torch.sqrt(var + eps)).reshape(z.shape) * gain + bias
        else:
            z = z + bias
        i, u, f, o = z.chunk(4, 1)
        c = sig(f + 1.0) * c + sig(i) * torch.tanh(u)
        h = sig(o) * torch.tanh(c)
        outs.append(h)
    return torch.stack(outs, 1), c, h


@pytest.mark.parametrize("layernorm", [True, False])
def test_oracle_against_torch_float64_autograd(layernorm):
    rng = np.random.default_rng(3)
    N, T, In, W = 3, 4, 5, 6
    arrs = dict(x=rng.normal(0, 1, (N, T, In)), c=rng.normal(0, 1, (N, W)), h=rng.normal(0, 1, (N, W)),
                kernel=rng.normal(0, 0.4, (In + W, 4 * W)), bias=rng.normal(0, 0.5, 4 * W),
                gain=rng.normal(1, 0.3, 4 * W))
    d_out, d_c, d_h = rng.normal(0, 1, (N, T, W)), rng.normal(0, 1, (N, W)), rng.normal(0, 1, (N, W))
    eps = 1e-3                                 # large enough to matter in the comparison
    ts = {k: torch.tensor(v, requires_grad=True) for k, v in arrs.items()}
    out, cT, hT = _torch_layer(ts["x"], ts["c"], ts["h"], ts["kernel"], ts["bias"], ts["gain"], layernorm, eps)
    (out * torch.tensor(d_out)).sum().add_((cT * torch.tensor(d_c)).sum()).add_((hT * torch.tensor(d_h)).sum()).backward()
    gain = arrs["gain"] if layernorm else None
    ro, rc, rh = lstm_layer_oracle.grouped_lstm(arrs["x"], arrs["c"], arrs["h"], arrs["kernel"], arrs["bias"], gain,
                                                layernorm, eps=eps)
    for got, t in ((ro, out), (rc, cT), (rh, hT)):
        np.testing.assert_allclose(got, t.detach().numpy(), rtol=1e-12, atol=1e-13)
    grads = lstm_layer_oracle.grouped_lstm_grad(arrs["x"], arrs["c"], arrs["h"], arrs["kernel"], arrs["bias"], gain,
                                                layernorm, d_out, d_c, d_h, eps=eps)
    for got, name in zip(grads, ("x", "c", "h", "kernel", "bias", "gain")):
        if name == "gain" and not layernorm:
            assert got is None
            continue
        np.testing.assert_allclose(got, ts[name].grad.numpy(), rtol=1e-11, atol=1e-12, err_msg=name)


def test_cell_oracle_against_torch_float64_autograd():
    rng = np.random.default_rng(4)
    N, In, W, fb = 3, 5, 6, 0.5
    arrs = dict(x=rng.normal(0, 1, (N, In)), c=rng.normal(0, 1, (N, W)), h=rng.normal(0, 1, (N, W)),
                kernel=rng.normal(0, 0.4, (In + W, 4 * W)), bias=rng.normal(0, 0.5, 4 * W))
    d_h, d_c = rng.normal(0, 1, (N, W)), rng.normal(0, 1, (N, W))
    ts = {k: torch.tensor(v, requires_grad=True) for k, v in arrs.items()}
    i, u, f, o = (torch.cat([ts["x"], ts["h"]], 1) @ ts["kernel"] + ts["bias"]).chunk(4, 1)
    cn = torch.sigmoid(f + fb) * ts["c"] + torch.sigmoid(i) * torch.tanh(u)
    hn = torch.sigmoid(o) * torch.tanh(cn)
    (hn * torch.tensor(d_h) + cn * torch.tensor(d_c)).sum().backward()
    rh, rc = lstm_layer_oracle.cell_step(arrs["x"], arrs["c"], arrs["h"], arrs["kernel"], arrs["bias"], fb)
    np.testing.assert_allclose(rh, hn.detach().numpy(), rtol=1e-12, atol=1e-13)
    np.testing.assert_allclose(rc, cn.detach().numpy(), rtol=1e-12, atol=1e-13)
    grads = lstm_layer_oracle.cell_step_grad(arrs["x"], arrs["c"], arrs["h"], arrs["kernel"], arrs["bias"], d_h, d_c,
                                             fb)
    for got, name in zip(grads, ("x", "c", "h", "kernel", "bias")):
        np.testing.assert_allclose(got, ts[name].grad.numpy(), rtol=1e-11, atol=1e-12, err_msg=name)
