"""ConvEdgeBias and cwise_linear on tensors past 2^31 elements, where 32-bit and 64-bit offsets part ways: the forward
and dx are checked whole for NaN (each output starts as NaN) and against float64 on sampled images (the first, the last,
both sides of offset 2^31, seeded random ones); dg / db and da / db whole against float64 sums formed on the device.
The edge case runs both data formats and inference in place on the same tensor."""
import numpy as np
import pytest
import torch

from blocksparse_b200.conv_bias import ConvEdgeBias, cwise_linear
from tests._util import _on_poisoned_output
from tests.test_large_offsets_gpu import _need, _no_nan, sample_ids

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
U, EPS = 2.0 ** -24, 2.0 ** -8
H = W = 64
K = 16
N = 2 ** 31 // (K * H * W) + 4                 # N * K * H * W = 2^31 + 2^18


def _within(got, ref, lim, what):
    err = np.abs(got - ref)
    assert (err <= lim).all(), "%s: worst %.3e vs bound %.3e" % (what, err.max(), lim[np.argmax(err - lim)])


def _device_sums(fn, n, step=256):
    """sum over images of fn(slice) in float64, formed on the device in slices."""
    out = None
    for i in range(0, n, step):
        r = fn(slice(i, i + step))
        out = r if out is None else out + r
    return out.cpu().numpy()


@pytest.mark.parametrize("fmt", ["NHWC", "NCHW"])
def test_edge_bias_past_2_31(fmt):
    _need(26, "a bf16 edge bias of 2^31 + 2^18 elements with its gradient")
    shape = [N, H, W, K] if fmt == "NHWC" else [N, K, H, W]
    op = ConvEdgeBias(shape, shape, [3, 3, K, K], data_format=fmt)
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = (torch.rand(shape, device="cuda", generator=gen) * 2 - 1).to(BF16)
    assert x.numel() > 2 ** 31
    g = torch.rand(op.shape, device="cuda", generator=gen) * 2 - 1
    b = torch.rand(op.shape, device="cuda", generator=gen) * 2 - 1
    ids = sample_ids(N, 2 ** 31 // (K * H * W), np.random.default_rng(1))
    P = H * W
    pe = torch.as_tensor(op._pos_edge).long().cuda()
    on = pe >= 0
    ge = g[pe.clamp(min=0)] if fmt == "NHWC" else g[:, pe.clamp(min=0)]          # per position (P, K) / (K, P)
    be = b[pe.clamp(min=0)] if fmt == "NHWC" else b[:, pe.clamp(min=0)]
    mask = on[:, None] if fmt == "NHWC" else on[None, :]
    view = lambda t: t.reshape(t.shape[0], P, K) if fmt == "NHWC" else t.reshape(t.shape[0], K, P)

    def ref_y(xs):
        xs = view(xs.double())
        return torch.where(mask, xs * ge.double() + be.double(), xs), torch.where(mask, xs.abs() * ge.abs().double() + be.abs().double(), xs.abs())

    y = _on_poisoned_output(lambda: op._forward(x, g, b, torch.empty_like(x), False))
    _no_nan(y, "y")
    r, m = ref_y(x[ids])
    _within(view(y[ids]).double().cpu().numpy(), r.cpu().numpy(), ((U + EPS) * m).cpu().numpy() + 1e-38, "y")
    dy = y
    del r, m
    dx, dg, db = _on_poisoned_output(lambda: op._backward(dy, x, g))
    _no_nan(dx, "dx")
    d, xs = view(dy[ids].double()), view(x[ids].double())
    _within(view(dx[ids]).double().cpu().numpy(), torch.where(mask, d * ge.double(), d).cpu().numpy(),
            ((U + EPS) * torch.where(mask, d.abs() * ge.abs().double(), d.abs())).cpu().numpy() + 1e-38, "dx")
    del dx
    onehot = (pe[:, None] == torch.arange(op.edgeBiasDim, device="cuda")[None, :]).double()          # (P, E)
    eq = "npk,pe->ek" if fmt == "NHWC" else "nkp,pe->ke"
    sg = _device_sums(lambda s: torch.einsum(eq, view(dy[s].double()) * view(x[s].double()), onehot), N)
    sga = _device_sums(lambda s: torch.einsum(eq, (view(dy[s].double()) * view(x[s].double())).abs(), onehot), N)
    sb = _device_sums(lambda s: torch.einsum(eq, view(dy[s].double()), onehot), N)
    sba = _device_sums(lambda s: torch.einsum(eq, view(dy[s].double()).abs(), onehot), N)
    L = N * op._max_count + 64
    _within(dg.double().cpu().numpy(), sg, (L + 1) * U * sga, "dg")
    _within(db.double().cpu().numpy(), sb, (L + 1) * U * sba, "db")
    del dy, y
    # inference in place: the edges of the sampled images change, the rest stays
    x0 = x[ids].clone()
    with torch.no_grad():
        op(x, g, b, inference=True)
    r, m = ref_y(x0)
    _within(view(x[ids]).double().cpu().numpy(), r.cpu().numpy(), ((U + EPS) * m).cpu().numpy() + 1e-38, "inference")


@pytest.mark.parametrize("shape", [(2 ** 31 // 64 + 1024, 64), (2 ** 31 // (48 * 4096) + 2, 48, 64, 64)],
                         ids=["nc", "ncdhw"])
def test_cwise_linear_past_2_31(shape):
    _need(26, "a bf16 cwise_linear of more than 2^31 elements with its gradient")
    C = shape[1]
    gen = torch.Generator(device="cuda").manual_seed(4)
    x = (torch.rand(shape, device="cuda", generator=gen) * 2 - 1).to(BF16)
    assert x.numel() > 2 ** 31
    a = torch.rand(C, device="cuda", generator=gen) * 2 - 1
    b = torch.rand(C, device="cuda", generator=gen) * 2 - 1
    bc = [1, C] + [1] * (len(shape) - 2)
    A, B = a.double().view(bc), b.double().view(bc)
    n = shape[0]
    cross = 2 ** 31 // (x.numel() // n)
    ids = sample_ids(n, cross, np.random.default_rng(2))
    y = _on_poisoned_output(lambda: cwise_linear(x, a, b))
    _no_nan(y, "y")
    xs = x[ids].double()
    _within(y[ids].double().cpu().numpy(), (A * xs + B).cpu().numpy(),
            ((U + EPS) * (A.abs() * xs.abs() + B.abs())).cpu().numpy() + 1e-38, "y")
    del y
    xr, ar, br = x.requires_grad_(), a.requires_grad_(), b.requires_grad_()
    dy = x.detach()
    dx, da, db = _on_poisoned_output(lambda: torch.autograd.grad(cwise_linear(xr, ar, br), (xr, ar, br), dy))
    _no_nan(dx, "dx")
    _within(dx[ids].double().cpu().numpy(), (A * xs).cpu().numpy(), ((U + EPS) * (A.abs() * xs.abs())).cpu().numpy()
            + 1e-38, "dx")
    del dx
    axes = [0] + list(range(2, len(shape)))
    sa = _device_sums(lambda s: (dy[s].double() ** 2).sum(axes), n, 4096)
    sb = _device_sums(lambda s: dy[s].double().sum(axes), n, 4096)
    sba = _device_sums(lambda s: dy[s].double().abs().sum(axes), n, 4096)
    L = x.numel() // C + 64
    _within(da.double().cpu().numpy(), sa, L * U * sa + 1e-30, "da")
    _within(db.double().cpu().numpy(), sb, L * U * sba + 1e-30, "db")
