"""cwise_linear and ConvEdgeBias at the margins of their kernel routes: the cwise_linear backward with D*H*W > 1 gives
each thread the same elements in the same order on the 16-byte and the scalar route, so misaligned inputs (which take
the scalar route) give bit-identical dx, da and db; a channel or spatial dim of size 0 has empty sums in the backward as
in the forward; and an edge op whose tables are not yet on the device refuses to make its first call inside CUDA graph
capture, with a ValueError rather than a CUDA error."""
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv_bias import ConvEdgeBias, _cwise_linear_grad, cwise_linear

pytestmark = pytest.mark.gpu


def _misaligned(t):
    """t's values in a contiguous tensor that starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


def _bits(t):
    return t.detach().reshape(-1).view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16], ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("shape", [(6, 24, 40, 40), (3, 5, 4096), (2, 7, 16, 9, 8)], ids=lambda s: "x".join(map(str, s)))
def test_grad_routes_bit_identical(dt, shape):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.rand(shape, device="cuda", generator=g) * 2 - 1).to(dt)
    dy = (torch.rand(shape, device="cuda", generator=g) * 2 - 1).to(dt)
    a = torch.rand(shape[1], device="cuda", generator=g) * 2 - 1
    b = torch.rand(shape[1], device="cuda", generator=g) * 2 - 1
    ref = _cwise_linear_grad(dy, x, a, b, True, True)
    assert _lib.last_kernel() == "cwise_linear_grad_ncdhw"
    xm, dym = _misaligned(x), _misaligned(dy)
    assert xm.data_ptr() % 16 and dym.data_ptr() % 16
    got = _cwise_linear_grad(dym, xm, a, b, True, True)
    for r, o, what in zip(ref, got, ("dx", "da", "db")):
        assert torch.equal(_bits(r), _bits(o)), what


@pytest.mark.parametrize("shape", [(3, 0, 5), (3, 4, 0, 6), (0, 4, 5)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("gain,relu", [(True, True), (False, True), (False, False)])
def test_empty_shapes(shape, gain, relu):
    C = shape[1]
    x = torch.randn(shape, device="cuda").requires_grad_()
    a = torch.randn(C, device="cuda").requires_grad_() if gain else None
    b = torch.randn(C, device="cuda").requires_grad_()
    y = cwise_linear(x, a, b, relu=relu)
    assert y.shape == x.shape
    y.backward(torch.ones_like(y))
    assert x.grad.shape == x.shape
    assert b.grad.shape == (C,) and not b.grad.any()
    if gain:
        assert a.grad.shape == (C,) and not a.grad.any()


def test_first_call_inside_capture_is_refused():
    ConvEdgeBias.Cache.clear()             # a fresh geometry entry: no device copies yet
    op = ConvEdgeBias([2, 9, 11, 8], [2, 9, 11, 8], [3, 3, 8, 8], data_format="NHWC")
    x = torch.randn(2, 9, 11, 8, device="cuda")
    g = torch.randn(op.shape, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError, match="capture"):
        with torch.cuda.graph(graph, stream=s):
            op(x, g, g)
    torch.cuda.synchronize()
    y = op(x, g, g)                          # outside capture the tables are copied and the op runs
    torch.cuda.synchronize()
    assert y.shape == x.shape
