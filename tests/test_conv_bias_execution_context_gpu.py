"""ConvEdgeBias and cwise_linear in the other ways users run them, each bit for bit against an eager run on the default
stream: on a side stream whose inputs are still being written behind a torch.cuda._sleep, in a CUDA graph replayed with
new inputs, and on cuda:1 while cuda:0 is current. Each case runs the forward and the backward through autograd, so the
gradient workspaces, their partial sums and the per-device tables are on the path; the edge case also runs inference
in place."""
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv_bias import ConvEdgeBias, cwise_linear

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 1 << 22
EDGE = ConvEdgeBias([4, 12, 10, 24], [4, 24, 20, 16], [3, 3, 16, 24], strides=[1, 2, 2, 1])
CASES = [(kind, dt) for kind in ("edge", "cwise_nc", "cwise_ncdhw") for dt in (torch.bfloat16, torch.float32)]
IDS = ["%s-%s" % (k, str(d).split(".")[-1]) for k, d in CASES]
SHAPES = {"edge": [4, 12, 10, 24], "cwise_nc": [96, 40], "cwise_ncdhw": [4, 40, 6, 9]}


def make(kind, dt, seed, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    r = lambda shape, t=dt: (torch.rand(shape, generator=g) * 2 - 1).to(t).to(device)
    x, dy = r(SHAPES[kind]), r(SHAPES[kind])
    pshape = EDGE.shape if kind == "edge" else [SHAPES[kind][1]]
    return [x, dy, r(pshape, torch.float32), r(pshape, torch.float32)]


def run(kind, x, dy, g, b):
    xr, gr, br = x.detach().requires_grad_(), g.detach().requires_grad_(), b.detach().requires_grad_()
    if kind == "edge":
        y = EDGE(xr, gr, br)
    else:
        y = cwise_linear(xr, gr, br, relu=True, bias_first=kind == "cwise_nc")
    out = [y] + list(torch.autograd.grad(y, (xr, gr, br), dy))
    if kind == "edge":
        xi = x.clone()
        with torch.no_grad():
            EDGE(xi, g, b, inference=True)
        out.append(xi)
    return out


def _bits(t):
    t = t.detach().reshape(-1)
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _same(got, ref, what):
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(_bits(a), _bits(b)), "%s: output %d differs" % (what, i)


@pytest.mark.parametrize("kind,dt", CASES, ids=IDS)
def test_side_stream(kind, dt):
    staging = make(kind, dt, 7)
    ref = run(kind, *staging)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = run(kind, *bufs)
    s.synchronize()
    _same(out, ref, kind)


@pytest.mark.parametrize("kind,dt", CASES, ids=IDS)
def test_graph_replay(kind, dt):
    static = make(kind, dt, 0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run(kind, *static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run(kind, *static)
    for i in range(1, 4):
        new = make(kind, dt, i)
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        _same(out, run(kind, *new), "%s replay %d" % (kind, i))


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="needs two visible GPUs: runs the ops on cuda:1 while cuda:0 is current")
@pytest.mark.parametrize("kind,dt", CASES, ids=IDS)
def test_second_gpu(kind, dt):
    torch.cuda.set_device(0)
    ref = run(kind, *make(kind, dt, 11, "cuda:0"))
    out = run(kind, *make(kind, dt, 11, "cuda:1"))
    assert torch.cuda.current_device() == 0
    assert all(t.device == torch.device("cuda:1") for t in out)
    _same(out, ref, kind + " on cuda:1")
    assert _lib.device_error() == 0
