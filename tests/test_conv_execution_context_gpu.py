"""BlocksparseConv and BlocksparseDeconv in the other ways users run them, each bit for bit against an eager run on the
default stream: on a side stream whose inputs are still being written behind a torch.cuda._sleep, in a CUDA graph
replayed with new inputs, and on cuda:1 while cuda:0 is current. Each case runs forward, backward (dI and dF) and
l2_normalize with its gradient, on an overlapping, non-uniform layout, so the multi-pass accumulator, its memset and
cast, the updat workspace and the per-device tables are all on the path."""
import numpy as np
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv import BlocksparseConv, BlocksparseDeconv

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 1 << 22
BCK = [[list(range(0, 12)), list(range(0, 8))], [list(range(10, 40)), list(range(8, 36))],
       [list(range(5, 21)), list(range(3, 19))]]
OPS = {"conv": BlocksparseConv(BCK, (3, 3), (6, 7), strides=(1, 2)),
       "deconv": BlocksparseDeconv(BCK, (3, 3), (6, 7), strides=(1, 2))}
CASES = [(name, dt) for name in OPS for dt in (torch.bfloat16, torch.float32)]
IDS = ["%s-%s" % (n, str(d).split(".")[-1]) for n, d in CASES]


def make(op, dt, seed, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    r = lambda shape: (torch.rand(shape, generator=g) * 2 - 1).to(dt).to(device)
    return [r([op.sizeF]), r(op.i_shape(4)), r(op.o_shape(4)), r([op.sizeF])]


def run(op, F, I, E, U):
    f, x = F.detach().requires_grad_(), I.detach().requires_grad_()
    y = op(f, x)
    df, dx = torch.autograd.grad(y, (f, x), E)
    f2 = F.detach().requires_grad_()
    w = op.l2_normalize(f2)
    dw, = torch.autograd.grad(w, (f2,), U)
    return [y, dx, df, w, dw]


def _bits(t):
    t = t.detach().reshape(-1)
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _same(got, ref, what):
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(_bits(a), _bits(b)), "%s: output %d differs" % (what, i)


@pytest.mark.parametrize("name,dt", CASES, ids=IDS)
def test_side_stream(name, dt):
    op = OPS[name]
    staging = make(op, dt, 7)
    ref = run(op, *staging)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = run(op, *bufs)
    s.synchronize()
    _same(out, ref, name)


@pytest.mark.parametrize("name,dt", CASES, ids=IDS)
def test_graph_replay(name, dt):
    op = OPS[name]
    static = make(op, dt, 0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run(op, *static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run(op, *static)
    for i in range(1, 4):
        new = make(op, dt, i)
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        _same(out, run(op, *new), "%s replay %d" % (name, i))


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="needs two visible GPUs: runs the conv on cuda:1 while cuda:0 is current")
@pytest.mark.parametrize("name,dt", CASES, ids=IDS)
def test_second_gpu(name, dt):
    op = OPS[name]
    torch.cuda.set_device(0)
    ref = run(op, *make(op, dt, 11, "cuda:0"))
    out = run(op, *make(op, dt, 11, "cuda:1"))
    assert torch.cuda.current_device() == 0
    assert all(t.device == torch.device("cuda:1") for t in out)
    _same(out, ref, name + " on cuda:1")
    assert _lib.device_error() == 0
