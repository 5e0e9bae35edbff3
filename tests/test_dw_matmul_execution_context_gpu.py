"""dw_matmul_large_n in the other ways users run it, each bit for bit against an eager run on the default stream: on a
side stream whose inputs are still being written behind a torch.cuda._sleep, in a CUDA graph replayed with new inputs,
and on cuda:1 while cuda:0 is current. The cases cover both routes, with and without the minibatch split (whose
workspace and second kernel are then on the path)."""
import pytest
import torch

from blocksparse_b200 import _lib, dw_matmul_large_n

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 1 << 22
CASES = [((65536, 64, 96), torch.float16, 0), ((4096, 512, 512), torch.bfloat16, 0),
         ((20000, 33, 70), torch.float32, 0), ((65536, 64, 96), torch.bfloat16, _lib.FLAG_FORCE_GENERIC)]
IDS = ["%s-%s-%s" % (s, str(d).split(".")[-1], "fma" if f else "auto") for s, d, f in CASES]


def make(shape, dt, seed, device="cuda"):
    N, C, K = shape
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand((N, n), generator=g) * 2 - 1).to(dt).to(device) for n in (C, K)]


def _same(a, b, what):
    assert torch.equal(a.view(torch.int32).cpu(), b.view(torch.int32).cpu()), what


@pytest.mark.parametrize("shape,dt,flags", CASES, ids=IDS)
def test_side_stream(shape, dt, flags):
    staging = make(shape, dt, 7)
    ref = dw_matmul_large_n(*staging, flags=flags)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = dw_matmul_large_n(*bufs, flags=flags)
    s.synchronize()
    _same(out, ref, "side stream")


@pytest.mark.parametrize("shape,dt,flags", CASES, ids=IDS)
def test_graph_replay(shape, dt, flags):
    static = make(shape, dt, 0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            dw_matmul_large_n(*static, flags=flags)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = dw_matmul_large_n(*static, flags=flags)
    for i in range(1, 4):
        new = make(shape, dt, i)
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        _same(out, dw_matmul_large_n(*new, flags=flags), "replay %d" % i)


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="needs two visible GPUs: runs the op on cuda:1 while cuda:0 is current")
@pytest.mark.parametrize("shape,dt,flags", CASES, ids=IDS)
def test_second_gpu(shape, dt, flags):
    torch.cuda.set_device(0)
    ref = dw_matmul_large_n(*make(shape, dt, 11, "cuda:0"), flags=flags)
    out = dw_matmul_large_n(*make(shape, dt, 11, "cuda:1"), flags=flags)
    assert torch.cuda.current_device() == 0
    assert out.device == torch.device("cuda:1")
    _same(out, ref, "cuda:1")
    assert _lib.device_error() == 0
