"""dw_matmul_large_n where N * C passes 2^31 elements (and each operand 4 GB): N = 2^25 + 64 rows of C = K = 64 fp16,
on both routes, elementwise against float64 within the bound of tests/test_dw_matmul_gpu.py."""
import pytest
import torch

from blocksparse_b200 import _lib, dw_matmul_large_n
from tests.test_dw_matmul_gpu import check_bound

pytestmark = pytest.mark.gpu

N, C, K = (1 << 25) + 64, 64, 64


def test_past_2_31_elements():
    assert N * C > 2 ** 31
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GB of free device memory")
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.empty((N, C), dtype=torch.float16, device="cuda")
    e = torch.empty((N, K), dtype=torch.float16, device="cuda")
    ref = torch.zeros((C, K), dtype=torch.float64, device="cuda")
    absref = torch.zeros_like(ref)
    step = 1 << 21
    for n0 in range(0, N, step):          # filled and reduced in float64 chunk by chunk, to stay within memory
        n1 = min(N, n0 + step)
        xs = torch.randn((n1 - n0, C), generator=g, device="cuda") + 0.1
        es = torch.randn((n1 - n0, K), generator=g, device="cuda") + 0.2
        x[n0:n1], e[n0:n1] = xs, es
        xd, ed = x[n0:n1].double(), e[n0:n1].double()
        ref += xd.t() @ ed
        absref += xd.abs().t() @ ed.abs()
    ref, absref = ref.cpu().numpy(), absref.cpu().numpy()
    for route, flags, kernel in (("tc", _lib.FLAG_FORCE_TC, "wgmma_dense_dw"),
                                 ("fma", _lib.FLAG_FORCE_GENERIC, "fma_dense_dw")):
        u = dw_matmul_large_n(x, e, flags=flags)
        assert _lib.last_kernel() == kernel
        torch.cuda.synchronize()
        assert _lib.device_error() == 0
        check_bound(u.cpu().numpy(), ref, absref, N, C, K, route == "tc", "N = %d %s" % (N, route))
