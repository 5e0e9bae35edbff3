"""Two-rank NCCL test of the data-parallel path ON THE GPU (skipped with fewer than two GPUs): every rank runs the
wgmma updat kernel on its minibatch shard, the partial dW is all-reduced (blocking, and on the side stream the
benchmark uses) in bf16 and in fp32, and the result is compared with the oracle's full-minibatch updat.  fprop of a
shard is checked against the oracle on that shard.  Run it on a machine with two GPUs: `python -m pytest tests/test_dist_nccl_gpu.py -m gpu`."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests._util import ref_errors

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, out):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
        from blocksparse_b200 import BlocksparseMatMul, _lib
        from blocksparse_b200 import dist as bdist
        from oracle.bsmm_oracle import MatmulOracle
        rng = np.random.default_rng(9)
        lay = (rng.random((16, 12)) < 0.3).astype(np.int32)
        lay[0, 0] = 1
        bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
        orc = MatmulOracle(lay, 32, 1)
        N = 1000                                              # 500 rows per rank
        W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).bfloat16()
        X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).bfloat16()
        E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).bfloat16()
        xs = bdist.shard_minibatch(X, 1).cuda()
        es = bdist.shard_minibatch(E, 1).cuda()
        ref = orc.updat(X.float().numpy(), E.float().numpy())
        errs = {}
        for name, dw_dtype in (("bf16", None), ("fp32", torch.float32)):
            dw = bsmm.updat([xs], [es], dw_dtype=dw_dtype)
            assert _lib.last_kernel().startswith("wgmma_updat"), _lib.last_kernel()
            bdist.allreduce_dw(dw)
            errs["blocking " + name] = ref_errors(dw.float().cpu().numpy(), ref)
            side = bdist.AllreduceStream(torch.device("cuda", rank))
            dw2 = bsmm.updat([xs], [es], dw_dtype=dw_dtype)
            side.reduce(dw2)
            y = bsmm.fprop(xs, W.cuda())                      # overlaps the reduction
            side.wait()
            errs["side-stream " + name] = ref_errors(dw2.float().cpu().numpy(), ref)
        a, b = bdist.shard_bounds(N, rank, world)
        errs["fprop shard"] = ref_errors(y.float().cpu().numpy(), orc.fprop(X.float().numpy()[a:b], W.float().numpy()))
        assert _lib.device_error() == 0
        out[rank] = errs
        dist.destroy_process_group()
    except Exception as e:                                      # surface the failure in the parent
        out[rank] = "error: %r" % (e,)
        raise


def test_two_rank_nccl_dw_allreduce_matches_full_batch_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    world = 2
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    for r in range(world):
        assert isinstance(out[r], dict), out[r]
        for what, (mx, l2) in out[r].items():
            tol = (4e-2, 1e-2) if "bf16" in what or "fprop" in what else (1e-2, 2e-3)   # fp32 dW: only the bf16 inputs round
            assert mx <= tol[0] and l2 <= tol[1], "rank %d %s: max %.3e l2 %.3e" % (r, what, mx, l2)
