"""Data-parallel use of the block-sparse matmul: the minibatch axis is sharded across ranks.

fprop and bprop are independent per minibatch column, so they need no communication.  updat reduces over
the minibatch: each rank produces the partial dW of its shard and the true dW is the SUM over ranks -- one
all-reduce per weight tensor (the reference leaves this to user code through its
AllreduceNccl op, examples/transformer/enwik8.py:220-231).  One process per GPU, torch.distributed (NCCL on
GPUs; the same code runs on gloo for the CPU tests of the host logic).
"""
import torch
import torch.distributed as dist


def shard_bounds(N, rank, world):
    """Contiguous, balanced [start, stop) of rank's slice of a minibatch of N columns (first N % world ranks get one more)."""
    base, extra = divmod(N, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_minibatch(t, feature_axis, rank=None, world=None):
    """Slice a (C, N) [axis 0] or (N, C) [axis 1] activation tensor to this rank's minibatch shard."""
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    N = t.shape[1] if feature_axis == 0 else t.shape[0]
    a, b = shard_bounds(N, rank, world)
    return t[:, a:b] if feature_axis == 0 else t[a:b]


def allreduce_dw(dw, group=None, average=False, async_op=False):
    """Sum (or average) the partial weight gradient over ranks, in place.  Returns the work handle if async_op."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return None
    work = dist.all_reduce(dw, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
    if average:
        if async_op:
            work.wait()
        dw.div_(dist.get_world_size(group))
    return work if async_op else None


def reserve_sms_for_nccl(n_sms=8, nccl_ctas=None):
    """Leave `n_sms` SMs to a concurrent NCCL kernel.

    NCCL is capped to that many CTAs (NCCL_MAX_CTAS) and the host-built updat schedule balances its tiles over
    sm_count - n_sms SMs (csrc/common.cuh:sm_margin, _lib.grid_sms), so a dW all-reduce on a side stream and the next
    block-sparse kernels can run side by side.
    Must be called before the first block-sparse op and before the process group is created; explicit environment
    settings win.  Returns the margin in effect.
    """
    import os
    os.environ.setdefault("BSMM_SM_MARGIN", str(int(n_sms)))
    margin = int(os.environ["BSMM_SM_MARGIN"])
    if margin > 0:
        os.environ.setdefault("NCCL_MAX_CTAS", str(int(nccl_ctas or margin)))
    return margin


def nccl_options():
    """ProcessGroupNCCL options for runs that overlap the dW all-reduce with the block-sparse kernels: the collective runs
    on a HIGH-PRIORITY stream.  The next compute kernel and the NCCL kernel become runnable at the same moment (when updat
    retires); with priority the NCCL CTAs are placed first instead of waiting for a whole compute grid to drain."""
    opts = dist.ProcessGroupNCCL.Options()
    opts.is_high_priority_stream = True
    return opts


class AllreduceStream(object):
    """Issue the dW all-reduce on a side stream ordered after the updat kernel by an event, so that the next layer's
    bprop overlaps it (the reference's AllreduceNccl pattern, src/nccl_op.cc:168,513)."""

    def __init__(self, device):
        self.stream = torch.cuda.Stream(device=device)
        self.pending = []

    def reduce(self, dw):
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            dist.all_reduce(dw)
        dw.record_stream(self.stream)          # allocated on the compute stream, consumed on this one
        self.pending.append(dw)
        return dw

    def wait(self):
        """Order the current stream after every reduction issued so far (device-side dependency, no host sync)."""
        if self.pending:
            torch.cuda.current_stream().wait_stream(self.stream)
        done, self.pending = self.pending, []
        return done
