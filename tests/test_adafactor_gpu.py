"""AdafactorOptimizer on the GPU, checked elementwise against the float64 oracle (oracle/adafactor_oracle.py) given the
same rounded inputs, bit for bit against itself in every execution context, and against the reference's own kernels.

Tolerance (REL below). Every cross-tile sum is added in fp64, so the fp32 rounding chains have a length fixed by the
tile shapes, not by the tensor: at most 40 fp32 additions (a thread's 32 squares of a 64 x 128 tile or 8192-element
chunk, then 8 levels of the block tree) for a sum of squares, 16 for a column sum and 9 for a row sum. Each sum is
then within 40 * 2^-24 of exact, rv and cv within that plus one rounding of the decayed update, and x within half of
their errors (square roots) plus two rsqrtf (2 ulp each) and three products. The update p_old - p_new, formed from fp32
params, also carries one rounding of p_new (2^-24 |p_new|). 64 * 2^-23 relative covers all of it with margin.
"""
import copy
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from blocksparse_b200 import AdafactorOptimizer, _lib, clip_by_global_norm
from oracle import adafactor_oracle as ao

pytestmark = pytest.mark.gpu

GDTYPES = [torch.float32, torch.float16, torch.bfloat16]
REL = 64 * 2.0 ** -23
SHAPES = [(1003,), (1, 1003), (3, 1), (37, 129), (64, 256), (256, 64), (300, 260), (0,), (5, 0)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")


def _np(t):
    return None if t is None else t.detach().double().cpu().numpy()


def _f32(v):
    return float(np.float32(v))


def _host_decay(beta2, d1, d2):
    f = np.float32
    return float(f(beta2) * (f(1) - f(d1)) / (f(1) - f(d2)))


def _view(shape, dtype, offset, rng, scale=1.0):
    """A tensor of `shape` at `offset` elements into a larger buffer (offset 1: no 16-byte access)."""
    n = int(np.prod(shape))
    base = torch.as_tensor(rng.normal(0, scale, n + offset + 3).astype(np.float32)).to(dtype).cuda()
    return base[offset:offset + n].view(shape)


def _set_state(opt, p, rng):
    """Random positive moments; returns (cv, rv) as float64 (rv None when unfactored)."""
    factored = p.dim() == 2 and p.shape[0] > 1
    cv = torch.as_tensor(rng.uniform(1e-3, 1e-2, p.shape[1] if factored else p.numel()).astype(np.float32)).cuda()
    opt.state[p]["cv"] = cv
    if factored:
        opt.state[p]["rv"] = torch.as_tensor(rng.uniform(1e-3, 1e-2, p.shape[0]).astype(np.float32)).cuda()
    return _np(cv), _np(opt.state[p].get("rv"))


def _close(got, ref, what, scale=None):
    if ref is None:
        assert got is None, what
        return
    tol = REL * np.abs(ref) + (0 if scale is None else scale)
    bad = np.abs(got - ref) > tol
    assert not bad.any(), "%s: %d of %d off, worst %.3e (tol %.3e)" % (
        what, bad.sum(), bad.size, np.abs(got - ref).max(), REL * np.abs(ref).max())


def _check(opt, p, p0, cv0, rv0, g_np, what, lr, decay, **kw):
    kw = {k: _f32(v) if isinstance(v, float) else v for k, v in kw.items()}
    pr, cvr, rvr = ao.adafactor(g_np, p0, cv0, rv0, lr=_f32(lr), decay=decay, **kw)
    pn = _np(p)
    _close(pn - p0, pr - p0, what + " update", scale=2.0 ** -24 * np.abs(pn))
    _close(_np(opt.state[p]["cv"]), cvr, what + " cv")
    _close(_np(opt.state[p].get("rv")), rvr, what + " rv")


def _opt(params, **kw):
    args = dict(learning_rate=0.01, beta2=0.9, epsilon=1e-30, zero_init_variables=True)     # decay == beta2
    args.update(kw)
    return AdafactorOptimizer(params, **args)


@pytest.mark.parametrize("gdtype", GDTYPES, ids=lambda d: str(d).replace("torch.", ""))
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_every_tensor_class_matches_oracle(shape, gdtype):
    rng = np.random.default_rng(sum(shape) + 7 * GDTYPES.index(gdtype))
    for offset in (0, 1):                                  # offset 1: the scalar path
        p = _view(shape, torch.float32, offset, rng, 0.5)
        g = _view(shape, gdtype, offset, rng, 0.1)
        opt = _opt([p])
        cv0, rv0 = _set_state(opt, p, rng)
        p0, g_np = _np(p), _np(g)
        opt.step(grads=[g])
        if p.numel() == 0:
            continue
        _check(opt, p, p0, cv0, rv0, g_np, "%s %s offset %d" % (shape, gdtype, offset), 0.01, _f32(0.9))


def test_grad_at_odd_offset_next_to_aligned_param():
    """Only the grad is misaligned: the tensor takes the scalar path as a whole."""
    rng = np.random.default_rng(5)
    p = torch.as_tensor(rng.normal(0, 1, (40, 132)).astype(np.float32)).cuda()
    g = _view((40, 132), torch.bfloat16, 1, rng, 0.1)
    opt = _opt([p])
    cv0, rv0 = _set_state(opt, p, rng)
    p0 = _np(p)
    opt.step(grads=[g])
    _check(opt, p, p0, cv0, rv0, _np(g), "odd grad", 0.01, _f32(0.9))


def test_more_tensors_than_one_table_mixed_classes():
    rng = np.random.default_rng(9)
    shapes = []
    for i in range(420):
        c = i % 4
        shapes.append([(int(rng.integers(1, 3000)),), (1, int(rng.integers(1, 500))), (0,),
                       (int(rng.integers(2, 70)), int(rng.integers(1, 300)))][c])
    ps = [_view(s, torch.float32, int(rng.integers(0, 2)), rng) for s in shapes]
    gs = [_view(s, GDTYPES[i % 3], 0, rng, 0.1) for i, s in enumerate(shapes)]
    opt = _opt(ps)
    olds = [(_np(p), *_set_state(opt, p, rng)) for p in ps]
    opt.step(grads=gs)
    for i, (p, g, (p0, cv0, rv0)) in enumerate(zip(ps, gs, olds)):
        if p.numel():
            _check(opt, p, p0, cv0, rv0, _np(g), "tensor %d %s" % (i, tuple(p.shape)), 0.01, _f32(0.9))


def _pair(rng):
    ps = [_view((96, 200), torch.float32, 0, rng), _view((777,), torch.float32, 0, rng)]
    gs = [_view(p.shape, torch.float16, 0, rng, 0.1) for p in ps]
    return ps, gs


@pytest.mark.parametrize("ns", [None, 0.5, 0.0, "other_device"])
def test_norm_scale(ns):
    rng = np.random.default_rng(13)
    if ns == "other_device":
        if torch.cuda.device_count() < 2:
            pytest.skip("needs two visible GPUs: norm_scale on cuda:1 for params on cuda:0")
        nst = torch.full((), 0.75, device="cuda:1")
    else:
        nst = None if ns is None else torch.full((), ns, device="cuda")
    ps, gs = _pair(rng)
    opt = _opt(ps)
    olds = [(p.clone(), *_set_state(opt, p, rng)) for p in ps]
    bits = [{k: v.clone() for k, v in opt.state[p].items()} for p in ps]
    opt.step(grads=gs, norm_scale=nst)
    if ns == 0.0:
        for p, (pb, _, _), st in zip(ps, olds, bits):
            assert torch.equal(p.view(torch.int32), pb.view(torch.int32))
            for k, v in st.items():
                assert torch.equal(opt.state[p][k].view(torch.int32), v.view(torch.int32)), k
        assert opt.param_groups[0]["decay1_power"] == 0.0                  # zero_init: the powers stay 0
        return
    scale = 1.0 if ns is None else (0.75 if ns == "other_device" else ns)
    for p, g, (pb, cv0, rv0) in zip(ps, gs, olds):
        _check(opt, p, _np(pb), cv0, rv0, _np(g), "norm_scale %s" % ns, 0.01, _f32(0.9), norm_scale=_f32(scale))


@pytest.mark.parametrize("case", ["saturate", "zero_infs_nans", "grad_scale", "clip_active", "clip_inactive"])
def test_conditioning_and_clipping(case):
    rng = np.random.default_rng(17)
    kw = dict(saturate=dict(saturate=0.05, zero_nans=True), zero_infs_nans=dict(zero_infs=True, zero_nans=True),
              grad_scale=dict(grad_scale=0.25), clip_active=dict(clip_thresh=0.05),
              clip_inactive=dict(clip_thresh=1e6))[case]
    for gdtype in GDTYPES:
        ps = [_view((70, 130), torch.float32, 0, rng), _view((5000,), torch.float32, 0, rng)]
        gs = [_view(p.shape, gdtype, 0, rng, 0.1) for p in ps]
        if case in ("saturate", "zero_infs_nans"):
            for g in gs:
                flat = g.view(-1)
                for v in ("inf", "-inf", "nan"):
                    flat[torch.as_tensor(rng.integers(0, flat.numel(), 20)).cuda()] = float(v)
        opt = _opt(ps, **kw)
        olds = [(_np(p), *_set_state(opt, p, rng)) for p in ps]
        opt.step(grads=gs)
        okw = dict(kw)
        for p, g, (p0, cv0, rv0) in zip(ps, gs, olds):
            assert torch.isfinite(p).all()
            _check(opt, p, p0, cv0, rv0, _np(g), "%s %s" % (case, gdtype), 0.01, _f32(0.9), **okw)
            if case.startswith("clip"):                  # active: the step's rms is cut to clip_thresh
                rms = np.sqrt(np.mean(((p0 - _np(p)) / 0.01) ** 2))
                assert (abs(rms - 0.05) < 1e-3) if case == "clip_active" else rms > 0.1, (case, rms)


@pytest.mark.parametrize("zero_init", [False, True])
def test_five_steps_from_the_state_each_leaves(zero_init):
    rng = np.random.default_rng(19)
    ps = [_view(s, torch.float32, 0, rng) for s in ((50, 300), (1, 999), (4097,))]
    beta2 = 0.8
    opt = AdafactorOptimizer(ps, learning_rate=0.02, beta2=beta2, zero_init_variables=zero_init)
    for t in range(5):
        gs = [_view(p.shape, torch.bfloat16, 0, rng, 0.1) for p in ps]
        grp = opt.param_groups[0]
        decay = _host_decay(beta2, grp["decay1_power"], grp["decay2_power"])
        olds = []
        for p in ps:
            st = opt.state[p]
            factored = p.dim() == 2 and p.shape[0] > 1
            if "cv" not in st:
                olds.append((_np(p), np.zeros(p.shape[1] if factored else p.numel()),
                             np.zeros(p.shape[0]) if factored else None))
            else:
                olds.append((_np(p), _np(st["cv"]), _np(st.get("rv"))))
        opt.step(grads=gs)
        for p, g, (p0, cv0, rv0) in zip(ps, gs, olds):
            _check(opt, p, p0, cv0, rv0, _np(g), "step %d %s" % (t, tuple(p.shape)), 0.02, decay)
    want = (0.0, 0.0) if zero_init else (beta2 ** 6, beta2 ** 7)
    assert opt.param_groups[0]["decay1_power"] == pytest.approx(want[0], rel=1e-5)
    assert opt.param_groups[0]["decay2_power"] == pytest.approx(want[1], rel=1e-5)


def test_bitwise_determinism_and_state_dict_resume():
    rng = np.random.default_rng(23)
    shapes = [(300, 260), (37, 129), (1003,)]
    init = [_view(s, torch.float32, 0, rng) for s in shapes]
    grads = [[_view(s, torch.float16, 0, rng, 0.1) for s in shapes] for _ in range(6)]
    runs = []
    for _ in range(2):
        ps = [p.clone() for p in init]
        opt = AdafactorOptimizer(ps, learning_rate=0.01, clip_thresh=0.5)
        for gs in grads:
            opt.step(grads=gs)
        runs.append((ps, opt))
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    ps = [p.clone() for p in init]
    opt = AdafactorOptimizer(ps, learning_rate=0.01, clip_thresh=0.5)
    for gs in grads[:3]:
        opt.step(grads=gs)
    saved = copy.deepcopy(opt.state_dict())
    ps2 = [p.detach().clone() for p in ps]
    opt2 = AdafactorOptimizer(ps2, learning_rate=0.3, clip_thresh=0.5)
    opt2.load_state_dict(saved)
    assert opt2.param_groups[0]["lr"] == 0.01
    for gs in grads[3:]:
        opt2.step(grads=gs)
    ref_ps, ref_opt = runs[0]
    for a, b in zip(ref_ps, ps2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        for k in ref_opt.state[a]:
            assert torch.equal(ref_opt.state[a][k].view(torch.int32), opt2.state[b][k].view(torch.int32)), k


def test_peak_memory_is_the_workspace_only():
    """A step allocates the workspace of partial sums and nothing of the param's size (no fp32 x temporary)."""
    rng = np.random.default_rng(29)
    p = _view((4096, 4096), torch.float32, 0, rng)
    g = _view((4096, 4096), torch.bfloat16, 0, rng, 0.1)
    opt = _opt([p])
    opt.step(grads=[g])                                     # state exists
    rows, cols = np.array([4096], np.int64), np.array([4096], np.int64)
    ws = _lib.load().bsmm_adafactor_workspace_bytes(1, rows.ctypes.data, cols.ctypes.data)
    assert ws < 0.03 * p.numel() * 4
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    opt.step(grads=[g])
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    rounded = -(-ws // (2 << 20)) * (2 << 20)               # the caching allocator hands out 2 MiB multiples here
    assert extra <= rounded and extra < p.numel(), (extra, ws)   # an fp32 x temporary would be 64 MiB


_LAUNCHES = """
import json, sys
sys.path.insert(0, %r)
import torch
from torch.profiler import ProfilerActivity, profile
from blocksparse_b200 import AdafactorOptimizer
g = torch.Generator().manual_seed(31)
shapes = [(int(torch.randint(2, 200, (), generator=g)), int(torch.randint(1, 300, (), generator=g))) for _ in range(150)]
ps = [torch.randn(s, generator=g).cuda() for s in shapes + [(1000,)] * 50]
gs = [torch.randn_like(p).half() for p in ps]
opt = AdafactorOptimizer(ps)
opt.step(grads=gs)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    opt.step(grads=gs)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_five_launches_per_step():
    """200 params of both classes in one table: exactly the five kernels, in order. The profile runs in a child process,
    so that its profiler session leaves this process's profiler state as it found it."""
    out = subprocess.run([sys.executable, "-c", _LAUNCHES % ROOT], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    k = json.loads(out.stdout.strip().splitlines()[-1])
    names = ["stats", "finish", "sumsq", "rate", "apply"]
    assert len(k) == 5 and all("mt_adafactor_" + n in s for n, s in zip(names, k)), k


def test_no_host_synchronisation():
    rng = np.random.default_rng(31)
    ps = [_view(s, torch.float32, 0, rng) for s in ((300, 260), (37, 129), (1003,))]
    gs = [torch.randn_like(p).half() for p in ps]
    opt = AdafactorOptimizer(ps)
    opt.step(grads=gs)                                      # state is created outside the check
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _, scale = clip_by_global_norm(gs)
        opt.step(grads=gs, norm_scale=scale)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ---- execution contexts, bit for bit against eager on cuda:0 -------------------------------------------------------------
def _make(seed, dev):
    g = torch.Generator().manual_seed(seed)
    rn = lambda s, dt=torch.float32, sc=1.0: (torch.randn(s, generator=g) * sc).to(dt).to(dev)
    return [rn((64, 96)), rn((1003,)), rn((37, 129)), rn((64, 96), torch.bfloat16, 0.1), rn((1003,), torch.float16, 0.1),
            rn((37, 129), torch.float32, 0.1)]


def _run(p1, p2, p3, g1, g2, g3):
    ps = [p1.clone(), p2.clone(), p3.clone()]
    opt = AdafactorOptimizer(ps, learning_rate=0.01, clip_thresh=0.5, zero_init_variables=True)
    _, scale = clip_by_global_norm([g1, g2, g3], clip_norm=1.0)
    opt.step(grads=[g1, g2, g3], norm_scale=scale)
    opt.step(grads=[g1, g2, g3])
    return ps + [v for p in ps for v in opt.state[p].values()]


def _same(got, ref, what):
    assert len(got) == len(ref), what
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape and torch.equal(a.view(torch.int32).cpu(), b.view(torch.int32).cpu()), (what, i)


def test_side_stream():
    staging = _make(7, "cuda")
    ref = _run(*staging)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 22)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = _run(*bufs)
    s.synchronize()
    _same(out, ref, "side stream")


def test_graph_replay():
    static = _make(0, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _run(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _run(*static)
    for i in range(1, 4):
        new = _make(i, "cuda")
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        _same(out, _run(*new), "replay %d" % i)


def test_graph_refuses_non_zero_decay_powers():
    p = torch.randn(64, 96, device="cuda")
    g = torch.randn(64, 96, device="cuda")
    opt = AdafactorOptimizer([p], learning_rate=0.01)
    opt.step(grads=[g])                                     # state exists: nothing to allocate under capture
    before, powers = p.clone(), dict(opt.param_groups[0])
    kernel = _lib.last_kernel()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError, match="zero_init_variables"):
        with torch.cuda.graph(graph):
            opt.step(grads=[g])
    assert torch.equal(p, before) and _lib.last_kernel() == kernel
    assert opt.param_groups[0]["decay1_power"] == powers["decay1_power"]
    opt.step(grads=[g])
    assert not torch.equal(p, before)


def test_two_host_threads():
    inputs = [_make(80 + i, "cuda") for i in range(2)]
    refs = [_run(*ins) for ins in inputs]
    torch.cuda.synchronize()
    barrier = threading.Barrier(2)
    results, errors = [None, None], []

    def worker(i):
        try:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.default_stream())
            barrier.wait()
            with torch.cuda.stream(s):
                results[i] = _run(*inputs[i])
            s.synchronize()
        except BaseException as e:
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for i in range(2):
        _same(results[i], refs[i], "thread %d" % i)


@two_gpus
def test_second_gpu():
    torch.cuda.set_device(0)
    ref = _run(*_make(11, "cuda:0"))
    out = _run(*_make(11, "cuda:1"))
    assert torch.cuda.current_device() == 0 and all(t.device == torch.device("cuda:1") for t in out)
    _same(out, ref, "cuda:1")


@two_gpus
def test_params_split_over_two_gpus():
    """One optimizer over params on cuda:0 and cuda:1 equals one per device, bit for bit; norm_scale from cuda:0."""
    torch.cuda.set_device(0)
    ins0 = _make(13, "cuda:0")
    ins1 = _make(13, "cuda:1")
    ps = [ins0[0].clone(), ins1[1].clone(), ins0[2].clone()]
    gs = [ins0[3], ins1[4], ins0[5]]
    qs = [p.clone() for p in ps]
    opt = AdafactorOptimizer(ps, learning_rate=0.01)
    o0, o1 = AdafactorOptimizer([qs[0], qs[2]], learning_rate=0.01), AdafactorOptimizer([qs[1]], learning_rate=0.01)
    scale = torch.full((), 0.75, device="cuda:0")
    for _ in range(2):
        opt.step(grads=gs, norm_scale=scale)
        o0.step(grads=[gs[0], gs[2]], norm_scale=scale)
        o1.step(grads=[gs[1]], norm_scale=scale.to("cuda:1"))
    for p, q, o in zip(ps, qs, (o0, o1, o0)):
        _same([p] + list(opt.state[p].values()), [q] + list(o.state[q].values()), "split")


# ---- element offsets past 2^31 ---------------------------------------------------------------------------------------------
def test_factored_param_past_two_to_the_31():
    """(65537, 32768) with a bf16 grad: 2^31 + 32768 elements. rv, cv, mean(rv) and rms are formed in float64 on the
    device in slices of rows; the rows on both sides of element 2^31 are checked elementwise. Peak: param 8.6 GB, grad
    4.3 GB, workspace 0.2 GB and float64 slices of 0.5 GB."""
    C, K = 65537, 32768
    need = C * K * 6 + (4 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB are free" % (need / 2 ** 30, free / 2 ** 30))
    gen = torch.Generator(device="cuda").manual_seed(3)
    p = torch.empty(C, K, device="cuda")
    g = torch.empty(C, K, device="cuda", dtype=torch.bfloat16)
    for r in range(0, C, 4096):
        p[r:r + 4096].normal_(0, 1, generator=gen)
        g[r:r + 4096] = torch.empty(min(4096, C - r), K, device="cuda").normal_(0, 0.1, generator=gen)
    rows = [(1 << 31) // K - 1, (1 << 31) // K]              # 65535 ends at element 2^31, 65536 starts there
    p_old = p[rows].double().cpu().numpy()
    eps, decay, lr = _f32(1e-30), _f32(0.9), _f32(0.01)
    opt = _opt([p])
    opt.step(grads=[g])
    rv_ref = torch.empty(C, dtype=torch.float64, device="cuda")
    colsum = torch.zeros(K, dtype=torch.float64, device="cuda")
    for r in range(0, C, 2048):
        sq = g[r:r + 2048].double().square() + eps
        rv_ref[r:r + 2048] = (1 - decay) * sq.mean(dim=1)
        colsum += sq.sum(dim=0)
    cv_ref = (1 - decay) * colsum / C
    rv_mean = rv_ref.mean()
    rms = 0.0
    for r in range(0, C, 2048):
        x = g[r:r + 2048].double() / (rv_ref[r:r + 2048, None] / rv_mean).sqrt() / cv_ref[None, :].sqrt()
        rms += float(x.square().sum())
    rms /= C * K
    rate = lr / max(1.0, np.sqrt(rms))
    _close(_np(opt.state[p]["rv"]), rv_ref.cpu().numpy(), "rv")
    _close(_np(opt.state[p]["cv"]), cv_ref.cpu().numpy(), "cv")
    x = g[rows].double() / (rv_ref[rows, None] / rv_mean).sqrt() / cv_ref[None, :].sqrt()
    upd_ref = (rate * x).cpu().numpy()
    pn = p[rows].double().cpu().numpy()
    _close(p_old - pn, upd_ref, "rows %s update" % rows, scale=2.0 ** -24 * np.abs(pn))
    assert _lib.device_error() == 0, _lib.device_error_text()


# ---- the reference's own kernels -------------------------------------------------------------------------------------------
REF_CASES = [((64, 256), t) for t in GDTYPES] + [((37, 129), t) for t in GDTYPES] + [((1003,), t) for t in GDTYPES]


@pytest.mark.parametrize("shape,gdtype", REF_CASES, ids=["%s-%s" % ("x".join(map(str, s)), str(d)[6:]) for s, d in REF_CASES])
def test_against_reference_kernels(shape, gdtype):
    """The reference's Adafactor launcher on the same state: it adds mean(rv) and mean(x^2) with atomics in any order and
    uses fast-math rsqrtf and division (prec-div / prec-sqrt off), so the bound is REL (64 ulps) on rv / cv and 4 * REL
    on the update, whose rate depends on both atomic sums."""
    from oracle import ref_adafactor as ra
    why = ra.missing()
    if why:
        pytest.skip(why)
    rng = np.random.default_rng(sum(shape))
    p = _view(shape, torch.float32, 0, rng)
    g = _view(shape, gdtype, 0, rng, 0.1)
    opt = _opt([p], clip_thresh=0.5)
    _set_state(opt, p, rng)
    cv0, rv0 = opt.state[p]["cv"].clone(), opt.state[p].get("rv")
    rv0 = None if rv0 is None else rv0.clone()
    p0 = p.clone()
    ns = torch.full((), 0.8, device="cuda")
    rp, rcv, rrv = ra.adafactor(g, p0, cv0, rv0, lr=0.01, decay=_f32(0.9), clip_thresh=0.5, norm_scale=ns)
    opt.step(grads=[g], norm_scale=ns)
    p0n = _np(p0)
    for got, ref, what, rel in ((_np(p) - p0n, _np(rp) - p0n, "update", 4 * REL), (_np(opt.state[p]["cv"]), _np(rcv), "cv", REL),
                                (_np(opt.state[p].get("rv")), _np(rrv), "rv", REL)):
        if ref is None:
            assert got is None
            continue
        err = np.abs(got - ref)
        tol = rel * np.abs(ref) + 2.0 ** -23 * np.abs(_np(p)).max() * (what == "update")
        assert (err <= tol).all(), "%s %s %s: worst %.3e" % (shape, gdtype, what, err.max())
