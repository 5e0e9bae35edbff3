"""AdamOptimizer, clip_by_global_norm and Ema on the GPU, checked against the float64 oracle (oracle/optimize_oracle.py)
given the same rounded inputs: every grad dtype, both moment formats, sizes with and without 16-byte access, storage
offsets, gates at every block size, norm_scale, multi-step power bookkeeping, state_dict resumption, launch counts and
the absence of host synchronisation."""
import copy

import numpy as np
import pytest
import torch

from blocksparse_b200 import AdamOptimizer, Ema, _lib, clip_by_global_norm, global_norm
from oracle import optimize_oracle as oo

pytestmark = pytest.mark.gpu

GDTYPES = [torch.float32, torch.float16, torch.bfloat16]
SIZES = [1, 3, 127, 1024, 1023 * 1024, 1024 * 1024, 8197, 65536 + 13]


def _np(t):
    return t.detach().double().cpu().numpy()


def _codes_np(t):
    return t.detach().cpu().numpy().view(np.uint16)


def _view(n, dtype, offset, rng, scale=1.0):
    """A tensor of n elements at `offset` elements into a larger buffer (offset 1: no 16-byte access)."""
    base = torch.as_tensor(rng.normal(0, scale, n + offset + 3).astype(np.float32)).to(dtype).cuda()
    return base[offset:offset + n]


def _state(opt, p, rng, codes, lo=0.0):
    """Fills the param's moments with random values (fp32, or 16-bit codes of random values); returns them as float64."""
    n = p.numel()
    m = rng.normal(0, 0.05, n)
    v = rng.uniform(lo, 0.01, n)
    if codes:
        mc, vc = oo.mean_encode(m), oo.var_encode(v)
        opt.state[p]["mean"] = torch.as_tensor(mc.view(np.int16).reshape(p.shape)).cuda()
        opt.state[p]["var"] = torch.as_tensor(vc.view(np.int16).reshape(p.shape)).cuda()
        return oo.mean_decode(mc).reshape(p.shape), oo.var_decode(vc).reshape(p.shape)
    opt.state[p]["mean"] = torch.as_tensor(m.astype(np.float32).reshape(p.shape)).cuda()
    opt.state[p]["var"] = torch.as_tensor(v.astype(np.float32).reshape(p.shape)).cuda()
    return _np(opt.state[p]["mean"]), _np(opt.state[p]["var"])


def _check_fp32(got, ref, what):
    tol = 1e-6 * max(np.abs(ref).max(), 1e-30)
    err = np.abs(got - ref).max()
    assert err <= tol, "%s: max err %.3e > %.3e" % (what, err, tol)


def _check_codes(got, ref_vals, enc, dec, mbits, what):
    """Every kernel code decodes to within half a code ulp (plus fp32 rounding, 1e-6 of the largest value) of the float64
    value, and at least 95 % equal the oracle's code. The rest sit where the exact value lies within fp32 rounding of a
    tie between two codes (inputs with few significant bits, such as decoded codes and 16-bit grads, put up to a few
    percent of the exact results there), or are near-zero means after cancellation, where the same absolute fp32 error
    spans several codes."""
    back = dec(got)
    bound = np.abs(ref_vals) * 2.0 ** -mbits + 1e-6 * np.abs(ref_vals).max()
    bad = np.flatnonzero(np.abs(back - ref_vals) > bound)
    assert not len(bad), "%s: %d codes off, e.g. %s for %s" % (what, len(bad), back[bad[:3]], ref_vals[bad[:3]])
    same = (got.astype(np.int64) == enc(ref_vals).astype(np.int64)).mean()
    assert same >= 0.95, "%s: only %.2f%% of codes equal the oracle's" % (what, 100 * same)


def _check_update(p_new, p_old, p_ref, what):
    upd, upd_ref = p_new - p_old, p_ref - p_old
    tol = 1e-5 * max(np.abs(upd_ref).max(), 1e-30)
    err = np.abs(upd - upd_ref).max()
    assert err <= tol, "%s: update err %.3e > %.3e" % (what, err, tol)


def _check_step(opt, p, p_old, m_old, v_old, g_np, codes, what, gate=None, bs=0, **kw):
    kw = {k: float(np.float32(v)) if isinstance(v, float) else v for k, v in kw.items()}     # the kernel's fp32 constants
    pr, mr, vr = oo.adam(g_np, p_old, m_old, v_old, gate=gate, bs=bs, **kw)
    _check_update(_np(p), p_old, pr, what + " p")
    m, v = opt.state[p]["mean"], opt.state[p]["var"]
    if codes:
        assert m.dtype == torch.int16
        _check_codes(_codes_np(m).ravel(), mr.ravel(), oo.mean_encode, oo.mean_decode, 9, what + " mean")
        _check_codes(_codes_np(v).ravel(), vr.ravel(), oo.var_encode, oo.var_decode, 10, what + " var")
    else:
        _check_fp32(_np(m), mr, what + " mean")
        _check_fp32(_np(v), vr, what + " var")


ADAM = dict(lr=0.1, beta1=0.9, beta2=0.999, epsilon=1e-8)


def _opt(params, **kw):
    args = dict(learning_rate=ADAM["lr"], beta1=ADAM["beta1"], beta2=ADAM["beta2"], epsilon=ADAM["epsilon"],
                zero_init_variables=True)             # lr_t == lr exactly
    args.update(kw)
    return AdamOptimizer(params, **args)


@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
@pytest.mark.parametrize("gdtype", GDTYPES, ids=lambda d: str(d).replace("torch.", ""))
@pytest.mark.parametrize("n", SIZES)
def test_dense_adam_matches_oracle(n, gdtype, codes):
    rng = np.random.default_rng(n + 7 * GDTYPES.index(gdtype) + 100 * codes)
    for offset in ((0, 1) if n < 1023 * 1024 else (0,)):
        p = _view(n, torch.float32, offset, rng, 0.5)
        g = _view(n, gdtype, offset, rng, 0.1)
        opt = _opt([p], fp16=codes)
        m0, v0 = _state(opt, p, rng, codes)
        p0, g_np = _np(p), _np(g)
        opt.step(grads=[g])
        _check_step(opt, p, p0, m0, v0, g_np, codes, "n %d offset %d" % (n, offset), **ADAM)


@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
@pytest.mark.parametrize("case", ["clip_sigma", "grad_scale", "zero_infs_nans", "saturate"])
def test_adam_conditioning(case, codes):
    rng = np.random.default_rng(11)
    n = 40000 + 5
    kw = dict(clip_sigma=dict(clip_sigmas=2.0), grad_scale=dict(grad_scale=0.25),
              zero_infs_nans=dict(zero_infs=True, zero_nans=True), saturate=dict(saturate=0.05, zero_nans=True))[case]
    okw = {"clip_sigma" if k == "clip_sigmas" else k: v for k, v in kw.items()}
    for gdtype in GDTYPES:
        p = _view(n, torch.float32, 0, rng, 0.5)
        g = _view(n, gdtype, 0, rng, 0.1)
        if case in ("zero_infs_nans", "saturate"):
            g[rng.integers(0, n, 50)] = float("inf")
            g[rng.integers(0, n, 50)] = float("-inf")
            g[rng.integers(0, n, 50)] = float("nan")
        opt = _opt([p], fp16=codes, **kw)
        m0, v0 = _state(opt, p, rng, codes)
        p0, g_np = _np(p), _np(g)
        opt.step(grads=[g])
        assert torch.isfinite(p).all()
        _check_step(opt, p, p0, m0, v0, g_np, codes, "%s %s" % (case, gdtype), **ADAM, **okw)


@pytest.mark.parametrize("zero_init", [False, True])
@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
def test_ten_steps_track_the_powers(zero_init, codes):
    rng = np.random.default_rng(21)
    ps = [_view(n, torch.float32, 0, rng, 0.5) for n in (9000, 300, 16384)]
    b1, b2, lr = 0.8, 0.95, 0.05
    opt = AdamOptimizer(ps, learning_rate=lr, beta1=b1, beta2=b2, fp16=codes, zero_init_variables=zero_init)
    for t in range(1, 11):
        gs = [_view(p.numel(), torch.float16, 0, rng, 0.1) for p in ps]
        olds = []
        for p in ps:
            if p not in opt.state:
                olds.append((_np(p), np.zeros(p.shape), np.zeros(p.shape)))
                continue
            m, v = opt.state[p]["mean"], opt.state[p]["var"]
            if m.dtype == torch.int16:
                olds.append((_np(p), oo.mean_decode(_codes_np(m)), oo.var_decode(_codes_np(v))))
            else:
                olds.append((_np(p), _np(m), _np(v)))
        opt.step(grads=gs)
        lr_t = lr if zero_init else oo.lr_t(lr, b1 ** t, b2 ** t)
        for p, g, (p0, m0, v0) in zip(ps, gs, olds):
            c = codes and p.numel() >= 8192
            _check_step(opt, p, p0, m0, v0, _np(g), c, "step %d n %d" % (t, p.numel()), lr=lr_t, beta1=b1, beta2=b2,
                        epsilon=1e-8)
    want = (0.0, 0.0) if zero_init else (b1 ** 11, b2 ** 11)
    assert opt.param_groups[0]["beta1_power"] == pytest.approx(want[0], rel=1e-5)
    assert opt.param_groups[0]["beta2_power"] == pytest.approx(want[1], rel=1e-5)


@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
def test_state_dict_resume_is_bit_identical(codes):
    rng = np.random.default_rng(31)
    ps = [_view(n, torch.float32, 0, rng) for n in (10000, 77, 4096 * 4)]
    grads = [[_view(p.numel(), torch.bfloat16, 0, rng, 0.1) for p in ps] for _ in range(8)]
    opt = AdamOptimizer(ps, learning_rate=0.01, fp16=codes, clip_sigmas=2.0)
    for gs in grads[:4]:
        opt.step(grads=gs)
    saved = copy.deepcopy(opt.state_dict())
    ps2 = [p.detach().clone() for p in ps]
    for gs in grads[4:]:
        opt.step(grads=gs)
    opt2 = AdamOptimizer(ps2, learning_rate=0.5, fp16=codes, clip_sigmas=2.0)
    opt2.load_state_dict(saved)
    assert opt2.param_groups[0]["lr"] == 0.01
    for gs in grads[4:]:
        opt2.step(grads=gs)
    for a, b in zip(ps, ps2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        for k in ("mean", "var"):
            x, y = opt.state[a][k], opt2.state[b][k]
            assert x.dtype == y.dtype and torch.equal(x.view(torch.int16), y.view(torch.int16))


@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
@pytest.mark.parametrize("bs", [8, 16, 32, 64])
def test_gated_adam_skips_pruned_blocks_and_steps_live_ones_once(bs, codes):
    rng = np.random.default_rng(bs + codes)
    blocks = max(8192 // (bs * bs) + 3, 40)
    p = torch.as_tensor(rng.normal(0, 1, (blocks, bs, bs)).astype(np.float32)).cuda()
    gate = rng.uniform(0.5, 1.5, blocks).astype(np.float32)
    gate[rng.random(blocks) < 0.4] = 0.0
    p.gate = torch.as_tensor(gate).cuda()
    dense = _view(3000, torch.float32, 1, rng)                 # a dense tensor in the same launch
    opt = _opt([p, dense], gated=True, fp16=codes)
    m0, v0 = _state(opt, p, rng, codes)
    dm0, dv0 = _state(opt, dense, rng, False)
    bits = {k: opt.state[p][k].clone() for k in ("mean", "var")}
    p0, pbits = _np(p), p.clone()
    g = torch.as_tensor(rng.normal(0, 0.1, p.shape).astype(np.float32)).half().cuda()
    gd = _view(3000, torch.float32, 0, rng, 0.1)
    d0 = _np(dense)
    opt.step(grads=[g, gd])
    dead = torch.as_tensor(gate == 0).cuda()
    assert torch.equal(p[dead].view(torch.int32), pbits[dead].view(torch.int32))
    for k in ("mean", "var"):
        assert torch.equal(opt.state[p][k][dead].view(torch.int16 if codes else torch.int32),
                           bits[k][dead].view(torch.int16 if codes else torch.int32))
    assert not torch.equal(p[~dead], pbits[~dead])
    c = codes and p.numel() >= 8192
    _check_step(opt, p, p0, m0, v0, _np(g), c, "gated bs %d" % bs, gate=gate, bs=bs, **ADAM)
    _check_step(opt, dense, d0, dm0, dv0, _np(gd), False, "dense next to gated", **ADAM)


def test_ungated_optimizer_ignores_the_gate():
    rng = np.random.default_rng(41)
    p = torch.as_tensor(rng.normal(0, 1, (4, 8, 8)).astype(np.float32)).cuda()
    p.gate = torch.zeros(4, device="cuda")
    opt = _opt([p])
    m0, v0 = _state(opt, p, rng, False)
    p0, g = _np(p), torch.randn_like(p)
    opt.step(grads=[g])
    _check_step(opt, p, p0, m0, v0, _np(g), False, "gate ignored", **ADAM)


@pytest.mark.parametrize("codes", [False, True], ids=["fp32_moments", "codes"])
def test_norm_scale(codes):
    rng = np.random.default_rng(51)
    ps = [_view(n, torch.float32, 0, rng) for n in (9000, 13)]
    gs = [_view(p.numel(), torch.float16, 0, rng, 0.1) for p in ps]
    opt = _opt(ps, fp16=codes, norm_scale=torch.zeros((), device="cuda"))
    olds = [(p.clone(), *_state(opt, p, rng, codes and p.numel() >= 8192)) for p in ps]
    mv = [(opt.state[p]["mean"].clone(), opt.state[p]["var"].clone()) for p in ps]
    opt.step(grads=gs)                                          # the constructor's scale: 0
    for p, (pb, _, _), (mb, vb) in zip(ps, olds, mv):
        assert torch.equal(p.view(torch.int32), pb.view(torch.int32))
        assert torch.equal(opt.state[p]["mean"], mb) and torch.equal(opt.state[p]["var"], vb)
    ns = torch.full((), 0.3, device="cuda")
    opt.step(grads=gs, norm_scale=ns)                           # overrides the constructor's
    for p, g, (pb, m0, v0) in zip(ps, gs, olds):
        _check_step(opt, p, _np(pb), m0, v0, _np(g), codes and p.numel() >= 8192, "norm_scale 0.3",
                    norm_scale=float(np.float32(0.3)), **ADAM)


def test_param_grad_and_many_tensors():
    """.grad is used when no grads are given; 300 tensors take two launches and are all stepped."""
    rng = np.random.default_rng(61)
    ps = [_view(int(n), torch.float32, int(o), rng) for n, o in zip(rng.integers(1, 3000, 300), rng.integers(0, 2, 300))]
    opt = _opt(ps)
    olds = [(_np(p), *_state(opt, p, rng, False)) for p in ps]
    for p in ps:
        p.grad = torch.randn_like(p)
    opt.step()
    for i, (p, (p0, m0, v0)) in enumerate(zip(ps, olds)):
        _check_step(opt, p, p0, m0, v0, _np(p.grad), False, "tensor %d" % i, **ADAM)


def _mixed(rng, count):
    out = []
    for i in range(count):
        n = int(rng.choice([0, 1, 5, 127, 1024, 8193, 70000, 1 << 20])) if count > 1 else 1 << 20
        out.append(_view(n, GDTYPES[i % 3], int(rng.integers(0, 2)), rng, float(rng.uniform(0.01, 2))))
    return out


@pytest.mark.parametrize("count", [1, 7, 300])
def test_clip_by_global_norm(count):
    rng = np.random.default_rng(count)
    gs = _mixed(rng, count)
    host = [_np(g) for g in gs]
    for kw in (dict(), dict(clip_norm=1e9, grad_scale=0.5), dict(saturate=0.5)):
        norm, scale = clip_by_global_norm(gs, **kw)
        assert norm.shape == () and scale.shape == () and norm.dtype == scale.dtype == torch.float32 and norm.is_cuda
        rn, rs = oo.global_norm(host, **kw)
        assert abs(norm.item() - rn) <= 1e-6 * rn, (kw, norm.item(), rn)
        assert abs(scale.item() - rs) <= 1e-6 * rs, (kw, scale.item(), rs)
        n2, s2 = clip_by_global_norm(gs, **kw)
        assert torch.equal(norm.view(torch.int32), n2.view(torch.int32)) and torch.equal(scale, s2)
    assert abs(global_norm(gs).item() - oo.global_norm(host)[0]) <= 1e-6 * oo.global_norm(host)[0]


@pytest.mark.parametrize("bad", ["inf", "-inf", "nan"])
def test_clip_by_global_norm_non_finite(bad):
    rng = np.random.default_rng(71)
    gs = _mixed(rng, 7)
    gs[3][0] = float(bad)
    norm, scale = clip_by_global_norm(gs)
    assert not torch.isfinite(norm).item() and scale.item() == 0.0
    norm, scale = clip_by_global_norm(gs, zero_infs=True, zero_nans=True)
    rn, rs = oo.global_norm([_np(g) for g in gs], zero_infs=True, zero_nans=True)
    assert torch.isfinite(norm).item() and abs(norm.item() - rn) <= 1e-6 * rn and abs(scale.item() - rs) <= 1e-6 * rs


def test_clip_by_global_norm_empty():
    for gs in ([], [torch.empty(0, device="cuda"), torch.empty(0, 3, device="cuda", dtype=torch.float16)]):
        norm, scale = clip_by_global_norm(gs)
        assert norm.item() == 0.0 and scale.item() == 1.0


def test_no_host_synchronisation():
    rng = np.random.default_rng(81)
    gs = _mixed(rng, 7)
    ps = [torch.zeros(g.shape, device="cuda") for g in gs]
    opt = AdamOptimizer(ps, fp16=True)
    ema = Ema()
    opt.step(grads=gs)                                          # moments and averages are created outside the check
    ema.apply(ps)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _, scale = clip_by_global_norm(gs)
        opt.step(grads=gs, norm_scale=scale)
        ema.apply(ps)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_launch_counts():
    rng = np.random.default_rng(91)
    ps = [_view(int(n), torch.float32, 0, rng) for n in rng.integers(1, 20000, 256)]
    gs = [torch.randn_like(p).half() for p in ps]
    opt = AdamOptimizer(ps, fp16=True)
    ema = Ema(fp16=True)
    opt.step(grads=gs)
    ema.apply(ps)
    norm_scale = clip_by_global_norm(gs)[1]
    k = _kernels(lambda: opt.step(grads=gs, norm_scale=norm_scale))
    assert len(k) == 1 and "mt_adam" in k[0], k
    k = _kernels(lambda: ema.apply(ps))
    assert len(k) == 1 and "mt_ema" in k[0], k
    k = _kernels(lambda: clip_by_global_norm(gs))
    assert len(k) <= 2 and all("mt_" in n for n in k), k


@pytest.mark.parametrize("gated", [False, True])
@pytest.mark.parametrize("fp16", [False, True])
def test_ema(fp16, gated):
    rng = np.random.default_rng(101 + fp16 + 2 * gated)
    bs = 16
    p1 = torch.as_tensor(rng.normal(0, 1, (50, bs, bs)).astype(np.float32)).cuda()
    gate = (rng.random(50) < 0.6).astype(np.float32)
    p1.gate = torch.as_tensor(gate).cuda()
    p2 = _view(1000 + 3, torch.float32, 1, rng)
    ema = Ema(decay=0.9, gated=gated, fp16=fp16)
    ema.apply([p1, p2])
    dt = torch.float16 if fp16 else torch.float32
    e1, e2 = ema.average(p1), ema.average(p2)
    assert e1.dtype == dt and ema.average(torch.zeros(1)) is None
    # first use: a copy of the param, then one update towards itself (a no-op up to rounding)
    assert torch.allclose(e1.float(), p1, rtol=1e-3 if fp16 else 1e-6, atol=0)
    before = [_np(e1), _np(e2)]
    bits = e1.clone()
    with torch.no_grad():
        p1.add_(torch.randn_like(p1))
        p2.add_(torch.randn_like(p2))
    ema.apply([p1, p2])
    for e, e0, p, g, what in ((e1, before[0], p1, gate if gated else None, "gated"), (e2, before[1], p2, None, "dense")):
        ref = oo.ema(e0, _np(p), 0.9, gate=g, bs=bs)
        if fp16:                                                # within one fp16 ulp
            assert np.all(np.abs(_np(e) - ref) <= np.abs(ref) * 2.0 ** -10 + 2.0 ** -24), what
        else:
            _check_fp32(_np(e), ref, "ema " + what)
    if gated:
        dead = torch.as_tensor(gate == 0).cuda()
        assert torch.equal(e1[dead].view(torch.int16 if fp16 else torch.int32),
                           bits[dead].view(torch.int16 if fp16 else torch.int32))
