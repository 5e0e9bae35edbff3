"""quantize, log_stats and the optimizers' qspecs on the GPU: bitwise against the NumPy oracle (oracle/quantize_oracle.py)
over every format, against the reference's own Quantize / QuantizationStats kernels where oracle/_ref has them, the
exponent sequence of the statistics schedule, stochastic rounding from the Philox state, autograd, AdamOptimizer and Ema,
side streams, replayed CUDA graphs, a second GPU and offsets past 2^31."""
import copy
import importlib

import numpy as np
import pytest
import torch

from blocksparse_b200 import AdamOptimizer, Ema, _lib, get_entropy, set_entropy
from blocksparse_b200.quantize import QuantizeSpec, log_stats, quantize, quantize_state, reset_quantize_states
from oracle import quantize_oracle as qo
from oracle import ref_quantize as rq
from tests.test_quantize_oracle import _inputs, _wraps

qm = importlib.import_module("blocksparse_b200.quantize")
pytestmark = pytest.mark.gpu
GB = 1 << 30


def _run(xs, spec, exps, ys=None):
    """quantize_tensors over CUDA tensors xs with exponent records exps (new schedules), into new tensors or ys."""
    ys = [torch.empty_like(x) for x in xs] if ys is None else ys
    qm.quantize_tensors(xs, ys, exps, [qm.new_schedule() for _ in xs], spec, ["t%d" % i for i in range(len(xs))])
    return ys


def _exp(e):
    return torch.full((), int(e), dtype=torch.int64, device="cuda")


def _misaligned(a, dtype):
    """a as a CUDA tensor of dtype that starts one element past a 16-byte boundary."""
    t = torch.as_tensor(a)
    buf = torch.empty(t.numel() + 1, dtype=dtype, device="cuda")
    v = buf[1:]
    v.copy_(t.to(dtype))
    return v


@pytest.mark.parametrize("ebits", range(1, 9))
def test_nonstochastic_fp32_and_bf16_match_the_oracle_bitwise(ebits):
    rng = np.random.default_rng(100 + ebits)
    for fbits in range(24):
        for denorm in (True, False):
            top = qo.top_exponent(ebits) - 127
            es = sorted({top, top + 5, (1 << (ebits - 1)) - 1, 127})
            x = [_inputs(rng, e, ebits, fbits, denorm, n=1001) for e in es]
            for xi in x:
                xi[:4] = [np.nan, -np.inf, np.inf, -np.nan]
            spec = QuantizeSpec(ebits=ebits, fbits=fbits, denorm=denorm, frequency=0)
            # one multi-tensor call over aligned and misaligned tensors, each at its own exponent
            xs = [torch.as_tensor(xi).cuda() for xi in x] + [_misaligned(xi, torch.float32) for xi in x]
            ys = _run(xs, spec, [_exp(e) for e in es] * 2)
            for i, (xi, e) in enumerate(list(zip(x, es)) * 2):
                ref = qo.quantize_bits(xi.view(np.uint32), e, ebits, fbits, denorm)
                got = ys[i].cpu().numpy().view(np.uint32)
                assert np.array_equal(got, ref), (ebits, fbits, denorm, e, np.flatnonzero(got != ref)[:5])
            if fbits > 7:
                continue
            xb = [torch.as_tensor(xi).bfloat16() for xi in x]
            xs = [t.cuda() for t in xb] + [_misaligned(t, torch.bfloat16) for t in xb]
            ys = _run(xs, spec, [_exp(e) for e in es] * 2)
            for i, (t, e) in enumerate(list(zip(xb, es)) * 2):
                bits = t.view(torch.int16).numpy().view(np.uint16)
                full = qo.quantize_bits(bits.astype(np.uint32) << 16, e, ebits, fbits, denorm)
                nan = np.isnan(t.float().numpy())
                ok = ((full & 0xFFFF) == 0) | nan  # everywhere but the no-denorm wrap-around corner
                assert np.all(ok | _wraps(t.float().numpy(), qo.fmt(e, ebits, fbits, denorm)))
                got = ys[i].cpu().view(torch.int16).numpy().view(np.uint16)
                assert np.array_equal(got[ok], (full >> 16).astype(np.uint16)[ok]), (ebits, fbits, denorm, e)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_nonstochastic_matches_the_reference_kernel(dtype):
    if not rq.available():
        pytest.skip(rq.missing())
    rng = np.random.default_rng(7)
    for ebits in range(1, 9):
        for fbits in range(8 if dtype == torch.bfloat16 else 24):
            for denorm in (True, False):
                top = qo.top_exponent(ebits) - 127
                for e in sorted({top, top + 4, (1 << (ebits - 1)) - 1, 127}):
                    xn = _inputs(rng, e, ebits, fbits, denorm, n=777)
                    xn[:2] = [np.inf, -np.inf]
                    x = torch.as_tensor(xn).to(dtype).cuda()
                    spec = QuantizeSpec(ebits=ebits, fbits=fbits, denorm=denorm, frequency=0)
                    ours = _run([x], spec, [_exp(e)])[0]
                    ref = rq.quantize(x, e, ebits, fbits, denorm)
                    a = ours.view(torch.int16 if dtype == torch.bfloat16 else torch.int32).cpu().numpy()
                    b = ref.view(torch.int16 if dtype == torch.bfloat16 else torch.int32).cpu().numpy()
                    keep = ~_wraps(x.float().cpu().numpy(), qo.fmt(e, ebits, fbits, denorm))
                    assert np.array_equal(a[keep], b[keep]), (ebits, fbits, denorm, e)


def test_stochastic_matches_the_oracle_and_advances_the_call():
    rng = np.random.default_rng(11)
    for dtype, fbits in ((torch.float32, 10), (torch.float32, 2), (torch.bfloat16, 5)):
        for stoch in (1, 2):
            spec = QuantizeSpec(ebits=6, fbits=fbits, stochastic=stoch, frequency=0)
            sizes = [1, 7, 4096 + 3, 100003]
            xn = [rng.normal(0, 2, n).astype(np.float32) for n in sizes]
            xs = [torch.as_tensor(a).to(dtype).cuda() for a in xn[:2]] + [_misaligned(a, dtype) for a in xn[2:]]
            state = set_entropy(1234 + stoch)
            call0 = int(state[1].item())
            ys = _run(xs, spec, [_exp(5)] * len(xs))
            assert int(get_entropy()[1].item()) == call0 + len(xs)
            for i, (x, y) in enumerate(zip(xs, ys)):
                xf = x.float().cpu().numpy()
                w = qo.philox_words(1234 + stoch, call0 + i, xf.size)
                ref = qo.quantize_bits(xf.view(np.uint32), 5, 6, fbits, True, words=w)
                lo = qo.quantize_bits(xf.view(np.uint32), 5, 6, fbits, True, words=np.zeros(xf.size, np.uint32))
                hi = qo.quantize_bits(xf.view(np.uint32), 5, 6, fbits, True,
                                      words=np.full(xf.size, 0xFFFFFFFF, np.uint32))
                got = y.float().cpu().numpy().view(np.uint32)
                assert np.array_equal(got, ref), (dtype, fbits, stoch, i)
                assert np.all((got == lo) | (got == hi))


def test_stochastic_rounding_is_unbiased():
    """2^24 draws of each of a few fixed values: the mean of the rounded values is within 6 standard errors of x (each
    draw is one of x's two grid neighbours, so its standard deviation is at most half an ulp)."""
    n = 1 << 24
    spec = QuantizeSpec(ebits=5, fbits=3, stochastic=2, frequency=0)
    set_entropy(99)
    for v in (1.03, 1.5 + 1 / 64, -2.2, 0.7):
        x = torch.full((n,), v, dtype=torch.float32, device="cuda")
        y = _run([x], spec, [_exp(15)])[0]
        xv = float(np.float32(v))
        ulp = 2.0 ** (np.floor(np.log2(abs(xv))) - 3)
        mean = y.double().mean().item()
        assert abs(mean - xv) <= 6 * (ulp / 2) / np.sqrt(n), (v, mean, xv)
        xb = np.array([xv], np.float32).view(np.uint32)
        lo = qo.quantize_bits(xb, 15, 5, 3, True, words=np.zeros(1, np.uint32)).view(np.float32)[0]
        hi = qo.quantize_bits(xb, 15, 5, 3, True, words=np.full(1, 0xFFFFFFFF, np.uint32)).view(np.float32)[0]
        assert set(np.unique(y.cpu().numpy()).tolist()) == {float(lo), float(hi)}


def _drift(rng, k, n=5003):
    return (rng.normal(0, 1, n) * 2.0 ** (k / 3.0 - 4)).astype(np.float32)


@pytest.mark.parametrize("mode", [0, 1])
def test_exponent_sequence_and_statistics_follow_the_oracle(mode):
    rng = np.random.default_rng(20 + mode)
    xs = [_drift(rng, k) for k in range(44)]
    for bias_pad in (0, 2, 3):
        for dtype, fbits in ((torch.float32, 5), (torch.bfloat16, 3)):
            spec = QuantizeSpec(ebits=5, fbits=fbits, frequency=8, mode=mode, bias_pad=bias_pad, stdv_mul=3.0)
            xin = [torch.as_tensor(x).to(dtype) for x in xs]
            ref = qo.run([x.float().numpy() for x in xin], dict(ebits=5, fbits=fbits, denorm=True, stoch=0, freq=8,
                                                               mode=mode, bias_pad=bias_pad, stdv_mul=3.0, emax=15))
            runs = []
            for _ in range(2):
                reset_quantize_states()
                outs = []
                for x, (qref, eref, sref) in zip(xin, ref):
                    y = quantize(x.cuda(), spec, name="seq")
                    st = quantize_state("seq")
                    assert int(st.exp_f.item()) == eref
                    got = y.float().cpu().numpy()
                    assert np.array_equal(got.view(np.uint32), qref.view(np.uint32))
                    if sref is not None:
                        s = st.stats_f.cpu().numpy()
                        np.testing.assert_allclose(s, np.array(sref, np.float64), rtol=1e-6, atol=1e-6)
                        outs.append(s.copy())
                runs.append(outs)
                assert st.calls_f == len(xs) and st.calls_b == 0
            assert len(runs[0]) == len([r for r in ref if r[2] is not None]) >= 10
            for a, b in zip(*runs):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_statistics_match_the_reference_kernel():
    if not rq.available():
        pytest.skip(rq.missing())
    rng = np.random.default_rng(5)
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        for n in (1, 1000, 1 << 20):
            x = torch.as_tensor(rng.normal(0, 30, n).astype(np.float32)).to(dtype).cuda()
            if n > 1:
                x[0] = float("nan")
            ours = qm.log_statistics(x, 40.0, 0.5).cpu().numpy()
            ref = rq.quantization_stats(x, 40.0, 0.5)
            orc = qo.stats(x.float().cpu().numpy(), 40.0, 0.5, half=dtype == torch.float16)
            np.testing.assert_allclose(ours, np.array(orc, np.float64), rtol=1e-6)
            assert ours[4] == ref[4]
            if n > 1:           # a NaN makes the sums inf in both (fp16 clamps it to 65504 first)
                assert np.isinf(ours[0]) == np.isinf(ref[0]) == (dtype != torch.float16)
                x[0] = 1.0
                ours = qm.log_statistics(x, 40.0, 0.5).cpu().numpy()
                ref = rq.quantization_stats(x, 40.0, 0.5)
            np.testing.assert_allclose(ours[:2], np.array(ref[:2], np.float64), rtol=1e-3)
            np.testing.assert_allclose(ours[2:4], np.array(ref[2:4], np.float64), rtol=1e-3, atol=1e-4)


def test_autograd_uses_the_backward_spec_and_state():
    reset_quantize_states()
    f, b = QuantizeSpec(ebits=4, fbits=3, frequency=0), QuantizeSpec(ebits=6, fbits=5, frequency=0, emax=3)
    rng = np.random.default_rng(1)
    xn, dn = rng.normal(0, 3, (37, 11)).astype(np.float32), rng.normal(0, 3, (37, 11)).astype(np.float32)
    x = torch.as_tensor(xn).cuda().requires_grad_()
    y = quantize(x, f, b, name="ag")
    y.backward(torch.as_tensor(dn).cuda())
    assert np.array_equal(y.detach().cpu().numpy(), qo.quantize(xn, 7, 4, 3, True))
    assert np.array_equal(x.grad.cpu().numpy(), qo.quantize(dn, 3, 6, 5, True))
    st = quantize_state("ag")
    assert (st.calls_f, st.calls_b, int(st.exp_f.item()), int(st.exp_b.item())) == (1, 1, 7, 3)
    quantize(x, f, b, name="ag")
    assert (st.calls_f, st.calls_b) == (2, 1)
    st.exp_b.fill_(-2)                      # the user may overwrite an exponent, as the reference's variable
    x.grad = None
    quantize(x, f, b, name="ag").backward(torch.as_tensor(dn).cuda())
    assert np.array_equal(x.grad.cpu().numpy(), qo.quantize(dn, -2, 6, 5, True))
    # the default spec of the gradient is the forward's, and an empty x launches nothing
    before = _lib.last_kernel()
    e = quantize(torch.empty(0, 3, device="cuda"), f, name="empty")
    assert e.shape == (0, 3) and _lib.last_kernel() == before


def _grads(rng, shapes):
    return [torch.as_tensor(rng.normal(0, 1, s).astype(np.float32)).cuda() for s in shapes]


SHAPES = [(64, 48), (1000,), (3, 5, 7), (8192 + 5,), (1,), (130, 33)]


def _oracle_inplace(t, spec, exp, sched, st_list):
    """The oracle's step for one tensor: the schedule, the statistics and exponent update, then the rounding."""
    hit = qo.Schedule(0)
    hit.freq, hit.count, hit.pow2, hit.pow2_count = spec.freq, *sched[:3]
    now = hit.step()
    sched[:3] = [hit.count, hit.pow2, hit.pow2_count]
    a = t.cpu().numpy()
    if now:
        s = qo.quant_stats(a, exp[0], spec.ebits, spec.fbits, spec.denorm)
        exp[0] = qo.next_exponent(s, spec.ebits, spec.mode, spec.bias_pad, spec.stdv_mul)
    t.copy_(torch.as_tensor(qo.quantize(a, exp[0], spec.ebits, spec.fbits, spec.denorm)))


def test_adam_qspecs_match_plain_steps_then_the_oracle():
    rng = np.random.default_rng(3)
    init = [torch.as_tensor(rng.normal(0, 0.1, s).astype(np.float32)).cuda() for s in SHAPES]
    specs = dict(param_qspec=QuantizeSpec(ebits=6, fbits=9, frequency=2, mode=1),
                 mean_qspec=QuantizeSpec(ebits=5, fbits=7, frequency=4),
                 var_qspec=QuantizeSpec(ebits=8, fbits=6, frequency=0, emax=-10))
    pq = [p.clone() for p in init]
    pr = [p.clone() for p in init]
    oq = AdamOptimizer(pq, learning_rate=0.01, **specs)
    orf = AdamOptimizer(pr, learning_rate=0.01)
    host = {k: [([s.emax], qm.new_schedule()) for _ in init] for k, s in specs.items()}
    for step in range(6):
        gs = _grads(rng, SHAPES)
        oq.step(grads=gs)
        orf.step(grads=gs)
        for i, p in enumerate(pr):
            st = orf.state[p]
            for kind, t in (("param_qspec", p), ("mean_qspec", st["mean"]), ("var_qspec", st["var"])):
                exp, sched = host[kind][i]
                _oracle_inplace(t, specs[kind], exp, sched, None)
        for a, b in zip(pq, pr):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), step
            for k in ("mean", "var"):
                assert torch.equal(oq.state[a][k].view(torch.int32), orf.state[b][k].view(torch.int32)), (step, k)
        for i, p in enumerate(pq):
            for kind in ("param", "mean", "var"):
                assert int(oq.state[p][kind + "_qexp"].item()) == host[kind + "_qspec"][i][0][0], (step, kind)
    # the state travels with state_dict(): integer records stay integers and the next step is bitwise the same
    sd = copy.deepcopy(oq.state_dict())      # torch's loader would otherwise share the fp32 moments
    p2 = [p.clone() for p in pq]
    o2 = AdamOptimizer(p2, learning_rate=0.01, **specs)
    o2.load_state_dict(sd)
    for a, b in zip(pq, p2):
        for kind in ("param", "mean", "var"):
            assert o2.state[b][kind + "_qexp"].dtype == torch.int64
            assert o2.state[b][kind + "_qsched"] == oq.state[a][kind + "_qsched"]
    gs = _grads(rng, SHAPES)
    oq.step(grads=gs)
    o2.step(grads=gs)
    for a, b in zip(pq, p2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_adam_launches_one_quantize_per_spec_per_256_tensors():
    n = 300
    ps = [torch.zeros(17 + i, device="cuda") for i in range(n)]
    spec = QuantizeSpec(ebits=5, fbits=4, frequency=1)
    opt = AdamOptimizer(ps, param_qspec=spec, mean_qspec=spec, var_qspec=spec)
    gs = [torch.ones_like(p) for p in ps]
    opt.step(grads=gs)
    names = _kernel_names(lambda: opt.step(grads=gs))
    assert sum("q_quantize" in k for k in names) == 3 * 2
    assert sum("q_stats_finish" in k for k in names) == 3 * 2
    assert sum("q_stats<" in k for k in names) == 3 * 2


def test_ema_qspec_matches_plain_ema_then_the_oracle():
    rng = np.random.default_rng(4)
    ps = [torch.as_tensor(rng.normal(0, 1, s).astype(np.float32)).cuda() for s in SHAPES]
    spec = QuantizeSpec(ebits=5, fbits=6, frequency=2, mode=1, bias_pad=1)
    eq, er = Ema(decay=0.9), Ema(decay=0.9)
    host = [([spec.emax], qm.new_schedule()) for _ in ps]
    for step in range(5):
        for p in ps:
            p.add_(torch.as_tensor(rng.normal(0, 0.1, p.shape).astype(np.float32)).cuda())
        eq.apply(ps, qspec=spec)
        er.apply(ps)
        for p, (exp, sched) in zip(ps, host):
            _oracle_inplace(er.average(p), spec, exp, sched, None)
            assert torch.equal(eq.average(p).view(torch.int32), er.average(p).view(torch.int32)), step
            assert int(eq.qstate[id(p)]["ema_qexp"].item()) == exp[0]


def _sequence(device, xs, spec, name, seed=7):
    """Eager quantize calls of xs on `device` from a fresh state and entropy seed; returns the outputs' bits."""
    reset_quantize_states()
    set_entropy(seed, device=device)
    with torch.cuda.device(device):
        return [quantize(x.to(device), spec, name=name).view(torch.int32).cpu() for x in xs]


SPECS = [QuantizeSpec(ebits=5, fbits=3, stochastic=2, frequency=0),
         QuantizeSpec(ebits=5, fbits=3, stochastic=2, frequency=1, mode=1),
         QuantizeSpec(ebits=4, fbits=2, frequency=1, bias_pad=1)]


@pytest.mark.parametrize("spec", SPECS, ids=["freq0", "freq1-mode1", "freq1-round"])
def test_side_stream_graph_replay_and_second_gpu(spec):
    rng = np.random.default_rng(6)
    xs = [torch.as_tensor(_drift(rng, 3 * k, 10007)) for k in range(6)]
    ref = _sequence("cuda:0", xs, spec, "ctx")
    # side stream
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        side = _sequence("cuda:0", xs, spec, "ctx")
    s.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(ref, side))
    # a replayed graph: the state exists before capture; each replay runs the captured launches
    reset_quantize_states()
    set_entropy(7)
    static_x = xs[0].cuda()
    qm._state("ctx", static_x.device, spec, spec)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_y = quantize(static_x, spec, name="ctx")
    outs = []
    for x in xs:
        static_x.copy_(x)
        graph.replay()
        outs.append(static_y.view(torch.int32).cpu())
    assert all(torch.equal(a, b) for a, b in zip(ref, outs))
    if torch.cuda.device_count() > 1:
        other = _sequence("cuda:1", xs, spec, "ctx")
        assert all(torch.equal(a, b) for a, b in zip(ref, other))


def test_capture_refuses_a_new_state_and_a_logfile(tmp_path):
    x = torch.ones(100, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError):
        with torch.cuda.graph(graph):
            quantize(x, QuantizeSpec(), name="never-created-before-capture")
    quantize(x, QuantizeSpec(logfile=str(tmp_path / "q.txt")), name="logged")
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(ValueError):
        with torch.cuda.graph(graph):
            quantize(x, QuantizeSpec(logfile=str(tmp_path / "q.txt")), name="logged")


def test_logfiles_follow_the_reference_columns(tmp_path):
    reset_quantize_states()
    rng = np.random.default_rng(8)
    path = str(tmp_path / "q.txt")
    spec = QuantizeSpec(ebits=5, fbits=2, frequency=4, logfile=path)
    xs = [_drift(rng, k, 999) for k in range(12)]
    ref = qo.run(xs, dict(ebits=5, fbits=2, denorm=True, stoch=0, freq=4, mode=0, bias_pad=2, stdv_mul=4.0, emax=15))
    for x in xs:
        quantize(torch.as_tensor(x).cuda(), spec, name="lg")
    rows = open(path).read().splitlines()
    assert rows[0].split("\t") == qm.QUANT_HEADERS
    hits = [(k + 1, r) for k, r in enumerate(ref) if r[2] is not None]
    assert len(rows) == 1 + len(hits)
    lo, hi = np.float32(np.finfo(np.float32).max), np.float32(0)
    for row, (count, (_, e, s)) in zip(rows[1:], hits):
        lo, hi = min(lo, s[4]), max(hi, s[4])
        want = qo.quant_log_row(s, e, 5, 2, True, lo, hi, count, "lg")
        got = row.split("\t")
        assert got[2:] == want.rstrip("\n").split("\t")[2:], (row, want)
    # log_stats: steps 1, 2, 4, 8, 16 ... forward, the same at bfreq backward, once per step value
    path = str(tmp_path / "s_%(timestamp)s.txt")
    x = torch.as_tensor(xs[0]).cuda().requires_grad_()
    for step in [1, 1, 2, 3, 4, 5, 8, 9, 16]:
        y = log_stats(x, torch.tensor(step), freq=8, bfreq=8, logfile=path, name="ls")
        y.backward(torch.ones_like(y))
    files = list(tmp_path.glob("s_*.txt"))
    assert len(files) == 1
    rows = open(files[0]).read().splitlines()
    assert rows[0].split("\t") == qm.STAT_HEADERS
    body = [r.split("\t") for r in rows[1:]]
    assert [int(r[-2]) for r in body] == [1, 1, 2, 2, 4, 4, 8, 8, 16, 16]
    assert [r[-1] for r in body[:2]] == ["ls", "ls_grad"]
    s = qo.stats(xs[0], 65504.0, 2.0 ** -24)
    assert body[0] == qo.stat_log_row(s, s[4], s[4], 1, "ls").rstrip("\n").split("\t")
    before = _lib.last_kernel()
    log_stats(x.detach(), 3, freq=8, name="ls2")             # not a logging step: nothing launched
    log_stats(x.detach(), 3, freq=0, name="ls3")
    assert _lib.last_kernel() == before


def _need(gb):
    free = torch.cuda.mem_get_info()[0]
    if free < gb * GB:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB are free" % (gb, free / GB))


def test_bf16_past_2_31_elements():
    n = (1 << 31) + 4096 + 5
    _need(2 * n * 2 / GB + 1)
    rng = np.random.default_rng(9)
    block = rng.normal(0, 4, 4096).astype(np.float32)
    b16 = torch.as_tensor(block).bfloat16()
    x = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    x[: n - 5].view(-1, 4096).copy_(b16.cuda().expand((n - 5) // 4096, 4096))
    x[n - 5:] = b16[:5].cuda()
    spec = QuantizeSpec(ebits=5, fbits=3, frequency=0)
    y = _run([x], spec, [_exp(4)])[0]
    ref = qo.quantize_bf16_bits(b16.view(torch.int16).numpy().view(np.uint16), 4, 5, 3, True)
    yv = y[: n - 5].view(-1, 4096)
    for r in (0, (1 << 31) // 4096 - 1, (1 << 31) // 4096, yv.shape[0] - 1):
        assert np.array_equal(yv[r].cpu().view(torch.int16).numpy().view(np.uint16), ref), r
    assert np.array_equal(y[n - 5:].cpu().view(torch.int16).numpy().view(np.uint16), ref[:5])
    del x, y
    torch.cuda.empty_cache()
