"""BlocksparseConv / BlocksparseDeconv on the GPU, elementwise against the float64 oracle (oracle/conv_oracle.py):
every fixture layout, every dtype pair, both kernel routes, several minibatch sizes; l2_normalize with and without gain
and its gradients; bitwise reproducibility (two runs, an SM margin); the kernel each route names."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv import BlocksparseConv, BlocksparseDeconv
from oracle import conv_oracle
from tests._util import ROOT
from tests.test_conv_oracle import FILES, load

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
PAIRS = [(F32, F32), (F16, F16), (BF16, BF16), (F16, F32), (F32, F16), (BF16, F32), (F32, BF16)]   # (F, I)
EPS = {F32: 2.0 ** -24, F16: 2.0 ** -11, BF16: 2.0 ** -8}
TINY = {F32: 2.0 ** -150, F16: 2.0 ** -25, BF16: 2.0 ** -134}     # half the subnormal spacing: rounding near zero


def make(name):
    z, BCK, kw = load(name)
    deconv = str(z["kind"]) == "deconv"
    op = (BlocksparseDeconv if deconv else BlocksparseConv)(BCK, tuple(z["TRS"]), tuple(z["DHW"]), **kw)
    orc = conv_oracle.Conv(BCK, tuple(z["TRS"]), tuple(z["DHW"]), deconv=deconv, **kw)
    return op, orc


def rand(shape, dtype, seed):
    g = np.random.default_rng(seed)
    return torch.as_tensor(g.uniform(-1, 1, shape).astype(np.float32)).to(dtype)


def bound(ref_abs, L, out_dtype, tc):
    """Accumulation: L fp32 roundings of partial sums bounded by the sum of |terms| (twice that on the tensor cores,
    whose adds may truncate); plus one rounding of the output, relative or, among subnormals, absolute."""
    return (2 if tc else 1) * L * 2.0 ** -24 * ref_abs + EPS[out_dtype] * ref_abs + TINY[out_dtype]


def assert_close(got, ref, ref_abs, L, out_dtype, tc, what):
    got = got.detach().double().cpu().numpy().reshape(ref.shape)
    err = np.abs(got - ref)
    lim = bound(ref_abs, L, out_dtype, tc)
    bad = err > lim
    assert not bad.any(), "%s: %d bad of %d, worst %.3e vs bound %.3e" % (
        what, bad.sum(), bad.size, err[bad].max(), lim[bad][np.argmax(err[bad])])


def run(op, orc, F, I, E, flags):
    """(y, dI, dF) of one forward / backward: through autograd on the default route, through the raw ops with
    flags (BSMM_FLAG_FORCE_GENERIC)."""
    if not flags:
        f, x = F.cuda().requires_grad_(), I.cuda().requires_grad_()
        y = op(f, x)
        y.backward(E.cuda().to(y.dtype))
        return y, x.grad, f.grad
    N = I.shape[0]
    C, _ = op._in_dims()
    K, _ = op._out_dims()
    f, x, e = F.cuda(), I.cuda().view(N, C, -1), E.cuda().to(I.dtype).view(N, K, -1)
    y = op._xprop(f, x, bprop=op.deconv, flags=flags)
    dI = op._xprop(f, e, bprop=not op.deconv, flags=flags)
    dF = op._updat(x, e, F.dtype, flags=flags) if op.deconv else op._updat(e, x, F.dtype, flags=flags)
    return y.view(op.o_shape(N)), dI.view(op.i_shape(N)), dF


def check_all(op, orc, N, fdt, idt, flags, seed=0):
    F = rand([op.sizeF], fdt, seed)
    I = rand(op.i_shape(N), idt, seed + 1)
    E = rand(op.o_shape(N), idt, seed + 2)
    tc = fdt == idt and idt != F32 and not flags
    y, dI, dF = run(op, orc, F, I, E, flags)
    Fb = orc.split_filter(F.double().numpy())
    Fa = orc.split_filter(np.abs(F.double().numpy()))
    In, En = I.double().numpy(), E.double().numpy()
    C, K = (op.K, op.C) if op.deconv else (op.C, op.K)
    assert y.dtype == idt and list(y.shape) == op.o_shape(N)
    assert_close(y, orc.fprop(Fb, In), orc.fprop(Fa, np.abs(In)), C * op.trs, idt, tc, "fprop")
    assert dI.dtype == idt and list(dI.shape) == op.i_shape(N)
    assert_close(dI, orc.bprop(Fb, En), orc.bprop(Fa, np.abs(En)), K * op.trs, idt, tc, "bprop")
    assert dF.dtype == fdt and dF.numel() == op.sizeF
    L = N * int(np.prod(op.MPQ if not op.deconv else op.DHW)) + 64
    assert_close(dF, orc.updat(En, In), orc.updat(np.abs(En), np.abs(In)), L, fdt, tc, "updat")


@pytest.mark.parametrize("name", FILES)
@pytest.mark.parametrize("fdt,idt", PAIRS, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("generic", [False, True])
def test_conv_every_layout_and_dtype(name, fdt, idt, generic):
    if generic and (fdt != idt or idt == F32):
        pytest.skip("only 16-bit F and I of one dtype have a second route")
    op, orc = make(name)
    check_all(op, orc, 2, fdt, idt, _lib.FLAG_FORCE_GENERIC if generic else 0)


@pytest.mark.parametrize("N", [1, 2, 28, 64])
@pytest.mark.parametrize("name", ["conv_cfg4.npz", "conv_cfg6.npz", "conv_cfg9.npz", "conv_rand.npz"])
@pytest.mark.parametrize("dt", [F32, BF16, F16], ids=lambda d: str(d).split(".")[-1])
def test_conv_batch_sizes(N, name, dt):
    op, orc = make(name)
    check_all(op, orc, N, dt, dt, 0, seed=N)


@pytest.mark.parametrize("name", FILES)
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("gain", [False, True])
@pytest.mark.parametrize("out32", [False, True])
def test_l2_normalize(name, dt, gain, out32):
    op, orc = make(name)
    if gain and (op.overlapC if op.deconv else op.overlapK):
        with pytest.raises(ValueError):
            op.l2_normalize(rand([op.sizeF], dt, 0).cuda(), gain=torch.ones(op.normSize, device="cuda"))
        return
    F = rand([op.sizeF], dt, 3)
    U = rand([op.sizeF], F32 if out32 else dt, 4)
    G = rand([op.normSize], F32, 5) if gain else None
    f = F.cuda().requires_grad_()
    g = G.cuda().requires_grad_() if gain else None
    y = op.l2_normalize(f, gain=g, dtype=F32 if out32 else None)
    assert y.dtype == (F32 if out32 else dt)
    y.backward(U.cuda())
    Fb, Ub = orc.split_filter(F.double().numpy()), orc.split_filter(U.double().numpy())
    Gn = None if G is None else G.double().numpy()
    ref = orc.l2_normalize(Fb, Gn)
    # longest row: C_b * trs per output channel (KCTRS), K_b * trs per input channel for the deconv (CKTRS)
    n = max(len(k) if op.deconv else len(c) for c, k in op.BCK) * op.trs
    assert_close(y, ref, np.abs(ref), n + 4, y.dtype, False, "l2")   # sum of squares, sqrt, divide, product
    d, dg = orc.l2_normalize_grad(Fb, Ub, Gn)
    mag, dg_mag = l2_grad_magnitude(orc, Fb, Ub, Gn)
    assert_close(f.grad, d, mag, 2 * n + 8, dt, False, "l2 grad")
    if gain:
        assert g.grad.dtype == F32
        assert_close(g.grad, dg, dg_mag, n + 4, F32, False, "l2 dgain")


def l2_grad_magnitude(orc, F, U, gain, epsilon=1e-12):
    """Per element, the l2 gradient's terms in absolute value: (|u g| + |x| sum|u x| |g| / m) / sqrt(m), and
    sum|u x| / sqrt(m) for dgain -- what the rounding errors of the fp32 sums scale with."""
    D, dg, off = [], [], 0
    for f, u in zip(F, U):
        r, du = np.abs(orc._rows(f)), np.abs(orc._rows(u))
        mx = np.maximum((r * r).sum(axis=(1, 2)), epsilon)
        s = (du * r).sum(axis=(1, 2))
        g = np.ones(len(r)) if gain is None else np.abs(gain[off:off + len(r)])
        d = (du * g[:, None, None] + r * (s * g / mx)[:, None, None]) / np.sqrt(mx)[:, None, None]
        D.append((np.moveaxis(d, 0, 1) if orc.deconv else d).ravel())
        dg.append(s / np.sqrt(mx))
        off += len(r)
    return np.concatenate(D), np.concatenate(dg)


def _digest(op, dt, flags):
    F = rand([op.sizeF], dt, 7).cuda()
    I = rand(op.i_shape(16), dt, 8).cuda()
    E = rand(op.o_shape(16), dt, 9).cuda()
    y, dI, dF = run(op, None, F, I, E, flags)
    return [t.detach().cpu().view(torch.int16 if t.element_size() == 2 else torch.int32).numpy().tobytes()
            for t in (y, dI, dF)]


@pytest.mark.parametrize("dt,flags", [(BF16, 0), (BF16, 1), (F32, 0)], ids=["wgmma", "generic16", "fp32"])
def test_bitwise_reproducible(dt, flags):
    for name in ("conv_cfg4.npz", "conv_rand.npz", "conv_cfg9.npz"):
        op, _ = make(name)
        a, b = _digest(op, dt, flags), _digest(op, dt, flags)
        assert a == b, name


def margin_digest():
    """sha256 of the outputs of three layouts on every route (run in a subprocess under an SM margin)."""
    import hashlib
    h = hashlib.sha256()
    for name in ("conv_cfg4.npz", "conv_rand.npz", "conv_cfg9.npz"):
        for dt, flags in ((BF16, 0), (BF16, 1), (F32, 0)):
            for b in _digest(make(name)[0], dt, flags):
                h.update(b)
    return h.hexdigest()


def test_bitwise_under_sm_margin():
    code = "import sys; sys.path.insert(0, %r); from tests.test_conv_gpu import margin_digest; print(margin_digest())" % ROOT
    outs = []
    for margin in ("0", "16"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, BSMM_SM_MARGIN=margin), cwd=ROOT,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(r.stdout.split()[-1])
    assert outs[0] == outs[1] == margin_digest()


@pytest.mark.parametrize("dt,flags,family", [(BF16, 0, "wgmma"), (F16, 0, "wgmma"), (BF16, 1, "fma"), (F32, 0, "fma")])
def test_last_kernel_names_route(dt, flags, family):
    op, _ = make("conv_cfg6.npz")
    F, I = rand([op.sizeF], dt, 0).cuda(), rand(op.i_shape(2), dt, 1).cuda()
    x = I.view(2, op.C, -1)
    op._xprop(F, x, False, flags=flags)
    assert _lib.last_kernel() == family + "_conv_xprop"
    e = op._xprop(F, x, False, flags=flags)
    op._updat(e, x, dt, flags=flags)
    assert _lib.last_kernel() == family + "_conv_updat"


# ---- the l2 kernels against the reference's own (oracle/ref/conv_l2norm.cu) ------------------------------------------
@pytest.mark.parametrize("name", FILES)
@pytest.mark.parametrize("dt", [F32, F16, BF16], ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("gain", [False, True])
def test_l2_normalize_against_reference_kernels(name, dt, gain):
    """y, the sums of squares, dF and dgain against L2NormalizeKCTRS / L2NormalizeCKTRS and their gradients. The
    reference scales by rsqrtf (an approximation) where the kernels here divide by sqrtf, so results agree to the
    fp32 sums' rounding plus one rounding of each side's output, not bit for bit."""
    from oracle import ref_conv
    why = ref_conv.missing()
    if why:
        pytest.skip(why)
    op, orc = make(name)
    if gain and (op.overlapC if op.deconv else op.overlapK):
        pytest.skip("no gain where the normalised rows overlap")
    F = rand([op.sizeF], dt, 13).cuda()
    U = rand([op.sizeF], dt, 14).cuda()
    G = rand([op.normSize], F32, 15).cuda() if gain else None
    f = F.clone().requires_grad_()
    g = G.clone().requires_grad_() if gain else None
    y = op.l2_normalize(f, gain=g)
    y.backward(U)
    ry, rss = ref_conv.l2_normalize(op, F, G)
    rdx, rdg = ref_conv.l2_normalize_grad(op, U, F, rss, G)
    n = max(len(k) if op.deconv else len(c) for c, k in op.BCK) * op.trs
    Fb, Ub = orc.split_filter(F.double().cpu().numpy()), orc.split_filter(U.double().cpu().numpy())
    Gn = None if G is None else G.double().cpu().numpy()
    mag = np.abs(orc.l2_normalize(Fb, Gn))
    rel = 2 * (n + 8) * 2.0 ** -24
    err = np.abs(y.detach().double().cpu().numpy() - ry.double().cpu().numpy())
    lim = rel * mag + 2 * EPS[dt] * mag + 2 * TINY[dt]
    assert (err <= lim).all(), "y: worst excess %.3e" % (err - lim).max()
    gmag, dgmag = l2_grad_magnitude(orc, Fb, Ub, Gn)
    err = np.abs(f.grad.double().cpu().numpy() - rdx.double().cpu().numpy())
    lim = 2 * rel * gmag + 2 * EPS[dt] * gmag + 2 * TINY[dt]
    assert (err <= lim).all(), "dF: worst excess %.3e" % (err - lim).max()
    if gain:
        err = np.abs(g.grad.double().cpu().numpy() - rdg.double().cpu().numpy())
        assert (err <= 2 * rel * dgmag + 1e-30).all(), "dgain: worst %.3e" % err.max()
