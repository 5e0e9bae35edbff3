"""Conv edge bias and cwise_linear without a GPU: the float64 oracle (oracle/conv_bias_oracle.py) and the package's
tables and checkers against fixtures recorded from the reference's own conv.py (tests/golden/make_golden_conv_bias.py),
the tables against a brute-force enumeration of padded taps (dilation > 1 included), the two reference quirks the
package does not inherit, pinned signatures and exports, every ValueError and the C entries' argument errors."""
import inspect
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._util import GOLDEN, ROOT, golden_files

sys.path.insert(0, GOLDEN)
from make_golden_conv import hash_values  # noqa: E402
from oracle import conv_bias_oracle as cbo  # noqa: E402
from blocksparse_b200 import _lib  # noqa: E402
from blocksparse_b200.conv_bias import ConvEdgeBias, conv_edge_bias_init, cwise_linear, deconv_edge_bias_init  # noqa

EDGE = golden_files("edge_bias_")
CWISE = golden_files("cwise_")
REF = os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference"


def edge_args(z):
    strides = z["strides"].tolist() or None
    y, x, w = z["y_shape"].tolist(), z["x_shape"].tolist(), z["w_shape"].tolist()
    fmt, deconv = str(z["data_format"]), bool(z["deconv"])
    return (x, y, w, strides, "SAME", fmt, None, deconv) if deconv else (y, x, w, strides, "SAME", fmt, None, deconv)


def edge_inputs(z, shape):
    io = z["io_shape"].tolist()
    size = int(np.prod(io))
    return (hash_values(size, 1).reshape(io), hash_values(size, 2).reshape(io),
            hash_values(int(np.prod(shape)), 3).reshape(shape), hash_values(int(np.prod(shape)), 4).reshape(shape))


def check(z, key, got, tol=1e-6):
    ref = z[key]
    np.testing.assert_allclose(np.asarray(got, np.float64).ravel()[z[key + "_idx"]], ref, rtol=tol,
                               atol=tol * max(1.0, np.abs(ref).max()), err_msg=key)


def ref_map(z):
    return np.split(z["map"], np.cumsum(z["map_sizes"])[:-1])


@pytest.mark.parametrize("name", EDGE)
def test_edge_oracle_matches_reference(name):
    z = np.load(os.path.join(GOLDEN, name))
    y, x, w, st, pad, fmt, dl, deconv = edge_args(z)
    orc = cbo.EdgeBias(y, x, w, st, pad, fmt, dl, deconv)
    assert list(orc.shape) == z["shape"].tolist() and orc.edgeEntries == int(z["entries"])
    assert [list(m) for m in orc.edgeBiasMap] == [m.tolist() for m in ref_map(z)]
    np.testing.assert_array_equal(orc.lut(), z["lut"])
    X, D, G, B = edge_inputs(z, orc.shape)
    check(z, "y", orc.edge_bias(X, G, B))
    dx, dg, db = orc.edge_bias_grad(D, X, G)
    check(z, "dx", dx)
    check(z, "dg", dg, 1e-5)       # the reference sums in float32
    check(z, "db", db, 1e-5)


@pytest.mark.parametrize("name", EDGE)
def test_edge_package_matches_reference(name):
    z = np.load(os.path.join(GOLDEN, name))
    args = edge_args(z)
    ConvEdgeBias.Cache.clear()
    op = ConvEdgeBias(*args)
    assert list(op.shape) == z["shape"].tolist() and op.edgeEntries == int(z["entries"])
    assert op.edgeBiasDim == len(z["map_sizes"])
    assert op.edgeBiasMap == [m.tolist() for m in ref_map(z)]
    np.testing.assert_array_equal(op.edgeBiasLut, z["lut"])                 # bit for bit at dilation 1
    assert ConvEdgeBias(*args)._entry is op._entry                         # cached per geometry
    X, D, G, B = edge_inputs(z, op.shape)
    check(z, "y", op.edge_bias_test(X, G, B))
    dx, dg, db = op.edge_bias_grad_test(D, X, G)
    check(z, "dx", dx)
    check(z, "dg", dg, 1e-5)
    check(z, "db", db, 1e-5)


def test_init_helpers_read_shapes():
    z = np.load(os.path.join(GOLDEN, "edge_bias_deconv.npz"))
    y, x, w = (torch.empty(z[k].tolist(), device="meta") for k in ("y_shape", "x_shape", "w_shape"))
    op = deconv_edge_bias_init(y, x, w, strides=[1, 2, 2, 1])
    assert list(op.shape) == z["shape"].tolist() and op.deconv
    z = np.load(os.path.join(GOLDEN, "edge_bias_stride2.npz"))
    y, x, w = (torch.empty(z[k].tolist(), device="meta") for k in ("y_shape", "x_shape", "w_shape"))
    assert list(conv_edge_bias_init(y, x, w, strides=[1, 2, 2, 1]).shape) == z["shape"].tolist()


@pytest.mark.parametrize("name", CWISE)
def test_cwise_oracle_matches_reference(name):
    z = np.load(os.path.join(GOLDEN, name))
    shape = tuple(z["shape"])
    C = shape[1]
    x = hash_values(int(np.prod(shape)), 5).reshape(shape)
    dy = hash_values(int(np.prod(shape)), 6).reshape(shape)
    a, b = hash_values(C, 7), hash_values(C, 8)
    for relu in (False, True):
        tag = "_relu" if relu else ""
        check(z, "y" + tag, cbo.cwise_linear(x, a, b, relu))
        dx, da, db = cbo.cwise_linear_grad(dy, x, a, b, relu)
        check(z, "dx" + tag, dx)
        check(z, "da" + tag, da, 1e-5)
        check(z, "db" + tag, db, 1e-5)


def test_cwise_bias_first_gradient_by_differences():
    """The bias_first gradient (restated from the reference kernel, which the NumPy checker lacks) against central
    differences of the forward."""
    rng = np.random.default_rng(0)
    x, dy = rng.normal(size=(3, 4, 5)), rng.normal(size=(3, 4, 5))
    a, b = rng.normal(size=4), rng.normal(size=4)
    dx, da, db = cbo.cwise_linear_grad(dy, x, a, b, relu=True, bias_first=True)
    f = lambda x_, a_, b_: np.sum(dy * cbo.cwise_linear(x_, a_, b_, relu=True, bias_first=True))
    h = 1e-6
    for c in range(4):
        e = np.eye(4)[c] * h
        assert abs((f(x, a + e, b) - f(x, a - e, b)) / (2 * h) - da[c]) < 1e-5
        assert abs((f(x, a, b + e) - f(x, a, b - e)) / (2 * h) - db[c]) < 1e-5
    ex = np.zeros_like(x)
    ex[1, 2, 3] = h
    assert abs((f(x + ex, a, b) - f(x - ex, a, b)) / (2 * h) - dx[1, 2, 3]) < 1e-5


def brute_pattern_map(y, x, w, st, fmt, dl, deconv):
    """Edge pattern lists by enumerating every (position, tap) pair: a tap is padded when the input coordinate it
    reads (conv), or the deconv-output coordinate it would come from, falls outside the image in some dim."""
    last = fmt[-1] == "C"
    sp = (lambda s: s[1:-1]) if last else (lambda s: s[2:])
    Y, X, S = sp(y), sp(x), w[:-2]
    st = [1] * len(S) if st is None else sp(st)
    dl = [1] * len(S) if dl is None else sp(dl)
    small, big = (X, Y) if deconv else (Y, X)          # the conv's output and input (the deconv's are swapped)
    pad = [max((q - 1) * s + (k - 1) * d + 1 - xx, 0) // 2 for k, q, xx, s, d in zip(S, small, big, st, dl)]
    out_dims = Y
    groups = {}
    for o, pos in enumerate(itertools.product(*[range(n) for n in out_dims])):
        key = []
        for tap in itertools.product(*[range(k) for k in S]):
            padded = False
            for i, (p, t) in enumerate(zip(pos, tap)):
                if deconv:          # output position p of the deconv receives tap (flipped) from q = (p - off) / s
                    q = p - ((S[i] - 1) * dl[i] - pad[i]) + (S[i] - 1 - t) * dl[i]
                    padded |= q % st[i] == 0 and not 0 <= q // st[i] < X[i]
                else:
                    c = p * st[i] - pad[i] + t * dl[i]
                    padded |= not 0 <= c < X[i]
            if padded:
                key.append(tap)
        if key:
            groups.setdefault(tuple(key), []).append(o)
    return sorted(groups.values(), key=lambda v: v[0])


@pytest.mark.parametrize("y,x,w,st,fmt,dl,deconv", [
    ([1, 8, 8, 4], [1, 8, 8, 4], [3, 3, 4, 4], None, "NHWC", [1, 2, 2, 1], False),
    ([1, 4, 9, 7], [1, 4, 9, 7], [3, 2, 4, 4], None, "NCHW", [1, 1, 3, 1], False),
    ([2, 6, 3], [2, 11, 3], [4, 3, 3], [1, 2, 1], "NWC", [1, 2, 1], False),
    ([1, 2, 3, 4, 5], [1, 2, 3, 4, 5], [3, 3, 3, 5, 5], None, "NDHWC", [1, 1, 2, 1, 1], False),
    ([1, 9, 11, 2], [1, 5, 6, 3], [3, 3, 2, 3], [1, 2, 2, 1], "NHWC", None, True),
    ([1, 3, 10, 12], [1, 2, 5, 4], [3, 3, 3, 2], [1, 1, 2, 3], "NCHW", [1, 1, 2, 1], True),
])
def test_tables_against_brute_force(y, x, w, st, fmt, dl, deconv):
    args = (x, y, w, st, "SAME", fmt, dl, True) if deconv else (y, x, w, st, "SAME", fmt, dl)
    op = ConvEdgeBias(*args)
    expect = brute_pattern_map(y, x, w, st, fmt, dl, deconv)
    assert op.edgeBiasMap == expect
    orc = cbo.EdgeBias(*args)
    assert [list(m) for m in orc.edgeBiasMap] == expect
    pos = np.full(int(np.prod(op.MPQ)), -1)
    for e, m in enumerate(expect):
        pos[m] = e
    np.testing.assert_array_equal(op._pos_edge, pos)


def test_quirk_dilated_same_padding():
    """The reference pads a dilated SAME conv by the undilated filter size: 8x8, 3x3, dilation 2 gives it 15 edge
    patterns where TensorFlow's padding of 2 gives 8."""
    args = ([1, 8, 8, 4], [1, 8, 8, 4], [3, 3, 4, 4], None, "SAME", "NHWC", [1, 2, 2, 1])
    assert ConvEdgeBias(*args).edgeBiasDim == 8
    assert cbo.EdgeBias(*args).edgeBiasDim == 8 and cbo.EdgeBias(*args).padding == [0, 2, 2]
    assert cbo.EdgeBias(*args, undilated_pad=True).edgeBiasDim == 15


def test_quirk_valid_has_no_edges():
    """The reference's constructor raises AttributeError for VALID; here the shape is (0, K) / (K, 0)."""
    op = ConvEdgeBias([1, 6, 6, 4], [1, 8, 8, 4], [3, 3, 4, 4], padding="VALID")
    assert op.shape == (0, 4) and op.edgeBiasDim == 0 and op.edgeBiasMap == [] and op.edgeEntries == 0
    assert ConvEdgeBias([1, 4, 6, 6], [1, 4, 8, 8], [3, 3, 4, 4], padding="VALID", data_format="NCHW").shape == (4, 0)


def test_signatures_and_exports():
    assert str(inspect.signature(ConvEdgeBias.__init__)) == (
        "(self, y_shape, x_shape, w_shape, strides=None, padding='SAME', data_format='NHWC', dilations=None, "
        "deconv=False)")
    assert str(inspect.signature(ConvEdgeBias.__call__)) == "(self, x, g, b, inference=False, bench=0, name=None)"
    assert str(inspect.signature(cwise_linear)) == "(x, gain=None, bias=None, relu=False, bias_first=False, use_tf=False)"
    for f in (conv_edge_bias_init, deconv_edge_bias_init):
        assert str(inspect.signature(f)) == "(y, x, w, strides=None, padding='SAME', data_format='NHWC', dilations=None)"
    import blocksparse_b200
    from blocksparse_b200 import conv, conv_bias
    assert conv_bias.__all__ == ["ConvEdgeBias", "conv_edge_bias_init", "deconv_edge_bias_init", "cwise_linear"]
    for n in conv_bias.__all__:
        assert getattr(blocksparse_b200, n) is getattr(conv_bias, n) is getattr(conv, n)
        assert n not in blocksparse_b200.__all__ and n not in conv.__all__
    assert isinstance(ConvEdgeBias.Cache, dict)


def test_package_does_not_import_oracle():
    code = "import sys, blocksparse_b200; print(any(m == 'oracle' or m.startswith('oracle.') for m in sys.modules))"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.split()[-1] == "False", r.stderr[-2000:]


@pytest.mark.parametrize("kw", [
    dict(data_format="NHCW"),
    dict(padding="FULL"),
    dict(padding=(1, 1)),
    dict(w_shape=[4, 4, 3, 3]),                            # KCRS, as the reference's own test passes for NCHW
    dict(w_shape=[3, 3, 4, 5]),                            # K mismatch
    dict(y_shape=[1, 8, 4]),                               # ranks disagree
    dict(w_shape=[3, 4, 4]),
    dict(strides=[1, 1]),
    dict(dilations=[1, 0, 1, 1]),
    dict(x_shape=[1, 8, 0, 4]),
])
def test_constructor_errors(kw):
    args = dict(y_shape=[1, 8, 8, 4], x_shape=[1, 8, 8, 4], w_shape=[3, 3, 4, 4])
    args.update(kw)
    with pytest.raises(ValueError):
        ConvEdgeBias(**args)


def test_call_errors_before_any_launch():
    op = ConvEdgeBias([1, 8, 8, 4], [1, 8, 8, 4], [3, 3, 4, 4])
    x, g = torch.zeros(2, 8, 8, 4), torch.zeros(op.shape)
    with pytest.raises(ValueError):
        op(x, g, g)                                        # CPU tensors
    with pytest.raises(ValueError):
        cwise_linear(torch.zeros(2, 3), torch.ones(3))      # CPU tensors
    with pytest.raises(ValueError):
        cwise_linear(torch.zeros(2, 3), use_tf=True)


def test_c_abi_argument_errors():
    lib = _lib.load()
    null, fake, E_ARG, E_LIMIT = None, 16, -3, -4
    # dtype, layout, pos_edge, lut, edges, entries, x, g, b, y, N, MPQ, K, inference, stream
    args = [0, 1, fake, fake, 8, 28, fake, fake, fake, fake, 2, 64, 4, 0, null]
    for i, v in ((0, 3), (1, 2), (2, null), (8, null), (4, 0), (5, 4), (5, 65), (6, null), (10, -1), (12, 0)):
        bad = list(args)
        bad[i] = v
        assert lib.bsmm_edge_bias(*bad) == E_ARG, (i, v)
    bad = list(args)
    bad[13], bad[9] = 1, 32                                # inference writes x in place
    assert lib.bsmm_edge_bias(*bad) == E_ARG
    bad = list(args)
    bad[4], bad[5], bad[11] = 70000, 70000, 2 ** 20
    assert lib.bsmm_edge_bias(*bad) == E_LIMIT
    bad = list(args)
    bad[11] = 2 ** 31
    assert lib.bsmm_edge_bias(*bad) == E_LIMIT
    # dtype, layout, pos_edge, lut, edges, entries, max_count, dy, x, g, dx, dg, db, ws, N, MPQ, K, stream
    gargs = [0, 1, fake, fake, 8, 28, 6, fake, fake, fake, fake, fake, fake, fake, 2, 64, 4, null]
    for i, v in ((6, 0), (6, 29), (8, null), (11, null), (13, null)):
        bad = list(gargs)
        bad[i] = v
        assert lib.bsmm_edge_bias_grad(*bad) == E_ARG, (i, v)
    assert lib.bsmm_edge_bias_grad_workspace_bytes(2, 8, 6, 4) == 2 * 1 * 8 * 4 * 4
    assert lib.bsmm_edge_bias_grad_workspace_bytes(-1, 8, 6, 4) == 0
    # dtype, x, a, b, y, N, C, DHW, relu, swap, stream
    cargs = [0, fake, fake, fake, fake, 2, 8, 16, 0, 0, null]
    for i, v in ((0, 7), (1, null), (4, null), (5, -1), (6, 0), (7, 0)):
        bad = list(cargs)
        bad[i] = v
        assert lib.bsmm_cwise_linear(*bad) == E_ARG, (i, v)
    bad = list(cargs)
    bad[2], bad[3] = null, null
    assert lib.bsmm_cwise_linear(*bad) == E_ARG
    bad = list(cargs)
    bad[5], bad[7] = 2 ** 40, 2 ** 30
    assert lib.bsmm_cwise_linear(*bad) == E_LIMIT
    # dtype, dy, xy, a, b, dx, da, db, ws, N, C, DHW, relu, swap, stream
    gargs = [0, fake, fake, fake, fake, fake, fake, fake, fake, 2, 8, 16, 0, 0, null]
    for i, v in ((6, null), (7, null), (2, null), (5, null), (8, null)):
        bad = list(gargs)
        bad[i] = v
        assert lib.bsmm_cwise_linear_grad(*bad) == E_ARG, (i, v)
    bad = list(gargs)
    bad[3], bad[6], bad[12] = null, null, 1                # relu without a gain reads y and writes dx
    bad[2] = null
    assert lib.bsmm_cwise_linear_grad(*bad) == E_ARG
    assert lib.bsmm_cwise_linear_grad_workspace_bytes(2, 8, 16) == 2 * 1 * 8 * 4
    assert lib.bsmm_cwise_linear_grad_workspace_bytes(100, 8, 1) == 2 * 13 * 8 * 4


def test_no_reference_line_in_new_sources():
    srcs = [os.path.join(REF, "src", f) for f in ("edge_bias_op_gpu.cu", "cwise_linear_op_gpu.cu")]
    if not all(os.path.isfile(p) for p in srcs):
        pytest.skip("no reference checkout")
    lines = set()
    for p in srcs:
        with open(p, errors="replace") as fh:
            lines.update(s for s in ("".join(line.split()) for line in fh) if len(s) >= 10)
    tracked = subprocess.run(["git", "ls-files", "oracle"], cwd=ROOT, capture_output=True, text=True)
    if tracked.returncode != 0:
        pytest.skip("not a git checkout")
    paths = sorted(set(tracked.stdout.split() + ["oracle/conv_bias_oracle.py", "oracle/ref_conv_bias.py",
                                                 "oracle/ref/conv_bias.cu", "oracle/ref/cwise_linear.cu"]))
    for path in paths:
        full = os.path.join(ROOT, path)
        if not os.path.isfile(full):
            continue
        with open(full, errors="replace") as fh:
            for n, line in enumerate(fh, 1):
                assert "".join(line.split()) not in lines, "%s:%d repeats a line of the reference sources" % (path, n)
