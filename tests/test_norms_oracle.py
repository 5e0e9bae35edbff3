"""The float64 layer norm oracle (oracle/norms_oracle.py) against the fixtures the reference's own checkers wrote
(tests/golden/norms_*.npz), against torch's float64 layer_norm and its autograd, and on a row whose mean dwarfs its
spread, where it stays exact while E[x^2] - E[x]^2 in fp32 does not. The package's NumPy checkers are held to the
oracle too."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import norms_oracle as orc
from tests._util import golden_files, GOLDEN
from blocksparse_b200 import norms

FILES = golden_files("norms_")


def test_fixtures_present():
    assert len(FILES) == 16
    tags = {f.split("_")[1] for f in FILES}
    assert tags == {"ax0", "ax1"}


@pytest.mark.parametrize("name", FILES)
def test_oracle_matches_reference_fixtures(name):
    d = np.load("%s/%s" % (GOLDEN, name))
    kw = dict(axis=int(d["axis"]), segments=int(d["segments"]), epsilon=float(d["epsilon"]), relu=bool(d["relu"]))
    y = orc.layer_norm(d["x"], d["g"], d["b"], **kw)
    dx, dg, db = orc.layer_norm_grad(d["dy"], d["x"], d["g"], d["b"], **kw)
    for got, ref in ((y, d["y"]), (dx, d["dx"]), (dg, d["dg"]), (db, d["db"])):
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    # the package's checkers restate the same maths
    cy = norms.layer_norm_test(d["x"], d["g"], d["b"], **kw)
    cdx, cdg, cdb = norms.layer_norm_grad_test(d["dy"], d["x"], d["g"], d["b"], **kw)
    for got, ref in ((cy, d["y"]), (cdx, d["dx"]), (cdg.ravel(), d["dg"]), (cdb.ravel(), d["db"])):
        np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("shape", [(5, 64), (3, 4, 33), (2, 1)])
@pytest.mark.parametrize("relu", [False, True])
def test_oracle_matches_torch_float64_last_axis(shape, relu):
    rng = np.random.default_rng(sum(shape))
    x = torch.tensor(rng.normal(1, 3, shape), requires_grad=True)
    K = shape[-1]
    g = torch.tensor(rng.uniform(0.5, 1.5, K), requires_grad=True)
    b = torch.tensor(rng.normal(0, 1, K), requires_grad=True)
    y = F.layer_norm(x, (K,), g, b, eps=1e-5)
    if relu:
        y = torch.relu(y)
    dy = torch.tensor(rng.normal(0, 1, shape))
    y.backward(dy)
    ref = orc.layer_norm(x.detach().numpy(), g.detach().numpy(), b.detach().numpy(), epsilon=1e-5, relu=relu)
    dx, dg, db = orc.layer_norm_grad(dy.numpy(), x.detach().numpy(), g.detach().numpy(), b.detach().numpy(),
                                     epsilon=1e-5, relu=relu)
    np.testing.assert_allclose(ref, y.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dx, x.grad.numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(dg, g.grad.numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(db, b.grad.numpy(), rtol=1e-10, atol=1e-10)


def test_oracle_first_axis_is_the_transposed_last_axis():
    rng = np.random.default_rng(3)
    x, dy = rng.normal(0, 1, (40, 7)), rng.normal(0, 1, (40, 7))
    g, b = rng.uniform(0.5, 1.5, 40), rng.normal(0, 1, 40)
    np.testing.assert_allclose(orc.layer_norm(x, g, b, axis=0), orc.layer_norm(x.T, g, b).T, rtol=1e-13, atol=1e-14)
    got, ref = orc.layer_norm_grad(dy, x, g, b, axis=0), orc.layer_norm_grad(dy.T, x.T, g, b)
    np.testing.assert_allclose(got[0], ref[0].T, rtol=1e-13, atol=1e-14)
    np.testing.assert_allclose(got[1], ref[1], rtol=1e-13, atol=1e-14)


def test_large_mean_is_stable_in_the_oracle_and_not_in_the_naive_fp32_variance():
    """|mean| = 1e4 std: the centred variance recovers std^2 to float64 precision; E[x^2] - E[x]^2 in fp32 loses it
    (fp32 carries 24 bits, and x^2 ~ 1e8 std^2 leaves none for the spread)."""
    rng = np.random.default_rng(7)
    std = 1.0
    x = (1e4 * std + rng.normal(0, std, (4, 1024))).astype(np.float32)
    x64 = x.astype(np.float64)
    true_var = x64.var(axis=1)
    mean, rstd = orc.statistics(x64, -1, 1, 0.0)
    np.testing.assert_allclose(1.0 / rstd[:, 0] ** 2, true_var, rtol=1e-10)
    naive = (x * x).mean(axis=1, dtype=np.float32) - np.square(x.mean(axis=1, dtype=np.float32))
    assert np.max(np.abs(naive - true_var) / true_var) > 0.1
