"""The float64 oracle of softmax_cross_entropy and the transposes (tests/_xent_oracle.py) against scipy's logsumexp and
torch's float64 cross_entropy with autograd, on CPU, including bad labels and -inf entries."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy.special import logsumexp

from tests import _xent_oracle as orc


def _torch_ref(x, labels, dy):
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    loss = F.cross_entropy(xt.reshape(-1, x.shape[-1]), torch.as_tensor(labels).reshape(-1).long(), reduction="none")
    loss.backward(torch.as_tensor(dy, dtype=torch.float64).reshape(-1))
    return loss.detach().numpy().reshape(x.shape[:-1]), xt.grad.numpy()


@pytest.mark.parametrize("shape", [(7,), (5, 1), (4, 10), (2, 3, 257), (3, 4096)])
def test_loss_lse_and_grad_match_scipy_and_torch(shape):
    rng = np.random.default_rng(sum(shape))
    x = rng.normal(0, 3, shape)
    K = shape[-1]
    labels = rng.integers(0, K, shape[:-1])
    if labels.size > 1:
        labels.reshape(-1)[0], labels.reshape(-1)[-1] = 0, K - 1
    dy = rng.normal(0, 1, shape[:-1])
    loss, lse = orc.softmax_cross_entropy(x, labels)
    assert loss.shape == lse.shape == shape[:-1]
    np.testing.assert_allclose(lse, logsumexp(x, axis=-1), rtol=1e-13, atol=1e-13)
    ref_loss, ref_grad = _torch_ref(x, labels, dy)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(orc.softmax_cross_entropy_grad(x, labels, dy), ref_grad, rtol=1e-12, atol=1e-14)


def test_infinite_logits_match_torch():
    """-inf entries get probability 0, a label at -inf gives +inf, an all -inf row gives NaN: as torch float64."""
    x = np.array([[0.5, -np.inf, 2.0, -np.inf], [1.0, -np.inf, 3.0, 0.0], [-np.inf] * 4, [-np.inf, -np.inf, 7.0, -np.inf]])
    labels = np.array([2, 1, 0, 2])
    dy = np.array([1.0, 0.5, 2.0, -1.5])
    loss, lse = orc.softmax_cross_entropy(x, labels)
    ref_loss, ref_grad = _torch_ref(x, labels, dy)
    np.testing.assert_allclose(loss, ref_loss, rtol=1e-13)
    assert np.isposinf(loss[1]) and np.isnan(loss[2]) and loss[3] == 0.0
    assert np.isneginf(lse[2])
    np.testing.assert_allclose(lse[[0, 1, 3]], logsumexp(x[[0, 1, 3]], axis=-1), rtol=1e-13)
    g = orc.softmax_cross_entropy_grad(x, labels, dy)
    np.testing.assert_allclose(g[[0, 1, 3]], ref_grad[[0, 1, 3]], rtol=1e-13, atol=1e-15)
    assert np.all(g[0, [1, 3]] == 0) and np.all(np.isnan(g[2])) and np.all(np.isnan(ref_grad[2]))


def test_out_of_range_labels_give_nan_rows_only():
    rng = np.random.default_rng(3)
    x = rng.normal(0, 1, (5, 6))
    labels = np.array([0, 6, -1, 5, 255])
    loss, lse = orc.softmax_cross_entropy(x, labels)
    bad = np.array([False, True, True, False, True])
    assert np.all(np.isnan(loss[bad])) and np.all(np.isnan(lse[bad]))
    assert np.all(np.isfinite(loss[~bad]))
    g = orc.softmax_cross_entropy_grad(x, labels, np.ones(5))
    assert np.all(np.isnan(g[bad])) and np.all(np.isfinite(g[~bad]))
    ref_loss, ref_grad = _torch_ref(x[~bad], labels[~bad], np.ones(2))
    np.testing.assert_allclose(loss[~bad], ref_loss, rtol=1e-13)
    np.testing.assert_allclose(g[~bad], ref_grad, rtol=1e-13, atol=1e-15)


def test_transposes_and_argument_checks():
    x = np.arange(2 * 3 * 5 * 7).reshape(2, 3, 5, 7)
    y = orc.transpose_0213(x)
    assert y.shape == (2, 5, 3, 7) and y.flags.c_contiguous
    np.testing.assert_array_equal(y, torch.as_tensor(x).permute(0, 2, 1, 3).numpy())
    np.testing.assert_array_equal(orc.transpose_0213(y), x)
    m = np.arange(12).reshape(3, 4)
    np.testing.assert_array_equal(orc.transpose_2d(m), m.T)
    for call in (lambda: orc.transpose_0213(m), lambda: orc.transpose_2d(x),
                 lambda: orc.softmax_cross_entropy(np.zeros((3, 4)), np.zeros(2, np.int64))):
        with pytest.raises(ValueError):
            call()
