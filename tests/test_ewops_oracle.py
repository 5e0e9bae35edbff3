"""The float64 oracle of bias_relu, dropout and embedding_lookup (oracle/ewops_oracle.py) against independent statements:
Random123's Philox4x32-10 known answers, torch float64 autograd and explicit loops. CPU only."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ewops_oracle as eo


@pytest.mark.parametrize("ctr,key,out", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(ctr, key, out):
    got = eo.philox4x32_10(np.array(ctr, np.uint32), np.array(key, np.uint32))
    assert [int(v) for v in got] == out


def test_mask_words_follow_the_counter_layout():
    """Bit e of the mask is word e % 4 of the Philox block e / 4 with counter (e / 4, call) and key seed, both 64-bit."""
    seed, call, M, kp = -5 * 2 ** 40 + 17, 2 ** 33 + 3, 77, 0.5
    bits = eo.unpack_mask(eo.dropout_mask(seed, call, M, kp), M)
    s, c = seed % 2 ** 64, call % 2 ** 64
    for e in (0, 1, 5, 31, 32, 76):
        g = e // 4
        u = eo.philox4x32_10(np.array([g & 0xffffffff, g >> 32, c & 0xffffffff, c >> 32], np.uint32),
                             np.array([s & 0xffffffff, s >> 32], np.uint32))[e % 4]
        assert bits[e] == (int(u) < int(kp * 2 ** 32))
    words = eo.dropout_mask(seed, call, M, kp).view(np.uint32)
    assert words[-1] >> (M % 32) == 0                     # bits past M are 0
    assert eo.unpack_mask(eo.dropout_mask(1, 2, 100, 1.0), 100).all()


@pytest.mark.parametrize("x_shape,mask_shape", [((6, 5), (1, 5)), ((4, 3, 7), (1, 3, 1)), ((2, 3, 4, 5), (2, 1, 4, 1)),
                                                ((2, 2, 3, 2, 3), (1, 2, 1, 2, 3)), ((3, 4), None)])
def test_broadcast_mask_against_a_loop(x_shape, mask_shape):
    rng = np.random.default_rng(0)
    ms = x_shape if mask_shape is None else mask_shape
    M = int(np.prod(ms))
    bits = rng.random(M) < 0.5
    words = eo.pack_mask(bits)
    x = rng.normal(size=x_shape)
    got = eo.dropout_apply(x, words, 0.7, mask_shape)
    for i in itertools.product(*[range(s) for s in x_shape]):
        m = 0
        for d, (ii, s) in enumerate(zip(i, ms)):
            m = m * s + (ii if s != 1 else 0)
        assert got[i] == (x[i] / 0.7 if bits[m] else 0.0)


@pytest.mark.parametrize("act", ["none", "relu", "fast_gelu"])
@pytest.mark.parametrize("axis,shape", [(-1, (5, 7)), (-1, (2, 3, 6)), (0, (6, 9)), (0, (4, 3, 5))])
def test_bias_relu_against_torch_autograd(act, axis, shape):
    rng = np.random.default_rng(1)
    x, dy = rng.normal(size=shape), rng.normal(size=shape)
    K = shape[axis]
    b = rng.normal(size=K)
    xt, bt = torch.tensor(x, requires_grad=True), torch.tensor(b, requires_grad=True)
    bb = bt.view((K,) + (1,) * (len(shape) - 1)) if axis == 0 else bt
    z = xt + bb
    y = torch.relu(z) if act == "relu" else z * torch.sigmoid(1.702 * z) if act == "fast_gelu" else z
    y.backward(torch.tensor(dy))
    kw = dict(axis=axis, relu=act == "relu", fast_gelu=act == "fast_gelu")
    np.testing.assert_allclose(eo.bias_relu(x, b, **kw), y.detach().numpy(), rtol=1e-13, atol=1e-13)
    dx, db = eo.bias_relu_grad(dy, x, b, **kw)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_embedding_against_torch():
    rng = np.random.default_rng(2)
    C, K = 11, 6
    emb = rng.normal(size=(C, K))
    idx = rng.integers(-3, C + 3, (4, 5))
    dy = rng.normal(size=(4, 5, K))
    ok = (idx >= 0) & (idx < C)
    et = torch.tensor(emb, requires_grad=True)
    y = F.embedding(torch.tensor(np.where(ok, idx, 0)), et) * torch.tensor(ok[..., None], dtype=torch.float64)
    y.backward(torch.tensor(dy))
    np.testing.assert_array_equal(eo.embedding_lookup(emb, idx), y.detach().numpy())
    np.testing.assert_allclose(eo.embedding_grad(dy, idx, C), et.grad.numpy(), rtol=1e-13, atol=1e-13)
    assert not eo.embedding_lookup(emb, idx)[~ok].any()
