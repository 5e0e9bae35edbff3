"""CPU restatement of the reference's block-sparse weight utilities -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py:
only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this package).

Each function follows the reference line by line (file:line relative to the openai/blocksparse source tree):
  l2_normalize / l2_normalize_grad   blocksparse/matmul.py:421-443 (l2_normalize_test, l2_normalize_grad_test); the gain
                                     variant follows the kernel comment src/blocksparse_l2_norm_op_gpu.cu:704-708
  block_norm / l2_decay / threshold_prune / prune_topk
                                     src/optimize_op_gpu.cu:891-952, 794-855, 1006-1070, 985-995 and the host wrapper
                                     src/optimize_op.cc:652-672 (keep = (uint)(blocks * (1 - sparsity) + 0.5))
  identity_init                      src/blocksparse_matmul_op_gpu.cu:2988-3015 (and the commented NumPy version matmul.py:320-329)
  reduced_dw                         test/blocksparse_reduced_dw_test.py:87-112 (the reference test's own NumPy expectation)
  SparseProj tables                  blocksparse/matmul.py:843-872
Parity status: pinned where the reference has NumPy code to import (l2_normalize_test / l2_normalize_grad_test:
tests/golden/make_golden.py records them in wutil_*.npz); the kernel-only ops have no reference-side NumPy and are
restated from the CUDA source (they are elementwise / per-block reductions).
"""
import numpy as np


def l2_normalize(fprop_list, W, bsize, gain=None, epsilon=1e-12):
    W = W.astype(np.float64).copy()
    ss_all = {}
    for k, lut in fprop_list:
        ws = [w for c, w in lut]
        if not ws:
            continue
        W2 = W[ws, :, :].reshape(-1, bsize)
        ss = np.sum(np.square(W2), axis=0, keepdims=True)
        norm = np.sqrt(np.maximum(ss, epsilon))
        g = 1.0 if gain is None else gain[k * bsize:(k + 1) * bsize][None, :]
        for w in ws:
            W[w, :, :] = W[w, :, :] / norm * g
        ss_all[k] = ss[0]
    return W, ss_all


def l2_normalize_grad(fprop_list, W, U, bsize, gain=None, epsilon=1e-12):
    """grad_x = (grad_y*g + x * (sum_sqr >= eps) * sum(-grad_y*g * x / norm^2)) / norm ; grad_g = sum(grad_y * x / norm)."""
    W = W.astype(np.float64)
    DX = np.zeros_like(W)
    U = U.astype(np.float64)
    K = max(k for k, _ in fprop_list) + 1
    DG = np.zeros(K * bsize)
    for k, lut in fprop_list:
        ws = [w for c, w in lut]
        if not ws:
            continue
        W2 = W[ws, :, :].reshape(-1, bsize)
        U2 = U[ws, :, :].reshape(-1, bsize)
        g = np.ones((1, bsize)) if gain is None else gain[k * bsize:(k + 1) * bsize][None, :].astype(np.float64)
        sum_sqr_w = np.sum(np.square(W2), axis=0, keepdims=True)
        max_w = np.maximum(sum_sqr_w, epsilon)
        norm_grad = (U2 * g + W2 * (sum_sqr_w >= epsilon) * np.sum(-U2 * g * W2 / max_w, axis=0, keepdims=True)) / np.sqrt(max_w)
        DG[k * bsize:(k + 1) * bsize] = np.sum(U2 * W2 / np.sqrt(max_w), axis=0)
        norm_grad = norm_grad.reshape(-1, bsize, bsize)
        for i, w in enumerate(ws):
            DX[w, :, :] = norm_grad[i]
    return DX, DG


def block_norm(W, norm="max"):
    W = W.astype(np.float64).reshape(W.shape[0], -1)
    return np.abs(W).max(axis=1) if norm == "max" else np.sqrt(np.square(W).sum(axis=1))


def l2_decay(W, gate=None, rate=0.05, epsilon=1e-12):
    out = W.astype(np.float64).copy()
    for b in range(W.shape[0]):
        if gate is not None and gate[b] == 0.0:
            continue
        p = out[b]
        decay = min(1.0 / np.sqrt(np.square(p).sum() + epsilon) * rate, 1.0)
        out[b] = p - p * decay
    return out


def threshold_prune(W, threshold, norm="max"):
    return (block_norm(W, norm) >= threshold).astype(np.float32)


def prune_topk(norms, sparsity):
    blocks = len(norms)
    keep = int(np.float32(blocks) * (np.float32(1.0) - np.float32(sparsity)) + np.float32(0.5))
    idx = np.argsort(-norms, kind="stable")
    gate = np.zeros(blocks, dtype=np.float32)
    gate[idx[:keep]] = 1.0
    return gate


def identity_init(updat_list, CB, KB, bsize, scale=1.0):
    W = np.zeros((len(updat_list), bsize, bsize), dtype=np.float32)
    for w, (cb, kb) in enumerate(updat_list):
        if (cb % KB) == (kb % CB):
            W[w] = np.eye(bsize, dtype=np.float32) * scale
    return W


def reduced_dw(XS, YS, scale, bsize, axis, norm, DWA=None, round_red=None):
    """test/blocksparse_reduced_dw_test.py:87-112. round_red, if given, maps X_RED / Y_RED to the values a kernel that
    stores them in a narrower dtype multiplies (e.g. rounding to float16); the returned X_RED / Y_RED are rounded too."""
    depth = len(XS)
    if axis == 0:
        bx, by, N = XS[0].shape[0] // bsize, YS[0].shape[0] // bsize, XS[0].shape[1]
        X_RED = np.zeros([bx, depth, N]); Y_RED = np.zeros([by, depth, N])
        for i in range(depth):
            X = XS[i].reshape([bx, bsize, N]); Y = YS[i].reshape([by, bsize, N])
            if norm == "max":
                X_RED[:, i, :] = np.max(np.abs(X), axis=1); Y_RED[:, i, :] = np.max(np.abs(Y), axis=1)
            else:
                X_RED[:, i, :] = np.sqrt(np.sum(np.square(X), axis=1)); Y_RED[:, i, :] = np.sqrt(np.sum(np.square(Y), axis=1))
        if round_red is not None:
            X_RED, Y_RED = round_red(X_RED), round_red(Y_RED)
        DW = np.dot(X_RED.reshape(bx, -1), Y_RED.reshape(by, -1).T) * scale
    else:
        bx, by, N = XS[0].shape[1] // bsize, YS[0].shape[1] // bsize, XS[0].shape[0]
        X_RED = np.zeros([depth, N, bx]); Y_RED = np.zeros([depth, N, by])
        for i in range(depth):
            X = XS[i].reshape([N, bx, bsize]); Y = YS[i].reshape([N, by, bsize])
            if norm == "max":
                X_RED[i] = np.max(np.abs(X), axis=2); Y_RED[i] = np.max(np.abs(Y), axis=2)
            else:
                X_RED[i] = np.sqrt(np.sum(np.square(X), axis=2)); Y_RED[i] = np.sqrt(np.sum(np.square(Y), axis=2))
        if round_red is not None:
            X_RED, Y_RED = round_red(X_RED), round_red(Y_RED)
        DW = np.dot(X_RED.reshape(-1, bx).T, Y_RED.reshape(-1, by)) * scale
    if DWA is not None:
        DW = DW + DWA
    return DW, X_RED, Y_RED
