"""Float64 NumPy restatement of the reference's Adafactor step (blocksparse/optimize.py:113-191, src/optimize_op_gpu.cu
Adafactor), written from its description, and of the host-side decay it is driven with.

Kept next to oracle/optimize_oracle.py, whose `condition` it uses. Inputs are taken as given (already rounded to their
storage dtype); every result is float64.
"""
import numpy as np

from .optimize_oracle import condition


def decay(beta2, decay1_power, decay2_power):
    """beta2 (1 - d1) / (1 - d2) (optimize.py:140)."""
    return beta2 * (1.0 - decay1_power) / (1.0 - decay2_power)


def adafactor(g, p, cv, rv, lr, decay, epsilon=1e-30, clip_thresh=1.0, grad_scale=1.0, norm_scale=1.0, saturate=0.0,
              zero_infs=False, zero_nans=False):
    """One step from the given state; returns (p, cv, rv). rv is None for an unfactored param (rank 1 or (1, K)), whose
    cv has one entry per element; a (C, K) param with C > 1 has rv [C] and cv [K]. norm_scale == 0 returns the inputs."""
    p = np.array(p, dtype=np.float64)
    cv = np.array(cv, dtype=np.float64)
    rv = None if rv is None else np.array(rv, dtype=np.float64)
    if norm_scale == 0:
        return p, cv, rv
    x = condition(g, saturate, zero_infs, zero_nans) * (grad_scale * norm_scale)
    if rv is None:
        x = x.reshape(-1)
        cv = decay * cv + (1 - decay) * (x * x + epsilon)
        x = x / np.sqrt(cv)
    else:
        sq = x * x + epsilon
        rv = decay * rv + (1 - decay) * sq.mean(axis=1)
        cv = decay * cv + (1 - decay) * sq.mean(axis=0)
        x = x / np.sqrt(rv / rv.mean())[:, None] / np.sqrt(cv)[None, :]
    rms = np.mean(x * x)
    p = p - (lr * x / max(1.0, np.sqrt(rms) / clip_thresh)).reshape(p.shape)
    return p, cv, rv
