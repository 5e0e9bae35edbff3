"""Synthetic block layouts of the reference's tests and benchmarks (host-side helpers, NumPy only).

  bernoulli_layout        i.i.d. Bernoulli(density) with the diagonal forced on
  barabasi_albert_layout  the skewed layout of test/blocksparse_matmul_bench.py:53-68: Barabasi-Albert adjacency
                          + identity + a dense m x m corner (networkx is not needed: the preferential-attachment
                          process is restated here)
  local_strided_layout    causal local + strided attention layout of BASELINE cfg 3 (enwik8.py:66-77 recipe)
"""
import numpy as np


def bernoulli_layout(rng, CB, KB, density):
    lay = (rng.random((CB, KB)) < density).astype(np.int32)
    for i in range(min(CB, KB)):
        lay[i, i] = 1
    return lay


def barabasi_albert_graph(n, m, rng):
    """Adjacency matrix of a Barabasi-Albert graph: nodes m..n-1 arrive one at a time and attach to m distinct
    existing nodes drawn with probability proportional to their degree (the first arrival attaches to nodes 0..m-1)."""
    adj = np.zeros((n, n), dtype=np.int32)
    targets = list(range(m))
    repeated = []                       # every node once per incident edge
    for src in range(m, n):
        for t in targets:
            adj[src, t] = adj[t, src] = 1
        repeated.extend(targets)
        repeated.extend([src] * m)
        chosen = set()
        while len(chosen) < m:
            chosen.add(repeated[int(rng.integers(len(repeated)))])
        targets = sorted(chosen)
    return adj


def barabasi_albert_m(n, density):
    """Smallest m whose layout reaches `density` (bench.py:53-58: blks = 2m(n-m) + m^2 + n - m)."""
    for m in range(1, max(2, n // 2)):
        if (2 * m * (n - m) + m * m + n - m) >= density * n * n:
            return m
    return max(1, n // 2 - 1)


def barabasi_albert_layout(n, density, rng):
    m = barabasi_albert_m(n, density)
    lay = barabasi_albert_graph(n, m, rng) + np.eye(n, dtype=np.int32)
    lay[0:m, 0:m] = 1
    return (lay != 0).astype(np.int32)


def local_strided_layout(ctx_blks, local=4, stride=8):
    """layout[q, k] = 1 iff k <= q and (q - k < local or k % stride == stride - 1)."""
    q = np.arange(ctx_blks)[:, None]
    k = np.arange(ctx_blks)[None, :]
    return ((k <= q) & ((q - k < local) | (k % stride == stride - 1))).astype(np.int32)
