"""Helpers the GPU fit tests share: contexts built under the environment switches pb200_create reads, start points near
the oracle's initial one, the oracle's per-iteration record, the trajectory comparison, and a host mirror of the grouped
kernel's chunk rule.  TEST INFRASTRUCTURE ONLY."""
import os

import numpy as np

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L


def ctx_with_env(**env):
    """A context created while ``env`` is set (the switches are read once, at pb200_create)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return L.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def grp_chunk(T, P, G, U=2):
    """Host mirror of fit_kernel.cuh grp_chunk: the grouped kernel's points per lane, -1 when no chunk keeps the bins of
    one step apart (the series then leaves the grouped kernel)."""
    c0 = (T + G - 1) // G
    for c in range(c0, c0 + 25):
        if all(U - 1 < (c * dl) % P < P - (U - 1) for dl in range(1, G)):
            return c
    return -1


def thetas(b, oopts, lay, rng, steep=False):
    """Per series of RaggedBatch ``b``: a point near the oracle's initial_theta, zero-padded to the layout's pstride, and
    the oracle's Prepared.  Returns ``(rows, [(prepared, theta)])``."""
    rows, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        if steep:
            # a steep falling logistic trend: k (t - m) = -520 t stays inside +-600 on the series' own t in [0, 1], so the
            # kernel takes its exp-ratio recurrence; past t ~ 1.36 exp(520 t) overflows a double
            th[0], th[1], th[2:2 + p.S] = -520.0, 0.0, 0.0
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        rows.append(row)
        preps.append((p, th))
    return np.array(rows), preps


def oracle_rows(ds, y, oopts):
    """The oracle's L-BFGS fit and its per-iteration record ``(iteration, f_k, alpha_k, n_evals)``."""
    rows = []
    fr = po.fit(ds, y, opts=oopts, algorithm="LBFGS", trace=rows)
    return fr, np.array(rows).reshape(-1, 4)


def assert_trajectory_head(tr, n_gpu, rows, what, n_head=6):
    """The first accepted iterations against the oracle, at the tolerances of test_lbfgs_trajectory_matches_oracle."""
    head = min(n_gpu, len(rows), n_head)
    assert head >= 1, what
    g, o = tr[:head], rows[:head]
    assert np.array_equal(g[:, 0], np.arange(1, head + 1)), what
    assert np.array_equal(g[:, 3], o[:, 3]), (what, g[:, 3], o[:, 3])
    df = np.abs(g[:, 1] - o[:, 1]) / np.maximum(1.0, np.abs(o[:, 1]))
    assert np.all(df <= 1e-11), (what, df)
    da = np.abs(g[:, 2] - o[:, 2]) / np.abs(o[:, 2])
    assert np.all(da <= 1e-7), (what, da)
