"""Numpy restatement of the Monte-Carlo interval sampler of ``csrc/mc_kernel.cuh``.

This is a statement of exactly what ``mc_kernel`` computes -- its own counter-based Philox4x32-10
stream, its per-model key, its changepoint and noise draws and its percentile rule -- so that the
kernel can be held to it draw for draw.  It is NOT fbprophet's stream: fbprophet draws from the
unseeded global numpy RNG (``prophet_oracle.predict_uncertainty`` restates that one), and the two
agree in distribution only (tests/test_mc_stream.py checks that they do).

Per model and draw ``j`` (0 <= j < n_samples), with ``S`` fitted changepoints and
``Tmax = max t`` over the future frame:

* key: ``model_key`` -- splitmix64 over the words of the model's record, folded with the seed;
* first simulated changepoint (only if ``Tmax > 1``): ``1 - log(u) / S``, ``u`` from the counter
  ``(j, 0xffffffff, 1, 0)``;
* the c-th simulated changepoint (c = 0, 1, ...) takes the counter ``(j, c, 1, 0)``: words 0, 1
  give its Laplace(0, lam) slope change ``-lam sign(u - 1/2) log(1 - 2 |u - 1/2|)``, words 2, 3
  the exponential gap ``-log(u) / S`` to the next one;
* noise at point h: Box-Muller from the counter ``(j, h >> 1, 0, 0)``,
  ``sqrt(-2 log u1) * (cos if h even else sin)(2 pi u2)``, times sigma_obs * y_scale;
* trend: the fitted changepoints first (the same k / m updates as Prophet.piecewise_linear /
  piecewise_logistic), then the simulated ones; ``yhat = trend (1 + s)`` (multiplicative) or
  ``trend + s y_scale`` (additive), plus the noise;
* bounds: numpy linear-interpolation percentiles at ``100 (1 -+ w) / 2``.
"""
from __future__ import annotations

import numpy as np

M64 = (1 << 64) - 1
M32 = np.uint64(0xFFFFFFFF)
MC_BINS = 256


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _bits(x) -> int:
    return int(np.asarray(x, np.float64).reshape(1).view(np.uint64)[0])


def model_key(seed: int, params_row, tchange_row, start_ns: int, t_scale_ns: int, y_scale: float, floor: float,
              cap: float):
    """(k0, k1) of one model: word i of (params[pstride], tchange[smax], start_ns, t_scale_ns, y_scale, floor, cap)
    contributes splitmix64(w_i ^ splitmix64(i)); the XOR of the contributions h gives splitmix64(h ^ splitmix64(seed))."""
    words = [int(w) for w in np.ascontiguousarray(params_row, np.float64).view(np.uint64)]
    words += [int(w) for w in np.ascontiguousarray(tchange_row, np.float64).view(np.uint64)]
    words += [int(start_ns) & M64, int(t_scale_ns) & M64, _bits(y_scale), _bits(floor), _bits(cap)]
    h = 0
    for i, w in enumerate(words):
        h ^= splitmix64(w ^ splitmix64(i))
    key = splitmix64(h ^ splitmix64(int(seed) & M64))
    return key & 0xFFFFFFFF, key >> 32


def philox4x32_10(k0: int, k1: int, c0, c1, c2, c3):
    """Philox4x32-10 of the counters (broadcast uint32 arrays) under the key (k0, k1): four uint64 arrays of 32-bit words."""
    c0, c1, c2, c3 = (x.astype(np.uint64) for x in np.broadcast_arrays(*(np.asarray(c, np.uint64) for c in (c0, c1, c2, c3))))
    a0, a1 = int(k0), int(k1)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    for _ in range(10):
        p0 = m0 * c0
        p1 = m1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(a0), p1 & M32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(a1), p0 & M32)
        a0 = (a0 + 0x9E3779B9) & 0xFFFFFFFF
        a1 = (a1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def u01(a, b):
    """Uniform in (0, 1) from two 32-bit words: the top 53 bits, offset by half a step."""
    v = ((a << np.uint64(32)) | b) >> np.uint64(11)
    return (v.astype(np.float64) + 0.5) * (1.0 / 9007199254740992.0)


def _seasonal(ds_ns, mask: int, beta) -> np.ndarray:
    """The packed Fourier terms of predict_kernel.cuh seasonal_term: yearly (10), weekly (3), daily (4) as the mask has them."""
    tau = (1e-9 * np.asarray(ds_ns, np.int64).astype(np.float64)) / 86400.0
    acc = np.zeros(tau.size)
    col = 0
    for bit, period, order in ((1, 365.25, 10), (2, 7.0, 3), (4, 1.0, 4)):
        if mask & bit:
            blk = np.zeros(tau.size)
            for i in range(order):
                arg = (2.0 * (i + 1)) * np.pi * tau / period
                blk = blk + np.sin(arg) * beta[col + 2 * i] + np.cos(arg) * beta[col + 2 * i + 1]
            acc = acc + blk
            col += 2 * order
    return acc


def draws(fitted, i: int, future_ds, floor: float, cap: float, logistic: bool, multiplicative: bool, n_samples: int,
          seed: int) -> np.ndarray:
    """[H, n_samples] draws of model row ``i`` of a FittedBatch (numpy arrays), as mc_kernel generates them.

    ``floor`` / ``cap`` are the per-model values handed to the predict call.  The future timestamps must be ascending
    (the kernel's requirement)."""
    pr = np.asarray(fitted.params[i], np.float64)
    smax = int(fitted.smax)
    S, mask = int(fitted.meta_i32[i, 1]), int(fitted.meta_i32[i, 3])
    start, t_scale = int(fitted.meta_i64[i, 0]), int(fitted.meta_i64[i, 1])
    y_scale = float(fitted.meta_f64[i, 0])
    ds = np.asarray(future_ds, np.int64)
    assert np.all(np.diff(ds) >= 0), "mc_kernel wants ascending future timestamps"
    H, n = ds.size, int(n_samples)
    k0, k1 = model_key(seed, pr, fitted.tchange[i], start, t_scale, y_scale, floor, cap)
    t = (ds - start).astype(np.float64) / float(t_scale)
    fl = float(floor) if logistic else 0.0
    cap_s = (float(cap) - fl) / y_scale if logistic else 0.0
    k, m, sigma = float(pr[0]), float(pr[1]), float(pr[2])
    delta = [float(pr[3 + s]) for s in range(S)]
    tc = [float(fitted.tchange[i, s]) for s in range(S)]
    # fitted changepoints: the state after the first s of them (load_model's gamma recurrence, then advance's updates)
    kh, mh, lam_acc, acc, kc = [k], [m], 0.0, 0.0, k
    for s in range(S):
        kn = kc + delta[s]
        if logistic:
            g = (tc[s] - m - acc) * (1.0 - kc / kn)
            acc += g
        else:
            g = -tc[s] * delta[s]
        kc = kn
        lam_acc += abs(delta[s])
        kh.append(kh[-1] + delta[s])
        mh.append(mh[-1] + g)
    lam = lam_acc / S + 1e-8
    rate = float(S)
    s_hist = np.searchsorted(np.array(tc), t, side="right") if S else np.zeros(H, np.int64)
    Tmax = t.max()
    # simulated changepoints: positions [n, C] and the (k, m) state after each
    nsim = np.zeros((n, H), np.int64)
    ks = np.full((n, 1), kh[-1])
    ms_ = np.full((n, 1), mh[-1])
    if Tmax > 1.0:
        pos, dl = simulated_changepoints(k0, k1, n, rate, lam, Tmax)
        C = pos.shape[1]
        kcol, mcol = [ks[:, 0]], [ms_[:, 0]]
        kk, mm = ks[:, 0].copy(), ms_[:, 0].copy()
        for c in range(C):
            kn = kk + dl[:, c]
            if logistic:
                mm = mm + (pos[:, c] - mm) * (1.0 - kk / kn)
            else:
                mm = mm + -pos[:, c] * dl[:, c]
            kk = kn
            kcol.append(kk)
            mcol.append(mm)
        ks, ms_ = np.stack(kcol, axis=1), np.stack(mcol, axis=1)
        for c in range(C):
            nsim += pos[:, c:c + 1] <= t[None, :]
    kt = np.where(nsim > 0, np.take_along_axis(ks, nsim, axis=1), np.array(kh)[s_hist][None, :])
    mt = np.where(nsim > 0, np.take_along_axis(ms_, nsim, axis=1), np.array(mh)[s_hist][None, :])
    with np.errstate(over="ignore"):
        tr = cap_s / (1.0 + np.exp(-kt * (t[None, :] - mt))) if logistic else kt * t[None, :] + mt
    tr = tr * y_scale + fl
    K = (20 if mask & 1 else 0) + (6 if mask & 2 else 0) + (8 if mask & 4 else 0)
    sd = _seasonal(ds, mask, pr[3 + smax:]) if K > 0 else np.zeros(H)
    yh = tr * (1.0 + sd[None, :]) if multiplicative else tr + sd[None, :] * y_scale
    return (yh + (sigma * y_scale) * noise(k0, k1, n, H)).T


def simulated_changepoints(k0: int, k1: int, n: int, rate: float, lam: float, Tmax: float):
    """Positions [n, C] and slope changes [n, C] of the first C simulated changepoints of draws 0..n-1, C large enough
    that every draw's last one lies past Tmax (the kernel generates them up to the last point only)."""
    draw = np.arange(n, dtype=np.uint64)
    r = philox4x32_10(k0, k1, draw, 0xFFFFFFFF, 1, 0)
    first = 1.0 - np.log(u01(r[0], r[1])) / rate
    C = max(8, int(2 * rate * (Tmax - 1.0) + 8 * np.sqrt(rate * (Tmax - 1.0) + 1.0)))
    r = philox4x32_10(k0, k1, draw[:, None], np.arange(C, dtype=np.uint64)[None, :], 1, 0)
    ul = u01(r[0], r[1]) - 0.5
    dl = -lam * np.where(ul < 0, -1.0, 1.0) * np.log(1.0 - 2.0 * np.abs(ul))
    gap = -np.log(u01(r[2], r[3])) / rate
    pos = np.cumsum(np.concatenate([first[:, None], gap[:, :-1]], axis=1), axis=1)   # sequential, as next_cp +=
    assert np.all(pos[:, -1] > Tmax), "a draw needs more simulated changepoints than were generated"
    return pos, dl


def noise(k0: int, k1: int, n: int, H: int) -> np.ndarray:
    """Standard normals [n, H] of the noise: Box-Muller, cos for even and sin for odd points of a counter pair."""
    draw = np.arange(n, dtype=np.uint64)
    h = np.arange(H, dtype=np.uint64)
    r = philox4x32_10(k0, k1, draw[:, None], (h >> np.uint64(1))[None, :], 0, 0)
    rad = np.sqrt(-2.0 * np.log(u01(r[0], r[1])))
    ang = 2.0 * np.pi * u01(r[2], r[3])
    return rad * np.where((h & np.uint64(1)) == 0, np.cos(ang), np.sin(ang))


_MASK_BIT = {"yearly": 1, "weekly": 2, "daily": 4}


def record(prep, k: float, m: float, sigma: float, delta, beta, smax: int, kmax: int, status: int = 0):
    """One fitted-model record in the library's layout (batched.FittedBatch rows) for parameters chosen by hand on the
    history of a prophet_oracle.Prepared: (params[pstride], tchange[smax], meta_i32[8], meta_i64[2], meta_f64[4])."""
    S, K = prep.S, prep.K
    params = np.zeros(3 + smax + kmax)
    params[:3] = k, m, sigma
    params[3:3 + S] = delta
    mask = sum(_MASK_BIT[s.name] for s in prep.seasonalities)
    if mask:
        params[3 + smax:3 + smax + K] = beta
    tchange = np.zeros(smax)
    tchange[:S] = prep.t_change
    mi32 = np.array([prep.T, S, prep.n_changepoints_real, mask, status, 0, 0, 0], np.int32)
    mi64 = np.array([prep.start_ns, prep.t_scale_ns], np.int64)
    mf64 = np.array([prep.y_scale, prep.floor, prep.cap_value, 0.0])
    return params, tchange, mi32, mi64, mf64


def stack(records, smax: int, kmax: int):
    """Records -> an object with FittedBatch's fields (numpy arrays)."""
    from types import SimpleNamespace
    cols = [np.stack([r[j] for r in records]) for j in range(5)]
    return SimpleNamespace(params=cols[0], tchange=cols[1], meta_i32=cols[2], meta_i64=cols[3], meta_f64=cols[4],
                           smax=smax, kmax=kmax)


def percentiles(width: float):
    return 100.0 * (1.0 - width) / 2.0, 100.0 * (1.0 + width) / 2.0


def bounds(d: np.ndarray, width: float):
    """(lower, upper) over the draws of each point: numpy's linear-interpolation percentiles."""
    lo_p, hi_p = percentiles(width)
    return (np.percentile(d, lo_p, axis=1, method="linear"), np.percentile(d, hi_p, axis=1, method="linear"))


def target_ranks(n: int, width: float):
    """The order statistics the kernel reads for the two bounds (launch_mc: lo_i, lo_i + 1, hi_i, hi_i + 1, clamped)."""
    lo_p, hi_p = percentiles(width)
    li, ui = lo_p / 100.0 * (n - 1), hi_p / 100.0 * (n - 1)
    lo_i, hi_i = int(np.floor(li)), int(np.floor(ui))
    return [lo_i, min(lo_i + 1, n - 1), hi_i, min(hi_i + 1, n - 1)]


def crowded_bin(d: np.ndarray, width: float) -> np.ndarray:
    """Per point, the most draws in one of the kernel's 256 histogram bins (between the row's min and max) that holds
    one of its target ranks.  Above 64 (MC_CAND) the kernel selects by its bitonic-sort fallback; 0 for a constant row,
    which needs no selection."""
    H, n = d.shape
    ranks = target_ranks(n, width)
    out = np.zeros(H, np.int64)
    for p in range(H):
        row = d[p]
        mn, mx = row.min(), row.max()
        if not mx > mn:
            continue
        b = np.minimum(255, ((row - mn) * (256.0 / (mx - mn))).astype(np.int64))
        cnt = np.bincount(b, minlength=MC_BINS)
        sb = np.sort(b)     # bins are monotone in the value: the k-th smallest value lies in the k-th smallest bin
        out[p] = max(cnt[sb[r]] for r in ranks)
    return out
