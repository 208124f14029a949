"""The restatement of mc_kernel's sampler (oracle/mc_stream.py) against fbprophet's process, in distribution.

The GPU suite (test_gpu_scorer.py) holds the kernel to the restatement draw for draw; these tests say that the process
the restatement describes -- exponential gaps instead of a Poisson count and sorted uniforms, Laplace slopes by the
inverse CDF, Box-Muller noise -- is fbprophet's predict_uncertainty process.  No GPU needed."""
import numpy as np
import pytest
from scipy import stats

from oracle import mc_stream as mcs
from oracle import prophet_oracle as po

N_BIG = 100_000
KEY = mcs.model_key(123, np.arange(5.0), np.arange(3.0), 10**18, 86400 * 10**9, 7.0, 0.0, 9.0)


def test_simulated_changepoint_count_is_poisson():
    S, Tmax = 25.0, 1.2
    pos, _ = mcs.simulated_changepoints(*KEY, N_BIG, S, 0.1, Tmax)
    cnt = (pos <= Tmax).sum(axis=1)
    mu = S * (Tmax - 1.0)
    assert abs(cnt.mean() - mu) <= 4 * np.sqrt(mu / N_BIG), cnt.mean()
    # variance of a Poisson(mu) sample variance: (mu + 2 mu^2) / n
    assert abs(cnt.var() - mu) <= 4 * np.sqrt((mu + 2 * mu * mu) / N_BIG), cnt.var()
    # and the whole distribution: chi-square over the bins holding >= 5 expected counts
    ks = np.arange(cnt.max() + 1)
    exp = stats.poisson.pmf(ks, mu) * N_BIG
    obs = np.bincount(cnt, minlength=ks.size).astype(float)
    keep = exp >= 5
    o = np.append(obs[keep], obs[~keep].sum())
    e = np.append(exp[keep], N_BIG - exp[keep].sum())
    assert stats.chisquare(o, e).pvalue > 1e-4


def test_simulated_changepoint_positions_are_uniform():
    S, Tmax = 25.0, 1.3
    pos, _ = mcs.simulated_changepoints(*KEY, N_BIG // 10, S, 0.1, Tmax)
    inside = pos[pos <= Tmax]
    assert inside.min() > 1.0
    assert stats.kstest((inside - 1.0) / (Tmax - 1.0), "uniform").pvalue > 1e-4


def test_slope_changes_are_laplace():
    lam = 0.037
    _, dl = mcs.simulated_changepoints(*KEY, N_BIG // 10, 25.0, lam, 1.1)
    x = dl[:, :10].ravel()
    assert stats.kstest(x, stats.laplace(0, lam).cdf).pvalue > 1e-4
    # a scale off by 2x is far outside
    assert stats.kstest(x, stats.laplace(0, 2 * lam).cdf).pvalue < 1e-10


def test_noise_is_standard_normal_and_pairs_are_independent():
    z = mcs.noise(*KEY, N_BIG // 4, 4)
    for h in range(4):
        assert stats.kstest(z[:, h], "norm").pvalue > 1e-4
    # cos / sin halves of one Box-Muller pair are uncorrelated normals, and so are different pairs
    c = np.corrcoef(z.T)
    assert np.max(np.abs(c - np.eye(4))) < 4 * 4 / np.sqrt(z.shape[0])


def test_key_is_a_function_of_the_record_and_the_seed():
    rec = (np.arange(5.0), np.arange(3.0), 10**18, 86400 * 10**9, 7.0, 0.0, 9.0)
    assert mcs.model_key(123, *rec) == KEY
    assert mcs.model_key(124, *rec) != KEY
    assert mcs.model_key(123 | (1 << 40), *rec) != KEY
    p = np.arange(5.0)
    p[4] = np.nextafter(p[4], 10.0)
    assert mcs.model_key(123, p, *rec[1:]) != KEY
    assert mcs.model_key(123, *rec[:6], 9.5) != KEY


def _model(growth, mode):
    """A hand-made model on 30 days of hourly history (weekly + daily seasonality, 25 changepoints)."""
    rng = np.random.RandomState(3)
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + 3600 * 10**9 * np.arange(720, dtype=np.int64)
    y = 100 + 10 * rng.rand(ds.size)
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode)
    p = po.prepare(ds, y, 0.0, 130.0, oopts)
    assert (p.S, p.K) == (25, 14)
    delta = 0.5 * rng.laplace(size=p.S)
    beta = 0.05 * rng.randn(p.K)
    k, m, sigma = (0.8, -0.2, 0.02) if growth == "logistic" else (0.1, 0.7, 0.02)
    fr = po.FitResult(prep=p, k=k, m=m, delta=delta, sigma_obs=sigma, beta=beta, theta=None, neg_logp=0.0, iters=0,
                      n_evals=0, ret=0)
    return p, fr, oopts, mcs.stack([mcs.record(p, k, m, sigma, delta, beta, 25, 14)], 25, 14)


@pytest.mark.parametrize("mode", ["multiplicative", "additive"])
@pytest.mark.parametrize("growth", ["logistic", "linear"])
def test_bounds_match_fbprophet_process(growth, mode):
    """The restatement's bounds and po.predict_uncertainty's (fbprophet's process on numpy's RNG) at the same sample size
    agree within a few Monte-Carlo standard errors, at points inside the history and up to 30 % past it."""
    n = 20_000
    p, fr, oopts, rec = _model(growth, mode)
    oopts.uncertainty_samples = n
    last = int(p.ds_sorted[-1])
    fut = np.concatenate([p.ds_sorted[[100, 500]], last + 3600 * 10**9 * np.array([1, 24, 72, 140, 216])])
    cap = 130.0
    pr = po.predict(fr, fut, 0.0, cap, oopts)
    un = po.predict_uncertainty(fr, fut, pr, np.random.RandomState(0), oopts)
    d = mcs.draws(rec, 0, fut, 0.0, cap, growth == "logistic", mode == "multiplicative", n, 99)
    lo, hi = mcs.bounds(d, oopts.interval_width)
    for q, mine, ref in ((0.1, lo, un["yhat_lower"]), (0.9, hi, un["yhat_upper"])):
        # standard error of a sample quantile: sqrt(q (1 - q) / n) / density, the density from the draws' own quantiles
        spread = (np.quantile(d, q + 0.02, axis=1) - np.quantile(d, q - 0.02, axis=1)) / 0.04
        se = np.sqrt(q * (1 - q) / n) * spread
        z = np.abs(mine - ref) / (np.sqrt(2.0) * se)
        assert np.all(z < 5.0), (growth, mode, q, z)
    # the trend spread past the history is the simulated changepoints' doing: it must be visible here
    assert (hi - lo)[-1] > 1.2 * (hi - lo)[2]
