"""Extra regressors without a GPU (DESIGN §19): make_regressor_options' validations and the library's limits, the
layout, the host standardisation rule against a restatement of pandas' semantics, and the oracle's column order and
prior scales."""
import numpy as np
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

import regressor_oracle as ro

DAY = 86400 * 10**9


@pytest.mark.parametrize("regs, kw, match", [
    ([dict(name="")], {}, r"regressors\[0\]\.name"),
    ([dict(name="x" * 16)], {}, r"regressors\[0\]\.name"),
    ([dict(name="a"), dict(name="a")], {}, r"regressors\[1\]\.name.*twice"),
    ([dict(name="a"), dict(name="trend")], {}, r"regressors\[1\]\.name.*reserved"),
    ([dict(name="price_lower")], {}, r"regressors\[0\]\.name.*reserved"),
    ([dict(name="weekly")], {}, r"regressors\[0\]\.name.*seasonality"),
    ([dict(name="monthly")], dict(seasonalities=[dict(name="monthly", period=30.5, fourier_order=3)]),
     r"regressors\[0\]\.name.*seasonality"),
    ([dict(name="a", prior_scale=0)], {}, r"regressors\[0\]\.prior_scale"),
    ([dict(name="a", prior_scale=-1.0)], {}, r"regressors\[0\]\.prior_scale"),
    ([dict(name="a", prior_scale="big")], {}, r"regressors\[0\]\.prior_scale"),
    ([dict(name="a", standardize="yes")], {}, r"regressors\[0\]\.standardize"),
    ([dict(name="a", mode="additive")], {}, r"regressors\[0\]\.mode"),
    ([dict(name="a", colour=1)], {}, r"regressors\[0\]: unknown"),
    ([dict(prior_scale=1.0)], {}, r"regressors\[0\]\.name is required"),
    (["a"], {}, r"regressors\[0\] must be a mapping"),
    ([dict(name=f"r{i}") for i in range(17)], {}, r"regressors: at most 16"),
    ([dict(name="a")], dict(holidays_prior_scale=0.0), r"holidays_prior_scale"),
])
def test_make_regressor_options_refuses(regs, kw, match):
    with pytest.raises(ValueError, match=match):
        batched.make_regressor_options(regs, **kw)


def test_mode_must_be_the_models():
    o = batched.make_regressor_options([dict(name="a", mode="additive")], seasonality_mode="additive")
    assert o.n_regressors == 1 and o.multiplicative == 0


def test_layout_counts_the_regressors():
    o = batched.make_regressor_options([dict(name="a"), dict(name="b"), dict(name="c")])
    lay = L.get_layout(o)
    assert (lay.smax, lay.kmax, lay.pstride) == (25, 34 + 3, 3 + 25 + 37)
    off = batched.make_regressor_options([dict(name="a"), dict(name="b")], yearly_seasonality=False,
                                         weekly_seasonality=False, daily_seasonality=False)
    assert L.get_layout(off).kmax == 2
    assert batched.seasonality_table(off) == []
    # with regressors the defaults are a table; without, version 3 is its version-2 part
    assert [e[0] for e in batched.seasonality_table(o)] == ["yearly", "weekly", "daily"]


@pytest.mark.parametrize("kw", [dict(), dict(yearly_seasonality=20),
                                dict(seasonalities=[dict(name="monthly", period=30.5, fourier_order=5)])])
def test_no_regressor_is_the_version_2_layout(kw):
    v2 = batched.make_table_options(**kw)
    v3 = batched.make_regressor_options([], **kw)
    a, b = L.get_layout(v2), L.get_layout(v3)
    assert [getattr(a, f) for f, _ in L.Layout._fields_] == [getattr(b, f) for f, _ in L.Layout._fields_]
    assert batched.seasonality_table(v2) == batched.seasonality_table(v3)


def test_limits():
    # K = 2 * 30 = 60 seasonal columns: 4 regressors fit, 5 do not
    kw = dict(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False,
              seasonalities=[dict(name="s", period=30.5, fourier_order=30)], n_changepoints=5)
    batched.make_regressor_options([dict(name=f"r{i}") for i in range(4)], **kw)
    with pytest.raises(ValueError, match="K = 60 columns and the 5 regressors"):
        batched.make_regressor_options([dict(name=f"r{i}") for i in range(5)], **kw)
    # P = 3 + 30 + 60 + 3 = 96 fits, 4 regressors make 97
    kw["n_changepoints"] = 30
    batched.make_regressor_options([dict(name=f"r{i}") for i in range(3)], **kw)
    with pytest.raises(ValueError, match=r"P = 3 \+ S \+ K \+ R = 97"):
        batched.make_regressor_options([dict(name=f"r{i}") for i in range(4)], **kw)


def test_library_refuses_what_python_would():
    import ctypes as C
    o = batched.make_regressor_options([dict(name="a"), dict(name="b")])
    o.regressors[1].name = b"a"
    assert L.load().pb200_get_layout(C.byref(o), C.byref(L.Layout())) == -1 and "twice" in L.last_error()
    o.regressors[1].name = b"b"
    o.regressors[1].standardize = 7
    assert L.load().pb200_get_layout(C.byref(o), C.byref(L.Layout())) == -1 and "standardize" in L.last_error()
    o.regressors[1].standardize = L.STD_AUTO
    o.n_regressors = 17
    assert L.load().pb200_get_layout(C.byref(o), C.byref(L.Layout())) == -4
    o.n_regressors = 2
    assert L.load().pb200_component_count(C.byref(o)) == -4 and "regressor" in L.last_error()


def _pandas_rule(x, standardize):
    """initialize_scales as fbprophet 0.5 writes it on a pandas Series: len(unique) < 2 -> no; 'auto' and
    set(unique) == {1, 0} -> no; else mean() and std() (ddof = 1, two-pass)."""
    u = np.unique(x)
    if len(u) < 2:
        return 0.0, 1.0
    if standardize == "auto":
        standardize = not (set(u.tolist()) == {1, 0})
    if not standardize:
        return 0.0, 1.0
    mu = np.mean(x)
    return mu, np.sqrt(np.sum((x - mu) ** 2) / (len(x) - 1))


@pytest.mark.parametrize("values, standardize, on", [
    (np.full(50, 3.25), "auto", False),
    (np.full(50, 3.25), True, False),                       # a forced standardize on a constant column
    ((np.arange(50) % 3 == 0).astype(float), "auto", False),
    ((np.arange(50) % 3 == 0).astype(float), True, True),
    (2.0 * (np.arange(50) % 3 == 0), "auto", True),        # {0, 2} is not binary
    (np.random.RandomState(1).randn(50) * 7 + 100, "auto", True),
    (np.random.RandomState(2).randn(50), False, False),
])
def test_host_standardisation_rule(values, standardize, on):
    sc = batched.regressor_scales(values[None, :], np.array([0, values.size]), [standardize])[0, 0]
    mu, sd = _pandas_rule(values, standardize)
    assert ((sc[0], sc[1]) != (0.0, 1.0)) == on
    assert abs(sc[0] - mu) <= 1e-13 * np.max(np.abs(values)) and abs(sc[1] - sd) <= 1e-12 * sd
    bad = values.copy()
    bad[7] = np.nan
    assert np.all(np.isnan(batched.regressor_scales(bad[None, :], np.array([0, bad.size]), [standardize])))


def _series(days=800):
    ds = np.datetime64("2019-01-01", "ns").astype(np.int64) + DAY * np.arange(days, dtype=np.int64)
    y = 100 + np.sin(np.arange(days) / 7.0) * 10
    return ds, y


@pytest.mark.parametrize("mode", ["additive", "multiplicative"])
def test_oracle_columns_order_and_sigmas(mode):
    ds, y = _series()
    opts = batched.make_regressor_options([dict(name="promo"), dict(name="price", prior_scale=0.5)],
                                          seasonalities=[dict(name="monthly", period=30.5, fourier_order=2)],
                                          seasonality_mode=mode, holidays_prior_scale=4.0)
    oopts = po.ProphetOptions(seasonality_mode=mode)
    reg = np.vstack([(np.arange(ds.size) % 5 == 0).astype(float), 10 + np.cos(np.arange(ds.size))])
    scale = np.array([[0.0, 1.0], [10.0, 2.0]])
    p, seas = ro.prepare(ds, y, 0.0, 1.1 * y.max(), oopts, {}, opts_custom(opts), reg, scale, ro.prior_scales(opts))
    # monthly (4), yearly (20), weekly (6), then the regressors; 800 daily points leave daily off
    assert [s[0] for s in seas] == ["monthly", "yearly", "weekly"]
    assert p.K == 4 + 20 + 6 + 2
    assert np.array_equal(p.X[:, -2], reg[0]) and np.allclose(p.X[:, -1], (reg[1] - 10.0) / 2.0, rtol=0, atol=0)
    assert np.array_equal(p.sigmas[-2:], [4.0, 0.5])          # holidays_prior_scale is the default prior
    assert np.array_equal(p.sigmas[:30], [10.0] * 30)
    mult = mode == "multiplicative"
    assert np.array_equal(p.s_m[-2:], [1.0, 1.0] if mult else [0.0, 0.0])
    assert np.array_equal(p.s_a[-2:], [0.0, 0.0] if mult else [1.0, 1.0])


def opts_custom(opts):
    return [dict(name=opts.seasonalities[i].name.decode(), period=opts.seasonalities[i].period,
                 fourier_order=opts.seasonalities[i].fourier_order) for i in range(opts.n_seasonalities)]


def test_oracle_every_seasonality_off_has_only_the_regressors():
    ds, y = _series()
    oopts = po.ProphetOptions()
    reg = np.vstack([np.linspace(0, 1, ds.size)] * 3)
    scale = np.tile([0.0, 1.0], (3, 1))
    p, seas = ro.prepare(ds, y, 0.0, 1.1 * y.max(), oopts, dict(yearly=False, weekly=False, daily=False), [], reg, scale,
                         np.array([10.0, 10.0, 1.0]))
    assert seas == [] and p.K == 3 and p.X.shape == (ds.size, 3)
    assert np.array_equal(p.sigmas, [10.0, 10.0, 1.0])
    assert np.array_equal(p.X, reg.T)


@pytest.mark.parametrize("custom", [[dict(name="monthly", period=30.5, fourier_order=5)],
                                    [dict(name="weekly", period=7.0, fourier_order=5)]])
def test_no_regressor_is_version_2_in_the_python_helpers(custom):
    """component_names, _with_mask (the backtest's cutoff options) and copy_options read a v3 options' table as they
    read the v2 one's."""
    v2 = batched.make_table_options(seasonalities=custom)
    v3 = batched.make_regressor_options([], seasonalities=custom)
    assert batched.component_names(v3) == batched.component_names(v2)
    for mask in range(8):
        c2, c3 = batched._with_mask(v2, mask), batched._with_mask(v3, mask)
        assert (c3.yearly, c3.weekly, c3.daily) == (c2.yearly, c2.weekly, c2.daily)
        assert c3.abi_version == L.ABI_VERSION_REGRESSORS and c3.n_seasonalities == len(custom)
        l2, l3 = L.get_layout(c2), L.get_layout(c3)
        assert (l2.smax, l2.kmax, l2.pstride) == (l3.smax, l3.kmax, l3.pstride)


def test_a_reg_scale_of_another_shape_is_refused():
    """predict reads the fit's reg_scale as [n][R][2] doubles: another shape or dtype is refused before the library
    is called."""
    opts = batched.make_regressor_options([dict(name="a"), dict(name="b")])
    lay = L.get_layout(opts)
    n, h = 3, 5
    fb = batched.FittedBatch(np.zeros((n, lay.pstride)), np.zeros((n, lay.smax)), np.zeros((n, 8), np.int32),
                             np.zeros((n, 2), np.int64), np.zeros((n, 4)), lay.smax, lay.kmax)
    fut = np.zeros((n, h), np.int64)
    freg = np.zeros((2, n, h))
    for rs in (None, np.zeros((n, 1, 2)), np.zeros((n, 2, 2), np.float32), np.zeros((n + 1, 2, 2))):
        fb.reg_scale = rs
        with pytest.raises(ValueError, match="reg_scale"):
            batched.predict_batch_host(None, opts, fb, fut, np.zeros(n), np.ones(n), regressors=freg)
