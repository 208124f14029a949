"""Seasonality tables without a GPU (DESIGN §18): make_table_options' validation and refusals, the layout and the
K / P limits, and the oracle's column order, name rule, int orders and per-column prior scales."""
import numpy as np
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

import seasonality_table as st

DAY = 86400 * 10**9


def test_default_restatements_are_the_v1_model():
    for kw in (dict(), dict(yearly_seasonality=10), dict(weekly_seasonality=3, daily_seasonality=4),
               dict(yearly_seasonality=True, weekly_seasonality=False)):
        o = batched.make_table_options(**kw)
        assert o.abi_version == L.ABI_VERSION_TABLE
        v1 = batched.make_options(**{k: (bool(v) if not isinstance(v, str) else v) for k, v in kw.items()})
        a, b = L.get_layout(o), L.get_layout(v1)
        assert (a.smax, a.kmax, a.pstride) == (b.smax, b.kmax, b.pstride)
    assert (o.yearly, o.weekly) == (1, 0)


def test_layout_follows_the_table():
    assert L.get_layout(batched.make_table_options(yearly_seasonality=20)).kmax == 40 + 6 + 8
    lay = L.get_layout(batched.make_table_options(seasonalities=[dict(name="monthly", period=30.5, fourier_order=5)]))
    assert (lay.kmax, lay.pstride) == (10 + 34, 3 + 25 + 44)
    lay = L.get_layout(batched.make_table_options(
        yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False,
        seasonalities=[dict(name="weekly2", period=7, fourier_order=3), dict(name="daily2", period=1, fourier_order=4)]))
    assert lay.kmax == 14
    # custom 'yearly' replaces the auto built-in at its own place and order
    lay = L.get_layout(batched.make_table_options(seasonalities=[dict(name="yearly", period=365.25, fourier_order=3)]))
    assert lay.kmax == 6 + 6 + 8


def test_limits_are_refused_with_the_value():
    with pytest.raises(ValueError, match="K = 66"):
        batched.make_table_options(yearly_seasonality=30, weekly_seasonality=3, daily_seasonality=False)
    ok = batched.make_table_options(yearly_seasonality=29, weekly_seasonality=3, daily_seasonality=False,
                                    n_changepoints=3)                   # K = 64, P = 3 + 3 + 64
    assert L.get_layout(ok).kmax == 64
    with pytest.raises(ValueError, match="P = 3 \\+ S \\+ K = 97"):
        batched.make_table_options(yearly_seasonality=29, weekly_seasonality=3, daily_seasonality=False,
                                   n_changepoints=30)
    with pytest.raises(ValueError, match="at most 8"):
        batched.make_table_options(seasonalities=[dict(name=f"s{i}", period=2 + i, fourier_order=1) for i in range(9)])
    with pytest.raises(ValueError, match="10 seasonalities"):
        batched.make_table_options(seasonalities=[dict(name=f"s{i}", period=2 + i, fourier_order=1) for i in range(7)])


@pytest.mark.parametrize("spec, match", [
    (dict(period=30.5, fourier_order=5), r"seasonalities\[0\]\.name is required"),
    (dict(name="m", fourier_order=5), r"seasonalities\[0\]\.period is required"),
    (dict(name="m", period=30.5), r"seasonalities\[0\]\.fourier_order is required"),
    (dict(name="m", period=0, fourier_order=5), r"seasonalities\[0\]\.period"),
    (dict(name="m", period=30.5, fourier_order=0), r"seasonalities\[0\]\.fourier_order"),
    (dict(name="m", period=30.5, fourier_order=2.5), r"seasonalities\[0\]\.fourier_order"),
    (dict(name="m", period=30.5, fourier_order=5, prior_scale=0), r"seasonalities\[0\]\.prior_scale"),
    (dict(name="m", period=30.5, fourier_order=5, mode="additive"), r"seasonalities\[0\]\.mode"),
    (dict(name="", period=30.5, fourier_order=5), r"seasonalities\[0\]\.name"),
    (dict(name="x" * 16, period=30.5, fourier_order=5), r"seasonalities\[0\]\.name"),
    (dict(name="m", period=30.5, fourier_order=5, condition_name="c"), r"seasonalities\[0\]: unknown"),
    (dict(name="m", period=30.5, fourier_order=None), r"seasonalities\[0\]\.fourier_order"),
    (dict(name="m", period="30", fourier_order=5), r"seasonalities\[0\]\.period must be a number"),
    (dict(name="m", period=30.5, fourier_order=5, prior_scale="x"), r"seasonalities\[0\]\.prior_scale"),
    (dict(name="trend", period=30.5, fourier_order=5), r"seasonalities\[0\]\.name: 'trend' is reserved"),
    (dict(name="yhat_lower", period=30.5, fourier_order=5), r"seasonalities\[0\]\.name"),
])
def test_bad_entries_name_the_key(spec, match):
    with pytest.raises(ValueError, match=match):
        batched.make_table_options(seasonalities=[spec])


def test_other_refusals():
    m = dict(name="m", period=30.5, fourier_order=5)
    with pytest.raises(ValueError, match="added twice"):
        batched.make_table_options(seasonalities=[m, m])
    with pytest.raises(ValueError, match="weekly_seasonality is 'auto'"):
        batched.make_table_options(weekly_seasonality=True, seasonalities=[dict(name="weekly", period=7, fourier_order=5)])
    with pytest.raises(ValueError, match="yearly_seasonality"):
        batched.make_table_options(yearly_seasonality=-1)
    with pytest.raises(ValueError, match="yearly_seasonality"):
        batched.make_table_options(yearly_seasonality="on")
    # the existing v1 options keep refusing non-default orders
    with pytest.raises(ValueError):
        batched.make_options(yearly_seasonality=20)


def test_oracle_column_order_name_rule_and_sigmas():
    ds = np.arange(800, dtype=np.int64) * DAY + 1_600_000_000 * 10**9
    y = 10 + np.sin(np.arange(800) / 9.0)
    custom = [dict(name="monthly", period=30.5, fourier_order=5), dict(name="quarterly", period=91.3125,
                                                                       fourier_order=2, prior_scale=0.1)]
    p, seas = st.prepare(ds, y, 0.0, 12.0, po.ProphetOptions(), {"yearly": 20}, custom)
    assert [s[0] for s in seas] == ["monthly", "quarterly", "yearly", "weekly"]     # daily auto-off on daily data
    assert [s[2] for s in seas] == [5, 2, 20, 3]
    assert p.K == 2 * (5 + 2 + 20 + 3)
    assert np.array_equal(p.sigmas, np.repeat([10.0, 0.1, 10.0, 10.0], [10, 4, 40, 6]))
    assert np.array_equal(p.X[:, :10], po.fourier_series(p.ds_sorted, 30.5, 5))
    assert np.array_equal(p.X[:, 14:54], po.fourier_series(p.ds_sorted, 365.25, 20))
    # a custom 'weekly' replaces the auto built-in and keeps its own place
    _, seas = st.prepare(ds, y, 0.0, 12.0, po.ProphetOptions(), {}, [dict(name="weekly", period=7, fourier_order=6)])
    assert [(s[0], s[2]) for s in seas] == [("weekly", 6), ("yearly", 10)]
    # an explicit order forces the built-in on where auto would disable it
    short = ds[:100]
    _, seas = st.prepare(short, y[:100], 0.0, 12.0, po.ProphetOptions(), {"yearly": 7}, [])
    assert [(s[0], s[2]) for s in seas] == [("yearly", 7), ("weekly", 3)]
    # per-column prior scales enter the objective's beta prior
    th = po.initial_theta(p)
    th[3 + p.S:] = 0.3
    _, f1, g1 = po.neg_logp_grad(th, p)
    p.sigmas = np.full(p.K, 10.0)
    _, f2, g2 = po.neg_logp_grad(th, p)
    q = slice(3 + p.S + 10, 3 + p.S + 14)
    assert np.allclose(g1[q] - g2[q], 0.3 / 0.01 - 0.3 / 100.0)
    assert np.isclose(f1 - f2, 4 * 0.5 * 0.09 * (1 / 0.01 - 1 / 100.0))


def test_numpy_bools_and_component_names():
    o = batched.make_table_options(yearly_seasonality=np.bool_(True), weekly_seasonality=np.bool_(False))
    assert (o.yearly, o.yearly_order, o.weekly) == (1, 0, 0)
    with pytest.raises(ValueError, match="yearly_seasonality"):
        batched.make_table_options(yearly_seasonality=20.0)
    o = batched.make_table_options(seasonalities=[dict(name="monthly", period=30.5, fourier_order=5),
                                                  dict(name="weekly", period=7, fourier_order=5)])
    assert batched.component_names(o) == L.COMPONENTS + ("monthly",)
    assert batched.component_names(batched.make_options()) == L.COMPONENTS
