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


# ---------------------------------------------------------------------------------------------------------------------
# the two oracle column sets (tests/seasonality_table.py) against a 60-digit evaluation
# ---------------------------------------------------------------------------------------------------------------------
PI60 = "3.14159265358979323846264338327950288419716939937510582097494459"
# (period, order) of the table cells of tests/test_gpu_table_instances.py and the built-ins' longest periods
REF_TABLES = ((1.0, 20), (0.5, 32), (0.25, 32), (1.0 / 24.0, 4), (30.5, 32), (365.25, 32))


def _dec_sincos(x):
    """sin, cos of the Decimal x at 60 digits: reduced by 2 pi, then Taylor series."""
    from decimal import Decimal, localcontext
    with localcontext() as ctx:
        ctx.prec = 60
        tp = 2 * Decimal(PI60)
        r = x - (x / tp).to_integral_value() * tp
        s, c, term, n = Decimal(0), Decimal(0), Decimal(1), 0
        while n < 80:                                   # |r| <= pi: term n is below 1e-70 by n = 80
            if n % 2 == 0:
                c += term if n % 4 == 0 else -term
            else:
                s += term if n % 4 == 1 else -term
            n += 1
            term = term * r / n
        return +s, +c


def _ref_points(seed, n):
    """(ds, period, order, harmonic) at n points over REF_TABLES: instants from 1970 to 2260, two in three of them
    between 2015 and 2030."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        per, o = REF_TABLES[j % len(REF_TABLES)]
        lo, hi = (16436, 21915) if j % 3 else (0, 106000)               # days since 1970
        ds = int(rng.integers(lo * DAY, hi * DAY))
        out.append((ds, per, o, int(rng.integers(1, o + 1)) if j % 4 else o))
    return out


def test_exact_columns_are_sin_cos_of_h_theta_to_half_an_ulp():
    """The "exact" columns are sin / cos(h theta) of the staged base angle correctly rounded (within 0.5 ulp and the
    extended-precision evaluation's 2^-11 ulp)."""
    from decimal import Decimal
    for ds, per, o, h in _ref_points(1, 300):
        d = np.array([ds], np.int64)
        th = st.base_angle(d, per)[0]
        assert th == 2.0 * 3.141592653589793 * ((1e-9 * float(ds)) / 86400.0) / per       # as the kernel stages it
        X = st.fourier_columns(d, per, o, "exact")[0]
        s, c = _dec_sincos(Decimal(th) * h)
        for got, ref in ((X[2 * h - 2], s), (X[2 * h - 1], c)):
            ulp = Decimal(float(np.spacing(abs(got))))
            assert abs(Decimal(got) - ref) <= ulp * Decimal(0.5 + 2.0**-11), (ds, per, h, got, ref)


def test_numpy_columns_differ_from_exact_by_their_argument_rounding():
    """fbprophet's columns take the argument 2.0 (i + 1) pi t / p rounded three times, the exact ones h theta with theta
    rounded twice (h theta itself is exact): the two arguments are within 3 + 2 relative roundings of the angle, each at
    most ulp(arg), so per column |numpy - exact| <= 5 ulp(arg_h) plus the two results' roundings (2^-52).  Measured up
    to 2.7 ulp(arg_h); at harmonic 32 of a 6-hour period on 2021 dates that is over 1e-9, which is why the fit kernel,
    whose recurrence follows h theta, is held to the exact columns."""
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + np.arange(0, 365 * 96, 37, dtype=np.int64) * 900 * 10**9
    worst = {}
    for per, o in REF_TABLES:
        Xn = st.fourier_columns(ds, per, o, "numpy")
        Xe = st.fourier_columns(ds, per, o, "exact")
        t = st.tau_days(ds)
        for h in range(1, o + 1):
            arg = 2.0 * h * np.pi * t / per
            d = np.abs(Xn[:, 2 * h - 2:2 * h] - Xe[:, 2 * h - 2:2 * h]).max(axis=1)
            ulp = np.spacing(np.abs(arg))
            assert np.all(d <= 5.0 * ulp + 2.0**-52), (per, h, np.max((d - 2.0**-52) / ulp))
            worst[(per, h)] = float(np.max(d / ulp))
    assert np.max(np.abs(st.fourier_columns(ds, 0.25, 32, "numpy") - st.fourier_columns(ds, 0.25, 32, "exact"))) > 1e-9
    assert max(worst.values()) > 1.0            # more than one rounding of the argument apart


def test_unknown_column_set_is_refused():
    with pytest.raises(ValueError, match="columns"):
        st.fourier_columns(np.zeros(2, np.int64), 7.0, 3, "float32")


# ---------------------------------------------------------------------------------------------------------------------
# predict_kernel.cuh sincos_reduced: its three FMA steps in exact rational arithmetic, with the kernel's own constants
# ---------------------------------------------------------------------------------------------------------------------
def _reduction_constants():
    """(1 / (2 pi), C1, C2, C3, guard) as sincos_reduced's source states them."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(L.__file__), "csrc", "predict_kernel.cuh")).read()
    body = src[src.index("void sincos_reduced("):]
    body = body[:body.index("\n}\n")]
    num = r"([0-9.]+(?:e[-+]?[0-9]+)?)"
    inv = float(re.search(r"rint\(x \* " + num + r"\)", body).group(1))
    guard = float(re.search(r"fabs\(k\) < " + num + r"\)", body).group(1))
    steps = re.findall(r"fma\(-k, " + num + r", (x|r)\);\s*//\s*(0x[0-9a-fp.+-]+)", body)
    assert [s[1] for s in steps] == ["x", "r", "r"], steps
    for dec, _, hx in steps:                              # each literal is the value its comment states
        assert float(dec) == float.fromhex(hx), (dec, hx)
    return (inv, *(float(s[0]) for s in steps), guard)


def _reduce(x, inv, c1, c2, c3, guard):
    """sincos_reduced's r for x with every fma rounded once, exactly (Fraction), or None where it falls back."""
    from fractions import Fraction
    k = float(np.rint(x * inv))
    if not abs(k) < guard:
        return k, None
    r = x
    for c in (c1, c2, c3):
        r = float(Fraction(r) - Fraction(k) * Fraction(c))     # CPython rounds int / int correctly: one fma
    return k, r


def test_sincos_reduced_matches_the_exact_reduction_over_its_whole_range():
    """r = x - k 2 pi within 4.5e-16 of the exact value (60-digit pi) for every k the guard admits, up to
    k = +-(2^21 - 1), and the first k past it takes the library's sincos; k C1 and k C2 are exact."""
    from decimal import Decimal
    from fractions import Fraction
    inv, c1, c2, c3, guard = _reduction_constants()
    assert guard == 2.0**21
    two_pi = 2 * Fraction(Decimal(PI60))
    rng = np.random.default_rng(7)
    top = float((guard - 0.5) * two_pi)
    xs = list(rng.uniform(-top, top, 20000))
    # the last admitted k (either sign), just inside and past the rounding boundary, and the first k that falls back
    for kk in (guard - 1, guard - 2, guard):
        for sgn in (1, -1):
            for off in (-0.5, -0.49999, 0.0, 0.49999, 0.5):
                xs.append(sgn * float((Fraction(int(kk)) + Fraction(off)) * two_pi))
    worst, fell_back, kmax = 0.0, set(), 0.0
    for x in xs:
        k, r = _reduce(x, inv, c1, c2, c3, guard)
        if r is None:
            fell_back.add(abs(k))
            continue
        assert abs(k) <= guard - 1
        kmax = max(kmax, abs(k))
        err = abs(Fraction(r) - (Fraction(x) - Fraction(k) * two_pi))
        worst = max(worst, float(err))
        assert err <= Fraction(4.5e-16), (x, k, float(err))
    assert kmax == guard - 1 and fell_back == {guard}, (kmax, fell_back)
    assert worst > 1e-16, worst
    for c in (c1, c2):                                    # 32 significant bits: k c exact in a double for k < 2^21
        m, _ = np.frexp(c)
        assert float(m * 2**32) == np.rint(m * 2**32), c


# ---------------------------------------------------------------------------------------------------------------------
# the recipes of tests/test_gpu_table_instances.py give their tables, grids and lengths
# ---------------------------------------------------------------------------------------------------------------------
def _table_cells():
    import test_gpu_table_instances as ti
    return ti


@pytest.mark.parametrize("name", ["daily20", "h12", "q6h_p96", "hourly", "gap", "mixed"])
def test_table_recipe_gives_its_mask_grid_and_length(name):
    ti = _table_cells()
    cell = ti.CELLS[name]
    series = ti.cell_series(name)
    assert len(series) == len(cell.lengths) == len(cell.masks) == len(cell.regular)
    ents = ti.entries(cell.table)
    builtin, custom = ti.options(cell.table, cell.growth, "additive", cell.ncp)[2:]
    if name == "daily20":
        assert cell.lengths == (13, 31, 32, 33, 101)
    for j, (ds, y) in enumerate(series):
        assert ds.size == cell.lengths[j] and y.dtype == np.int32 and np.all(np.diff(ds) >= 0), (name, j)
        seas = st.seasonalities(ds, builtin, custom, 10.0)
        assert st.table_mask(seas, ents) == cell.masks[j], (name, j, seas)
        d = np.diff(ds)
        regular = bool(np.all(d == d[0]) and d[0] > 0)
        assert regular == cell.regular[j], (name, j)
        if regular and cell.step is not None:
            assert d[0] == cell.step
        if not regular:
            assert np.sum(d == 0) == 1                                  # one duplicate timestamp
        if name in ("q6h_p96", "hourly"):
            assert d[d > 0].min() == 15 * 60 * 10**9
        p, _ = st.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), po.ProphetOptions(n_changepoints=cell.ncp),
                          builtin, custom)
        if name in ("h12", "q6h_p96"):
            assert p.K == 64
        if name == "q6h_p96" and j == 0:
            assert p.S + p.K + 3 == 96 == L.get_layout(ti.options("q6h", "linear", "additive", 29)[0]).pstride
    if name == "hourly":
        assert (ds[-1] - ds[0]) == 30 * DAY
    if name == "mixed":
        assert [ds.size >= 800 for ds, _ in series] == [False, True, False, True]


def test_table_cells_reach_both_reduction_bands_and_the_fall_back():
    """The predict cells' highest harmonic arguments: hourly (1/24, 4) in [8e6, 2^21 2 pi), past the range the reduction
    was first checked over; q6h (0.25, 32) past 2^21 2 pi, the library sincos."""
    ti = _table_cells()
    guard = 2.0**21 * 2.0 * np.pi
    for name, per, o, lo, hi in (("hourly", 1.0 / 24.0, 4, 8e6, guard), ("q6h_p96", 0.25, 32, guard, np.inf)):
        ds = np.concatenate([s[0] for s in ti.cell_series(name)])
        arg = 2.0 * o * np.pi * st.tau_days(ds) / per
        assert lo <= arg.min() and arg.max() < hi, (name, arg.min(), arg.max())


def test_reuse_batch_masks_rise_and_fall():
    ti = _table_cells()
    series = ti._reuse_series()
    builtin, custom = ti.options("gap", "logistic", "multiplicative", 25)[2:]
    ents = ti.entries("gap")
    masks = tuple(st.table_mask(st.seasonalities(ds, builtin, custom, 10.0), ents) for ds, _ in series)
    assert masks == ti.REUSE_MASKS
    K = [sum(2 * e[2] for j, e in enumerate(ents) if (m >> j) & 1) for m in masks]
    assert any(a < b for a, b in zip(K, K[1:])) and any(a > b for a, b in zip(K, K[1:])), K
