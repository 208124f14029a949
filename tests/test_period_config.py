"""Forecast totals per calendar period (DESIGN §17) without a GPU: the calendar functions the kernel runs
(pb200_period_host, csrc/calendar.cuh) against pandas' ``to_period``, the alias parser ``batched.period_rule``, the slot
bound and its refusal of unrepresentable period starts, the reference tests/period_oracle.py, and the scorer's
``forecast.aggregate_period`` key."""
import re

import numpy as np
import pandas as pd
import pytest

import period_oracle as pdo
import window_oracle as wo
from oracle import mc_stream as mcs
from time_series_spark_b200 import batched
from time_series_spark_b200.jobs.prophet_scorer import ProphetScorer, aggregate_period, aggregate_rule

DAY = 86400 * 10**9
MONTHS = ("JAN", "FEB", "MAR", "APR", "MAY", "JUN", "JUL", "AUG", "SEP", "OCT", "NOV", "DEC")
DAYS = ("MON", "TUE", "WED", "THU", "FRI", "SAT", "SUN")
MONTH_ALIASES = ["M"] + [f"Q-{m}" for m in MONTHS] + [f"Y-{m}" for m in MONTHS]       # all 25 month rules


def _ns(s):
    return int(pd.Timestamp(s).value)


def _instants():
    """1679-01-01 .. 2262-04-01: every month start and +-1 ns around it, Feb 28 / 29 -> Mar 1 of 1900, 2000, 2024 and
    2100, instants around 1970-01-01, and 300 000 random instants; sorted, distinct."""
    starts = pd.date_range("1679-01-01", "2262-04-01", freq="MS").values.astype("datetime64[ns]").astype(np.int64)
    extra = []
    for y in (1900, 2000, 2024, 2100):
        for s in (f"{y}-02-28", f"{y}-02-28 23:59:59.999999999", f"{y}-03-01", f"{y}-03-01 00:00:00.000000001"):
            extra.append(_ns(s))
        if y % 4 == 0 and (y % 100 != 0 or y % 400 == 0):
            extra += [_ns(f"{y}-02-29"), _ns(f"{y}-02-29 12:00")]
    extra += [-DAY, -1, 0, 1, DAY - 1, DAY, _ns("1969-12-31 23:59:59.999999999"), _ns("1969-12-01"), _ns("1969-10-01")]
    rng = np.random.RandomState(0)
    rand = rng.randint(_ns("1679-01-01"), _ns("2262-04-01"), size=300_000, dtype=np.int64)
    ds = np.concatenate([starts, starts - 1, starts + 1, np.array(extra, np.int64), rand])
    return np.unique(ds[(ds >= _ns("1679-01-01")) & (ds < _ns("2262-04-01"))])


_DS = _instants()


@pytest.mark.parametrize("alias", MONTH_ALIASES)
def test_period_host_matches_pandas(alias):
    """The kernel's period_of / period_start (run on the host) partition the instants as pandas' to_period(alias) does,
    and every period starts at its start_time."""
    kind, months, shift = batched.period_rule(alias)
    assert kind == "months"
    period, start = batched.periods_host(_DS, months, shift)
    per = pd.DatetimeIndex(_DS.astype("datetime64[ns]")).to_period(alias)
    off = period - np.asarray(per.asi8, np.int64)
    assert np.all(off == off[0]), alias                         # the same partition, in the same order
    assert np.array_equal(start, per.start_time.values.astype("datetime64[ns]").astype(np.int64)), alias
    assert np.all(start <= _DS)


@pytest.mark.parametrize("day", DAYS)
def test_week_aliases_are_the_fixed_seven_day_rule(day):
    """W-<DAY> is 7D from the day after <DAY>: the tuple aggregate_rule gives for 7D with that origin, and the windows
    are pandas' weekly periods with their start times."""
    alias = f"W-{day}"
    kind, width, origin = batched.period_rule(alias)
    assert kind == "fixed" and width == 7 * DAY and 0 <= origin < 7 * DAY
    o = pd.Timestamp(origin)
    assert o.dayofweek == (DAYS.index(day) + 1) % 7
    cfg = {"io": {"aggregates": "a"}, "forecast": {"aggregate": "7D", "aggregate_origin": str(o.date())}}
    assert aggregate_rule(cfg) == (width, origin)
    ds = _DS[::50]
    first, start = wo.window_runs(ds, width, origin)
    pfirst, pstart = pdo.period_runs(ds, alias)
    assert np.array_equal(first, pfirst) and np.array_equal(start, pstart)
    if day == "SUN":
        assert batched.period_rule("W") == (kind, width, origin) and o == pd.Timestamp("1970-01-05")


def test_period_rule_accepts_the_period_aliases():
    assert batched.period_rule("M") == ("months", 1, 0)
    assert batched.period_rule("Q") == batched.period_rule("Q-DEC") == ("months", 3, 0)
    assert batched.period_rule("Y") == batched.period_rule("Y-DEC") == ("months", 12, 0)
    assert batched.period_rule("Q-NOV") == ("months", 3, 1)
    assert batched.period_rule("Q-JAN") == ("months", 3, 2)
    assert batched.period_rule("Y-JUN") == ("months", 12, 6)
    assert batched.period_rule("Y-JAN") == ("months", 12, 11)


@pytest.mark.parametrize("alias", ["D", "h", "7D", "MS", "QS", "A", "B", "2M", "2Q", "ME", "QE", "YE", "m", "q-nov",
                                   "Q-FOO", "W-JAN", "M-JAN", "W-", "", " M", 5, None])
def test_period_rule_refuses_other_aliases(alias):
    with pytest.raises(ValueError, match=re.escape(repr(alias))):
        batched.period_rule(alias)


def test_period_slots_bound_and_unrepresentable_starts():
    first = np.array([_ns("2021-01-31 23:00"), _ns("1969-11-15")], np.int64)
    last = np.array([_ns("2021-05-01"), _ns("1970-03-01")], np.int64)
    assert batched.period_slots(first, last, 1, 0) == 5             # 2021-01 .. 2021-05, 1969-11 .. 1970-03
    assert batched.period_slots(first, last, 3, 1) == 3             # Q-NOV: Sep-Nov 1969, Dec-Feb, Mar-May
    assert batched.period_slots(first[:0], last[:0], 1, 0) == 1
    # Y-JAN's period of 1678-01 starts 1677-02-01, before the earliest int64-ns instant
    early = np.array([_ns("1678-01-15")], np.int64)
    with pytest.raises(ValueError, match="1677-09-21"):
        batched.period_slots(early, early + DAY, 12, 11)
    assert batched.period_slots(early, early + DAY, 12, 0) == 1     # Y-DEC: 1678-01-01 is representable
    lo = np.array([int(pd.Timestamp.min.value)], np.int64)          # 1677-09-21 00:12:43: September starts before it
    with pytest.raises(ValueError, match="starts before"):
        batched.period_slots(lo, lo, 1, 0)
    for months, shift in ((2, 0), (3, 3), (12, -1), (0, 0)):
        with pytest.raises(ValueError, match="months"):
            batched.periods_host(first, months, shift)


def test_period_oracle_against_brute_force():
    """period_sums on a daily frame over New Year: runs by (year, month) of each point, sums point by point."""
    ds = _ns("2023-11-20") + DAY * np.arange(80, dtype=np.int64)
    d = np.random.RandomState(1).randn(80, 23) * 5.0 + 1.0
    start, pts, lo, hi = pdo.period_sums(d, ds, "M", 0.8)
    keys = [(t.year, t.month) for t in pd.DatetimeIndex(ds.astype("datetime64[ns]"))]
    runs = sorted(set(keys))
    assert pts.tolist() == [keys.count(k) for k in runs] == [11, 31, 31, 7]
    assert start.tolist() == [_ns(f"{y}-{m:02d}-01") for y, m in runs]
    lo_p, hi_p = mcs.percentiles(0.8)
    j0 = 0
    for j, n in enumerate(pts):
        s = np.zeros(23)
        for h in range(j0, j0 + n):
            s = s + d[h]
        j0 += n
        assert lo[j] == np.percentile(s, lo_p) and hi[j] == np.percentile(s, hi_p)
    e = pdo.period_sums(np.zeros((0, 4)), np.zeros(0, np.int64), "Q", 0.8)
    assert all(a.size == 0 for a in e)


def _cfg(io_aggregates=True, **fc):
    io = {"models": "/nonexistent/models", "forecasts": "f"}
    if io_aggregates:
        io["aggregates"] = "a"
    return {"io": io, "forecast": {"periods": 4, "frequency": "h", **fc}}


def test_aggregate_period_key():
    assert aggregate_period(_cfg()) is None
    assert aggregate_period(_cfg(aggregate_period="M")) == ("months", 1, 0)
    assert aggregate_period(_cfg(aggregate_period="Q-NOV")) == ("months", 3, 1)
    assert aggregate_period(_cfg(aggregate_period="W-SUN")) == ("fixed", 7 * DAY, 4 * DAY)
    assert aggregate_rule(_cfg(aggregate_period="M")) is None       # the fixed-width key is not set


@pytest.mark.parametrize("cfg", [
    _cfg(aggregate_period="M", aggregate="1D"),
    _cfg(aggregate_period="M", aggregate_origin="1970-01-05"),
    _cfg(aggregate_period="M", components=True),
    _cfg(aggregate_period="M", quantiles=[0.5]),
    _cfg(io_aggregates=False, aggregate_period="M"),
    _cfg(aggregate_period="MS"),
    _cfg(aggregate_period="2M"),
])
def test_aggregate_period_refusals_name_the_key_before_anything_is_read(cfg):
    with pytest.raises(ValueError, match="forecast.aggregate_period"):
        aggregate_period(cfg)
    with pytest.raises(ValueError, match="forecast.aggregate_period"):
        ProphetScorer.score(None, cfg)                             # io.models does not exist: nothing was read
