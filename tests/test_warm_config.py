"""CPU tests of warm starts (DESIGN §11): the host restatement of where a series starts (batched.warm_start), the warm
oracle (tests/warm_oracle.py), and the modeler job's ``io.warm_start`` handling (jobs/prophet_modeler.py)."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record
from time_series_spark_b200.jobs import prophet_modeler as pm

import warm_oracle as wo

NS_MIN = 60 * 10**9
NS_DAY = 86400 * 10**9
T0 = 1_600_000_000 * 10**9


def _history(T, step_min=15, seed=0):
    rng = np.random.RandomState(seed)
    ds = T0 + np.arange(T, dtype=np.int64) * step_min * NS_MIN
    tt = np.arange(T) * step_min / 1440.0
    y = 100 + 2 * tt + 20 * np.sin(2 * np.pi * tt) + 5 * np.sin(2 * np.pi * tt / 7) + rng.randn(T)
    return ds, np.round(y)


def _prep(T, step_min=15, seed=0):
    ds, y = _history(T, step_min, seed)
    return po.prepare(ds, y, 0.0, y.max() * 1.1, po.ProphetOptions())


def _record(p, lay, seed=1):
    """A model record with finite values, sized to prepared history ``p``."""
    rng = np.random.RandomState(seed)
    row = np.zeros(lay.pstride)
    row[:2] = rng.randn(2)
    row[2] = 0.05
    row[3:3 + p.S] = 0.01 * rng.randn(p.S)
    row[3 + lay.smax:3 + lay.smax + p.K] = 0.1 * rng.randn(p.K)
    meta = np.array([p.t.size, p.S, p.n_changepoints_real, wo.season_mask(p), 31, 5, 9, 0], np.int32)
    return row, meta


def _batch(rows, metas, lay):
    n = len(rows)
    return batched.FittedBatch(np.array(rows), np.zeros((n, lay.smax)), np.array(metas), np.zeros((n, 2), np.int64),
                               np.zeros((n, 4)), lay.smax, lay.kmax)


def test_host_rule_covers_every_reason_code():
    opts = batched.make_options()
    lay = L.get_layout(opts)
    # (old history, new history): the new one decides S and the mask
    cases = {
        "same": ((1440, 15), (1536, 15)),
        "S 24 -> 25": ((32, 15), (33, 15)),               # floor(0.8 T) - 1 changepoints around n_changepoints + 1
        "S 25 -> 24": ((33, 15), (32, 15)),
        "weekly on": ((1340, 15), (1345, 15)),            # the span crosses 14 days
        "daily on": ((190, 15), (193, 15)),               # the span crosses 2 days
    }
    rows, metas, S, mask, want = [], [], [], [], []
    for name, ((To, so), (Tn, sn)) in cases.items():
        po_, pn = _prep(To, so), _prep(Tn, sn)
        r, m = _record(po_, lay)
        rows.append(r)
        metas.append(m)
        S.append(pn.S)
        mask.append(wo.season_mask(pn))
        want.append(L.WARM_USED if name == "same" else L.WARM_SHAPE)
    assert (S[1], S[2]) == (25, 24) and (mask[3], mask[4]) == (6, 4)
    assert (metas[1][1], metas[2][1], metas[3][3], metas[4][3]) == (24, 25, 4, 0)
    pn = _prep(1536)
    base, meta = _record(pn, lay)
    bad_cols = {"k nan": (0, np.nan), "m +inf": (1, np.inf), "delta -inf": (3 + 4, -np.inf),
                "beta nan": (3 + lay.smax + pn.K - 1, np.nan), "sigma 0": (2, 0.0), "sigma < 0": (2, -1e-3),
                "sigma nan": (2, np.nan), "sigma inf": (2, np.inf)}
    for col, v in bad_cols.values():
        r = base.copy()
        r[col] = v
        rows.append(r)
        metas.append(meta)
        S.append(pn.S)
        mask.append(wo.season_mask(pn))
        want.append(L.WARM_BAD)
    # values past S and K are not the model's: they do not matter
    r = base.copy()
    r[3 + pn.S:3 + lay.smax] = np.nan
    rows.append(r), metas.append(meta), S.append(pn.S), mask.append(wo.season_mask(pn)), want.append(L.WARM_USED)
    # no previous model; a series that is not optimised; a failed previous fit
    for st, fitted in ((-1, True), (31, False), (L.ST_LSFAIL, True)):
        m = meta.copy()
        m[4] = st
        rows.append(base.copy()), metas.append(m), S.append(pn.S), mask.append(wo.season_mask(pn))
        want.append(L.WARM_NONE)
    fitted = np.ones(len(rows), bool)
    fitted[-2] = False
    init = _batch(rows, metas, lay)
    codes, x = batched.warm_start(init, np.array(S), np.array(mask), fitted)
    assert codes.tolist() == want
    used = np.flatnonzero(codes == L.WARM_USED)
    assert np.all(np.isnan(x[codes != L.WARM_USED]))
    for i in used:
        s, K = S[i], int(batched._seasonal_k(mask[i]))
        r = init.params[i]
        assert x[i, :3 + s + K].tobytes() == np.concatenate((r[:2], r[3:3 + s], [np.log(r[2])],
                                                               r[3 + lay.smax:3 + lay.smax + K])).tobytes()
        assert np.all(np.isnan(x[i, 3 + s + K:]))


def test_warm_oracle_from_the_cold_start_is_the_cold_fit():
    ds, y = _history(288)
    p = po.prepare(ds, y, 0.0, y.max() * 1.1, po.ProphetOptions())
    for alg in ("LBFGS+Newton", "LBFGS"):
        a = po.fit(ds, y, algorithm=alg)
        b = wo.fit(ds, y, algorithm=alg, init=po.initial_theta(p))
        assert a.theta.tobytes() == b.theta.tobytes() and (a.neg_logp, a.iters, a.n_evals, a.ret) == \
            (b.neg_logp, b.iters, b.n_evals, b.ret)
    with pytest.raises(ValueError):
        wo.fit(ds, y, init=np.zeros(3))


def test_warm_oracle_never_ends_above_its_start():
    ds, y = _history(384, seed=3)
    old = po.fit(ds[:-96], y[:-96])
    p = po.prepare(ds, y, 0.0, y.max() * 1.1, po.ProphetOptions())
    assert old.prep.S == p.S and wo.season_mask(old.prep) == wo.season_mask(p)
    x0 = old.theta
    err, f0, _ = po.neg_logp_grad(x0, p)
    assert err == 0
    warm = wo.fit(ds, y, init=x0)
    assert warm.ret > 0 and warm.neg_logp <= f0
    # from its own optimum the fit stays there
    again = wo.fit(ds, y, init=warm.theta)
    assert again.ret > 0 and again.neg_logp <= warm.neg_logp


# ---- the job's io.warm_start ----
def _table(keys, opts, status=31, **over):
    """A models table with one record per (series_id, dim_id) key; row i's k is i (to follow rows through a join)."""
    lay = L.get_layout(opts)
    n = len(keys)
    params = np.zeros((n, lay.pstride))
    params[:, 0] = np.arange(n)
    params[:, 2] = 0.1
    mi = np.zeros((n, 8), np.int32)
    mi[:, 1], mi[:, 3], mi[:, 4] = lay.smax, 6, status
    fb = batched.FittedBatch(params, np.zeros((n, lay.smax)), mi, np.zeros((n, 2), np.int64), np.zeros((n, 4)),
                             lay.smax, lay.kmax)
    o2 = L.Options.from_buffer_copy(opts)
    for k, v in over.items():
        setattr(o2, k, v)
    sid = np.array([k[0] for k in keys], np.int32)
    did = np.array([k[1] for k in keys], np.int32)
    return pa.table({"series_id": pa.array(sid, pa.int32()), "dim_id": pa.array(did, pa.int32()),
                     "floor": pa.array(np.zeros(n, np.float32)), "cap": pa.array(np.ones(n, np.float32)),
                     "model": model_record.encode(fb, np.zeros(n, np.int64), o2)})


@pytest.mark.parametrize("over", [{"growth": L.GROWTH_LINEAR}, {"multiplicative": 0}, {"yearly": 0}, {"weekly": 1},
                                  {"daily": 0}, {"n_changepoints": 10}])
def test_option_mismatch_names_the_key(over):
    opts = batched.make_options()
    t = _table([(1, 2)], opts, **over)
    with pytest.raises(ValueError, match="io.warm_start"):
        pm.warm_start_init(t, opts, np.array([1], np.int32), np.array([2], np.int32))


def test_duplicate_keys_name_the_first_group():
    opts = batched.make_options()
    t = _table([(5, 1), (7, 3), (5, 2), (7, 3), (5, 1)], opts)
    with pytest.raises(ValueError, match=r"io.warm_start.*first offender: series_id 7, dim_id 3; 2 group"):
        pm.warm_start_init(t, opts, np.array([5], np.int32), np.array([1], np.int32))


def test_join_equals_a_dictionary_join_on_shuffled_keys():
    opts = batched.make_options()
    lay = L.get_layout(opts)
    rng = np.random.RandomState(11)
    keys = [(int(s), int(d)) for s in range(40) for d in (-3, 0, 7, 2**31 - 1)]
    rng.shuffle(keys)
    table_keys = keys[:120]                           # the table: 120 groups ...
    groups = keys[60:] + [(999, 1), (-5, -5)]         # ... the input: 102 groups, 60 of them in the table
    rng.shuffle(groups)
    t = _table(table_keys, opts)
    sid = np.array([g[0] for g in groups], np.int32)
    did = np.array([g[1] for g in groups], np.int32)
    init, unmatched = pm.warm_start_init(t, opts, sid, did)
    row_of = {k: i for i, k in enumerate(table_keys)}
    assert unmatched == sum(k not in set(groups) for k in table_keys) == 60
    assert init.n == len(groups) and (init.smax, init.kmax) == (lay.smax, lay.kmax)
    for j, g in enumerate(groups):
        if g in row_of:
            assert init.params[j, 0] == row_of[g] and init.meta_i32[j, 4] == 31
        else:
            assert init.meta_i32[j, 4] < 0 and np.all(init.params[j] == 0)
    empty, un = pm.warm_start_init(t.slice(0, 0), opts, sid, did)
    assert un == 0 and np.all(empty.meta_i32[:, 4] < 0)


def test_report_line_counts_every_reason():
    w = np.array([L.WARM_USED, L.WARM_USED, L.WARM_NONE, L.WARM_SHAPE, L.WARM_BAD, L.WARM_SHAPE], np.int32)
    line = pm.warm_report(w, 4)
    assert line == ("Warm start: 2 series warm; cold: 1 without a previous model or not optimised, 2 whose changepoints "
                    "or seasonalities changed, 1 with unusable previous values; 4 table row(s) matched no input group")


def test_init_of_the_wrong_shape_is_refused():
    opts = batched.make_options()
    lay = L.get_layout(opts)
    fb = _batch([np.zeros(lay.pstride)] * 2, [np.zeros(8, np.int32)] * 2, lay)
    with pytest.raises(ValueError, match="init has 2 rows"):
        batched._check_init(fb, 3, lay)
    small = batched.FittedBatch(np.zeros((3, 10)), np.zeros((3, 5)), np.zeros((3, 8), np.int32),
                                np.zeros((3, 2), np.int64), np.zeros((3, 4)), 5, 2)
    with pytest.raises(ValueError, match="smax 5"):
        batched._check_init(small, 3, lay)
    with pytest.raises(ValueError, match="FittedBatch"):
        batched._check_init(np.zeros((3, lay.pstride)), 3, lay)
