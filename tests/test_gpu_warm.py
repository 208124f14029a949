"""GPU tests of warm starts (pb200_fit_warm_device / _host, batched.fit_batch_device(init=...), the modeler's
``io.warm_start``; DESIGN §11).  Contexts are pinned to the kernel families of test_gpu_tune.py."""
import os
import subprocess
import sys

import numpy as np
import pyarrow.parquet as pq
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

import warm_oracle as wo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPM = 1.1
FIELDS = ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")
PREP_ERRORS = (L.ST_TOO_FEW, L.ST_CAP_LE_FLOOR, L.ST_BAD_INPUT, L.ST_BAD_PRIOR, L.ST_CONST_LINEAR)

FAMILIES = {
    "g8": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 8, "PB200_PLAIN_GROUP": 1},
    "g16": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 16, "PB200_PLAIN_GROUP": 1},
    "tab32": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 0},
    "rot32": {"PB200_LC0_MAX": 1 << 30, "PB200_NO_TAB": 1},
    "default": {},
}


def _ctx_with_env(**env):
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


@pytest.fixture(scope="module")
def ctx_for():
    cache = {}

    def get(family, **more):
        env = dict(FAMILIES[family], **more)
        key = tuple(sorted((k, str(v)) for k, v in env.items()))
        if key not in cache:
            cache[key] = _ctx_with_env(**env)
        return cache[key]

    yield get
    for c in cache.values():
        c.close()


def _join(parts):
    offs = np.concatenate(([0], np.cumsum([p.offsets[-1] for p in parts]))).astype(np.int64)
    o = np.concatenate([p.offsets[:-1] + s for p, s in zip(parts, offs[:-1])] + [offs[-1:]]).astype(np.int64)
    n = o.size - 1
    return synth.RaggedBatch(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), o,
                             np.concatenate([p.ds for p in parts]), np.concatenate([p.y for p in parts]))


def _lsfail_batch():
    return _join([synth.config4(n=500_000, lo=i, hi=i + 1) for i in synth.CONFIG4_LSFAIL_IDS] + [synth.config4(n=23)])


def _tight_opts():
    o = batched.make_options(algorithm="LBFGS", max_iter=20000)
    o.tol_rel_grad = o.tol_rel_obj = o.tol_grad = o.tol_param = 0.0
    o.tol_obj = 1e-13
    o.algorithm = L.ALG_LBFGS_NEWTON
    return o


CASES = {
    "g8": ("g8", lambda: synth.config3(n=24), batched.make_options),
    "g16": ("g16", lambda: synth.config3(n=24), batched.make_options),
    "tab32": ("tab32", lambda: synth.config3(n=12), batched.make_options),
    "rot32": ("rot32", lambda: synth.config3(n=12), batched.make_options),
    "default_4_warps": ("default", lambda: synth.config3(n=12), batched.make_options),
    "plain_g8": ("g8", lambda: synth.config4(n=32), batched.make_options),
    "newton": ("default", lambda: synth.config4(n=12), lambda: batched.make_options(algorithm="Newton")),
    "lbfgs_newton_retry": ("default", _lsfail_batch, _tight_opts),
}


def _dev(b):
    import torch
    return torch.from_numpy(b.ds).cuda(), torch.from_numpy(b.y).cuda()


def _fit(ctx, opts, b, init=None):
    ds, y = _dev(b)
    return batched.fit_batch_device(ctx, opts, ds, y, b.offsets, 0.0, CAPM, init=init).to_host()


def _fit_prior(ctx, opts, b):
    """pb200_fit_prior_device called directly: the cold fit the warm entry point must equal without an init."""
    import torch
    ds, y = _dev(b)
    lay = L.get_layout(opts)
    n = b.n
    out = [torch.empty((n, lay.pstride), dtype=torch.float64, device="cuda"),
           torch.empty((n, lay.smax), dtype=torch.float64, device="cuda"),
           torch.empty((n, 8), dtype=torch.int32, device="cuda"), torch.empty((n, 2), dtype=torch.int64, device="cuda"),
           torch.empty((n, 4), dtype=torch.float64, device="cuda")]
    torch.cuda.synchronize()
    L.check(L.load().pb200_fit_prior_device(ctx.handle, batched.C.byref(opts), ds.data_ptr(), y.data_ptr(),
                                            batched._y_dtype(y), b.offsets.ctypes.data, n, 0.0, CAPM, None, None,
                                            *(t.data_ptr() for t in out)), "pb200_fit_prior_device")
    ctx.synchronize()
    return batched.FittedBatch(*(t.cpu().numpy() for t in out), lay.smax, lay.kmax)


def _same(fa, fb):
    return all(getattr(fa, k).tobytes() == getattr(fb, k).tobytes() for k in FIELDS)


def _rows_equal(fa, ia, fb, ib):
    return all(getattr(fa, k)[ia].tobytes() == getattr(fb, k)[ib].tobytes() for k in FIELDS)


def _fitted_mask(f):
    """Series the fit optimises (rule 2's "not optimised": a prep error or the constant-linear shortcut)."""
    return ~np.isin(f.meta_i32[:, 4], PREP_ERRORS)


def _crafted_init(cold, lay):
    """Previous models for the rows of ``cold``: every fourth its own record (self-warm), the others broken one way
    each (every cold reason code)."""
    init = batched.FittedBatch(*(getattr(cold, k).copy() for k in FIELDS), cold.smax, cold.kmax)
    for i in range(cold.n):
        r = i % 8
        if r == 1:
            init.meta_i32[i, 4] = -1                        # no previous model
        elif r == 2:
            init.meta_i32[i, 1] += 1 if init.meta_i32[i, 1] < lay.smax else -1      # S differs
        elif r == 3:
            init.meta_i32[i, 3] ^= 2                        # the weekly seasonality differs
        elif r == 5:
            init.params[i, 0] = np.nan
        elif r == 6:
            init.params[i, 3 + lay.smax] = np.inf if init.meta_i32[i, 3] else -np.inf
        elif r == 7:
            init.params[i, 2] = 0.0 if i % 16 == 7 else -1.0
    return init


@pytest.mark.parametrize("case", list(CASES))
def test_warm_fit_per_family(ctx_for, case):
    family, mk, mko = CASES[case]
    ctx, b, opts = ctx_for(family), mk(), mko()
    lay = L.get_layout(opts)
    cold = _fit_prior(ctx, opts, b)
    # no init, and an init without any previous model: the cold fit, byte for byte
    none = _fit(ctx, opts, b)
    assert _same(none, cold) and none.warm is None
    empty = batched.FittedBatch(*(np.zeros_like(getattr(cold, k)) for k in FIELDS), cold.smax, cold.kmax)
    empty.meta_i32[:, 4] = -1
    e = _fit(ctx, opts, b, init=empty)
    assert _same(e, cold) and np.all(e.warm == L.WARM_NONE)
    # every reason code; the cold fall-backs are the cold fit, the codes are the host rule's
    init = _crafted_init(cold, lay)
    got = _fit(ctx, opts, b, init=init)
    codes, _ = batched.warm_start(init, cold.meta_i32[:, 1], cold.meta_i32[:, 3], _fitted_mask(cold))
    assert got.warm.tolist() == codes.tolist(), case
    fitted = _fitted_mask(cold)
    for want in (L.WARM_USED, L.WARM_NONE, L.WARM_SHAPE, L.WARM_BAD):
        assert np.any(codes[fitted] == want), (case, want)
    for i in np.flatnonzero(codes != L.WARM_USED):
        assert _rows_equal(got, i, cold, i), (case, int(i))
    # self-warm: a fit from its own optimum does not rise above it
    for i in np.flatnonzero(codes == L.WARM_USED):
        st = int(got.meta_i32[i, 4])
        assert st >= 0, (case, int(i), st)
        f0 = cold.meta_f64[i, 3]
        assert got.meta_f64[i, 3] <= f0 + 1e-12 * max(1.0, abs(f0)), (case, int(i), got.meta_f64[i, 3], f0)


def _appended(b, drop):
    """(the histories without their last ``drop`` rows, the full histories)."""
    parts = [b.take(i, i + 1) for i in range(b.n)]
    short = []
    for p in parts:
        T = int(p.offsets[-1])
        short.append(synth.RaggedBatch(p.series_id, p.dim_id, np.array([0, T - drop], np.int64), p.ds[:T - drop],
                                       p.y[:T - drop]))
    return _join(short), b


@pytest.mark.parametrize("family", ["g8", "g16", "tab32", "rot32", "default"])
def test_warm_trajectory_against_the_oracle(ctx_for, family):
    ctx = ctx_for(family)
    b = synth.config3(n=4 if family in ("g8", "g16") else 2)
    old_b, new_b = _appended(b, 10)
    opts = batched.make_options()
    old = _fit(ctx, opts, old_b)
    init = batched.FittedBatch(*(getattr(old, k) for k in FIELDS), old.smax, old.kmax)
    cold = _fit(ctx, opts, new_b)
    codes, x = batched.warm_start(init, cold.meta_i32[:, 1], cold.meta_i32[:, 3], _fitted_mask(cold))
    assert np.all(codes == L.WARM_USED)
    for max_iter, cap in ((1, 2), (6, 8)):
        o = batched.make_options(max_iter=max_iter)
        fb, tr = batched.fit_batch_warm_host(ctx, o, new_b.ds, new_b.y, new_b.offsets, 0.0, CAPM, init, trace_cap=cap)
        assert np.all(fb.warm == L.WARM_USED)
        for i in range(new_b.n):
            a, e = new_b.offsets[i], new_b.offsets[i + 1]
            P = int(cold.meta_i32[i, 1]) + int(batched._seasonal_k(cold.meta_i32[i, 3])) + 3
            trace = []
            r = wo.fit(new_b.ds[a:e], new_b.y[a:e].astype(np.float64), opts=po.ProphetOptions(max_iter=max_iter),
                       algorithm="LBFGS", trace=trace, init=x[i, :P])
            ot = np.array(trace).reshape(-1, 4)
            head = min(int(fb.meta_i32[i, 5]), len(ot), max_iter)
            assert head >= 1, (family, i)
            gt = tr[i, :head]
            assert np.array_equal(gt[:, 0], np.arange(1, head + 1)) and np.array_equal(gt[:, 3], ot[:head, 3]), (family, i)
            assert np.all(np.abs(gt[:, 1] - ot[:head, 1]) <= 1e-11 * np.maximum(1.0, np.abs(ot[:head, 1]))), (family, i)
            assert np.all(np.abs(gt[:, 2] - ot[:head, 2]) <= 1e-7 * np.abs(ot[:head, 2])), (family, i)
            if max_iter == 1:
                assert fb.meta_i32[i, 6] == r.n_evals, (family, i)


@pytest.mark.parametrize("case", ["newton", "lbfgs_newton_retry"])
def test_newton_from_the_warm_point_against_the_oracle(ctx_for, case):
    family, mk, mko = CASES[case]
    ctx, b, opts = ctx_for(family), mk(), mko()
    lay = L.get_layout(opts)
    cold = _fit_prior(ctx, opts, b)
    init = batched.FittedBatch(*(getattr(cold, k).copy() for k in FIELDS), cold.smax, cold.kmax)
    init.params[:, 3:] *= 0.5                              # a start point away from the optimum
    init.params[:, 0] *= 1.1
    got = _fit(ctx, opts, b, init=init)
    codes, x = batched.warm_start(init, cold.meta_i32[:, 1], cold.meta_i32[:, 3], _fitted_mask(cold))
    assert got.warm.tolist() == codes.tolist()
    rows = [0] if case == "lbfgs_newton_retry" else range(b.n)
    oopts = po.ProphetOptions(max_iter=opts.max_iter, tol_obj=opts.tol_obj, tol_rel_obj=opts.tol_rel_obj,
                              tol_grad=opts.tol_grad, tol_rel_grad=opts.tol_rel_grad, tol_param=opts.tol_param)
    for i in rows:
        assert codes[i] == L.WARM_USED
        a, e = b.offsets[i], b.offsets[i + 1]
        P = int(cold.meta_i32[i, 1]) + int(batched._seasonal_k(cold.meta_i32[i, 3])) + 3
        alg = "Newton" if case == "newton" else "LBFGS+Newton"
        r = wo.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=oopts, algorithm=alg, init=x[i, :P])
        st = int(got.meta_i32[i, 4])
        assert st >= 0 and (st == L.ST_NEWTON) == (r.ret == po.TERM_NEWTON), (case, i, st, r.ret)
        f = got.meta_f64[i, 3]
        assert abs(f - r.neg_logp) <= 1e-4 * max(1.0, abs(r.neg_logp)), (case, i, f, r.neg_logp)


def test_warm_series_bits_do_not_depend_on_their_neighbours(ctx_for):
    b = synth.config3(n=12)
    opts = batched.make_options()
    old_b, new_b = _appended(b, 10)
    ref_ctx = ctx_for("g8")
    old = _fit(ref_ctx, opts, old_b)
    lay = L.get_layout(opts)
    init = batched.FittedBatch(*(getattr(old, k).copy() for k in FIELDS), old.smax, old.kmax)
    init.meta_i32[1::3, 4] = -1                            # cold neighbours in the same warps
    full = _fit(ref_ctx, opts, new_b, init=init)
    assert np.all(full.warm[0::3] == L.WARM_USED) and np.all(full.warm[1::3] == L.WARM_NONE)

    def sub(idx):
        parts = _join([new_b.take(int(i), int(i) + 1) for i in idx])
        ini = batched.FittedBatch(*(getattr(init, k)[idx] for k in FIELDS), init.smax, init.kmax)
        return parts, ini

    perm = np.random.RandomState(4).permutation(new_b.n)
    for ctx in (ref_ctx, ctx_for("g8", PB200_FIT_GRID_MAX=1), ctx_for("g8", PB200_FIT_GRID_MAX=3)):
        for idx in (perm, np.array([0]), np.array([3, 1, 0])):
            parts, ini = sub(idx)
            got = _fit(ctx, opts, parts, init=ini)
            for j, i in enumerate(idx):
                assert _rows_equal(got, j, full, i), (int(i), idx.tolist())
                assert got.warm[j] == full.warm[i]


def test_absurd_start_point_is_an_init_error(ctx_for):
    b = synth.config3(n=8)
    opts = batched.make_options()
    for family in ("g8", "tab32", "default"):
        ctx = ctx_for(family)
        cold = _fit(ctx, opts, b)
        init = batched.FittedBatch(*(getattr(cold, k).copy() for k in FIELDS), cold.smax, cold.kmax)
        init.params[::2, 2] = 1e-300                           # finite and > 0: used, but the likelihood overflows
        got = _fit(ctx, opts, b, init=init)
        assert np.all(got.warm == L.WARM_USED)
        assert np.all(got.meta_i32[::2, 4] == L.ST_INIT_ERROR), (family, got.meta_i32[:, 4])
        assert np.all(got.meta_i32[1::2, 4] >= 0)


# ---- the job ----
def _write_tree(root, gi, drop=0):
    d = os.path.join(root, "series_id=751")
    os.makedirs(d, exist_ok=True)
    keep = np.ones(gi["y"].size, bool)
    if drop:
        for dim in np.unique(gi["dim_id"]):
            idx = np.flatnonzero(gi["dim_id"] == dim)
            keep[idx[np.argsort(gi["ds_ns"][idx], kind="stable")][-drop:]] = False     # the group's 10 latest rows
    ts = gi["ds_ns"][keep].astype("datetime64[ns]").astype("datetime64[s]")
    lines = [f"{int(a)},{str(t).replace('T', ' ')},{int(q)}" for a, t, q in zip(gi["dim_id"][keep], ts, gi["y"][keep])]
    with open(os.path.join(d, "part.csv"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return root


def _run(drv, cfg, tmp_path, name):
    import yaml
    path = tmp_path / f"{name}.yaml"
    path.write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", f"time_series_spark_b200.{drv}", str(path)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (drv, r.stdout[-2000:], r.stderr[-2000:])
    return r.stdout


def test_job_warm_starts_the_golden_fixture(tmp_path, golden_input):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    gi = golden_input
    short = _write_tree(str(tmp_path / "short"), gi, drop=10)
    full = _write_tree(str(tmp_path / "full"), gi)
    model = {"floor": 0, "cap_multiplier": 1.1}
    old = str(tmp_path / "old_models")
    ProphetModeler.model(None, {"io": {"input": short, "models": old}, "model": model})
    warm_cfg = {"io": {"input": full, "models": str(tmp_path / "warm_models"), "warm_start": old}, "model": model}
    out = _run("modeler_driver", warm_cfg, tmp_path, "warm")
    assert "Warm start: 2 series warm; cold: 0 without" in out and "; 0 table row(s) matched no input group" in out
    t = pq.read_table(warm_cfg["io"]["models"])
    assert t.column_names == ["series_id", "dim_id", "floor", "cap", "model"] and t.num_rows == 2
    # in place: the previous table is the output
    inplace = str(tmp_path / "inplace")
    ProphetModeler.model(None, {"io": {"input": short, "models": inplace}, "model": model})
    ip_cfg = {"io": {"input": full, "models": inplace, "warm_start": inplace}, "model": model}
    out = _run("modeler_driver", ip_cfg, tmp_path, "inplace")
    assert "Warm start: 2 series warm" in out
    ti = pq.read_table(inplace)
    assert ti.num_rows == 2 and ti.sort_by("dim_id")["model"].to_pylist() == t.sort_by("dim_id")["model"].to_pylist()
    # the scorer reads the warm table unchanged
    sc = {"io": {"models": inplace, "forecasts": str(tmp_path / "fc")}, "forecast": {"periods": 12, "frequency": "15min"}}
    _run("scorer_driver", sc, tmp_path, "score")
    import pyarrow.dataset as pads
    assert pads.dataset(sc["io"]["forecasts"], format="csv").to_table().num_rows == 24


def test_job_warm_start_through_the_driver_on_a_synth_tree(tmp_path):
    b = synth.config3(n=3)
    old_b, new_b = _appended(b, 10)

    def tree(bb, root):
        for i in range(bb.n):
            d = root / f"series_id={300 + i}"
            d.mkdir(parents=True)
            a, e = bb.offsets[i], bb.offsets[i + 1]
            ts = bb.ds[a:e].astype("datetime64[ns]").astype("datetime64[s]")
            (d / "part.csv").write_text("".join(f"4,{str(x).replace('T', ' ')},{int(q)}\n" for x, q in zip(ts, bb.y[a:e])))
        return str(root)

    model = {"floor": 0, "cap_multiplier": 1.1}
    models = str(tmp_path / "models")
    _run("modeler_driver", {"io": {"input": tree(old_b, tmp_path / "old"), "models": models}, "model": model}, tmp_path, "a")
    out = _run("modeler_driver", {"io": {"input": tree(new_b, tmp_path / "new"), "models": models, "warm_start": models},
                                  "model": model}, tmp_path, "b")
    assert "Warm start: 3 series warm" in out
    t = pq.read_table(models)
    assert sorted(t["series_id"].to_pylist()) == [300, 301, 302]
    bad = {"io": {"input": str(tmp_path / "new"), "models": str(tmp_path / "m2"), "warm_start": models},
           "model": dict(model, n_changepoints=10)}
    import yaml
    path = tmp_path / "bad.yaml"
    path.write_text(yaml.safe_dump(bad))
    r = subprocess.run([sys.executable, "-m", "time_series_spark_b200.modeler_driver", str(path)], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "io.warm_start" in r.stderr
