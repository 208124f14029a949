"""The *_host entry points against their device twins (GPU).

A *_host call copies its numpy arrays to the device, runs the device body and copies the results back.  (a) Each host fit
and predict returns byte for byte what its *_device twin returns for the same arrays, where no other test compares the
two (sums, period sums, quantiles, components and the in-sample predict are compared in their own files).  (b) Each
*_host entry point returns the same code for the argument edge cases below: null outputs, zero and negative sizes, a bad
trace_cap, regressor options on an entry point without regressors, and the order in which the host and device calls
check their arguments."""
import ctypes as C

import numpy as np
import pytest

from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

pytestmark = pytest.mark.gpu

OK, E_ARG, E_UNSUPPORTED = 0, -1, -4
FIELDS = ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")
CAPM = 1.1
DAY = 86400 * 10**9
REGS = [dict(name="promo"), dict(name="price", prior_scale=0.5)]


def _same_bytes(a, b, what):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    b = b.detach().cpu().numpy() if hasattr(b, "detach") else np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert a.tobytes() == b.tobytes(), what


def _same_models(fa, fb):
    for k in FIELDS:
        _same_bytes(getattr(fa, k), getattr(fb, k), k)


@pytest.fixture(scope="module")
def batch():
    return synth.config2(n=48, T=400, seed=11)


@pytest.fixture(scope="module")
def dev(batch):
    import torch
    return (torch.as_tensor(batch.ds, device="cuda"), torch.as_tensor(batch.y, device="cuda"))


def _cap(b, scale=1.3):
    return np.array([b.y[b.offsets[i]:b.offsets[i + 1]].max() * scale for i in range(b.n)], np.float64)


def _reg_values(b, R=2, seed=4):
    rng = np.random.RandomState(seed)
    cols = [(rng.rand(b.ds.size) < 0.2).astype(np.float64), 10.0 + rng.randn(b.ds.size)]
    return np.ascontiguousarray(np.stack(cols[:R]))


def _future(b, h=30):
    return batched.make_future(b.ds[b.offsets[1:] - 1], h, DAY)


# ---- (a) host and device twins give the same bytes ----

def test_fit_host_matches_fit_device(gpu_ctx, batch, dev):
    import torch
    opts = batched.make_options()
    cap = _cap(batch)
    fh = batched.fit_batch_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM, cap=cap)
    lay = L.get_layout(opts)
    n = batch.n
    fd = batched.FittedBatch(torch.empty((n, lay.pstride), dtype=torch.float64, device="cuda"),
                             torch.empty((n, lay.smax), dtype=torch.float64, device="cuda"),
                             torch.empty((n, 8), dtype=torch.int32, device="cuda"),
                             torch.empty((n, 2), dtype=torch.int64, device="cuda"),
                             torch.empty((n, 4), dtype=torch.float64, device="cuda"), lay.smax, lay.kmax)
    cap_d = torch.as_tensor(cap, device="cuda")
    torch.cuda.synchronize()
    rc = L.load().pb200_fit_device(gpu_ctx.handle, C.byref(opts), dev[0].data_ptr(), dev[1].data_ptr(),
                                   batched._y_dtype(dev[1]), batched._np_ptr(batch.offsets), n, 0.0, CAPM,
                                   cap_d.data_ptr(), fd.params.data_ptr(), fd.tchange.data_ptr(), fd.meta_i32.data_ptr(),
                                   fd.meta_i64.data_ptr(), fd.meta_f64.data_ptr())
    assert rc == OK, L.last_error()
    gpu_ctx.synchronize()
    assert np.all(fh.meta_i32[:, 4] >= 0), fh.meta_i32[:, 4]
    _same_models(fh, fd)


def test_fit_warm_host_matches_fit_warm_device(gpu_ctx, batch, dev):
    import torch
    opts = batched.make_options()
    cap = _cap(batch)
    # the previous models: fits of the first 80 % of each history
    keep = [np.arange(batch.offsets[i], batch.offsets[i] + (batch.offsets[i + 1] - batch.offsets[i]) * 4 // 5)
            for i in range(batch.n)]
    idx = np.concatenate(keep)
    off0 = np.concatenate([[0], np.cumsum([k.size for k in keep])]).astype(np.int64)
    init = batched.fit_batch_host(gpu_ctx, opts, batch.ds[idx], batch.y[idx], off0, 0.0, CAPM, cap=cap)
    rng = np.random.RandomState(2)
    prior = np.stack([rng.uniform(0.01, 0.5, batch.n), rng.uniform(1.0, 10.0, batch.n)], axis=1)
    fh, _ = batched.fit_batch_warm_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM, init=init, cap=cap,
                                        prior=prior)
    fd = batched.fit_batch_device(gpu_ctx, opts, dev[0], dev[1], batch.offsets, 0.0, CAPM,
                                  cap=torch.as_tensor(cap, device="cuda"), prior=torch.as_tensor(prior, device="cuda"),
                                  init=init)
    assert np.all(fh.meta_i32[:, 4] >= 0), fh.meta_i32[:, 4]
    assert np.any(fh.warm == L.WARM_USED), fh.warm
    _same_models(fh, fd)
    _same_bytes(fh.warm, fd.warm, "warm")


def test_fit_regressors_host_matches_fit_regressors_device(gpu_ctx, batch, dev):
    import torch
    opts = batched.make_regressor_options(REGS)
    reg = _reg_values(batch)
    cap = _cap(batch)
    fh = batched.fit_batch_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM, cap=cap, regressors=reg)
    fd = batched.fit_batch_device(gpu_ctx, opts, dev[0], dev[1], batch.offsets, 0.0, CAPM,
                                  cap=torch.as_tensor(cap, device="cuda"), regressors=torch.as_tensor(reg, device="cuda"))
    assert np.all(fh.meta_i32[:, 4] >= 0), fh.meta_i32[:, 4]
    _same_models(fh, fd)
    _same_bytes(fh.reg_scale, fd.reg_scale, "reg_scale")


def test_fit_trace_host_model_matches_fit_host(gpu_ctx, batch):
    opts = batched.make_options()
    fh = batched.fit_batch_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM)
    ft, trace = batched.fit_batch_trace_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM, trace_cap=64)
    _same_models(fh, ft)
    assert np.any(trace[:, 0, 0] == 1.0)         # the trajectory was recorded


@pytest.mark.parametrize("intervals", [False, True])
def test_predict_host_matches_predict_device(gpu_ctx, batch, intervals):
    import torch
    opts = batched.make_options()
    fh = batched.fit_batch_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM)
    fut = _future(batch)
    cap32 = fh.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    floor = np.zeros(batch.n)
    ph = batched.predict_batch_host(gpu_ctx, opts, fh, fut, floor, cap32, seed=7, intervals=intervals)
    fdev = batched.FittedBatch(*[torch.as_tensor(getattr(fh, k), device="cuda") for k in FIELDS], fh.smax, fh.kmax)
    pd = batched.predict_batch_device(gpu_ctx, opts, fdev, torch.as_tensor(fut, device="cuda"),
                                      torch.as_tensor(floor, device="cuda"), torch.as_tensor(cap32, device="cuda"),
                                      seed=7, intervals=intervals)
    for k in ("yhat", "yhat_int") + (("yhat_lower", "yhat_upper") if intervals else ()):
        _same_bytes(getattr(ph, k), getattr(pd, k), k)
    assert (ph.yhat_lower is None) == (not intervals)


def test_predict_regressors_host_matches_predict_regressors_device(gpu_ctx, batch):
    import torch
    opts = batched.make_regressor_options(REGS)
    fh = batched.fit_batch_host(gpu_ctx, opts, batch.ds, batch.y, batch.offsets, 0.0, CAPM, regressors=_reg_values(batch))
    fut = _future(batch)
    rng = np.random.RandomState(9)
    freg = np.ascontiguousarray(np.stack([(rng.rand(*fut.shape) < 0.2).astype(np.float64),
                                          10.0 + rng.randn(*fut.shape)]))
    cap32 = fh.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    floor = np.zeros(batch.n)
    ph = batched.predict_batch_host(gpu_ctx, opts, fh, fut, floor, cap32, seed=5, regressors=freg)
    fdev = batched.FittedBatch(*[torch.as_tensor(getattr(fh, k), device="cuda") for k in FIELDS], fh.smax, fh.kmax,
                               reg_scale=torch.as_tensor(fh.reg_scale, device="cuda"))
    pd = batched.predict_batch_device(gpu_ctx, opts, fdev, torch.as_tensor(fut, device="cuda"),
                                      torch.as_tensor(floor, device="cuda"), torch.as_tensor(cap32, device="cuda"),
                                      seed=5, regressors=torch.as_tensor(freg, device="cuda"))
    for k in ("yhat", "yhat_int", "yhat_lower", "yhat_upper"):
        _same_bytes(getattr(ph, k), getattr(pd, k), k)


# ---- (b) the return codes of the *_host entry points at their argument edges ----

class _Args:
    """4 series, their fitted models (plain and with regressors), and room for every output of the *_host entry points.
    Each case below builds the raw argument list of one call from these; a missing array is passed as NULL."""

    def __init__(self, ctx):
        b = synth.config2(n=4, T=200, seed=3)
        self.b, self.n = b, b.n
        self.opts, self.reg_opts = batched.make_options(), batched.make_regressor_options(REGS)
        self.ds, self.y, self.off = b.ds, np.ascontiguousarray(b.y), b.offsets
        self.reg = _reg_values(b)
        self.m = batched.fit_batch_host(ctx, self.opts, b.ds, b.y, b.offsets, 0.0, CAPM)
        self.mr = batched.fit_batch_host(ctx, self.reg_opts, b.ds, b.y, b.offsets, 0.0, CAPM, regressors=self.reg)
        n, lay = b.n, L.get_layout(self.reg_opts)          # the wider layout: room for either model
        self.out = [np.zeros((n, lay.pstride)), np.zeros((n, lay.smax)), np.zeros((n, 8), np.int32),
                    np.zeros((n, 2), np.int64), np.zeros((n, 4))]
        self.trace, self.rsc, self.warm = np.zeros((n, 8, 4)), np.zeros((n, 2, 2)), np.zeros(n, np.int32)
        self.f, self.grad = np.zeros(n), np.zeros((n, lay.pstride))
        self.H = 6
        self.fut = np.ascontiguousarray(b.ds[b.offsets[1:] - 1][:, None] + DAY * np.arange(1, self.H + 1))
        self.freg = np.ascontiguousarray(np.stack([np.zeros((n, self.H)), np.full((n, self.H), 10.0)]))
        self.floor = np.zeros(n)
        self.cap = np.ascontiguousarray(self.m.meta_f64[:, 2])
        self.yhat, self.lo, self.hi = np.zeros((n, self.H)), np.zeros((n, self.H)), np.zeros((n, self.H))
        self.yint = np.zeros((n, self.H), np.int32)
        self.comp, self.tlo, self.thi = np.zeros((16, n, self.H)), np.zeros((n, self.H)), np.zeros((n, self.H))
        self.wmax = 8
        self.win = [np.zeros(n, np.int32), np.zeros((n, 8), np.int64), np.zeros((n, 8), np.int32), np.zeros((n, 8)),
                    np.zeros((n, 8), np.int64), np.zeros((n, 8)), np.zeros((n, 8))]
        self.pct, self.quant = np.array([10.0, 50.0, 90.0]), np.zeros((3, n, self.H))
        rows = int(b.offsets[-1])
        self.yhat_rows, self.lo_rows, self.hi_rows = np.zeros(rows), np.zeros(rows), np.zeros(rows)
        self.zero_off = np.zeros(n + 1, np.int64)
        self.neg_off = np.array([0] * n + [-1], np.int64)


def _p(a):
    return None if a is None else a.ctypes.data


def _with(opts, **kw):
    o = batched.copy_options(opts)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _fit(a, ctx, opts=None, n=None, ds=True, y_dtype=None, params=True):
    """pb200_fit_host's arguments: [ctx, opts, ds, y, y_dtype, offsets, n, floor, cap_multiplier, cap, <5 records>]"""
    out = [_p(v) for v in a.out]
    if not params:
        out[0] = None
    return [ctx, C.byref(opts or a.opts), _p(a.ds) if ds else None, _p(a.y),
            batched._y_dtype(a.y) if y_dtype is None else y_dtype, _p(a.off), a.n if n is None else n, 0.0, CAPM, None,
            *out]


def _pred(a, ctx, opts=None, n=None, h=None, yhat=True, bounds=True):
    """pb200_predict_host's arguments: [ctx, opts, <5 records>, n, future_ds, horizon, floor, cap, seed, yhat, lower, upper,
    yhat_int]; the model is the regressor fit for the regressor options"""
    m = a.mr if opts is a.reg_opts else a.m
    recs = [_p(np.ascontiguousarray(getattr(m, k))) for k in FIELDS]
    return [ctx, C.byref(opts or a.opts), *recs, a.n if n is None else n, _p(a.fut), a.H if h is None else h,
            _p(a.floor), _p(a.cap), 1, _p(a.yhat) if yhat else None, _p(a.lo) if bounds else None,
            _p(a.hi) if bounds else None, _p(a.yint)]


def _hist(lib, a, x, n=None, off="off", ds=True, yhat=True, params=True):
    recs = [_p(np.ascontiguousarray(getattr(a.m, k))) for k in FIELDS]
    if not params:
        recs[0] = None
    return lib.pb200_predict_history_host(x, C.byref(a.opts), *recs, a.n if n is None else n, _p(a.ds) if ds else None,
                                          _p(getattr(a, off)) if off else None, _p(a.floor), _p(a.cap), 1,
                                          _p(a.yhat_rows) if yhat else None, _p(a.lo_rows), _p(a.hi_rows))


def _cases():
    """pytest params (call(lib, args, ctx) -> code, expected code), the codes as the parent of the staging helper
    returned them"""
    c = []

    def add(name, expected, fn):
        c.append(pytest.param(fn, expected, id=name))

    fit = lambda lib, a, x, **kw: lib.pb200_fit_host(*_fit(a, x, **kw))                 # noqa: E731
    add("fit-ok", OK, fit)
    add("fit-null-ctx", E_ARG, lambda lib, a, x: fit(lib, a, None))
    add("fit-n0-nulls", OK, lambda lib, a, x: fit(lib, a, x, n=0, ds=False, params=False))
    add("fit-n-negative", E_ARG, lambda lib, a, x: fit(lib, a, x, n=-1))
    add("fit-null-params", E_ARG, lambda lib, a, x: fit(lib, a, x, params=False))
    add("fit-null-ds", E_ARG, lambda lib, a, x: fit(lib, a, x, ds=False))
    add("fit-y-dtype", E_ARG, lambda lib, a, x: fit(lib, a, x, y_dtype=3))
    add("fit-regressor-options", E_UNSUPPORTED, lambda lib, a, x: fit(lib, a, x, opts=a.reg_opts))
    add("fit-bad-options", E_UNSUPPORTED, lambda lib, a, x: fit(lib, a, x, opts=_with(a.opts, n_changepoints=31)))

    # pb200_fit_trace_host (no cap): trace_cap in 1 .. 2^26 / n, checked before any copy
    def trace(lib, a, x, tr, cap_, n=None):
        f = _fit(a, x, n=n)
        return lib.pb200_fit_trace_host(*f[:9], *f[10:], _p(tr), cap_)
    add("trace-ok", OK, lambda lib, a, x: trace(lib, a, x, a.trace, 8))
    add("trace-cap-0", E_ARG, lambda lib, a, x: trace(lib, a, x, a.trace, 0))
    add("trace-cap-too-large", E_ARG, lambda lib, a, x: trace(lib, a, x, a.trace, (1 << 26) // a.n + 1))
    add("trace-null", E_ARG, lambda lib, a, x: trace(lib, a, x, None, 8))
    add("trace-n0-null-cap-0", OK, lambda lib, a, x: trace(lib, a, x, None, 0, n=0))

    # pb200_fit_warm_host: [..., cap, prior, init_params, init_meta, <records>, warm, trace, trace_cap]
    def warm(lib, a, x, init=False, meta=False, tr=None, cap_=0, n=None):
        f = _fit(a, x, n=n)
        ip = _p(np.ascontiguousarray(a.m.params)) if init else None
        im = _p(np.ascontiguousarray(a.m.meta_i32)) if meta else None
        return lib.pb200_fit_warm_host(*f[:10], None, ip, im, *f[10:], _p(a.warm), _p(tr), cap_)
    add("warm-ok", OK, lambda lib, a, x: warm(lib, a, x, init=True, meta=True))
    add("warm-init-without-meta", E_ARG, lambda lib, a, x: warm(lib, a, x, init=True))
    add("warm-init-without-meta-n0", OK, lambda lib, a, x: warm(lib, a, x, init=True, n=0))
    add("warm-trace-cap-0", E_ARG, lambda lib, a, x: warm(lib, a, x, tr=a.trace, cap_=0))
    add("warm-trace-ok", OK, lambda lib, a, x: warm(lib, a, x, tr=a.trace, cap_=8))

    # pb200_fit_regressors_host: [..., cap, reg, reg_scale, <records>, trace, trace_cap]; untraced unless both are set
    def regfit(lib, a, x, reg=True, rsc=True, tr=None, cap_=0, opts=None):
        f = _fit(a, x, opts=opts or a.reg_opts)
        return lib.pb200_fit_regressors_host(*f[:10], _p(a.reg) if reg else None, _p(a.rsc) if rsc else None, *f[10:],
                                             _p(tr), cap_)
    add("regfit-ok", OK, regfit)
    add("regfit-null-values", E_ARG, lambda lib, a, x: regfit(lib, a, x, reg=False))
    add("regfit-null-scale", E_ARG, lambda lib, a, x: regfit(lib, a, x, rsc=False))
    add("regfit-trace-cap-0-untraced", OK, lambda lib, a, x: regfit(lib, a, x, tr=a.trace, cap_=0))
    add("regfit-trace-cap-too-large", E_ARG, lambda lib, a, x: regfit(lib, a, x, tr=a.trace, cap_=(1 << 26) // a.n + 1))
    add("regfit-plain-options-no-values", OK, lambda lib, a, x: regfit(lib, a, x, reg=False, rsc=False, opts=a.opts))

    # pb200_objective_host: [ctx .. cap_multiplier, theta, f, grad, meta_i32]
    def obj(lib, a, x, opts=None, n=None, f=True, theta=True):
        g = _fit(a, x, opts=opts, n=n)
        th = _p(np.ascontiguousarray(a.m.params)) if theta else None
        return lib.pb200_objective_host(*g[:9], th, _p(a.f) if f else None, _p(a.grad), _p(a.out[2]))
    add("objective-ok", OK, obj)
    add("objective-null-f", E_ARG, lambda lib, a, x: obj(lib, a, x, f=False))
    add("objective-null-theta", E_ARG, lambda lib, a, x: obj(lib, a, x, theta=False))
    add("objective-n0-null-f", OK, lambda lib, a, x: obj(lib, a, x, n=0, f=False))
    add("objective-regressor-options", E_UNSUPPORTED, lambda lib, a, x: obj(lib, a, x, opts=a.reg_opts))

    # pb200_objective_regressors_host: [ctx .. cap_multiplier, reg, reg_scale, theta, f, grad, meta_i32]
    def objreg(lib, a, x, reg=True):
        g = _fit(a, x, opts=a.reg_opts)
        return lib.pb200_objective_regressors_host(*g[:9], _p(a.reg) if reg else None, _p(a.rsc),
                                                   _p(np.ascontiguousarray(a.mr.params)), _p(a.f), _p(a.grad), _p(a.out[2]))
    add("objective-regressors-ok", OK, objreg)
    add("objective-regressors-null-values", E_ARG, lambda lib, a, x: objreg(lib, a, x, reg=False))

    # pb200_predict_host: without sums, n_models == 0 or horizon == 0 returns OK whatever the other size
    pred = lambda lib, a, x, **kw: lib.pb200_predict_host(*_pred(a, x, **kw))           # noqa: E731
    add("predict-ok", OK, pred)
    add("predict-no-intervals", OK, lambda lib, a, x: pred(lib, a, x, bounds=False))
    add("predict-null-ctx", E_ARG, lambda lib, a, x: pred(lib, a, None))
    add("predict-n0-h-negative", OK, lambda lib, a, x: pred(lib, a, x, n=0, h=-1))
    add("predict-n-negative-h0", OK, lambda lib, a, x: pred(lib, a, x, n=-1, h=0))
    add("predict-n-negative", E_ARG, lambda lib, a, x: pred(lib, a, x, n=-1))
    add("predict-h-negative", E_ARG, lambda lib, a, x: pred(lib, a, x, h=-1))
    add("predict-null-yhat", E_ARG, lambda lib, a, x: pred(lib, a, x, yhat=False))
    add("predict-regressor-options", E_UNSUPPORTED, lambda lib, a, x: pred(lib, a, x, opts=a.reg_opts))
    add("predict-samples-1", E_UNSUPPORTED, lambda lib, a, x: pred(lib, a, x, opts=_with(a.opts, uncertainty_samples=1)))
    add("predict-samples-1-no-intervals", OK,
        lambda lib, a, x: pred(lib, a, x, opts=_with(a.opts, uncertainty_samples=1), bounds=False))
    add("predict-width-nan", E_ARG, lambda lib, a, x: pred(lib, a, x, opts=_with(a.opts, interval_width=float("nan"))))
    # ... where the device twin refuses a negative horizon
    add("predict-device-n0-h-negative", E_ARG, lambda lib, a, x: lib.pb200_predict_device(*_pred(a, x, n=0, h=-1)))

    # pb200_predict_regressors_host: [.. seed, future_reg, reg_scale, yhat ..]
    def predreg(lib, a, x, freg=True, rsc=True):
        p = _pred(a, x, opts=a.reg_opts)
        return lib.pb200_predict_regressors_host(*p[:13], _p(a.freg) if freg else None,
                                                 _p(np.ascontiguousarray(a.mr.reg_scale)) if rsc else None, *p[13:])
    add("predict-regressors-ok", OK, predreg)
    add("predict-regressors-null-values", E_ARG, lambda lib, a, x: predreg(lib, a, x, freg=False))
    add("predict-regressors-null-scale", E_ARG, lambda lib, a, x: predreg(lib, a, x, rsc=False))

    # pb200_predict_components_host: [.., yhat_int, components, trend_lower, trend_upper]
    def comp(lib, a, x, planes=True, thi=True):
        return lib.pb200_predict_components_host(*_pred(a, x), _p(a.comp) if planes else None, _p(a.tlo),
                                                 _p(a.thi) if thi else None)
    add("components-ok", OK, comp)
    add("components-null-planes", E_ARG, lambda lib, a, x: comp(lib, a, x, planes=False))
    add("components-trend-lower-alone", E_ARG, lambda lib, a, x: comp(lib, a, x, thi=False))

    # pb200_predict_quantiles_host: the quantile arguments are checked before the sizes
    def quant(lib, a, x, n_q=3, pct=True, **kw):
        return lib.pb200_predict_quantiles_host(*_pred(a, x, **kw), n_q, _p(a.pct) if pct else None, _p(a.quant))
    add("quantiles-ok", OK, quant)
    add("quantiles-nq-0-n0-h0", E_ARG, lambda lib, a, x: quant(lib, a, x, n_q=0, n=0, h=0))
    add("quantiles-null-percentiles", E_ARG, lambda lib, a, x: quant(lib, a, x, pct=False))
    add("quantiles-samples-1-before-sizes", E_UNSUPPORTED,
        lambda lib, a, x: quant(lib, a, x, n=-1, opts=_with(a.opts, uncertainty_samples=1)))
    add("quantiles-n-negative", E_ARG, lambda lib, a, x: quant(lib, a, x, n=-1))

    # pb200_predict_sums_host: with sums, n_models == 0 returns OK only after the window arguments are checked
    def sums(lib, a, x, width=2 * DAY, wmax=None, n_windows=True, **kw):
        w = [_p(v) for v in a.win]
        if not n_windows:
            w[0] = None
        return lib.pb200_predict_sums_host(*_pred(a, x, **kw), width, int(a.b.ds[0]), a.wmax if wmax is None else wmax, *w)
    add("sums-ok", OK, sums)
    add("sums-h0", OK, lambda lib, a, x: sums(lib, a, x, h=0))
    add("sums-n0", OK, lambda lib, a, x: sums(lib, a, x, n=0))
    add("sums-n0-wmax-0", E_ARG, lambda lib, a, x: sums(lib, a, x, n=0, wmax=0))
    add("sums-n0-width-0", E_ARG, lambda lib, a, x: sums(lib, a, x, n=0, width=0))
    add("sums-n0-null-output", E_ARG, lambda lib, a, x: sums(lib, a, x, n=0, n_windows=False))
    add("sums-n-negative", E_ARG, lambda lib, a, x: sums(lib, a, x, n=-1))
    add("sums-h-negative", E_ARG, lambda lib, a, x: sums(lib, a, x, h=-1))

    # pb200_predict_period_sums_host
    def psums(lib, a, x, months=1, shift=0, **kw):
        return lib.pb200_predict_period_sums_host(*_pred(a, x, **kw), months, shift, a.wmax, *[_p(v) for v in a.win])
    add("period-sums-ok", OK, psums)
    add("period-sums-months-0-n0", E_ARG, lambda lib, a, x: psums(lib, a, x, months=0, n=0))
    add("period-sums-shift-out-of-range-n0", E_ARG, lambda lib, a, x: psums(lib, a, x, months=3, shift=3, n=0))

    # pb200_predict_history_host: a null ds is accepted when the frames hold 0 rows
    add("history-ok", OK, _hist)
    add("history-n0-null-offsets", OK, lambda lib, a, x: _hist(lib, a, x, n=0, off=None))
    add("history-n-negative", E_ARG, lambda lib, a, x: _hist(lib, a, x, n=-1))
    add("history-null-offsets", E_ARG, lambda lib, a, x: _hist(lib, a, x, off=None))
    add("history-zero-rows-null-ds", OK, lambda lib, a, x: _hist(lib, a, x, off="zero_off", ds=False, yhat=False))
    add("history-rows-negative", E_ARG, lambda lib, a, x: _hist(lib, a, x, off="neg_off"))
    add("history-null-ds", E_ARG, lambda lib, a, x: _hist(lib, a, x, ds=False))
    add("history-null-params", E_ARG, lambda lib, a, x: _hist(lib, a, x, params=False))
    return c


@pytest.fixture(scope="module")
def args(gpu_ctx):
    return _Args(gpu_ctx)


@pytest.mark.parametrize("call, expected", _cases())
def test_host_entry_point_return_codes(gpu_ctx, args, call, expected):
    rc = call(L.load(), args, gpu_ctx.handle)
    assert rc == expected, (rc, L.last_error())
