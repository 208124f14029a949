"""Cost of the forecast totals per calendar period (DESIGN §17): config-#3-fitted models x a 15-minute frame of 8 832
points (92 days, three or four calendar months), 1000 draws.

    python tools/bench_period_sums.py [--n 20000] [--reps 5]

Five legs, alternated rep by rep after one warm-up call each, timed with CUDA events on the context's stream: (1) predict
alone; (2) pointwise 1000-draw intervals (predict + mc_kernel); (3) daily totals (the fixed-width rule 1D); (4) monthly
totals (rule M: mc_sum_kernel's calendar instance); (5) quarterly totals (rule Q).  (4) - (3) is what the calendar
windows cost over fixed-width ones: one period_of per staged point in place of one 64-bit floor division.  Checks at full
size that the M call's yhat_sum is the ordered sum of its own yhat over each period, and that the scorer's W-SUN rule
(batched.period_rule) gives the rows of its 7D rule from 1970-01-05.  Prints one JSON line with the card's name, power
limit and SM clock read in the same run.  A timed call is the whole batched.* call: its output allocations (from torch's
caching allocator) and, for the totals, the copy of each frame's first and last point that sizes the slots.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_aggregate import _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402
from time_series_spark_b200.jobs.prophet_scorer import aggregate_rule  # noqa: E402

FIELDS = ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper")


def _same(x, y):
    """Bit for bit, NaN (an empty slot) equal to NaN."""
    if not x.is_floating_point():
        return torch.equal(x, y)
    return bool(torch.equal(x.view(torch.int64), y.view(torch.int64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000, help="models: fitted config-#3 series tiled up to this count")
    ap.add_argument("--fit", type=int, default=4096, help="config-#3 series fitted")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    H, STEP, DAY = 8832, 15 * 60 * 10**9, 86400 * 10**9
    b = synth.config3(n=min(a.fit, a.n))
    fb = batched.fit_batch_device(ctx, batched.make_options(), torch.from_numpy(b.ds).to(dev),
                                  torch.from_numpy(b.y).to(dev), b.offsets, 0.0, 1.1)
    idx = torch.arange(a.n, device=dev) % fb.n
    sub = batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)),
                              fb.smax, fb.kmax)
    last = torch.from_numpy(b.ds[b.offsets[1:] - 1].copy()).to(dev)[idx]
    fut = (last[:, None] + STEP * torch.arange(1, H + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
    fl = torch.zeros(a.n, dtype=torch.float64, device=dev)
    cap = sub.meta_f64[:, 2].float().double().contiguous()
    o_det = batched.make_options(uncertainty_samples=0)
    o_mc = batched.make_options(uncertainty_samples=1000)
    torch.cuda.synchronize(dev)
    out = {}

    def run(k):
        if k == "predict":
            return batched.predict_batch_device(ctx, o_det, sub, fut, fl, cap, seed=1, intervals=False)
        if k == "intervals":
            return batched.predict_batch_device(ctx, o_mc, sub, fut, fl, cap, seed=1, intervals=True)
        if k == "daily_sums":
            return batched.predict_sums_device(ctx, o_mc, sub, fut, fl, cap, DAY, 0, seed=1)
        _, months, shift = batched.period_rule({"month_sums": "M", "quarter_sums": "Q"}[k])
        return batched.predict_period_sums_device(ctx, o_mc, sub, fut, fl, cap, months, shift, seed=1)

    legs = ["predict", "intervals", "daily_sums", "month_sums", "quarter_sums"]
    for k in legs:                            # warm-up: module load, shared-memory attribute, allocator
        out[k] = run(k)
    ctx.synchronize()
    # M: yhat_sum is the ordered sum of the call's own yhat over each period
    fc, ws = out["month_sums"]
    yh = fc.yhat.cpu().numpy()
    nw, pts, ysum = ws.n_windows.cpu().numpy(), ws.points.cpu().numpy(), ws.yhat_sum.cpu().numpy()
    ordered = True
    for i in range(a.n):
        off = 0
        for j in range(int(nw[i])):
            ordered &= bool(np.add.accumulate(yh[i, off:off + pts[i, j]])[-1] == ysum[i, j])
            off += int(pts[i, j])
        ordered &= off == H
    month_counts = [int(nw.min()), int(nw.max())]
    del out
    # W-SUN through period_rule against 7D from 1970-01-05 through aggregate_rule
    _, w_width, w_origin = batched.period_rule("W-SUN")
    width7, origin7 = aggregate_rule({"io": {"aggregates": "a"},
                                      "forecast": {"aggregate": "7D", "aggregate_origin": "1970-01-05"}})
    _, wk = batched.predict_sums_device(ctx, o_mc, sub, fut, fl, cap, w_width, w_origin, seed=1)
    _, fx = batched.predict_sums_device(ctx, o_mc, sub, fut, fl, cap, width7, origin7, seed=1)
    week_identity = (w_width, w_origin) == (width7, origin7) and all(_same(getattr(wk, f), getattr(fx, f)) for f in FIELDS)
    del wk, fx
    torch.cuda.empty_cache()
    st = torch.cuda.ExternalStream(ctx.stream, device=dev)
    times = {k: [] for k in legs}
    clock = None
    for r in range(a.reps):
        for k in legs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            res = run(k)
            e1.record(st)
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
            del res
            if r == a.reps - 1 and k == "month_sums":
                clock = _smi()
    ms = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = {"workload": f"{a.n} fitted config-#3 models x {H} 15-min points (92 days), 1000 draws", "reps": a.reps,
           "median_ms": ms, "min_ms": {k: min(v) for k, v in times.items()}, "max_ms": {k: max(v) for k, v in times.items()},
           "months_per_model": month_counts,
           "month_minus_daily_ms": ms["month_sums"] - ms["daily_sums"],
           "month_yhat_sum_is_ordered_sum_of_yhat": bool(ordered), "w_sun_equals_7d_from_1970_01_05": bool(week_identity),
           "gpu": clock}
    print(json.dumps(res))
    if not (ordered and week_identity):
        raise SystemExit("the period sums disagree with their identities")


if __name__ == "__main__":
    main()
