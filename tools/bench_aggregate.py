"""Cost of the forecast window totals on config #5 (100k fitted models x 672 15-min periods, 1000 draws; DESIGN §13).

    python tools/bench_aggregate.py [--models 100000] [--reps 5]

Five legs, alternated rep by rep after one warm-up call each, timed with CUDA events on the context's stream:
(1) predict alone; (2) pointwise 1000-draw intervals (predict + mc_kernel); (3) daily totals (predict + mc_sum_kernel,
7-8 windows per model); (4) totals at a width of 15 minutes (672 one-point windows: the selections of leg 2 through
mc_sum_kernel); (5) one window over the whole frame.  (3) - (1) is what the feature costs; (2) - (3) and (4) - (3) bound
the share of the selection in leg 2, (5) - (1) is the draw generation with one selection.  The models are fitted
config-#3 series tiled up to --models, as bench.py's scorer section does.  Also checks that leg 4's bounds are leg 2's
byte for byte and that every leg leaves yhat / yhat_int byte for byte.  Prints one JSON line with the card's name, power
limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402


def _smi():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as exc:       # the numbers still stand; say why the card could not be read
        return {"error": repr(exc)}


class SumsLeg:
    """pb200_predict_sums_device into buffers allocated once, so that a timed call is the launches alone."""

    def __init__(self, ctx, opts, fitted, fut, fl, cap, width_ns, wmax):
        n, h = fut.shape
        dev = fut.device
        f64 = dict(dtype=torch.float64, device=dev)
        self.yhat = torch.empty((n, h), **f64)
        self.yhat_int = torch.empty((n, h), dtype=torch.int32, device=dev)
        self.ws = batched.WindowSums(
            torch.zeros(n, dtype=torch.int32, device=dev), torch.empty((n, wmax), dtype=torch.int64, device=dev),
            torch.empty((n, wmax), dtype=torch.int32, device=dev), torch.empty((n, wmax), **f64),
            torch.empty((n, wmax), dtype=torch.int64, device=dev), torch.empty((n, wmax), **f64), torch.empty((n, wmax), **f64))
        w = self.ws
        self.args = (ctx.handle, C.byref(opts), fitted.params.data_ptr(), fitted.tchange.data_ptr(),
                     fitted.meta_i32.data_ptr(), fitted.meta_i64.data_ptr(), fitted.meta_f64.data_ptr(), n,
                     fut.data_ptr(), h, fl.data_ptr(), cap.data_ptr(), 1, self.yhat.data_ptr(), None, None,
                     self.yhat_int.data_ptr(), int(width_ns), 0, int(wmax), w.n_windows.data_ptr(), w.start.data_ptr(),
                     w.points.data_ptr(), w.yhat_sum.data_ptr(), w.quantity_sum.data_ptr(), w.lower.data_ptr(),
                     w.upper.data_ptr())
        self.keep = (opts, fitted, fut, fl, cap)

    def __call__(self):
        L.check(L.load().pb200_predict_sums_device(*self.args), "pb200_predict_sums_device")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", type=int, default=100_000)
    ap.add_argument("--fit", type=int, default=4096, help="config-#3 series fitted and tiled up to --models")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    H, STEP, DAY = 672, 15 * 60 * 10**9, 86400 * 10**9
    b = synth.config3(n=a.fit)
    fb = batched.fit_batch_device(ctx, batched.make_options(), torch.from_numpy(b.ds).to(dev),
                                  torch.from_numpy(b.y).to(dev), b.offsets, 0.0, 1.1)
    idx = torch.arange(a.models, device=dev) % fb.n
    sub = batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)),
                              fb.smax, fb.kmax)
    last = torch.from_numpy(b.ds[b.offsets[1:] - 1].copy()).to(dev)[idx]
    fut = (last[:, None] + STEP * torch.arange(1, H + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
    fl = torch.zeros(a.models, dtype=torch.float64, device=dev)
    cap = sub.meta_f64[:, 2].float().double().contiguous()
    o_det = batched.make_options(uncertainty_samples=0)
    o_mc = batched.make_options(uncertainty_samples=1000)
    ends = fut[:, [0, -1]].cpu().numpy()
    whole = 4 * 10**18                        # wider than any int64 timestamp after 1970: one window
    sums = {"daily_sums": SumsLeg(ctx, o_mc, sub, fut, fl, cap, DAY, batched.window_slots(ends[:, 0], ends[:, 1], DAY, 0)),
            "one_point_sums": SumsLeg(ctx, o_mc, sub, fut, fl, cap, STEP, H),
            "whole_frame_sum": SumsLeg(ctx, o_mc, sub, fut, fl, cap, whole, 1)}
    torch.cuda.synchronize(dev)
    bufs = {"predict": batched.predict_batch_device(ctx, o_det, sub, fut, fl, cap, seed=1, intervals=False),
            "intervals": batched.predict_batch_device(ctx, o_mc, sub, fut, fl, cap, seed=1, intervals=True)}

    def run(k):
        if k in sums:
            sums[k]()
        else:
            batched.predict_batch_device(ctx, o_mc if k == "intervals" else o_det, sub, fut, fl, cap, seed=1,
                                         intervals=k == "intervals", sync=False, out=bufs[k])

    legs = ["predict", "intervals", "daily_sums", "one_point_sums", "whole_frame_sum"]
    for k in legs:                            # warm-up: module load, shared-memory attribute, first touch of the outputs
        run(k)
    ctx.synchronize()
    one = sums["one_point_sums"]
    identity1 = (torch.equal(one.ws.lower, bufs["intervals"].yhat_lower) and torch.equal(one.ws.upper, bufs["intervals"].yhat_upper)
                 and torch.equal(one.ws.yhat_sum, bufs["predict"].yhat)
                 and torch.equal(one.ws.quantity_sum, bufs["predict"].yhat_int.long()))
    identity2 = all(torch.equal(s.yhat, bufs["predict"].yhat) and torch.equal(s.yhat_int, bufs["predict"].yhat_int)
                    for s in sums.values()) and torch.equal(bufs["intervals"].yhat, bufs["predict"].yhat)
    nw = sums["daily_sums"].ws.n_windows
    st = torch.cuda.ExternalStream(ctx.stream, device=dev)
    times = {k: [] for k in legs}
    clock = None
    for r in range(a.reps):
        for k in legs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            run(k)
            e1.record(st)
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
            if r == a.reps - 1 and k == "intervals":
                clock = _smi()
    ms = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out = {"workload": f"{a.models} fitted config-#3 models x {H} 15-min periods, 1000 draws", "reps": a.reps,
           "median_ms": ms, "min_ms": {k: min(v) for k, v in times.items()}, "max_ms": {k: max(v) for k, v in times.items()},
           "daily_windows_per_model": [int(nw.min()), int(nw.max())],
           "daily_sums_extra_ms": ms["daily_sums"] - ms["predict"],
           "selection_share_of_intervals_ms": [ms["intervals"] - ms["daily_sums"], ms["one_point_sums"] - ms["daily_sums"]],
           "one_point_windows_equal_pointwise_intervals": bool(identity1),
           "yhat_and_yhat_int_unchanged": bool(identity2), "gpu": clock}
    print(json.dumps(out))
    if not (identity1 and identity2):
        raise SystemExit("the window sums disagree with pb200_predict_device")


if __name__ == "__main__":
    main()
