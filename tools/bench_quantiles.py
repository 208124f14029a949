"""Cost of forecast quantiles at many levels on config #5 (100k fitted models x 672 15-min periods, 1000 draws;
DESIGN §15).

    python tools/bench_quantiles.py [--models 100000] [--reps 5]

Seven legs, alternated rep by rep after one warm-up call each, timed with CUDA events on the context's stream:
(1) predict alone; (2) pointwise intervals (predict + mc_kernel); (3) Q = 2 planes at the interval's own percentiles and
no bounds (pb200_predict_quantiles_device); (4) deciles (Q = 9); (5) Q = 19 (0.05 ... 0.95); (6) Q = 32; (7) one
whole-frame window total (predict + mc_sum_kernel: the draw generation with one selection per model, DESIGN §13's
baseline).  (k) - (7) is the selection cost of leg k beyond generation.  Checks that leg 3's planes are leg 2's bounds byte for byte at full size and
that every leg leaves yhat / yhat_int byte for byte.  Prints one JSON line with the card's name, power limit and SM clock
read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_aggregate import SumsLeg, _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402


class QuantLeg:
    """pb200_predict_quantiles_device at raw percentiles into buffers allocated once."""

    def __init__(self, ctx, opts, fitted, fut, fl, cap, pct):
        n, h = fut.shape
        dev = fut.device
        self.pct = np.ascontiguousarray(pct, dtype=np.float64)
        self.yhat = torch.empty((n, h), dtype=torch.float64, device=dev)
        self.yhat_int = torch.empty((n, h), dtype=torch.int32, device=dev)
        self.planes = torch.empty((self.pct.size, n, h), dtype=torch.float64, device=dev)
        self.args = (ctx.handle, C.byref(opts), fitted.params.data_ptr(), fitted.tchange.data_ptr(),
                     fitted.meta_i32.data_ptr(), fitted.meta_i64.data_ptr(), fitted.meta_f64.data_ptr(), n,
                     fut.data_ptr(), h, fl.data_ptr(), cap.data_ptr(), 1, self.yhat.data_ptr(), None, None,
                     self.yhat_int.data_ptr(), int(self.pct.size), self.pct.ctypes.data, self.planes.data_ptr())
        self.keep = (opts, fitted, fut, fl, cap)

    def __call__(self):
        L.check(L.load().pb200_predict_quantiles_device(*self.args), "pb200_predict_quantiles_device")


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
    H, STEP = 672, 15 * 60 * 10**9
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
    w = o_mc.interval_width
    quant = {"q2_bounds": QuantLeg(ctx, o_mc, sub, fut, fl, cap, [100.0 * (1.0 - w) / 2.0, 100.0 * (1.0 + w) / 2.0]),
             "q9_deciles": QuantLeg(ctx, o_mc, sub, fut, fl, cap, [10.0 * k for k in range(1, 10)]),
             "q19": QuantLeg(ctx, o_mc, sub, fut, fl, cap, [5.0 * k for k in range(1, 20)]),
             "q32": QuantLeg(ctx, o_mc, sub, fut, fl, cap, np.linspace(1.0, 99.0, 32))}
    whole = SumsLeg(ctx, o_mc, sub, fut, fl, cap, 4 * 10**18, 1)
    torch.cuda.synchronize(dev)
    bufs = {"predict": batched.predict_batch_device(ctx, o_det, sub, fut, fl, cap, seed=1, intervals=False),
            "intervals": batched.predict_batch_device(ctx, o_mc, sub, fut, fl, cap, seed=1, intervals=True)}

    def run(k):
        if k in quant:
            quant[k]()
        elif k == "whole_frame_sum":
            whole()
        else:
            batched.predict_batch_device(ctx, o_mc if k == "intervals" else o_det, sub, fut, fl, cap, seed=1,
                                         intervals=k == "intervals", sync=False, out=bufs[k])

    legs = ["predict", "intervals", "q2_bounds", "q9_deciles", "q19", "q32", "whole_frame_sum"]
    for k in legs:                            # warm-up: module load, shared-memory attribute, first touch of the outputs
        run(k)
    ctx.synchronize()
    q2 = quant["q2_bounds"]
    identity1 = torch.equal(q2.planes[0], bufs["intervals"].yhat_lower) and torch.equal(q2.planes[1], bufs["intervals"].yhat_upper)
    identity2 = all(torch.equal(q.yhat, bufs["predict"].yhat) and torch.equal(q.yhat_int, bufs["predict"].yhat_int)
                    for q in quant.values()) and torch.equal(bufs["intervals"].yhat, bufs["predict"].yhat)
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
            if r == a.reps - 1 and k == "q9_deciles":
                clock = _smi()
    ms = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    gen = ms["whole_frame_sum"]
    nq = {"q2_bounds": 2, "q9_deciles": 9, "q19": 19, "q32": 32}
    out = {"workload": f"{a.models} fitted config-#3 models x {H} 15-min periods, 1000 draws", "reps": a.reps,
           "median_ms": ms, "min_ms": {k: min(v) for k, v in times.items()}, "max_ms": {k: max(v) for k, v in times.items()},
           "selection_ms_beyond_generation": {k: ms[k] - gen for k in ["intervals", *nq]},
           "selection_ms_per_level": {k: (ms[k] - gen) / q for k, q in nq.items()},
           "q2_planes_equal_interval_bounds": bool(identity1), "yhat_and_yhat_int_unchanged": bool(identity2),
           "gpu": clock}
    print(json.dumps(out))
    if not (identity1 and identity2):
        raise SystemExit("the quantile planes disagree with pb200_predict_device")


if __name__ == "__main__":
    main()
