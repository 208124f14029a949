"""The scorer's future-regressor join (DESIGN §20) and what it adds to a forecast.

    python tools/bench_regressor_jobs.py [--models 100000] [--horizon 672] [--rows 700] [--reps 5] [--out FILE]

A table of ``--rows`` 15-minute rows per group (the last ``--horizon`` of them on the forecast grid, the rest before it)
with R = 2 values (a 0/1 flag and a price), in group order, for ``--models`` models.  Legs, each timed with CUDA events
on the context's stream after one warm-up call, alternated rep by rep:
  pack      pack_groups_cuda of the table (upload, sort check, [R, rows] planes)
  join      pb200_join_future_regressors_device alone
  predict0  predict_batch_device without regressors (the default model's fits tiled)
  predict2  predict_batch_device with the two regressors (a table model's fits tiled, the joined values)
  mc0, mc2  the same with 1000-draw intervals
Medians in ms, the join's bytes moved over its time, and the card's name and power limit read in the same run; one JSON
line on stdout (and in ``--out``).
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import torch  # noqa: E402

from bench_aggregate import _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402
from time_series_spark_b200.pack import pack_groups_cuda  # noqa: E402

M15 = 15 * 60 * 10**9
OFF = dict(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False)
TABLE = [dict(name="weekly2", period=7, fourier_order=3), dict(name="daily2", period=1, fourier_order=4)]


def _timed(st, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(st)
    fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b)


def _tile(fb, n):
    idx = torch.arange(n, device=fb.params.device) % fb.n
    return batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                               fb.meta_f64)), fb.smax, fb.kmax,
                               reg_scale=None if fb.reg_scale is None else fb.reg_scale[idx].contiguous())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", type=int, default=100000)
    ap.add_argument("--horizon", type=int, default=672)
    ap.add_argument("--rows", type=int, default=700)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, H, rows = a.models, a.horizon, a.rows
    ctx = L.Context(0)
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    st = torch.cuda.ExternalStream(ctx.stream)
    # the fits whose forecasts are timed: 256 config #3 series, default model and table + flag + price
    b = synth.config3(n=256)
    dsd, yd = torch.from_numpy(b.ds).to(dev), torch.from_numpy(b.y.astype(np.int32)).to(dev)
    reg = torch.stack([((dsd // (6 * 3600 * 10**9)) % 3 == 0).double(), 2.0 + torch.sin(dsd.double() / 2e14)])
    o0 = batched.make_options(uncertainty_samples=1000)
    o2 = batched.make_regressor_options([dict(name="promo"), dict(name="price")], seasonalities=TABLE,
                                        uncertainty_samples=1000, **OFF)
    f0 = _tile(batched.fit_batch_device(ctx, o0, dsd, yd, b.offsets, 0.0, 1.1), n)
    f2 = _tile(batched.fit_batch_device(ctx, o2, dsd, yd, b.offsets, 0.0, 1.1, regressors=reg.contiguous()), n)
    last = torch.from_numpy(b.offsets[1:] - 1).to(dev)
    last = dsd[last][torch.arange(n, device=dev) % b.n]
    fut = (last[:, None] + M15 * torch.arange(1, H + 1, device=dev)[None, :]).contiguous()
    # the table: rows per group ending at the grid's last point, in group order
    t = (last[:, None] + M15 * torch.arange(H - rows + 1, H + 1, device=dev)[None, :]).reshape(-1).cpu().numpy()
    sid = np.repeat(np.arange(n, dtype=np.int32), rows)
    tab = pa.table({"series_id": pa.array(sid), "dim_id": pa.array(np.zeros(n * rows, np.int32)),
                    "ds": pa.array(t, pa.int64()).cast(pa.timestamp("ns")),
                    "promo": pa.array(((t // (6 * 3600 * 10**9)) % 3 == 0).astype(np.float64)),
                    "price": pa.array(2.0 + np.sin(t / 2e14))})
    group = torch.arange(n, dtype=torch.int64, device=dev)
    floor = torch.zeros(n, dtype=torch.float64, device=dev)
    cap = f0.meta_f64[:, 2].contiguous()
    state = {}

    def pack():
        state["pk"] = pack_groups_cuda(tab, device=dev, y_col=None, reg_cols=["promo", "price"])

    def join():
        pk = state["pk"]
        state["freg"] = batched.join_future_regressors_device(ctx, pk.ds, pk.offsets, pk.regressors, group, fut)[0]

    legs = {
        "pack": pack, "join": join,
        "predict0": lambda: batched.predict_batch_device(ctx, o0, f0, fut, floor, cap, intervals=False),
        "predict2": lambda: batched.predict_batch_device(ctx, o2, f2, fut, floor, cap, intervals=False,
                                                         regressors=state["freg"]),
        "mc0": lambda: batched.predict_batch_device(ctx, o0, f0, fut, floor, cap, intervals=True),
        "mc2": lambda: batched.predict_batch_device(ctx, o2, f2, fut, floor, cap, intervals=True,
                                                    regressors=state["freg"]),
    }
    for fn in legs.values():
        fn()
    assert int(torch.isnan(state["freg"]).sum()) == 0
    times = {k: [] for k in legs}
    for _ in range(a.reps):
        for k, fn in legs.items():
            times[k].append(_timed(st, fn))
    med = {k: float(np.median(v)) for k, v in times.items()}
    # join traffic: the grid (8 B) and 2 values (16 B) out per point, the points' searched rows (about log2(rows) 8-byte
    # loads each, mostly L2 hits) left out: the lower bound of what it moves
    join_bytes = n * H * (8 + 2 * 8) + n * 16
    out = {"models": n, "horizon": H, "rows_per_group": rows, "R": 2, "reps": a.reps, "ms_median": med,
           "ms_all": times, "join_min_GBps": join_bytes / (med["join"] * 1e-3) / 1e9, "gpu": _smi()}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
