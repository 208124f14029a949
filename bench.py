#!/usr/bin/env python
"""Headline benchmark: series fitted / second on BASELINE.json config #3
(50k synthetic series x 1440 15-min points, logistic growth with cap, multiplicative
weekly+daily seasonality -- the reference's hard-coded Prophet(...) at prophet_modeler.py:65).

    python bench.py --gpus N --steps K --warmup W            # this framework (one rank per GPU)
    python bench.py --impl reference --gpus N --steps K --warmup W   # CPU arm: the oracle port on the usable host cores

A "step" = one batched fit of the rank's shard.  `value` = whole-job series/s with inputs resident in HBM
(CUDA events on the library's stream, max over ranks); `e2e` = the same through pb200_fit_host with pinned
HOST buffers (H2D + D2H inside the timed region).

Scaling.  The headline is 50k synthetic series x 1440 points at 1/2/4/8 H100: the SAME 50k
series split over the ranks (contiguous row-balanced ranges, dist.shard_bounds; no data-path collective), i.e.
STRONG scaling -- that is the headline `value` at N > 1 (`"scaling": "strong"`).  The weak-scaling figure
(every rank its own 50k series) is measured in the same run and reported under `weak`.
`--scaling weak` makes the weak figure the headline instead.  Prints ONE JSON line on rank 0.

`--dump-outputs DIR` writes what the last timed step returned (rank 0's fitted-model arrays) as DIR/<name>.npy, so that
two builds can be compared output for output on the same seeded inputs.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_SERIES = 50_000
T_POINTS = 1440
METRIC = "series fitted/sec at 50k x 1440pts"
UNIT = "series/s"
WORKLOAD = "config#3: 50k synthetic series x 1440 15-min pts, logistic growth w/ cap (x1.1), multiplicative weekly+daily"
# SURVEY 8(d): algorithmic bytes per series = T*(8 B ds + 4 B y) in + params/meta out
ALG_BYTES_PER_SERIES = T_POINTS * 12 + (8 * 62 + 8 * 25 + 8 * 4 + 2 * 8 + 4 * 8)
# flops per objective+gradient evaluation (SURVEY 8d): ~T*(4K+28), K=14
FLOPS_PER_EVAL = T_POINTS * (4 * 14 + 28)
HBM_FALLBACK_GBS = 3350.0      # H100 SXM data sheet (HBM3, 700 W card)
FP64_PEAK_GFLOPS = 132 * 64 * 2 * 1.98    # 132 SMs x 64 DFMA/clk x 2 flop x max SM clock (GHz): 33.5 TFLOP/s


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            d = json.load(open(p))
            for k in ("hbm_gbs", "hbm_gb_s", "hbm_GBps"):
                if k in d:
                    return float(d[k]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return HBM_FALLBACK_GBS, "fallback (H100 SXM data sheet 3.35 TB/s)"


def usable_cores() -> dict:
    """Host threads this process may actually use (affinity x cgroup quota), see time_series_spark_b200/dist.py."""
    from time_series_spark_b200.dist import usable_cores as f
    return f()


def _build_digest():
    """Digest of the CUDA sources + nvcc flags the library is built from (time_series_spark_b200/build.py)."""
    try:
        from time_series_spark_b200.build import _sources_digest
        return _sources_digest()[:16]
    except Exception:
        return None


def dump_outputs(dirpath: str, fitted) -> None:
    """The fitted-model arrays of the last timed step as DIR/<name>.npy (float64; 50k series: ~40 MB in all).
    meta_i64 holds start_ns / t_scale_ns in whole seconds, which float64 holds exactly up to ~4.6e9 s (the year 2115)."""
    os.makedirs(dirpath, exist_ok=True)
    for name in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64"):
        np.save(os.path.join(dirpath, f"{name}.npy"), np.ascontiguousarray(getattr(fitted, name), dtype=np.float64))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx.append(float(f[1]))
            except ValueError:
                continue
            for nm, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": float(np.max(mx)) if mx else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def _real_fbprophet():
    """BASELINE.md section 2: prefer a real fbprophet / prophet install (or baseline/_ref) when one exists.
    None in this image (no network, no JVM) -- the probe is what would flip `kind` to "reference"."""
    ref = os.path.join(ROOT, "baseline", "_ref")
    if os.path.isdir(ref) and ref not in sys.path:
        sys.path.insert(0, ref)
    for mod in ("fbprophet", "prophet"):
        try:
            m = __import__(mod)
            return mod, getattr(m, "__version__", "?")
        except Exception:
            continue
    return None


# ------------------------------------------------------------------------------------------
# CPU arm: the oracle port on the host cores
# ------------------------------------------------------------------------------------------
def cpu_baseline(n_sample: int, cores: dict, batch=None):
    """Fits series [0, n_sample) of config #3 with the plain-C oracle (oracle/prophet_oracle.c: same
    algorithm, per-segment sums, gcc -O2) on the usable host threads.  Generation is outside the timing."""
    from oracle import c_oracle as co
    from time_series_spark_b200 import synth
    co.load()
    b = batch if batch is not None else synth.config3(n=N_SERIES, lo=0, hi=n_sample)
    y = b.y.astype(np.float64)
    nthreads = cores["usable"]
    t0 = time.perf_counter()
    _, _, info = co.fit_batch(b.ds, y, b.offsets, 0.0, 1.1, nthreads=nthreads)
    wall = time.perf_counter() - t0
    n = b.n
    real = _real_fbprophet()
    return {"value": n / wall, "unit": UNIT, "cores": nthreads, "per_core": n / wall / nthreads, "kind": "port",
            "host": cores, "real_fbprophet_importable": real,
            "sample": f"first {n} series of the workload, oracle/prophet_oracle.c (plain-C float64 restatement of "
                      f"fbprophet 0.5 + Stan L-BFGS with the same O(T*K) segment-sum objective as the GPU kernel; "
                      f"NOT fbprophet itself: parity unpinned), {nthreads} OpenMP threads "
                      f"(usable of {cores['logical']} logical), {wall:.2f} s wall",
            "mean_evals": float(info[:, 2].mean())}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    from time_series_spark_b200 import synth
    cores = usable_cores()
    n_sample = int(os.environ.get("PB200_CPU_SAMPLE", str(max(256, 16 * cores["usable"]))))
    batch = synth.config3(n=N_SERIES, lo=0, hi=n_sample)
    for _ in range(args.warmup):
        cpu_baseline(min(n_sample, cores["usable"]), cores, batch.take(0, min(n_sample, cores["usable"])))
    t0 = time.perf_counter()
    last = None
    for _ in range(args.steps):
        last = cpu_baseline(n_sample, cores, batch)
    wall = time.perf_counter() - t0
    value = args.steps * n_sample / wall
    last["value"] = value
    last["per_core"] = value / cores["usable"]
    line = {"impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * wall / args.steps,
            "higher_is_better": True, "scaling": "strong" if args.scaling != "weak" else "weak", "vs_baseline": None,
            "dtype": "f64", "data": "synthetic",
            "config": {"workload": WORKLOAD, "sample_series_per_step": n_sample,
                       "note": "fbprophet/pystan/pyspark are not installable here (no network, no JVM); the CPU arm is "
                               "the C oracle port of the same algorithm on the usable host cores"},
            "cpu_baseline": last,
            "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))
    return 0


# ------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------
def _kernel_name(variants: dict, group_g: int, opts_growth_logistic=True) -> str:
    """The dominant fit kernel of the last step from the variant counts the library reports."""
    if not variants:
        return "none"
    top = max(variants, key=variants.get)
    logi = "true" if opts_growth_logistic else "false"
    if top == "day_table":
        if group_g:
            return (f"pb200::grp::fit_group_kernel<{group_g}, {logi}, true, true>  ({group_g} lanes per series, {32 // group_g} series "
                    f"per warp, logistic, weekly 3 + daily 4 harmonics, day-table + exp-ratio recurrence)")
        return f"pb200::fit_kernel<32, {logi}, 0, 3, 4, 3>  (warp per series, day-table variant)"
    return {"planes": f"pb200::fit_kernel<32, {logi}, 0, 3, 4, 0>", "rotation": f"pb200::fit_kernel<32, {logi}, 0, 3, 4, 1>",
            "week_table": f"pb200::fit_kernel<32, {logi}, 0, 3, 4, 2>"}[top]


def run_gpu(args):
    import torch
    import torch.distributed as dist
    from time_series_spark_b200 import _lib as L
    from time_series_spark_b200 import batched, synth
    from time_series_spark_b200 import dist as pdist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise RuntimeError("bench.py needs an H100: there is no CPU fallback for the product path")
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    n_total = int(os.environ.get("PB200_BENCH_SERIES", str(N_SERIES)))
    ctx = L.Context(local)
    opts = batched.make_options()          # reference defaults: logistic, multiplicative
    dev = torch.device("cuda", local)
    lib_stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
    group_env = int(os.environ.get("PB200_GROUP", "-1"))
    no_tab = os.environ.get("PB200_NO_TAB") == "1"

    def group_of(n):           # the library's dispatch (capi.cu): 8 lanes per series from 16384 series on, 16 below
        if no_tab:
            return 0
        if group_env >= 0:
            return group_env if group_env in (8, 16, 32) else 0
        return 8 if n >= int(os.environ.get("PB200_GROUP_MIN", "16384")) else 16

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def allmax(x: float) -> float:
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def allsum(x: float) -> float:
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    def timed_fit(b, steps, warmup, sampler=None):
        """K resident-input fits of batch b on this rank; returns (ms max over ranks, this rank's ms, out, launches)."""
        ds_d, y_d = torch.from_numpy(b.ds).to(dev), torch.from_numpy(b.y).to(dev)
        out = batched.fit_batch_device(ctx, opts, ds_d, y_d, b.offsets, 0.0, 1.1)     # allocs + first touch
        for _ in range(warmup):
            batched.fit_batch_device(ctx, opts, ds_d, y_d, b.offsets, 0.0, 1.1, out=out, sync=False)
        ctx.synchronize()
        barrier()
        if sampler:
            sampler.start()
        l0 = ctx.launch_count
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(lib_stream):
            ev0.record(lib_stream)
            for _ in range(steps):
                batched.fit_batch_device(ctx, opts, ds_d, y_d, b.offsets, 0.0, 1.1, out=out, sync=False)
            ev1.record(lib_stream)
        ctx.synchronize()
        barrier()
        ms = ev0.elapsed_time(ev1)
        return allmax(ms), ms, out, ctx.launch_count - l0

    # ---- headline: strong scaling (the same n_total series split over the ranks) ----
    strong = args.scaling != "weak"
    if strong:
        full_offsets = np.arange(n_total + 1, dtype=np.int64) * T_POINTS
        lo, hi = pdist.shard_bounds(full_offsets, world)[rank]
        b = synth.config3(n=n_total, lo=lo, hi=hi)
    else:
        lo = rank * n_total
        b = synth.config3(n=world * n_total, lo=lo, hi=lo + n_total)
    n_mine = b.n
    sampler = ClockSampler(local)
    ms_max, ms_mine, out, launches = timed_fit(b, args.steps, args.warmup, sampler)
    n_job = int(allsum(float(n_mine)))
    host = out.to_host()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, host)
    vc = ctx.last_fit_variant_counts()          # which fit-kernel variant the series of the last step ran on
    variants = {name: int(vc[i].sum()) for i, name in enumerate(("planes", "rotation", "week_table", "day_table")) if vc[i].sum()}
    st = host.meta_i32[:, 4]
    evals = host.meta_i32[:, 6].astype(np.float64)
    fitted_ok = int((st >= 0).sum())
    # per-rank tail: the straggler series (100 .. 3000 evaluations) bound a rank's step once its queue is empty
    rank_ms = [torch.zeros(1, dtype=torch.float64, device=dev) for _ in range(world)]
    if world > 1:
        dist.all_gather(rank_ms, torch.tensor([ms_mine], dtype=torch.float64, device=dev))
        rank_ms = [float(t.item()) for t in rank_ms]
    else:
        rank_ms = [ms_mine]

    # ---- e2e: pinned host buffers through pb200_fit_host, copies inside the timed region ----
    ds_h = torch.from_numpy(b.ds).pin_memory()
    y_h = torch.from_numpy(b.y).pin_memory()
    ds_np, y_np = ds_h.numpy(), y_h.numpy()
    batched.fit_batch_host(ctx, opts, ds_np, y_np, b.offsets, 0.0, 1.1)
    e2e_steps = max(1, min(args.steps, 3))
    barrier()
    t0 = time.perf_counter()
    for _ in range(e2e_steps):
        res_h = batched.fit_batch_host(ctx, opts, ds_np, y_np, b.offsets, 0.0, 1.1)
    torch.cuda.synchronize()
    e2e_s = allmax(time.perf_counter() - t0)
    clocks = sampler.stop()
    h2d = int(b.ds.nbytes + b.y.nbytes + b.offsets.nbytes + 2 * 4 * n_mine)
    d2h = int(res_h.params.nbytes + res_h.tchange.nbytes + res_h.meta_i32.nbytes + res_h.meta_i64.nbytes + res_h.meta_f64.nbytes)

    # ---- the other scaling mode, measured in the same run (N > 1 only) ----
    other = None
    if world > 1 and os.environ.get("PB200_BENCH_SKIP_OTHER") != "1":
        try:
            if strong:
                lo2 = rank * n_total
                b2 = synth.config3(n=world * n_total, lo=lo2, hi=lo2 + n_total)
            else:
                full_offsets = np.arange(n_total + 1, dtype=np.int64) * T_POINTS
                lo2, hi2 = pdist.shard_bounds(full_offsets, world)[rank]
                b2 = synth.config3(n=n_total, lo=lo2, hi=hi2)
            steps2 = max(2, min(args.steps, 5))
            ms2, _, _, _ = timed_fit(b2, steps2, 1)
            n2 = int(allsum(float(b2.n)))
            other = {"scaling": "weak" if strong else "strong", "value": n2 * steps2 / (ms2 * 1e-3), "unit": UNIT,
                     "global_series": n2, "series_per_gpu": b2.n, "ms_per_step": ms2 / steps2, "steps": steps2}
            del b2
        except Exception as exc:
            other = {"error": repr(exc)}

    # ---- secondary: BASELINE.json configs #2, #4, #5 (driver-run numbers next to the headline) ----
    sec = {}
    if os.environ.get("PB200_BENCH_SKIP_SECONDARY") != "1":
        sec = _secondary(args, ctx, lib_stream, dev, rank, world, out, b, barrier, allmax, allsum)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return 0
    value = n_job * args.steps / (ms_max * 1e-3)
    peak, peak_src = _peaks()
    per_launch_s = ms_max * 1e-3 / args.steps
    achieved = n_mine * ALG_BYTES_PER_SERIES / per_launch_s / 1e9
    digest = _build_digest()
    gflops = n_mine * float(evals.mean()) * FLOPS_PER_EVAL / per_launch_s / 1e9
    cores = usable_cores()
    cpu = cpu_baseline(int(os.environ.get("PB200_CPU_SAMPLE", str(max(256, 16 * cores["usable"])))), cores) if world == 1 else None
    mean_ms = float(np.mean(rank_ms))
    l2_mb = torch.cuda.get_device_properties(dev).L2_cache_size / 2**20
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_max / args.steps, "higher_is_better": True, "scaling": "strong" if strong else "weak",
        "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": {"workload": WORKLOAD, "series_per_gpu": n_mine, "points_per_series": T_POINTS,
                   "global_series": n_job, "parallelism": f"series-sharded x{world} (contiguous row-balanced ranges), no data-path collective",
                   "l2": f"inputs {(b.ds.nbytes + b.y.nbytes) / 1e6:.0f} MB per GPU vs {l2_mb:.0f} MB L2; every step re-reads them "
                         f"from HBM (L2 serves the per-series workspace of the resident series, as much of it as fits)",
                   "mean_objective_evals_per_series": float(evals.mean()), "max_objective_evals": int(evals.max()),
                   "series_with_model": fitted_ok, "fit_kernel_variants": variants, "build_digest": digest},
        "e2e": {"value": n_job * e2e_steps / e2e_s, "unit": UNIT, "h2d_bytes_per_step": h2d,
                "d2h_bytes_per_step": d2h, "api": "pb200_fit_host (C ABI, pinned host buffers)", "steps": e2e_steps},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "rank_tail": {"ms_per_step_by_rank": [m / args.steps for m in rank_ms], "max_over_mean": (max(rank_ms) / mean_ms) if mean_ms else None,
                      "limiter": "no collective on the data path: a rank's step ends with its slowest series "
                                 "(max evaluations per series x per-evaluation latency), which does not shrink with the shard"},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "peak_source": peak_src,
                     "kernel": _kernel_name(variants, group_of(n_mine)),
                     "algorithmic_bytes_per_launch": n_mine * ALG_BYTES_PER_SERIES,
                     "note": "ds/y are read from HBM once per series; the ~700 objective evaluations stream the "
                             "series' y (8 B/point) from the per-series workspace: the kernel is FP64-issue / latency bound, "
                             "not HBM bound; see fp64 below (model flops of the plain T x K formulation -- the day-table "
                             "variant executes fewer)",
                     "fp64": {"achieved_gflops": gflops, "peak_gflops": FP64_PEAK_GFLOPS, "frac": gflops / FP64_PEAK_GFLOPS,
                              "flops_per_eval_model": FLOPS_PER_EVAL}},
    }
    if other is not None:
        line[other.get("scaling", "other")] = other
    line["secondary"] = sec
    if cpu is not None:
        line["cpu_baseline"] = cpu
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


def _secondary(args, ctx, lib_stream, dev, rank, world, out, b, barrier, allmax, allsum):
    """Driver-run numbers for the other BASELINE.json configs.  Every entry: resident inputs, CUDA events on the
    library stream, max over ranks; sizes are the configs' own (strong split over the ranks)."""
    import torch
    from time_series_spark_b200 import batched, synth
    from time_series_spark_b200 import dist as pdist
    sec = {}

    def timed(fn, reps):
        fn()
        ctx.synchronize()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(lib_stream):
            e0.record(lib_stream)
            for _ in range(reps):
                fn()
            e1.record(lib_stream)
        ctx.synchronize()
        barrier()
        return allmax(e0.elapsed_time(e1)) * 1e-3 / reps

    # ---- config #2: 1k x 365 daily, linear growth + yearly (K = 26), one GPU's worth of work split over the ranks ----
    try:
        n2 = 1000
        offs = np.arange(n2 + 1, dtype=np.int64) * 365
        lo, hi = pdist.shard_bounds(offs, world)[rank]
        b2 = synth.config2(n=n2, lo=lo, hi=hi)
        o2 = batched.make_options(growth="linear", yearly_seasonality=True)
        ds2, y2 = torch.from_numpy(b2.ds).to(dev), torch.from_numpy(b2.y).to(dev)
        out2 = batched.fit_batch_device(ctx, o2, ds2, y2, b2.offsets, 0.0, 1.1)
        t2 = timed(lambda: batched.fit_batch_device(ctx, o2, ds2, y2, b2.offsets, 0.0, 1.1, out=out2, sync=False), 5)
        ok2 = int(allsum(float((out2.meta_i32[:, 4] >= 0).sum().item())))
        sec["config2"] = {"workload": "1k synthetic series x 365 daily pts, linear growth + yearly + weekly seasonality (K = 26)",
                          "series_per_s": n2 / t2, "ms_per_step": t2 * 1e3, "series_with_model": ok2, "n_gpus": world}
    except Exception as exc:
        sec["config2"] = {"error": repr(exc)}

    # ---- config #4: 500k ragged short series (48..96 points), no seasonality ----
    try:
        n4 = int(os.environ.get("PB200_BENCH_C4_SERIES", "500000"))
        per = (n4 + world - 1) // world
        lo, hi = min(rank * per, n4), min((rank + 1) * per, n4)
        b4 = synth.config4(n=n4, lo=lo, hi=hi)
        ds4, y4 = torch.from_numpy(b4.ds).to(dev), torch.from_numpy(b4.y).to(dev)
        out4 = batched.fit_batch_device(ctx, batched.make_options(), ds4, y4, b4.offsets, 0.0, 1.1)
        o4 = batched.make_options()
        t4 = timed(lambda: batched.fit_batch_device(ctx, o4, ds4, y4, b4.offsets, 0.0, 1.1, out=out4, sync=False), 2)
        st4 = out4.meta_i32[:, 4]
        sec["config4"] = {"workload": "500k ragged series x 48..96 15-min pts (span < 2 d: no seasonality, K = 1)",
                          "series_per_s": n4 / t4, "ms_per_step": t4 * 1e3, "n_gpus": world, "global_series": n4,
                          "series_with_model": int(allsum(float((st4 >= 0).sum().item()))),
                          "newton_retries": int(allsum(float((st4 == 60).sum().item()))),
                          "dropped": int(allsum(float((st4 < 0).sum().item())))}
        del ds4, y4, out4, b4
    except Exception as exc:
        sec["config4"] = {"error": repr(exc)}

    # ---- config #5: scorer, 100k fitted models x 672 15-min periods (include_history=False), strong split ----
    try:
        H = 672
        n5 = int(os.environ.get("PB200_BENCH_SCORER_MODELS", "100000"))
        per = (n5 + world - 1) // world
        n_det = min(per, n5 - min(rank * per, n5))
        # models: this rank's fitted config-#3 models, tiled up to its share of the 100k
        reps = (n_det + out.n - 1) // max(out.n, 1)
        idx = torch.arange(n_det, device=dev) % out.n
        sub = batched.FittedBatch(out.params[idx].contiguous(), out.tchange[idx].contiguous(), out.meta_i32[idx].contiguous(),
                                  out.meta_i64[idx].contiguous(), out.meta_f64[idx].contiguous(), out.smax, out.kmax)
        last_np = b.ds[b.offsets[1:] - 1]
        last = torch.from_numpy(np.ascontiguousarray(last_np)).to(dev)[idx]
        fut = (last[:, None] + (15 * 60 * 10**9) * torch.arange(1, H + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
        fl_d = torch.zeros(n_det, dtype=torch.float64, device=dev)
        cap_d = sub.meta_f64[:, 2].float().double().contiguous()
        o_det = batched.make_options(uncertainty_samples=0)
        o_mc = batched.make_options(uncertainty_samples=1000)
        buf_det = batched.predict_batch_device(ctx, o_det, sub, fut, fl_d, cap_d, intervals=False)
        t_det = timed(lambda: batched.predict_batch_device(ctx, o_det, sub, fut, fl_d, cap_d, intervals=False, sync=False,
                                                           out=buf_det), 5)
        n_mc = min(n_det, int(os.environ.get("PB200_BENCH_MC_MODELS", str(n_det))))
        sub_mc = batched.FittedBatch(sub.params[:n_mc], sub.tchange[:n_mc], sub.meta_i32[:n_mc], sub.meta_i64[:n_mc],
                                     sub.meta_f64[:n_mc], sub.smax, sub.kmax)
        fut_mc, fl_mc, cap_mc = fut[:n_mc].contiguous(), fl_d[:n_mc].contiguous(), cap_d[:n_mc].contiguous()
        buf_mc = batched.predict_batch_device(ctx, o_mc, sub_mc, fut_mc, fl_mc, cap_mc, seed=1, intervals=True)
        t_mc = timed(lambda: batched.predict_batch_device(ctx, o_mc, sub_mc, fut_mc, fl_mc, cap_mc, seed=1, intervals=True,
                                                          sync=False, out=buf_mc), 1)
        n_mc_job = int(allsum(float(n_mc)))
        ent = {"workload": "scorer: 100k fitted models x 672 15-min periods, include_history=False",
               "models": n5, "horizon": H, "n_gpus": world,
               "forecast_points_per_s": n5 * H / t_det, "deterministic_ms": t_det * 1e3,
               "with_1000_draw_intervals_points_per_s": n_mc_job * H / t_mc, "mc_models": n_mc_job, "mc_ms": t_mc * 1e3,
               "note": "deterministic yhat + int epilogue is what the reference's scorer keeps (prophet_scorer.py:86); the "
                       "1000-draw intervals are computed by Prophet.predict and dropped there"}
        if world > 1:
            # the one collective north_star names: gather of the final forecast frame (series_id, dim_id, ds, yhat) to rank 0
            import torch.distributed as dist
            yint = buf_det.yhat_int.reshape(-1)
            cols = [yint, fut.reshape(-1)]
            nmax = int(allmax(float(yint.numel())))
            staged = []
            for c in cols:                                   # receive buffers allocated once, like a job that scores every day
                pad = torch.zeros(nmax, dtype=c.dtype, device=dev)
                pad[:c.numel()] = c
                staged.append((pad, [torch.empty_like(pad) for _ in range(world)] if rank == 0 else None))

            def gather_frame():
                for pad, bufs in staged:
                    dist.gather(pad, bufs, dst=0)

            gather_frame()                                   # warm-up: NCCL sets up its peer connections on first use
            reps = 3
            torch.cuda.synchronize()
            barrier()
            g0 = time.perf_counter()
            for _ in range(reps):
                gather_frame()
            torch.cuda.synchronize()
            barrier()
            gs = allmax(time.perf_counter() - g0) / reps
            got = sum(int(x.numel()) * x.element_size() for _, bufs in staged for x in (bufs or []))
            remote = got * (world - 1) // world
            ent["nccl_gather_to_rank0"] = {"seconds": gs, "bytes": got, "bytes_from_peers": remote,
                                           "GB_per_s_from_peers": remote / gs / 1e9 if gs > 0 else None, "reps": reps,
                                           "columns": "yhat int32 + ds int64 (ids are implied by rank order)"}
            del staged
            ent["forecast_points_per_s_incl_gather"] = n5 * H / (t_det + gs)
        sec["config5"] = ent
    except Exception as exc:      # the headline must not depend on the secondary metrics
        sec["config5"] = {"error": repr(exc)}
    return sec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--scaling", default="strong", choices=["strong", "weak"],
                    help="what `value` means at N > 1: the same 50k series split over the ranks (north_star), or 50k per rank")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the fitted-model arrays of the last timed step (rank 0) to DIR/<name>.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup
    if args.impl == "reference":
        return run_reference(args)
    return run_gpu(args)


if __name__ == "__main__":
    sys.exit(main())
