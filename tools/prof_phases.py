"""Dev helper: where the grouped fit kernel's warps spend their cycles, on config-3 series resident in HBM.

    PB200_VARIANT=clk PB200_NVCC_EXTRA="-DPB200_PHASE_CLOCKS" python -m time_series_spark_b200.build
    PB200_VARIANT=clk PB200_GRP_PAD=24576 python tools/prof_phases.py [n_series] [reps]

Times `reps` fits (CUDA events, after one warm-up fit) and samples nvidia-smi (read-only queries: memory / SM utilisation,
SM clock, power) while they run.  With a build that has the phase clocks (-DPB200_PHASE_CLOCKS), it also prints each
phase's share of the kernel's warp cycles (clock64 per warp, summed over the warps; pb200::grp::PhaseClock), and the
point pass's step loops in cycles per two-point step next to the rest of the pass per evaluation round.  The clocks
add instructions to the kernel: compare step times between builds without them.  PB200_GRP_PAD pads each CTA's shared
memory so that fewer CTAs fit an SM (24576: 4 per SM for G = 8).
"""
import ctypes as C
import json
import os
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_series_spark_b200 import _lib as L, batched, synth  # noqa: E402

PHASES = ["total", "fetch", "eval_setup", "point_pass", "eval_finalize", "ls_step", "post_accept", "ls_begin", "write_record",
          "point_pass.cp_async_wait", "post_accept.history_wait", "drain", "point_pass.step_loops", "rounds", "warps",
          "point_pass.steps", "post_accept.calls", "accepts"]
EXCLUSIVE = PHASES[1:9]
COUNTS = ("rounds", "warps", "point_pass.steps", "post_accept.calls", "accepts")


class Smi:
    Q = "utilization.gpu,utilization.memory,clocks.sm,power.draw"

    def __init__(self):
        self.rows, self.p = [], None

    def __enter__(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", "--id=0", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                      stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=lambda: [self.rows.append(ln) for ln in self.p.stdout], daemon=True)
            self.t.start()
        except OSError:
            self.p = None
        return self

    def __exit__(self, *exc):
        if self.p:
            self.p.terminate()
            self.p.wait(timeout=5)

    def summary(self):
        v = []
        for ln in self.rows:
            try:
                v.append([float(x) for x in ln.split(",")])
            except ValueError:
                pass
        if not v:
            return None
        a = np.array(v)
        return {k: float(np.median(a[:, i])) for i, k in enumerate(("util_gpu_pct", "util_mem_pct", "sm_mhz", "power_w"))} | {"samples": len(v)}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    lib = L.load()
    read = getattr(lib, "pb200_dev_phase_clocks", None)
    if read is not None:
        read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
        read.restype = C.c_int
    ctx = L.Context(0)
    b = synth.config3(n=n)
    opts = batched.make_options()
    ds, y = torch.from_numpy(b.ds).cuda(), torch.from_numpy(b.y).cuda()
    out = batched.fit_batch_device(ctx, opts, ds, y, b.offsets, 0.0, 1.1)
    ctx.synchronize()
    buf = (C.c_ulonglong * len(PHASES))()
    if read is not None:
        read(buf, len(PHASES), 1)
    stream = torch.cuda.ExternalStream(ctx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with Smi() as smi:
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(reps):
                batched.fit_batch_device(ctx, opts, ds, y, b.offsets, 0.0, 1.1, out=out, sync=False)
            e1.record(stream)
        ctx.synchronize()
    ms = e0.elapsed_time(e1) / reps
    res = {"variant": os.environ.get("PB200_VARIANT", ""), "grp_pad": int(os.environ.get("PB200_GRP_PAD", "0")),
           "l2_keep_pct": os.environ.get("PB200_L2_KEEP_PCT"), "n": n, "reps": reps, "ms_per_step": ms,
           "series_per_s": n / ms * 1e3, "evals_mean": float(out.meta_i32[:, 6].double().mean().item()), "smi": smi.summary()}
    if read is not None:
        read(buf, len(PHASES), 0)
        c = dict(zip(PHASES, (int(x) for x in buf)))
        tot = max(c["total"], 1)
        res["warp_cycle_share"] = {k: round(c[k] / tot, 4) for k in PHASES[1:] if k not in COUNTS}
        res["warp_cycle_share"]["(exclusive phases sum)"] = round(sum(c[k] for k in EXCLUSIVE) / tot, 4)
        res["cycles_per_round_per_warp"] = tot / max(c["rounds"], 1)
        res["wait_cycles_per_round_per_warp"] = c["point_pass.cp_async_wait"] / max(c["rounds"], 1)
        # the point pass split into its step loops (per two-point step of a warp) and the rest: seasonal table, bins'
        # gradient and the reductions (per evaluation round)
        res["step_loop_cycles_per_step"] = c["point_pass.step_loops"] / max(c["point_pass.steps"], 1)
        res["steps_per_round"] = c["point_pass.steps"] / max(c["rounds"], 1)
        res["pass_rest_cycles_per_round"] = (c["point_pass"] - c["point_pass.step_loops"]) / max(c["rounds"], 1)
        # warp cycles per evaluation round of every phase (shares alone do not compare builds routine by routine), and
        # g_post_accept per call: a warp's call serves every group of it whose line search was accepted that round
        res["cycles_per_round"] = {k: round(c[k] / max(c["rounds"], 1), 1) for k in PHASES[1:13] if k not in COUNTS}
        res["post_accept_cycles_per_call"] = c["post_accept"] / max(c["post_accept.calls"], 1)
        res["post_accept_calls_per_round"] = c["post_accept.calls"] / max(c["rounds"], 1)
        res["accepts_per_call"] = c["accepts"] / max(c["post_accept.calls"], 1)
        # the grid is SMs x the occupancy query's CTAs per SM when the batch fills it
        res["ctas_per_sm"] = c["warps"] / reps / torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps(res))


if __name__ == "__main__":
    main()
