"""Dev helper: config-3 (or, with AB_CONFIG=c4, config-4) fit under several context environments in one process (same inputs), e.g.
    python tools/ab_env.py 50000 3 g8: g16:PB200_GROUP=16 tab32:PB200_GROUP=0 notab:PB200_NO_TAB=1
prints timings, the kernel-variant counts and how the results compare with the first configuration."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from time_series_spark_b200 import synth, batched, _lib as L
n = int(sys.argv[1]) if len(sys.argv) > 1 else 50000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
specs = sys.argv[3:] or ["base:"]
KNOWN = ("PB200_NO_TAB", "PB200_GROUP", "PB200_GRP_PAD", "PB200_PLAIN_GROUP", "PB200_LC0_MAX")
cfg = os.environ.get("AB_CONFIG", "c3")          # c3 (50k x 1440 shape) or c4 (short ragged series, no seasonality)
b = synth.config4(n=n) if cfg == "c4" else synth.config3(n=n); opts = batched.make_options()
mask = 0 if cfg == "c4" else 6
if os.environ.get("AB_STEP_MIN"):                       # same values on another regular grid (e.g. 30 min: table period 48)
    T0 = int(b.offsets[1] - b.offsets[0])
    b.ds[:] = np.tile(b.ds[0] + int(os.environ["AB_STEP_MIN"]) * 60 * 10**9 * np.arange(T0, dtype=np.int64), n)
ds = torch.from_numpy(b.ds).cuda(); y = torch.from_numpy(b.y).cuda()
res = {}
for spec in specs:
    name, _, kv = spec.partition(":")
    for k in KNOWN:
        os.environ.pop(k, None)
    for item in filter(None, kv.split(",")):
        k, _, v = item.partition("=")
        os.environ[k] = v
    ctx = L.Context(0)
    out = None
    for r in range(reps):
        torch.cuda.synchronize(); t = time.time()
        out = batched.fit_batch_device(ctx, opts, ds, y, b.offsets, 0.0, 1.1, out=out)
        dt = time.time() - t
        print(f"{name} n={n} rep{r}: {dt*1e3:.2f} ms  {n/dt:.0f} series/s, evals/series {out.meta_i32[:,6].double().mean().item():.1f}", flush=True)
    print(name, "variant counts (planes, rotation, week table, day table):", ctx.last_fit_variant_counts()[:, mask].tolist())
    res[name] = (out.params.cpu().numpy().copy(), out.meta_f64[:, 3].cpu().numpy().copy(), out.meta_i32[:, 4].cpu().numpy().copy())
    ctx.close()
first = specs[0].partition(":")[0]
p0, f0, s0 = res[first]
for name, (p, f, s) in res.items():
    if name == first:
        continue
    rel = np.abs(f - f0) / np.abs(f0)
    print(f"{name} vs {first}: params bit-identical on {int((p == p0).all(axis=1).sum())}/{n} series; objective at optimum "
          f"median rel {np.median(rel):.2e} max {rel.max():.2e}; status equal on {int((s == s0).sum())}/{n}")
