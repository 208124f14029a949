"""Generates the committed golden fixtures from a checkout of the reference repository:

    python tests/golden/make_golden.py <path to mageky/time-series-spark>

  model_input_751.npz      the reference's only data fixture
                           (tests/fixtures/model-input/series_id=751/sample-model-input.csv,
                           config #1 of BASELINE.json) as three arrays; tests rebuild the
                           header-less hive-partitioned CSV from it byte for byte.
  fixture_751_oracle.npz   outputs of oracle/prophet_oracle.py on its two series: scaling meta,
                           initial point, objective+gradient at the initial point and at three
                           seeded random points, the Stan-L-BFGS optimum, in-sample yhat and the
                           40-step 15-min forecast the reference's scorer test asks for
                           (tests/unit/prophet_scorer_test.py:37-39).

The reference pins NO numerical value (its tests assert counts and column names only) and
fbprophet/pystan cannot be installed here, so these vectors pin the ORACLE (a restatement of
the published algorithm), not fbprophet itself: parity stays "unpinned" in that sense.
"""
import os
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import prophet_oracle as po  # noqa: E402

FIXTURE = os.path.join("tests", "fixtures", "model-input", "series_id=751", "sample-model-input.csv")


def main():
    src = os.path.join(sys.argv[1], FIXTURE)
    raw = open(src, "rb").read()
    df = pd.read_csv(src, header=None, names=["dim_id", "ds", "y"], parse_dates=["ds"])
    ds_ns = df["ds"].values.astype("datetime64[ns]").astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "model_input_751.npz"), dim_id=df["dim_id"].values.astype(np.int32),
                        ds_ns=ds_ns, y=df["y"].values.astype(np.int32), n_bytes=np.int64(len(raw)),
                        trailing_newline=np.bool_(raw.endswith(b"\n")))
    out = {}
    opts = po.ProphetOptions()
    for dim in (91, 155):
        g = df[df["dim_id"] == dim]
        d = g["ds"].values.astype("datetime64[ns]").astype(np.int64)
        y = g["y"].values.astype(np.float64)
        cap = y.max() * 1.1                                   # prophet_modeler.py:59
        p = po.prepare(d, y, 0.0, cap, opts)
        th0 = po.initial_theta(p)
        rng = np.random.RandomState(751 + dim)
        pts = [th0] + [th0 + 0.05 * rng.randn(th0.size) for _ in range(3)]
        fs, gs = [], []
        for th in pts:
            err, f, gr = po.neg_logp_grad(th, p)
            assert err == 0
            fs.append(f)
            gs.append(gr)
        fr = po.fit(d, y, 0.0, None, opts)
        fut = po.make_future_ns(fr.last_ds_ns, 40, 15 * 60 * 10**9)
        cap32 = float(np.float32(cap))                        # prophet_scorer.py:47 reads FloatType
        pred = po.predict(fr, fut, 0.0, cap32, opts)
        insample = po.predict(fr, p.ds_sorted, 0.0, cap, opts)
        k = f"d{dim}_"
        out.update({k + "y_scale": p.y_scale, k + "cap": cap, k + "cap32": cap32, k + "T": p.T, k + "S": p.S,
                    k + "K": p.K, k + "t_change": p.t_change, k + "theta0": th0, k + "points": np.array(pts),
                    k + "f": np.array(fs), k + "g": np.array(gs), k + "theta_opt": fr.theta,
                    k + "neg_logp": fr.neg_logp, k + "iters": fr.iters, k + "n_evals": fr.n_evals, k + "ret": fr.ret,
                    k + "k": fr.k, k + "m": fr.m, k + "delta": fr.delta, k + "beta": fr.beta,
                    k + "sigma_obs": fr.sigma_obs, k + "future_ns": fut, k + "yhat_future": pred["yhat"],
                    k + "yhat_int": po.scorer_epilogue(pred["yhat"], 0.0), k + "yhat_insample": insample["yhat"],
                    k + "trend_future": pred["trend"]})
    np.savez_compressed(os.path.join(HERE, "fixture_751_oracle.npz"), **out)
    print("wrote", sorted(os.listdir(HERE)))


if __name__ == "__main__":
    main()
