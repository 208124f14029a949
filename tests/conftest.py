import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def pytest_sessionstart(session):
    """The CUDA library is a build artefact (git-ignored): compile it in-tree if this checkout has none
    (nvcc cross-compiles without a GPU; a no-op when the sources are unchanged)."""
    from time_series_spark_b200 import build as _build
    try:
        _build.build()
    except Exception as exc:                      # keep collecting: the tests that need it will say why
        if not os.path.exists(_build.LIB):
            print(f"[conftest] libprophet_b200.so is missing and could not be built: {exc}")


@pytest.fixture(scope="session")
def golden_input():
    return np.load(os.path.join(GOLDEN, "model_input_751.npz"))


@pytest.fixture(scope="session")
def golden_oracle():
    return np.load(os.path.join(GOLDEN, "fixture_751_oracle.npz"))


def write_model_input(dirpath, gi) -> str:
    """Rebuilds the reference's fixture tree tests/fixtures/model-input/series_id=751/
    sample-model-input.csv (header-less ``dim_id,timestamp,quantity``) from the golden arrays."""
    d = os.path.join(dirpath, "model-input", "series_id=751")
    os.makedirs(d, exist_ok=True)
    ts = gi["ds_ns"].astype("datetime64[ns]").astype("datetime64[s]")
    lines = [f"{int(a)},{str(t).replace('T', ' ')},{int(q)}" for a, t, q in zip(gi["dim_id"], ts, gi["y"])]
    text = "\n".join(lines) + ("\n" if bool(gi["trailing_newline"]) else "")
    with open(os.path.join(d, "sample-model-input.csv"), "w") as f:
        f.write(text)
    return os.path.join(dirpath, "model-input")


@pytest.fixture()
def model_input_dir(tmp_path, golden_input):
    return write_model_input(str(tmp_path), golden_input)


@pytest.fixture(scope="session")
def gpu_ctx():
    from time_series_spark_b200 import _lib as L
    return L.Context(0)
