"""``python -m time_series_spark_b200.backtest_driver <config.yaml>``: backtest every series of the modeler's input
(jobs/prophet_backtest.py; example config/example_backtest_app_config.yaml)."""
import sys

import yaml

from .jobs.prophet_backtest import ProphetBacktester

if __name__ == "__main__":
    if len(sys.argv) != 2:
        print("arg1 must be the config YAML")
        sys.exit(1)
    with open(sys.argv[1]) as file:
        config = yaml.safe_load(file)
    print(f"config: {config}")
    ProphetBacktester.run(None, config)
