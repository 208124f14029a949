"""``python -m time_series_spark_b200.tuner_driver <config.yaml>``: tune every series' prior scales and fit its model
(jobs/prophet_tuner.py; example config/example_tuner_app_config.yaml)."""
import sys

import yaml

from .jobs.prophet_tuner import ProphetTuner

if __name__ == "__main__":
    if len(sys.argv) != 2:
        print("arg1 must be the config YAML")
        sys.exit(1)
    with open(sys.argv[1]) as file:
        config = yaml.safe_load(file)
    print(f"config: {config}")
    ProphetTuner.run(None, config)
