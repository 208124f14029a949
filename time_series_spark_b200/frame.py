"""Minimal DataFrame stand-in over a pyarrow.Table.

The reference drives its per-series operators through a handful of Spark DataFrame calls
(``groupby(...).apply(udf)`` src/jobs/prophet_modeler.py:139-141, src/jobs/prophet_scorer.py:159-161;
``count``/``columns``/``filter``/``select(...).distinct()``/``collect`` in tests/unit/*.py).
There is no Spark (no JVM) on the GPU path, so this class offers exactly that subset on an
Arrow table; ``groupby(keys).apply(op)`` hands ALL groups to the batched operator at once
instead of one pandas frame per Python worker.
"""
from __future__ import annotations

import re
from typing import List, Sequence

import pyarrow as pa
import pyarrow.compute as pc


class Frame:
    def __init__(self, table: pa.Table):
        self.table = table

    # -- Spark-like surface ------------------------------------------------------------
    @property
    def columns(self) -> List[str]:
        return list(self.table.column_names)

    def count(self) -> int:
        return self.table.num_rows

    def select(self, *cols: str) -> "Frame":
        return Frame(self.table.select(list(cols)))

    def distinct(self) -> "Frame":
        if self.table.num_rows == 0:
            return self
        return Frame(self.table.group_by(self.table.column_names).aggregate([]))

    def filter(self, expr: str) -> "Frame":
        """Conjunctions of ``col = <int>`` (all the reference's tests use)."""
        mask = None
        for clause in re.split(r"\s+and\s+", expr.strip(), flags=re.IGNORECASE):
            m = re.fullmatch(r"\s*(\w+)\s*=\s*(-?\d+)\s*", clause)
            if not m:
                raise ValueError(f"unsupported filter clause: {clause!r}")
            c = pc.equal(self.table[m.group(1)], int(m.group(2)))
            mask = c if mask is None else pc.and_(mask, c)
        return Frame(self.table.filter(mask))

    def withColumnRenamed(self, old: str, new: str) -> "Frame":
        return Frame(self.table.rename_columns([new if c == old else c for c in self.table.column_names]))

    def collect(self) -> list:
        cols = [self.table[c].to_pylist() for c in self.table.column_names]
        return [tuple(r) for r in zip(*cols)]

    def groupby(self, *keys: str) -> "GroupedFrame":
        return GroupedFrame(self, list(keys))

    def toPandas(self):
        return self.table.to_pandas()

    def __repr__(self):
        return f"Frame({self.table.schema}, rows={self.table.num_rows})"


class GroupedFrame:
    def __init__(self, frame: Frame, keys: Sequence[str]):
        self.frame, self.keys = frame, list(keys)

    def apply(self, op) -> Frame:
        """``op`` is a batched grouped-map operator (see jobs.prophet_modeler.model_time_series)."""
        if not hasattr(op, "apply_batched"):
            raise TypeError("groupby().apply() needs a batched operator with .apply_batched(table, keys)")
        return Frame(op.apply_batched(self.frame.table, self.keys))
