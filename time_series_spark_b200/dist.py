"""Multi-GPU sharding: one process per GPU (torchrun), series partitioned across ranks.

The reference parallelises over (series_id, dim_id) groups only -- one Spark task per group
after a hash shuffle (src/jobs/prophet_modeler.py:139-141, src/jobs/prophet_scorer.py:159-161,
README.md:119-130).  Groups never interact, so the GPU equivalent is a contiguous range
shard of the sorted group list balanced by ROWS (not by group count: ragged batches), no
collective during fit/predict, and -- optionally -- one gather of the final forecast frame to
rank 0 over NCCL (the only collective; otherwise each rank writes its own part file exactly
like Spark's output directory).
"""
from __future__ import annotations

import os
from typing import List, Tuple

import numpy as np


def world() -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from the torchrun environment (1 process if unset)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def usable_cores() -> dict:
    """Host threads this process may actually use: CPU affinity intersected with the cgroup CPU quota --
    NOT os.cpu_count(), which reports the machine (a GPU lease that owns 16 of a box's 128 cores)."""
    logical = os.cpu_count() or 1
    try:
        aff = len(os.sched_getaffinity(0))
    except Exception:
        aff = logical
    quota = None
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    quota = float(txt[0]) / float(txt[1])
            else:
                q = float(txt[0])
                if q > 0:
                    quota = q / float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            break
        except Exception:
            continue
    use = aff if quota is None else max(1, min(aff, int(quota + 0.5)))
    return {"usable": use, "logical": logical, "affinity": aff, "cgroup_quota": quota}


def size_host_pools() -> int:
    """pyarrow's CPU / IO pools default to os.cpu_count() threads PER PROCESS; under a cgroup quota, and with one
    process per GPU, that oversubscribes the lease several times over and the CSV parse of every rank slows down
    (2-rank modeler run: read 1.29 s against 0.69 s for ONE rank reading twice the rows).  Give this rank its share
    of the threads the lease really owns.  Returns the thread count set."""
    import pyarrow as pa
    local_ws = int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1")))
    n = max(1, usable_cores()["usable"] // max(local_ws, 1))
    pa.set_cpu_count(n)
    pa.set_io_thread_count(max(2, min(8, n)))
    return n


def shard_bounds(offsets: np.ndarray, world_size: int) -> List[Tuple[int, int]]:
    """Contiguous group ranges [lo, hi) per rank with balanced row counts.

    Rank r gets the groups whose row-midpoint falls in the r-th equal slice of the rows, so
    every group goes to exactly one rank and empty shards are possible only when there are
    fewer groups than ranks."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = offsets.size - 1
    if world_size <= 1 or n == 0:
        return [(0, n)] + [(n, n)] * (max(world_size, 1) - 1)
    total = int(offsets[-1])
    mid = (offsets[:-1] + offsets[1:]) / 2.0
    if total == 0:
        cuts = np.linspace(0, n, world_size + 1).astype(np.int64)
    else:
        edges = total * np.arange(1, world_size, dtype=np.float64) / world_size
        cuts = np.concatenate(([0], np.searchsorted(mid, edges, side="left"), [n])).astype(np.int64)
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(world_size)]


def init_process_group(backend: str | None = None):
    """Initialises torch.distributed from the torchrun environment (nccl on GPU, gloo on CPU)."""
    import torch
    import torch.distributed as dist
    rank, ws, local = world()
    if ws <= 1 or dist.is_initialized():
        return
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    if backend == "nccl":
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        dist.init_process_group(backend)


def gather_rows(arrays: List[np.ndarray], dst: int = 0, device=None) -> List[np.ndarray] | None:
    """Gathers row-aligned arrays (same length per rank, lengths differ across ranks) to ``dst``
    in rank order: the final-forecast-frame gather.  Uses the initialised process group (NCCL
    moves GPU tensors over NVLink; gloo moves CPU tensors).  Returns None on other ranks."""
    import torch
    import torch.distributed as dist
    rank, ws, local = world()
    if ws <= 1 or not dist.is_initialized():
        return list(arrays)
    backend = dist.get_backend()
    dev = torch.device("cuda", local) if backend == "nccl" else torch.device("cpu")
    n_local = int(arrays[0].shape[0]) if arrays else 0
    counts = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(ws)]
    dist.all_gather(counts, torch.tensor([n_local], dtype=torch.int64, device=dev))
    counts = [int(c.item()) for c in counts]
    nmax = max(counts) if counts else 0
    out = []
    for a in arrays:
        a = np.ascontiguousarray(a)
        t = torch.from_numpy(a.view(np.int64) if a.dtype.kind == "M" else a)
        pad = torch.zeros((nmax,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        pad[:n_local] = t.to(dev)
        bufs = [torch.empty_like(pad) for _ in range(ws)] if rank == dst else None
        dist.gather(pad, bufs, dst=dst)
        if rank == dst:
            parts = [b[:c].cpu().numpy() for b, c in zip(bufs, counts)]
            out.append(np.concatenate(parts, axis=0))
    return out if rank == dst else None


def barrier():
    """Barrier over the initialised process group (no-op for a single process)."""
    import torch.distributed as dist
    if world()[1] > 1 and dist.is_initialized():
        dist.barrier()


def prepare_output_dir(path: str):
    """mode='overwrite' for a directory of per-rank part files: rank 0 clears it, everybody waits."""
    import shutil
    rank, ws, _ = world()
    if rank == 0:
        if os.path.isdir(path):
            shutil.rmtree(path)
        os.makedirs(path, exist_ok=True)
    barrier()
    os.makedirs(path, exist_ok=True)
