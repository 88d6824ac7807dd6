"""Multi-GPU sharding for batched image streams (SURVEY §8(e)).

The reference has no distributed layer at all (§2: "NONE exist").  The path shards embarrassingly: a
unit is one image / camera frame, the batch is split contiguously across ranks, every rank runs the same
single-GPU kernels on its shard, and there is NO per-frame communication.  The only collectives are
  * ONE broadcast (rank 0 → all, NCCL over NVLink/NVSwitch) of the small parameter block an op instance
    needs — homography / affine (9 / 6 f32), normalisation mean & inv_std (6 f32), filter taps — at plan
    creation, never per frame;
  * optionally ONE all-reduce(SUM) of six integers for a *global* `std_mean` over a sharded batch (the
    per-shard sums are exact integers, so the global statistic is order-independent and exact).

One process per GPU (`torch.distributed`, backend "nccl"; "gloo" on CPU-only hosts for the tests).
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import torch
import torch.distributed as td


@dataclass(frozen=True)
class Shard:
    rank: int
    world_size: int
    start: int
    stop: int

    @property
    def count(self) -> int:
        return self.stop - self.start


def shard_range(n_items: int, rank: int, world_size: int) -> Shard:
    """Contiguous split of `n_items` units; the first `n_items % world_size` ranks take one extra."""
    if world_size <= 0 or not (0 <= rank < world_size):
        raise ValueError(f"bad rank/world_size {rank}/{world_size}")
    base, rem = divmod(n_items, world_size)
    start = rank * base + min(rank, rem)
    stop = start + base + (1 if rank < rem else 0)
    return Shard(rank, world_size, start, stop)


def is_initialized() -> bool:
    return td.is_available() and td.is_initialized()


def rank() -> int:
    return td.get_rank() if is_initialized() else 0


def world_size() -> int:
    return td.get_world_size() if is_initialized() else 1


_numa_state: dict = {}


def gpu_cpu_affinity(index: int) -> list[int]:
    """CPUs local to GPU `index` (NVML's ideal affinity = the cores of the NUMA node its PCIe root hangs off)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = [64 * w + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1]
        return [c for c in cpus if c < ncpu]
    except Exception:
        return []


def _node_of_cpu(cpu: int) -> int | None:
    try:
        for name in os.listdir(f"/sys/devices/system/cpu/cpu{cpu}"):
            if name.startswith("node") and name[4:].isdigit():
                return int(name[4:])
    except OSError:
        pass
    return None


def bind_to_gpu_numa(index: int) -> dict:
    """Pin this process (threads created later inherit it) to the CPUs of the GPU's NUMA node and prefer that node for
    memory, BEFORE any pinned host buffer is allocated: page-locked staging memory is then first-touched on the socket
    the GPU's PCIe root belongs to, so host<->device copies never cross the inter-socket link (ranks sharing a socket
    otherwise slow each other's e2e step).
    Returns what was done (reported by bench.py); every step is best effort."""
    info = {"gpu": index, "cpus": None, "node": None, "mempolicy": None}
    cpus = gpu_cpu_affinity(index)
    try:
        allowed = os.sched_getaffinity(0)
        cpus = [c for c in cpus if c in allowed]
        if cpus:
            os.sched_setaffinity(0, cpus)
            info["cpus"] = f"{len(cpus)} cpus ({min(cpus)}..{max(cpus)})"
    except (AttributeError, OSError) as e:
        info["cpus"] = f"unchanged ({e})"
    node = _node_of_cpu(cpus[0]) if cpus else None
    info["node"] = node
    if node is not None:
        try:  # set_mempolicy(MPOL_PREFERRED = 1, nodemask, maxnode) — x86_64 syscall 238
            import ctypes

            libc = ctypes.CDLL(None, use_errno=True)
            mask = (ctypes.c_ulong * 16)()
            mask[node // 64] = 1 << (node % 64)
            rc = libc.syscall(238, 1, mask, 16 * 64 + 1)
            info["mempolicy"] = "preferred" if rc == 0 else f"errno {ctypes.get_errno()}"
        except Exception as e:  # no libc syscall wrapper: first-touch under the affinity above still places pages locally
            info["mempolicy"] = f"skipped ({e})"
    _numa_state.update(info)
    return info


def numa_binding() -> dict:
    return dict(_numa_state)


def init_from_env(backend: str | None = None, bind_numa: bool = True) -> torch.device:
    """Join the job described by RANK / WORLD_SIZE / LOCAL_RANK / MASTER_ADDR / MASTER_PORT (torchrun).
    Returns this rank's device.  A single-process run (no WORLD_SIZE) does not create a process group.
    With `bind_numa` the process is first bound to its GPU's NUMA node (see bind_to_gpu_numa)."""
    ws = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    cuda = torch.cuda.is_available()
    dev = torch.device(f"cuda:{local}") if cuda else torch.device("cpu")
    if cuda:
        if bind_numa:
            bind_to_gpu_numa(local)
        torch.cuda.set_device(dev)
    if ws > 1 and not is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        kw = {}
        if cuda:
            kw["device_id"] = dev
        td.init_process_group(backend or ("nccl" if cuda else "gloo"), **kw)
    return dev


def _comm_device(dev: torch.device | None) -> torch.device:
    if dev is not None:
        return dev
    if is_initialized() and td.get_backend() == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def broadcast_params(params: dict[str, list[float]] | None, src: int = 0, device: torch.device | None = None) -> dict[str, list[float]]:
    """Rank `src` passes {name: floats}; every rank returns the same dict with f32-exact values.  The keys and
    lengths (the plan's layout) must be known to all ranks — non-source ranks pass a dict of the same
    shape (values ignored) — so the whole block travels as ONE f32 broadcast."""
    if params is None:
        raise ValueError("every rank passes the parameter layout (values are taken from `src`)")
    keys = sorted(params)
    flat = [float(v) for k in keys for v in params[k]]
    if world_size() == 1:
        t = torch.tensor(flat, dtype=torch.float32)
    else:
        t = torch.tensor(flat, dtype=torch.float32, device=_comm_device(device))
        td.broadcast(t, src=src)
    vals = t.cpu().tolist()
    out, i = {}, 0
    for k in keys:
        n = len(params[k])
        out[k] = vals[i:i + n]
        i += n
    return out


def all_reduce_sums(sums: torch.Tensor) -> torch.Tensor:
    """Global `std_mean` accumulators: element-wise SUM of each rank's int64[6] (Σp, Σp²)."""
    if world_size() == 1:
        return sums
    t = sums.clone()
    if td.get_backend() == "gloo":
        t = t.cpu()
    td.all_reduce(t, op=td.ReduceOp.SUM)
    return t.to(sums.device)


def max_over_ranks(value: float, device: torch.device | None = None) -> float:
    """Multi-GPU timings are reported as the max over ranks (never wall clock of one rank)."""
    if world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=_comm_device(device))
    td.all_reduce(t, op=td.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device: torch.device | None = None) -> float:
    if world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=_comm_device(device))
    td.all_reduce(t, op=td.ReduceOp.SUM)
    return float(t.item())


def barrier(device: torch.device | None = None) -> None:
    if world_size() > 1:
        if td.get_backend() == "nccl":
            td.barrier(device_ids=[torch.cuda.current_device()])
        else:
            td.barrier()
