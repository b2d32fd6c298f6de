"""Process bootstrap: one process per GPU, ``torch.distributed`` for the plumbing.

Reference: the top of every chapter's ``main()`` — ``rank = $RANK``, ``local_rank = rank %
device_count``, ``set_device``, ``init_process_group(rank, world_size, device_id=device)``
(``02-distributed-data-parallel/train_llm.py:36-41``), the mpirun variant reading
``OMPI_COMM_WORLD_*`` (``03-job-launchers/README.md:127-132``), the deepspeed launcher's
``--local_rank`` (``03R:178-190``), and the ordered-execution guards ``rank0_first``
(``02:272-280``), local-rank-0-first (``05-training-llama-405b/train_llm.py:415-423``) and
``rank_ordered`` (``06-tensor-parallel/train_llm.py:346-353``).

NCCL (over NVLink / NVSwitch) is the backend on GPUs and carries bootstrap, barriers and
cold-path collectives; the hot-path collectives are this package's own NVLink kernels
(``parallel/symm.py``, ``csrc/comm.cu``).  ``gloo`` is used on CPU (tests, toy).
"""
from __future__ import annotations

import dataclasses
import datetime
import os
from contextlib import contextmanager
from typing import Optional

import torch
import torch.distributed as dist


@dataclasses.dataclass
class DistEnv:
    rank: int
    local_rank: int
    world_size: int
    device: torch.device
    distributed: bool

    @property
    def is_main(self):
        return self.rank == 0


def _env_int(*names, default=None):
    for n in names:
        v = os.environ.get(n)
        if v is not None and v != "":
            return int(v)
    return default


def detect_rank_world():
    """RANK/WORLD_SIZE from torchrun, else OpenMPI, else slurm, else single process."""
    rank = _env_int("RANK", "OMPI_COMM_WORLD_RANK", "SLURM_PROCID", default=0)
    world = _env_int("WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "SLURM_NTASKS", default=1)
    local = _env_int("LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "SLURM_LOCALID", default=None)
    return rank, world, local


def init_distributed(device_type: Optional[str] = None, local_rank: Optional[int] = None,
                     timeout_s: Optional[int] = None, force: bool = False) -> DistEnv:
    # collective timeout: long enough for a rank-0-first model download, short enough that a wedged job dies with
    # a stack instead of burning an allocation (DTG_DIST_TIMEOUT_S overrides; bench.py sets 150 s)
    if timeout_s is None:
        timeout_s = int(os.environ.get("DTG_DIST_TIMEOUT_S", "600"))
    rank, world, env_local = detect_rank_world()
    if device_type is None:
        device_type = "cuda" if torch.cuda.is_available() else "cpu"
    if device_type == "cuda":
        n = torch.cuda.device_count()
        if local_rank is None:
            local_rank = env_local if env_local is not None else rank % n
        device = torch.device(f"cuda:{local_rank}")
        torch.cuda.set_device(device)
    else:
        local_rank = env_local if env_local is not None else rank
        device = torch.device("cpu")
    distributed = world > 1 or force or "MASTER_ADDR" in os.environ
    if distributed and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        kwargs = dict(rank=rank, world_size=world, timeout=datetime.timedelta(seconds=timeout_s))
        if device_type == "cuda":
            # eager communicator bound to the device, as the reference does with device_id=
            dist.init_process_group(backend="nccl", device_id=device, **kwargs)
        else:
            dist.init_process_group(backend="gloo", **kwargs)
    return DistEnv(rank=rank, local_rank=local_rank, world_size=world, device=device, distributed=distributed)


def barrier():
    if dist.is_available() and dist.is_initialized():
        dist.barrier()


@contextmanager
def rank_ordered(should_go_first: bool):
    """Processes for which ``should_go_first`` holds run the body, then everyone else does."""
    if should_go_first:
        yield
    barrier()
    if not should_go_first:
        yield
    barrier()


def rank0_first():
    r = dist.get_rank() if dist.is_initialized() else 0
    return rank_ordered(r == 0)


def local_rank0_first(local_rank: Optional[int] = None):
    if local_rank is None:
        _, _, local_rank = detect_rank_world()
        local_rank = local_rank or 0
    return rank_ordered(local_rank == 0)


def storage_first(path: str, env: DistEnv):
    """Who goes first depends on the storage: rank 0 on a shared mount, local-rank 0 on
    node-local disks (reference ``02-distributed-data-parallel/README.md:340-364``)."""
    shared = os.path.ismount(path)
    return rank_ordered(env.rank == 0 if shared else env.local_rank == 0)


def shutdown():
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()
