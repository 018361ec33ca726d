"""Process-wide runtime: one process per GPU (the analogue of one Spark executor), one mb_ctx.

torch is plumbing here: it owns device buffers (so NCCL via torch.distributed can move them) and
the stream; every kernel that touches matrix data is launched by libmarlin_b200.so.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _native as nat


class Runtime:
    _instance: Optional["Runtime"] = None

    def __init__(self, device_index: Optional[int] = None):
        if not torch.cuda.is_available():
            raise nat.MarlinError(nat.MB_ERR_CUDA, "no CUDA device visible: marlin_b200 runs on H100 (sm_90a) only and has "
                                  "no CPU fallback")
        if device_index is None:
            device_index = int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count()
        self.device_index = device_index
        self.device = torch.device("cuda", device_index)
        torch.cuda.set_device(self.device)
        self.lib = nat.load()
        self.ctx = nat.c_ctx()
        nat.check(self.lib.mb_init(device_index, C.byref(self.ctx)))
        self.sync_stream()

    @classmethod
    def get(cls) -> "Runtime":
        if cls._instance is None:
            cls._instance = Runtime()
        return cls._instance

    @classmethod
    def available(cls) -> bool:
        return torch.cuda.is_available()

    def sync_stream(self) -> None:
        """Launch on torch's current stream so torch.distributed collectives and our kernels order correctly."""
        nat.check(self.lib.mb_set_stream(self.ctx, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))

    def set_fp64_mode(self, mode: str = "native", slices: int = 6) -> None:
        """'native' (DMMA, IEEE fp64 — default), 'int8x7' (int8 tensor cores, 7-bit digit planes) or 'int8x8'
        (8-bit digit planes).  See include/marlin_b200.h: mb_set_fp64_mode."""
        code = {"native": 0, "int8x7": 1, "int8x8": 2}[mode]
        nat.check(self.lib.mb_set_fp64_mode(self.ctx, code, slices))

    def set_dmma_reference(self, on: bool) -> None:
        """Test and measurement hook, off by default: run the m8n8k4 reference instances of the fp64 DMMA kernels instead
        of the m16n8k4 ones.  See include/marlin_b200.h: mb_set_dmma_reference."""
        nat.check(self.lib.mb_set_dmma_reference(self.ctx, 1 if on else 0))

    def launch_count(self) -> int:
        return int(self.lib.mb_launch_count(self.ctx))

    def synchronize(self) -> None:
        nat.check(self.lib.mb_synchronize(self.ctx))


# ---- distributed plumbing (torch.distributed; NCCL on GPUs, gloo in CPU tests) ----
def world() -> tuple:
    """(rank, world_size) — (0, 1) when torch.distributed is not initialised."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1
