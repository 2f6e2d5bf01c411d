"""Process-level runtime: one process drives one GPU.

Stands in for the reference's Runtime singleton (sparse/runtime.py:56-130: library registration,
processor counts, eager NCCL bring-up when more than one GPU is present).  Here a process owns
exactly one device; multi-GPU runs are one process per GPU under torchrun, glued together by
`torch.distributed` (see dist.py).  `LEGATE_SPARSE_NUM_PROCS` keeps its reference meaning
(runtime.py:61-63): it overrides the shard count used by the row-block partitioner.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib

_TORCH_OF_NP = {
    np.dtype(np.float32): torch.float32,
    np.dtype(np.float64): torch.float64,
    np.dtype(np.int32): torch.int32,
    np.dtype(np.int64): torch.int64,
    np.dtype(np.complex64): torch.complex64,
    np.dtype(np.complex128): torch.complex128,
    np.dtype(np.bool_): torch.bool,
    np.dtype(np.int8): torch.int8,
    np.dtype(np.int16): torch.int16,
    np.dtype(np.uint8): torch.uint8,
    np.dtype(np.float16): torch.float16,
}
_NP_OF_TORCH = {v: k for k, v in _TORCH_OF_NP.items()}

SUPPORTED_VALUE_DTYPES = (np.dtype(np.float32), np.dtype(np.float64))


def torch_dtype(dt) -> torch.dtype:
    if isinstance(dt, torch.dtype):
        return dt
    return _TORCH_OF_NP[np.dtype(dt)]


def numpy_dtype(dt) -> np.dtype:
    if isinstance(dt, torch.dtype):
        return _NP_OF_TORCH[dt]
    return np.dtype(dt)


def vt_code(dt) -> int:
    code = _VT_OF_TORCH.get(dt) if isinstance(dt, torch.dtype) else None
    if code is not None:   # every launch asks: skip the numpy dtype comparisons
        return code
    dt = numpy_dtype(dt)
    if dt == np.float32:
        return _lib.F32
    if dt == np.float64:
        return _lib.F64
    raise NotImplementedError(
        f"legate.sparse_b200 kernels are built for float32/float64; got {dt} "
        "(complex dtypes of the reference's dispatch table are not implemented)"
    )


def idx_code(dt) -> int:
    code = _IDX_OF_TORCH.get(dt) if isinstance(dt, torch.dtype) else None
    if code is not None:
        return code
    dt = numpy_dtype(dt)
    if dt == np.int32:
        return _lib.I32
    if dt == np.int64:
        return _lib.I64
    raise TypeError(f"index arrays must be int32 or int64, got {dt}")


_VT_OF_TORCH = {torch.float32: _lib.F32, torch.float64: _lib.F64}
_IDX_OF_TORCH = {torch.int32: _lib.I32, torch.int64: _lib.I64}


class Runtime:
    def __init__(self):
        self._ws = {}
        self._l2 = {}
        self._num_procs_override = None
        env = os.environ.get("LEGATE_SPARSE_NUM_PROCS")
        if env is not None:
            self._num_procs_override = int(env)
            print(f"Overriding LEGATE_SPARSE_NUM_PROCS to {self._num_procs_override}")

    # -- device ---------------------------------------------------------------------------------
    @property
    def has_cuda(self) -> bool:
        return torch.cuda.is_available()

    @property
    def device(self) -> torch.device:
        """Device that holds matrices/vectors: the current CUDA device, or the host when no GPU is
        visible (construction / format logic only -- every compute entry point requires CUDA)."""
        if self.has_cuda:
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device("cpu")

    def require_cuda(self, what: str) -> None:
        if not self.has_cuda:
            raise RuntimeError(
                f"{what}: no CUDA device is visible. legate.sparse_b200 has no CPU fallback; "
                "the hot path runs only as sm_90a kernels from libb200sparse.so."
            )

    def stream_ptr(self) -> int:
        # the raw handle, without building a torch.cuda.Stream object: every launch asks, and at SpMV sizes the
        # object costs as much host time as the rest of the launch path
        return torch._C._cuda_getCurrentRawStream(torch.cuda.current_device())

    def workspace(self) -> torch.Tensor:
        """Reduction workspace (b2s_ws_bytes), one per (device, stream), zero-filled once."""
        key = (torch.cuda.current_device(), self.stream_ptr())
        ws = self._ws.get(key)
        if ws is None:
            ws = torch.zeros(int(_lib.lib.b2s_ws_bytes()), dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
        return ws

    def device_info(self, device: int | None = None):
        self.require_cuda("device_info")
        out = (_lib.c_i64 * 4)()
        dev = torch.cuda.current_device() if device is None else device
        _lib.check(_lib.lib.b2s_device_info(dev, out), "b2s_device_info")
        return {"sm_count": out[0], "l2_bytes": out[1], "cc": out[2], "max_smem_optin": out[3]}

    def l2_bytes(self) -> int:
        """L2 size of the current device, queried once per device: the column-split thresholds are fractions of it."""
        dev = torch.cuda.current_device()
        v = self._l2.get(dev)
        if v is None:
            v = self._l2[dev] = int(self.device_info(dev)["l2_bytes"])
        return v

    # -- processor counts (reference: runtime.num_procs / num_gpus) ----------------------------------
    @property
    def num_gpus(self) -> int:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size()
        return 1 if self.has_cuda else 0

    @property
    def num_procs(self) -> int:
        if self._num_procs_override is not None:
            return self._num_procs_override
        return max(self.num_gpus, 1)


runtime = Runtime()


# -- array plumbing ---------------------------------------------------------------------------------
def is_device_array(a) -> bool:
    return isinstance(a, torch.Tensor)


def to_device(a, dtype=None, copy: bool = False) -> torch.Tensor:
    """numpy / torch / sequence -> contiguous tensor on runtime.device."""
    dev = runtime.device
    if isinstance(a, torch.Tensor):
        t = a
        if dtype is not None and t.dtype != torch_dtype(dtype):
            t = t.to(torch_dtype(dtype))
            copy = False
        if t.device != dev:
            t = t.to(dev, non_blocking=True)
            copy = False
        if not t.is_contiguous():
            t = t.contiguous()
            copy = False
        return t.clone() if copy else t
    arr = np.asarray(a)
    if dtype is not None and arr.dtype != numpy_dtype(dtype):
        arr = arr.astype(numpy_dtype(dtype))
    arr = np.ascontiguousarray(arr)
    if not arr.flags.writeable:
        arr = arr.copy()
    t = torch.from_numpy(arr)
    if dev.type == "cuda":
        return t.to(dev, non_blocking=True)
    return t.clone() if copy else t


def to_host(t) -> np.ndarray:
    if isinstance(t, torch.Tensor):
        return t.detach().cpu().numpy()
    return np.asarray(t)


def ptr(t: torch.Tensor | None) -> int | None:
    if t is None:
        return None
    return t.data_ptr()
