"""Enums mirrored from csrc/glb/types.h and buffer introspection helpers."""
from __future__ import annotations

import enum
from typing import Any, Tuple

import numpy as np


class DataType(enum.IntEnum):
    INT8 = 0
    UINT8 = 1
    INT32 = 2
    INT64 = 3
    UINT64 = 4
    FLOAT32 = 5
    FLOAT64 = 6
    FLOAT16 = 7
    BFLOAT16 = 8
    UINT32 = 9
    INT16 = 10
    FLOAT8_E4M3 = 11
    FLOAT8_E5M2 = 12


class ReduceOp(enum.IntEnum):
    SUM = 1
    PRODUCT = 2
    MAX = 3
    MIN = 4
    CUSTOM = 1000


class Algorithm(enum.IntEnum):
    UNSPECIFIED = 0
    RING = 1
    BCUBE = 2


_NP = {
    np.dtype(np.int8): DataType.INT8,
    np.dtype(np.uint8): DataType.UINT8,
    np.dtype(np.int16): DataType.INT16,
    np.dtype(np.int32): DataType.INT32,
    np.dtype(np.uint32): DataType.UINT32,
    np.dtype(np.int64): DataType.INT64,
    np.dtype(np.uint64): DataType.UINT64,
    np.dtype(np.float32): DataType.FLOAT32,
    np.dtype(np.float64): DataType.FLOAT64,
    np.dtype(np.float16): DataType.FLOAT16,
}

_SIZES = {
    DataType.INT8: 1, DataType.UINT8: 1, DataType.INT16: 2, DataType.FLOAT16: 2, DataType.BFLOAT16: 2,
    DataType.INT32: 4, DataType.UINT32: 4, DataType.FLOAT32: 4, DataType.INT64: 8, DataType.UINT64: 8,
    DataType.FLOAT64: 8, DataType.FLOAT8_E4M3: 1, DataType.FLOAT8_E5M2: 1,
}


def _torch_map():
    import torch

    return {
        torch.int8: DataType.INT8, torch.uint8: DataType.UINT8, torch.int16: DataType.INT16,
        torch.int32: DataType.INT32, torch.int64: DataType.INT64, torch.float32: DataType.FLOAT32,
        torch.float64: DataType.FLOAT64, torch.float16: DataType.FLOAT16, torch.bfloat16: DataType.BFLOAT16,
        torch.bool: DataType.UINT8,
        # numpy has no FP8 dtype: these two formats are reachable through torch tensors only.
        torch.float8_e4m3fn: DataType.FLOAT8_E4M3, torch.float8_e5m2: DataType.FLOAT8_E5M2,
    }


def element_size(dt: DataType) -> int:
    return _SIZES[DataType(dt)]


def is_torch(x: Any) -> bool:
    return type(x).__module__.startswith("torch") and hasattr(x, "data_ptr")


def describe(x: Any) -> Tuple[int, int, DataType, bool]:
    """(address, element count, dtype, is_cuda) of a contiguous numpy array or torch tensor."""
    if is_torch(x):
        if not x.is_contiguous():
            raise ValueError("tensor must be contiguous")
        dt = _torch_map().get(x.dtype)
        if dt is None:
            raise TypeError(f"unsupported dtype {x.dtype}")
        return x.data_ptr(), x.numel(), dt, x.is_cuda
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise ValueError("array must be C-contiguous")
        if x.dtype not in _NP:
            raise TypeError(f"unsupported dtype {x.dtype}")
        return x.ctypes.data, x.size, _NP[x.dtype], False
    raise TypeError(f"unsupported buffer type {type(x)!r}")


def nbytes(x: Any) -> int:
    _, n, dt, _ = describe(x)
    return n * element_size(dt)
