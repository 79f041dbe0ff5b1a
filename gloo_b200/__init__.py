"""gloo_b200 — a Hopper-native (H100, sm_90a) collective-communications library with the
capabilities and API surface of pytorch/gloo.

Layers (see DESIGN.md):
  _C                  native core (C++17 + CUDA sm_90a), built in-tree by build.py
  gloo_b200.ops       collectives API for numpy arrays / torch tensors (host + CUDA)
  gloo_b200.parallel  consumers: DDP gradient sync, ZeRO/FSDP shard ops, TP, MoE
                      dispatch/combine, Ulysses / ring sequence parallel helpers
  gloo_b200.models    reference workloads used by smoke() / benchmarks
  gloo_b200.utils     launch helpers, rendezvous from torchrun env, timing
"""
from __future__ import annotations

import importlib
import os
import sys



def _load_native():
    try:
        return importlib.import_module("gloo_b200._C")
    except ImportError as first:
        # Build on demand (source checkout without a prior `python build.py`).
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        if os.path.exists(os.path.join(root, "build.py")) and os.environ.get("GLB_NO_AUTOBUILD") != "1":
            sys.path.insert(0, root)
            try:
                import build as _build  # type: ignore

                _build.build()
            finally:
                sys.path.pop(0)
            return importlib.import_module("gloo_b200._C")
        raise first


_C = _load_native()

from ._C import (  # noqa: E402
    BaseContext,
    Context,
    ContextFactory,
    EnforceError,
    FileStore,
    GlbError,
    HashStore,
    RedisStore,
    InvalidOperationError,
    IoError,
    PrefixStore,
    Store,
    TimeoutError,
)
from .types import DataType, ReduceOp, Algorithm  # noqa: E402

__version__ = _C.__version__
build_config = _C.build_config
from .ops.host import (  # noqa: E402
    allgather,
    allgatherv,
    allreduce,
    alltoall,
    alltoallv,
    barrier,
    broadcast,
    gather,
    gatherv,
    reduce,
    reduce_scatter,
    scatter,
)
from .utils.launch import create_device, init_context, spawn_threads  # noqa: E402

__all__ = [
    "Context", "BaseContext", "ContextFactory", "Store", "HashStore", "FileStore", "PrefixStore", "RedisStore",
    "GlbError", "IoError", "TimeoutError", "InvalidOperationError", "EnforceError",
    "DataType", "ReduceOp", "Algorithm",
    "allreduce", "reduce", "reduce_scatter", "broadcast", "allgather", "allgatherv", "alltoall",
    "alltoallv", "gather", "gatherv", "scatter", "barrier",
    "create_device", "init_context", "spawn_threads",
]
