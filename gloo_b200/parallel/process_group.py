"""``torch.distributed`` backend "glb".

PyTorch reaches pytorch/gloo through ``ProcessGroupGloo`` (``backend="gloo"``); this module is
the same door for this library::

    import gloo_b200.parallel.process_group          # registers the backend
    torch.distributed.init_process_group("glb", init_method="tcp://127.0.0.1:29500",
                                         rank=rank, world_size=size)
    torch.distributed.all_reduce(t)                  # CPU tensor: host transport
    torch.distributed.all_reduce(t.cuda())           # CUDA tensor: fused NVLink kernel

Rendezvous goes through the c10d store handed to the backend (wrapped as a ``gb.Store``), so
``env://``, ``tcp://`` and ``file://`` all work. CPU tensors use the host collectives;
CUDA tensors use ``gloo_b200.ops.cuda.CudaContext`` of their device (created on first use,
collectively) and are asynchronous on the current stream, like NCCL work; ``ReduceOp.AVG``
is applied inside the collective kernel (fused scale epilogue), not as a second pass.
Point-to-point ``send``/``recv`` return asynchronous work objects: host tensors go through the
transport (``wait()`` completes them), CUDA tensors travel over NVLink on dedicated send /
receive streams (``wait()`` orders the caller's stream after the transfer, as with NCCL), so
the usual "every rank posts isend, then irecv" pattern cannot deadlock.

Every method mirrors the signature c10d calls on a Python ``ProcessGroup``
(torch/testing/_internal/distributed/multi_threaded_pg.py is the reference for that).
"""
from __future__ import annotations

import os
from datetime import timedelta
from typing import Dict, Optional

import torch
import torch.distributed as dist
from torch._C._distributed_c10d import (
    AllgatherOptions,
    AllreduceOptions,
    AllToAllOptions,
    BarrierOptions,
    BroadcastOptions,
    GatherOptions,
    ReduceOptions,
    ReduceScatterOptions,
    ScatterOptions,
    _create_work_from_future,
)
from torch.futures import Future

from .. import _C
from ..ops import host as H
from ..types import ReduceOp

BACKEND_NAME = "glb"
_P2P_PREFIX = 0x7D  # slot prefix of send/recv issued through the process group


class _C10dStore(_C.Store):
    """A c10d store seen through the ``gb.Store`` interface (set / get / wait)."""

    def __init__(self, store):
        _C.Store.__init__(self)
        self._s = store

    def set(self, key, value):
        self._s.set(key, bytes(value))

    def get(self, key):
        return bytes(self._s.get(key))

    def wait(self, keys, timeout_ms):
        self._s.wait(list(keys), timedelta(milliseconds=max(1, int(timeout_ms))))


def _done(result=None):
    fut = Future()
    fut.set_result(result)
    return _create_work_from_future(fut)


class _HostP2pWork(dist.Work):
    """A posted host send / receive: completes in wait() (the transport progresses it in the
    background), keeps the buffer and the tensors alive until then."""

    def __init__(self, buf, is_send: bool, keep, on_done=None, src: int = -1):
        super().__init__()
        self._buf, self._is_send, self._keep, self._on_done, self._src = buf, is_send, keep, on_done, src
        self._done = False

    def wait(self, timeout=None):
        if not self._done:
            if self._is_send:
                self._buf.wait_send()
            else:
                got = self._buf.wait_recv()
                if got is not None and isinstance(got, int):
                    self._src = got
            if self._on_done is not None:
                self._on_done()
            self._done = True
            self._keep = None
        return True

    def is_completed(self):
        return self._done

    def is_success(self):
        return True

    def source_rank(self):
        self.wait()
        return self._src

    def _source_rank(self):
        return self.source_rank()

    def __del__(self):
        # A posted operation must not outlive its buffer: finish it if the caller dropped the work.
        try:
            self.wait()
        except Exception:  # noqa: BLE001
            pass


class _StreamWork(dist.Work):
    """A CUDA transfer enqueued on a side stream: wait() makes the caller's stream wait for it."""

    def __init__(self, event, keep, src: int = -1):
        super().__init__()
        self._event, self._keep, self._src = event, keep, src

    def wait(self, timeout=None):
        torch.cuda.current_stream().wait_event(self._event)
        return True

    def is_completed(self):
        return self._event.query()

    def is_success(self):
        return True

    def synchronize(self):
        self._event.synchronize()

    def source_rank(self):
        return self._src

    def _source_rank(self):
        return self._src


class _RecvWork(dist.Work):
    """Completed work of a receive; carries the sender's rank for recv-from-any."""

    def __init__(self, src: int):
        super().__init__()
        self._src = src

    def wait(self, timeout=None):
        return True

    def is_completed(self):
        return True

    def is_success(self):
        return True

    def source_rank(self):
        return self._src

    def _source_rank(self):
        return self._src


def _op(reduce_op) -> ReduceOp:
    R = dist.ReduceOp
    for theirs, ours in ((R.SUM, ReduceOp.SUM), (R.AVG, ReduceOp.SUM), (R.PRODUCT, ReduceOp.PRODUCT),
                         (R.MIN, ReduceOp.MIN), (R.MAX, ReduceOp.MAX)):
        if reduce_op == theirs:
            return ours
    raise NotImplementedError(f"glb backend: reduce op {reduce_op} is not supported (sum, avg, product, min, max)")


def _is_avg(reduce_op) -> bool:
    return reduce_op == dist.ReduceOp.AVG


_FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)


def _divide_(t, n: int):
    """t /= n in place. torch has no division kernel for FP8 tensors, so those take a float32
    round trip (one rounding, like the fused scale of the CUDA kernels)."""
    if t.dtype in _FP8:
        t.copy_(t.float().div_(n))
    else:
        t.div_(n)


class GlbProcessGroup(dist.ProcessGroup):
    def __init__(self, store, rank: int, world_size: int, timeout: timedelta):
        super().__init__(rank, world_size)
        self._rank, self._world = rank, world_size
        self._timeout_ms = max(1000, int(timeout.total_seconds() * 1000)) if timeout else 30 * 60 * 1000
        iface = os.environ.get("GLB_SOCKET_IFNAME") or os.environ.get("GLOO_SOCKET_IFNAME") or ""
        # No interface named: bind this host's own name (falls back to loopback when the name
        # does not resolve, e.g. in a container), so that ranks on other hosts can reach it -
        # the same rule ProcessGroupGloo applies.
        device = _C.create_tcp_device("", iface, False, 1)
        self.ctx = _C.Context(rank, world_size, 2)
        self.ctx.set_timeout(self._timeout_ms)
        self.ctx.connect_full_mesh(_C10dStore(store), device)
        self._cuda: Dict[int, object] = {}
        self._p2p_streams: Dict[int, tuple] = {}

    # ---- plumbing -------------------------------------------------------------------------
    def getBackendName(self):
        return BACKEND_NAME

    def size(self):
        return self._world

    def rank(self):
        return self._rank

    def __repr__(self):
        return f"GlbProcessGroup(rank={self._rank}, world_size={self._world})"

    def _cc(self, tensor):
        """The CudaContext of the tensor's device (first use is collective on every rank)."""
        from ..ops import cuda as gcu

        idx = tensor.device.index if tensor.device.index is not None else torch.cuda.current_device()
        if idx not in self._cuda:
            # torch tensors are not registered with the peer context, so they travel through
            # its staging pool (GLB_PG_STAGE_MB, default 128). Every collective takes any size:
            # a payload larger than the pool streams through it.
            stage = int(os.environ.get("GLB_PG_STAGE_MB", "128")) << 20
            with torch.cuda.device(idx):
                self._cuda[idx] = gcu.CudaContext(self.ctx, idx, stage_bytes=stage)
        return self._cuda[idx]

    @staticmethod
    def _contig(t):
        return t if t.is_contiguous() else t.contiguous()

    # ---- collectives ------------------------------------------------------------------------
    def allreduce(self, tensor_list, opts=AllreduceOptions()):
        tensors = tensor_list if isinstance(tensor_list, (list, tuple)) else [tensor_list]
        op = _op(opts.reduceOp)
        for t in tensors:
            w = self._contig(t)
            if w.is_cuda:
                # AVG is the kernel's scale epilogue: one launch, no second pass over the data.
                fused = _is_avg(opts.reduceOp) and w.is_floating_point()
                self._cc(w).allreduce(w, op=op, average=fused)
                if _is_avg(opts.reduceOp) and not fused:
                    _divide_(w, self._world)
            else:
                H.allreduce(self.ctx, w, op=op)
                if _is_avg(opts.reduceOp):
                    _divide_(w, self._world)
            if w is not t:
                t.copy_(w)
        return _done(tensors)

    def allreduce_coalesced(self, tensor_list, opts=AllreduceOptions()):
        return self.allreduce(tensor_list, opts)

    def broadcast(self, tensor_list, opts=BroadcastOptions()):
        tensors = tensor_list if isinstance(tensor_list, (list, tuple)) else [tensor_list]
        for t in tensors:
            w = self._contig(t)
            if w.is_cuda:
                self._cc(w).broadcast(w, root=opts.rootRank)
            else:
                H.broadcast(self.ctx, w, root=opts.rootRank)
            if w is not t:
                t.copy_(w)
        return _done(tensors)

    def _allgather_base(self, output_tensor, input_tensor, opts=AllgatherOptions()):
        out, inp = self._contig(output_tensor), self._contig(input_tensor)
        if out.is_cuda:
            self._cc(out).allgather(out.view(-1), inp.view(-1))
        else:
            H.allgather(self.ctx, out.view(-1), inp.view(-1))
        if out is not output_tensor:
            output_tensor.copy_(out)
        return _done(output_tensor)

    def allgather(self, output_tensors, input_tensor, opts=AllgatherOptions()):
        inputs = input_tensor if isinstance(input_tensor, (list, tuple)) else [input_tensor]
        for outs, inp in zip(output_tensors, inputs):
            flat = torch.empty(self._world * inp.numel(), dtype=inp.dtype, device=inp.device)
            self._allgather_base(flat, inp.reshape(-1))
            for r, o in enumerate(outs):
                o.copy_(flat[r * inp.numel():(r + 1) * inp.numel()].view_as(o))
        return _done(output_tensors)

    def allgather_into_tensor_coalesced(self, output_tensor_list, input_tensor_list, opts=AllgatherOptions()):
        for o, i in zip(output_tensor_list, input_tensor_list):
            self._allgather_base(o, i)
        return _done(output_tensor_list)

    def _reduce_scatter_base(self, output_tensor, input_tensor, opts=ReduceScatterOptions()):
        out, inp = self._contig(output_tensor), self._contig(input_tensor)
        op = _op(opts.reduceOp)
        if out.is_cuda:
            fused = _is_avg(opts.reduceOp) and out.is_floating_point()
            self._cc(out).reduce_scatter(out.view(-1), inp.view(-1), op=op, scale=1.0 / self._world if fused else 1.0)
            if _is_avg(opts.reduceOp) and not fused:
                _divide_(out, self._world)
        else:
            H.reduce_scatter(self.ctx, out.view(-1), inp.view(-1), op=op)
            if _is_avg(opts.reduceOp):
                _divide_(out, self._world)
        if out is not output_tensor:
            output_tensor.copy_(out)
        return _done(output_tensor)

    def reduce_scatter(self, output_tensor, scatter_list, opts=ReduceScatterOptions()):
        outs = output_tensor if isinstance(output_tensor, (list, tuple)) else [output_tensor]
        for out, parts in zip(outs, scatter_list):
            flat = torch.cat([p.reshape(-1) for p in parts])
            self._reduce_scatter_base(out, flat, opts)
        return _done(outs)

    def reduce_scatter_tensor_coalesced(self, output_tensors, input_tensors, opts=ReduceScatterOptions()):
        for o, i in zip(output_tensors, input_tensors):
            self._reduce_scatter_base(o, i, opts)
        return _done(output_tensors)

    def alltoall_base(self, output_buffer, input_buffer, output_split_sizes, input_split_sizes,
                      opts=AllToAllOptions()):
        out, inp = self._contig(output_buffer), self._contig(input_buffer)
        row = inp.numel() // inp.shape[0] if inp.dim() > 0 and inp.shape[0] > 0 else 1
        if not output_split_sizes and not input_split_sizes:
            if out.is_cuda:
                self._cc(out).alltoall(out.view(-1), inp.view(-1))
            else:
                H.alltoall(self.ctx, out.view(-1), inp.view(-1))
        else:
            ic = [int(s) * row for s in (input_split_sizes or [inp.shape[0] // self._world] * self._world)]
            oc = [int(s) * row for s in (output_split_sizes or [out.shape[0] // self._world] * self._world)]
            if out.is_cuda:
                self._cc(out).alltoallv(out.view(-1), oc, inp.view(-1), ic)
            else:
                H.alltoallv(self.ctx, out.view(-1), oc, inp.view(-1), ic)
        if out is not output_buffer:
            output_buffer.copy_(out)
        return _done(output_buffer)

    def alltoall(self, output_tensor_list, input_tensor_list, opts=AllToAllOptions()):
        ic = [t.numel() for t in input_tensor_list]
        oc = [t.numel() for t in output_tensor_list]
        inp = torch.cat([t.reshape(-1) for t in input_tensor_list])
        out = torch.empty(sum(oc), dtype=inp.dtype, device=inp.device)
        if out.is_cuda:
            self._cc(out).alltoallv(out, oc, inp, ic)
        else:
            H.alltoallv(self.ctx, out, oc, inp, ic)
        off = 0
        for t, n in zip(output_tensor_list, oc):
            t.copy_(out[off:off + n].view_as(t))
            off += n
        return _done(output_tensor_list)

    def reduce(self, tensor_list, opts=ReduceOptions()):
        tensors = tensor_list if isinstance(tensor_list, (list, tuple)) else [tensor_list]
        op = _op(opts.reduceOp)
        for t in tensors:
            w = self._contig(t)
            if w.is_cuda:
                res = torch.empty_like(w)
                self._cc(w).reduce(res, w, root=opts.rootRank, op=op)
                if self._rank == opts.rootRank:
                    w.copy_(res)
            else:
                H.reduce(self.ctx, w, root=opts.rootRank, op=op)
            if _is_avg(opts.reduceOp) and self._rank == opts.rootRank:
                _divide_(w, self._world)
            if w is not t:
                t.copy_(w)
        return _done(tensors)

    def gather(self, output_tensors, input_tensors, opts=GatherOptions()):
        inputs = input_tensors if isinstance(input_tensors, (list, tuple)) else [input_tensors]
        root = opts.rootRank
        for i, inp in enumerate(inputs):
            w = self._contig(inp).reshape(-1)
            flat = torch.empty(self._world * w.numel(), dtype=w.dtype, device=w.device) if self._rank == root else None
            if w.is_cuda:
                # every rank passes an output on the CUDA path (only the root's is written)
                buf = flat if flat is not None else torch.empty(self._world * w.numel(), dtype=w.dtype, device=w.device)
                self._cc(w).gather(buf, w, root=root)
            else:
                H.gather(self.ctx, w, flat, root=root)
            if self._rank == root:
                for r, o in enumerate(output_tensors[i]):
                    o.copy_(flat[r * w.numel():(r + 1) * w.numel()].view_as(o))
        return _done(output_tensors)

    def scatter(self, output_tensors, input_tensors, opts=ScatterOptions()):
        outs = output_tensors if isinstance(output_tensors, (list, tuple)) else [output_tensors]
        root = opts.rootRank
        for i, out in enumerate(outs):
            w = self._contig(out)
            if w.is_cuda:
                flat = torch.cat([p.reshape(-1) for p in input_tensors[i]]) if self._rank == root else None
                self._cc(w).scatter(w.view(-1), flat, root=root)
            else:
                parts = [self._contig(p).reshape(-1) for p in input_tensors[i]] if self._rank == root else None
                H.scatter(self.ctx, w.view(-1), parts, root=root)
            if w is not out:
                out.copy_(w)
        return _done(outs)

    def barrier(self, opts=BarrierOptions()):
        for idx in self._cuda:
            torch.cuda.current_stream(idx).synchronize()
        H.barrier(self.ctx)
        return _done(None)

    # ---- point to point ---------------------------------------------------------------------
    def _slot(self, src: int, dst: int, tag: int) -> int:
        # One ordered stream of messages per (src, dst, tag); the transport matches FIFO per slot.
        return _C.slot_build(_P2P_PREFIX, int(tag) & 0xFFFFFFFF, 0)

    def _side_streams(self, idx: int):
        """(send stream, recv stream) of a device: p2p kernels wait for their peer on the device,
        so they must not queue behind each other or behind the caller's compute."""
        if idx not in self._p2p_streams:
            from ..ops import cuda as gcu

            self._p2p_streams[idx] = (gcu.new_stream(idx), gcu.new_stream(idx))
        return self._p2p_streams[idx]

    def _cuda_p2p(self, t, peer: int, is_send: bool):
        cc = self._cc(t)
        idx = cc.device
        side = self._side_streams(idx)[0 if is_send else 1]
        cur = torch.cuda.current_stream(idx)
        w = self._contig(t) if is_send else (t if t.is_contiguous() else torch.empty_like(t, memory_format=torch.contiguous_format))
        side.wait_stream(cur)
        if is_send:
            cc.send(w, peer, stream=side)
        else:
            cc.recv(w, peer, stream=side)
            if w is not t:
                with torch.cuda.stream(side):
                    t.copy_(w)
        w.record_stream(side)
        t.record_stream(side)
        ev = torch.cuda.Event()
        ev.record(side)
        return _StreamWork(ev, (w, t), src=peer if not is_send else -1)

    def send(self, tensors, dstRank, tag=0):
        work = None
        for t in tensors:
            if t.is_cuda:
                work = self._cuda_p2p(t.detach(), dstRank, True)
                continue
            h = self._contig(t).detach()
            buf = self.ctx.create_unbound_buffer(h.data_ptr(), h.numel() * h.element_size())
            buf.send(dstRank, self._slot(self._rank, dstRank, tag))
            work = _HostP2pWork(buf, True, (h, t))
        return work if work is not None else _done(None)

    def recv(self, tensors, srcRank, tag=0):
        work = None
        for t in tensors:
            if t.is_cuda:
                work = self._cuda_p2p(t, srcRank, False)
                continue
            h = t if t.is_contiguous() else torch.empty(t.shape, dtype=t.dtype)
            buf = self.ctx.create_unbound_buffer(h.data_ptr(), h.numel() * h.element_size())
            buf.recv(srcRank, self._slot(srcRank, self._rank, tag))
            work = _HostP2pWork(buf, False, (h, t), on_done=(lambda h=h, t=t: t.copy_(h)) if h is not t else None,
                                src=srcRank)
        return work if work is not None else _done(None)

    def recv_anysource(self, tensors, tag=0):
        work = None
        for t in tensors:
            if t.is_cuda:
                raise NotImplementedError("glb backend: recv from any source is a host-transport feature; CUDA tensors "
                                          "travel over NVLink and match in posting order per peer (as with NCCL)")
            h = t if t.is_contiguous() else torch.empty(t.shape, dtype=t.dtype)
            buf = self.ctx.create_unbound_buffer(h.data_ptr(), h.numel() * h.element_size())
            buf.recv([r for r in range(self._world) if r != self._rank], self._slot(-1, self._rank, tag))
            work = _HostP2pWork(buf, False, (h, t), on_done=(lambda h=h, t=t: t.copy_(h)) if h is not t else None)
        return work if work is not None else _RecvWork(-1)

    def shutdown(self):
        try:
            self.ctx.close_connections()
        except Exception:  # noqa: BLE001 - shutting down anyway
            pass


def _create(store, rank: int, world_size: int, timeout: Optional[timedelta] = None):
    return GlbProcessGroup(store, rank, world_size, timeout or timedelta(minutes=30))


def register() -> None:
    """Idempotent registration of the "glb" backend with torch.distributed."""
    if BACKEND_NAME.upper() in getattr(dist.Backend, "backend_list", []) or \
            BACKEND_NAME in getattr(dist.Backend, "backend_list", []):
        return
    dist.Backend.register_backend(BACKEND_NAME, _create, devices=["cpu", "cuda"])


register()
