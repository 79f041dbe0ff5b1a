"""CUDA-buffer collectives over NVLink peer memory.

``CudaContext`` wraps the native PeerContext (topology exchange + symmetric pool)
and offers the collective suite for torch CUDA tensors. A tensor is either

* *registered* (``ctx.register(t)`` or allocated with ``ctx.empty(...)``): kernels
  read/write the peers' copies directly (zero-copy, NVLS-capable when symmetric);
* anything else: staged through the per-rank pool (``stage_bytes``) inside the same call.
  every collective takes any size: beyond the pool's bulk region (the pool minus two one-shot
  halves) the payload streams through it in one pipelined kernel.

Every method is asynchronous on the current torch stream unless ``stream`` is given,
and must be called in the same order on every rank.
"""
from __future__ import annotations

import weakref
from typing import Any, Dict, List, Optional, Sequence, Tuple

from .. import _C
from ..types import DataType, ReduceOp, describe, element_size

_cu = _C.cuda

ALGOS = {"auto": 0, "one_shot": 1, "two_shot": 2, "nvls": 3, "ll": 4, "pipelined": 5, "hybrid": 6, "ring": 10, "ring_chunked": 11,
         "halving_doubling": 12, "bcube": 13, "halving_doubling_pipelined": 14}


def _torch_dtype_to_glb(dtype) -> DataType:
    import torch

    return {torch.float32: DataType.FLOAT32, torch.float16: DataType.FLOAT16, torch.bfloat16: DataType.BFLOAT16,
            torch.float64: DataType.FLOAT64, torch.float8_e4m3fn: DataType.FLOAT8_E4M3,
            torch.float8_e5m2: DataType.FLOAT8_E5M2}[dtype]


def _stream(stream) -> int:
    if stream is None:
        import torch

        return torch.cuda.current_stream().cuda_stream
    if isinstance(stream, int):
        return stream
    return stream.cuda_stream


def _algo(a) -> int:
    return ALGOS[a] if isinstance(a, str) else int(a)


def new_stream(device: Optional[int] = None, high_priority: bool = False):
    """A dedicated CUDA stream as a torch ExternalStream (never shared through torch's pool)."""
    import torch

    device = torch.cuda.current_device() if device is None else device
    raw = _cu.create_stream(int(device), high_priority)
    return torch.cuda.ExternalStream(raw, device=device)


class _SymmetricStorage:
    """Exposes a PeerBuffer through __cuda_array_interface__ so torch can wrap it."""

    def __init__(self, buf, nbytes: int):
        self.buf = buf
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (buf.ptr, False), "version": 3, "strides": None,
        }


class CudaContext:
    def __init__(self, ctx, device: Optional[int] = None, stage_bytes: int = 0, use_vmm: bool = True,
                 use_nvls: bool = True):
        import torch

        if device is None:
            device = torch.cuda.current_device()
        self.ctx = ctx
        self.device = int(device)
        with torch.cuda.device(self.device):
            # One PeerContext per (context, device), shared with the old-style CUDA classes
            # (it is an attachment of the context): symmetric tensors allocated here are
            # recognised by CudaAllreduce* / CudaBroadcastOneToAll and get the NVLS path.
            self.pc = _cu.peer_context_for(ctx, self.device, stage_bytes, use_vmm, use_nvls)
        self.rank, self.size = self.pc.rank, self.pc.size
        # base ptr -> (PeerBuffer | weakref to the symmetric storage, nbytes)
        self._reg: Dict[int, Tuple[Any, int]] = {}

    # ---- memory -------------------------------------------------------------------------
    def register(self, tensor):
        """Collective: make ``tensor``'s memory addressable by every rank."""
        ptr, n, dt, cuda = describe(tensor)
        assert cuda, "register() needs a CUDA tensor"
        nbytes = n * element_size(dt)
        buf = self.pc.register_buffer(ptr, nbytes)
        self._reg[ptr] = (buf, nbytes)
        return buf

    def empty(self, shape, dtype):
        """Collective: allocate a symmetric tensor (peer-mapped, NVLS-bound when available)."""
        import math

        import torch

        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        n = math.prod(shape)
        es = torch.empty((), dtype=dtype).element_size()
        nbytes = max(16, n * es)
        buf = self.pc.alloc_symmetric(nbytes)
        store = _SymmetricStorage(buf, nbytes)
        flat = torch.as_tensor(store, device=f"cuda:{self.device}")
        t = flat[: n * es].view(dtype).view(shape)
        # The tensor keeps `store` (and through it the PeerBuffer) alive; when the last view
        # dies the symmetric memory and its multicast binding are released.
        self._reg[buf.ptr] = (weakref.ref(store), nbytes)
        return t

    def lookup(self, tensor) -> Tuple[Optional[Any], int]:
        """(PeerBuffer, byte offset) if ``tensor`` lies inside a registered region."""
        # torch reports data_ptr() 0 for an empty tensor; its place inside the storage still
        # decides the path, which must match the peers' (e.g. a rank that receives nothing in an
        # alltoallv into a registered buffer).
        ptr = tensor.data_ptr() if tensor.numel() else \
            tensor.untyped_storage().data_ptr() + tensor.storage_offset() * tensor.element_size()
        nbytes = tensor.numel() * tensor.element_size()
        dead = []
        found = (None, 0)
        for base, (ref, size) in self._reg.items():
            buf = ref
            if isinstance(ref, weakref.ref):
                store = ref()
                if store is None:
                    dead.append(base)
                    continue
                buf = store.buf
            if base <= ptr and ptr + nbytes <= base + size:
                found = (buf, ptr - base)
                break
        for b in dead:
            del self._reg[b]
        return found

    # ---- info ---------------------------------------------------------------------------
    def describe(self) -> str:
        return self.pc.describe()

    def topology(self):
        return self.pc.topology()

    def nvls_available(self) -> bool:
        return self.pc.nvls_available()

    # ---- collectives ----------------------------------------------------------------------
    def barrier(self, stream=None):
        _cu.barrier(self.pc, _stream(stream))

    def allreduce(self, tensor, op: ReduceOp = ReduceOp.SUM, algo="auto", out=None, stream=None, scale: float = 1.0,
                  average: bool = False, extra: Sequence = (), blocks: int = 0, unroll: int = 0, tile: int = 0):
        """In place on ``tensor`` (or tensor -> out), ONE kernel launch.

        ``scale`` / ``average`` (= 1/size) are applied to the fp32 accumulator inside the
        collective kernel, before the single rounding to the output dtype. ``out`` may have a
        different dtype (float32 <-> float16 / bfloat16, FP8 -> float32 / bfloat16 and
        float32 / bfloat16 -> FP8): registered tensors of any size, plain tensors up to the LL
        limit. FP8 results round to nearest even and saturate to the format's largest finite
        value. ``extra``: more local tensors of the same shape that are
        folded into the reduction and overwritten with the result (multi-pointer semantics).
        ``blocks`` / ``unroll`` / ``tile`` pin the launch shape (tuner)."""
        ptr, n, dt, _ = describe(tensor)
        s = _stream(stream)
        if average:
            scale = scale / self.size
        ex = [t.data_ptr() for t in extra]
        if out is None or out.data_ptr() == ptr:
            buf, off = self.lookup(tensor)
            if buf is not None:
                _cu.allreduce_registered(self.pc, buf, off, n, int(dt), int(op), _algo(algo), s, scale, ex, blocks,
                                         unroll, tile)
                return tensor
            _cu.allreduce(self.pc, ptr, ptr, n, int(dt), int(op), _algo(algo), s, scale, -1, ex, blocks, tile, unroll)
            return tensor
        _, _, odt, _ = describe(out)
        if odt != dt:
            ibuf, ioff = self.lookup(tensor)
            obuf, ooff = self.lookup(out)
            if ibuf is not None and obuf is not None and not ex:
                _cu.allreduce_cast(self.pc, ibuf, ioff, obuf, ooff, n, int(dt), int(odt), int(op), s, scale, blocks)
                return out
            _cu.allreduce(self.pc, ptr, out.data_ptr(), n, int(dt), int(op), _algo(algo), s, scale, int(odt), ex, blocks,
                          tile, unroll)
            return out
        _cu.allreduce(self.pc, ptr, out.data_ptr(), n, int(dt), int(op), _algo(algo), s, scale, -1, ex, blocks, tile, unroll)
        return out

    def plan(self, tensor, op: ReduceOp = ReduceOp.SUM) -> dict:
        """What ``algo="auto"`` resolves to for this tensor (variant + launch shape)."""
        _, n, dt, _ = describe(tensor)
        buf, off = self.lookup(tensor)
        kind = 2 if buf is None else (0 if (buf.has_multicast and off % 16 == 0) else 1)
        return _cu.plan_allreduce(self.pc, n * element_size(dt), int(dt), int(op), kind)

    @staticmethod
    def _norm_fp8_out(name, partial, norm, out, out_scales, shape):
        """The FP8 form's checks of ``out`` / ``out_scales`` (``shape``: out's shape): ``(quant, out)``,
        with ``out`` allocated when not given. An FP8 ``out`` needs ``out_scales``."""
        import torch

        fp8 = (torch.float8_e4m3fn, torch.float8_e5m2)
        if out_scales is None:
            if out is not None and out.dtype in fp8:
                raise ValueError(f"{name}: an FP8 out needs out_scales (float32 {(*shape[:-1], 1)})")
            return False, out
        form = f"the FP8 form takes float8_e4m3fn out {tuple(shape)} and float32 out_scales {(*shape[:-1], 1)}"
        if norm is None:
            raise ValueError(f"{name}: out_scales needs a norm; {form}")
        if shape[-1] % 16:
            raise ValueError(f"{name}: the FP8 out needs rows of a multiple of 16 elements, got {shape[-1]}")
        if out is None:
            out = torch.empty(tuple(shape), dtype=torch.float8_e4m3fn, device=partial.device)
        for key, t, dtype, want in (("out", out, torch.float8_e4m3fn, tuple(shape)),
                                    ("out_scales", out_scales, torch.float32, (*shape[:-1], 1))):
            if not isinstance(t, torch.Tensor) or t.dtype != dtype:
                raise ValueError(f"{name}: {key} must be a {dtype} tensor, got {getattr(t, 'dtype', type(t))}; {form}")
            if not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != want:
                raise ValueError(f"{name}: {key} must be a contiguous CUDA tensor of shape {want}, got "
                                 f"{tuple(t.shape)} on {t.device}{'' if t.is_contiguous() else ', not contiguous'}")
        return True, out

    def allreduce_residual_norm(self, partial, residual, weight=None, norm_bias=None, *, norm: Optional[str] = "rms",
                                eps: float = 1e-6, bias=None, residual_out=None, out=None, algo="auto", stream=None,
                                out_scales=None):
        """The row-parallel output step of tensor parallelism in ONE kernel launch: allreduce of the
        partial sums, ``+ bias``, ``+ residual`` and the next norm.

        For every row (the last dimension is the hidden size H): ``residual_out = round(sum over ranks
        of partial + bias + residual)`` in fp32, rounded once; ``out`` = RMSNorm (``norm="rms"``:
        ``x / sqrt(mean(x^2) + eps) * weight``) or LayerNorm (``norm="layer"``: ``(x - mean) /
        sqrt(var + eps) * weight + norm_bias``) of that rounded ``residual_out``, statistics in fp32,
        rounded once. ``norm=None`` writes ``residual_out`` only.

        Every tensor is float32, bfloat16 or float16 (one dtype), contiguous and 16-byte aligned; H *
        element size is a multiple of 16 bytes and H is at most ``MAX_NORM_HIDDEN`` (16384).
        ``residual``, ``bias``, ``weight`` and ``norm_bias`` must be the same on every rank; every rank
        then gets the same bytes. ``residual_out`` defaults to ``residual`` (in place); ``out`` is
        allocated when not given. ``algo``: ``"auto"`` (the allreduce's choice for a plain tensor of
        the same size), ``"ll"``, ``"one_shot"`` or ``"two_shot"``. Invalid arguments raise
        ``ValueError`` before anything is launched.

        FP8 ``out`` for an FP8 GEMM: passing ``out_scales`` (float32, shape ``out.shape[:-1] + (1,)``,
        the ``(M, 1)`` row-wise scales of ``scaled_mm``) makes ``out`` float8_e4m3fn codes (allocated
        when not given) of the row ``o`` that the call without it writes, in the same launch: per
        row ``amax = max(max |o|, 1e-4)``, ``out = e4m3(o * (448 / amax))`` (round to nearest even,
        saturating) and ``out_scales = amax / 448``, so ``o ~= out * out_scales``. It needs a norm and
        H a multiple of 16; ``residual_out`` is what the call without it writes. torch reproduces
        every byte: ``(o.float() * (448.0 / a)).to(torch.float8_e4m3fn)`` and ``a /
        torch.full_like(a, 448.0)`` with ``a = o.float().abs().amax(-1, keepdim=True).clamp_min(1e-4)``.

        Returns ``(residual_out, out)``, or ``residual_out`` when ``norm`` is None."""
        import torch

        kinds = {None: 0, "rms": 1, "layer": 2}
        if norm not in kinds:
            raise ValueError(f"allreduce_residual_norm: norm must be 'rms', 'layer' or None, got {norm!r}")
        if algo not in ("auto", "ll", "one_shot", "two_shot"):
            raise ValueError(f"allreduce_residual_norm: algo must be auto, ll, one_shot or two_shot, got {algo!r}")
        if norm != "layer" and norm_bias is not None:
            raise ValueError("allreduce_residual_norm: norm_bias needs norm='layer'")
        if norm is None and weight is not None:
            raise ValueError("allreduce_residual_norm: weight needs a norm")
        if partial.dim() == 0:
            raise ValueError("allreduce_residual_norm: partial must have a hidden dimension")
        H = partial.shape[-1]
        if residual_out is None:
            residual_out = residual
        quant, out = self._norm_fp8_out("allreduce_residual_norm", partial, norm, out, out_scales, tuple(partial.shape))
        if norm is not None and out is None:
            out = torch.empty_like(partial, memory_format=torch.contiguous_format)
        named = {"partial": partial, "residual": residual, "residual_out": residual_out, "out": out, "bias": bias,
                 "weight": weight, "norm_bias": norm_bias}
        for name, t in named.items():
            if t is None or (quant and name == "out"):
                continue
            if not t.is_cuda or t.dtype != partial.dtype or not t.is_contiguous():
                raise ValueError(f"allreduce_residual_norm: {name} must be a contiguous CUDA tensor of {partial.dtype}, "
                                 f"got {t.dtype} on {t.device}{'' if t.is_contiguous() else ', not contiguous'}")
            want = (H,) if name in ("bias", "weight", "norm_bias") else tuple(partial.shape)
            if tuple(t.shape) != want:
                raise ValueError(f"allreduce_residual_norm: {name} has shape {tuple(t.shape)}, expected {want}")
        _, _, dt, _ = describe(partial)
        ptr = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
        _cu.allreduce_residual_norm(self.pc, ptr(partial), ptr(residual), ptr(residual_out), ptr(out), ptr(bias),
                                    ptr(weight), ptr(norm_bias), partial.numel() // max(H, 1), H, int(dt), kinds[norm],
                                    float(eps), _algo(algo), _stream(stream), ptr(out_scales))
        return residual_out if norm is None else (residual_out, out)

    def reduce_scatter_residual_norm(self, partial, residual, weight=None, norm_bias=None, *,
                                     norm: Optional[str] = "rms", eps: float = 1e-6, bias=None, residual_out=None,
                                     out=None, gather_out: bool = True, stream=None, out_scales=None):
        """The row-parallel output step of sequence parallelism in ONE kernel launch: reduce-scatter
        of the partial sums over token shards, ``+ bias``, ``+ residual`` and the next norm, whose
        output is optionally allgathered.

        ``partial`` is ``(T, ...)`` with T = P * Ts on every rank; this rank owns rows ``[rank * Ts,
        (rank + 1) * Ts)`` along dim 0, and ``residual`` / ``residual_out`` are that shard, shape
        ``(Ts, ...)``. ``residual_out = round(sum over ranks of partial[shard rows] + bias +
        residual)`` and ``out`` = the norm of it, with the sum order, rounding and limits of
        :meth:`allreduce_residual_norm`, so the bytes equal the matching rows of its outputs.
        ``out`` has ``partial``'s shape with ``gather_out`` (every rank gets every shard, shard q at
        rows ``q * Ts``) and ``residual``'s shape without. ``bias``, ``weight`` and ``norm_bias`` must
        be the same on every rank. ``residual_out`` defaults to ``residual`` (in place); ``out`` is
        allocated when not given. Invalid arguments raise ``ValueError`` before anything is launched.

        ``out_scales``: the FP8 form of :meth:`allreduce_residual_norm`, with ``out``'s rows (with
        ``gather_out`` every shard's codes and scales, shard q at rows ``q * Ts``); the gathered rows
        travel as H code bytes and one scale each.

        Returns ``(residual_out, out)``, or ``residual_out`` when ``norm`` is None."""
        import torch

        kinds = {None: 0, "rms": 1, "layer": 2}
        name = "reduce_scatter_residual_norm"
        if norm not in kinds:
            raise ValueError(f"{name}: norm must be 'rms', 'layer' or None, got {norm!r}")
        if norm != "layer" and norm_bias is not None:
            raise ValueError(f"{name}: norm_bias needs norm='layer'")
        if norm is None and weight is not None:
            raise ValueError(f"{name}: weight needs a norm")
        if partial.dim() < 2:
            raise ValueError(f"{name}: partial must have a token and a hidden dimension")
        T, H = partial.shape[0], partial.shape[-1]
        if T % self.size:
            raise ValueError(f"{name}: {T} rows do not split into {self.size} equal shards")
        shard = (T // self.size, *partial.shape[1:])
        if residual_out is None:
            residual_out = residual
        quant, out = self._norm_fp8_out(name, partial, norm, out, out_scales,
                                        tuple(partial.shape) if gather_out else shard)
        if norm is not None and out is None:
            out = torch.empty(tuple(partial.shape) if gather_out else shard, dtype=partial.dtype, device=partial.device)
        named = {"partial": partial, "residual": residual, "residual_out": residual_out, "out": out, "bias": bias,
                 "weight": weight, "norm_bias": norm_bias}
        for key, t in named.items():
            if t is None or (quant and key == "out"):
                continue
            if not t.is_cuda or t.dtype != partial.dtype or not t.is_contiguous():
                raise ValueError(f"{name}: {key} must be a contiguous CUDA tensor of {partial.dtype}, "
                                 f"got {t.dtype} on {t.device}{'' if t.is_contiguous() else ', not contiguous'}")
            if key in ("bias", "weight", "norm_bias"):
                want = (H,)
            elif key == "partial" or (key == "out" and gather_out):
                want = tuple(partial.shape)
            else:
                want = shard
            if tuple(t.shape) != want:
                raise ValueError(f"{name}: {key} has shape {tuple(t.shape)}, expected {want}")
        _, _, dt, _ = describe(partial)
        ptr = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
        _cu.reduce_scatter_residual_norm(self.pc, ptr(partial), ptr(residual), ptr(residual_out), ptr(out), ptr(bias),
                                         ptr(weight), ptr(norm_bias), partial.numel() // max(H, 1), H, int(dt),
                                         kinds[norm], float(eps), bool(gather_out), _stream(stream), ptr(out_scales))
        return residual_out if norm is None else (residual_out, out)

    def reduce_scatter_residual_norm_backward(self, grad_out, residual_out, grad_residual_out=None, weight=None, *,
                                              norm: str, eps: float = 1e-6, gather_out: bool = True,
                                              grad_partial=None, grad_residual=None, grad_weight=None,
                                              grad_norm_bias=None, grad_bias=None, stream=None):
        """The backward of :meth:`reduce_scatter_residual_norm` with a norm, in ONE kernel launch
        per chunk: the reduce-scatter of a gathered ``out``'s gradient, the norm's backward on
        this rank's shard, the add of ``residual_out``'s gradient and the allgather of the sum.

        ``residual_out`` is the forward's saved shard ``(Ts, ...)``; ``grad_residual_out`` its
        gradient (None counts as zero); ``grad_out`` the gradient of ``out``: ``(T, ...)`` with
        ``gather_out`` (this rank's partial of it), ``(Ts, ...)`` without. ``norm``, ``eps``,
        ``weight`` and ``gather_out`` are the forward's. Per row, in fp32, with ``g`` the sum over
        ranks of ``grad_out`` (rank order) and the statistics recomputed exactly as the forward
        computed them: ``grad_residual = round(grad_residual_out + the norm's input gradient)``.
        ``grad_partial`` ``(T, ...)`` gets every rank's ``grad_residual`` shards (shard q at rows
        ``q * Ts``), the same bytes on every rank: the gradient of ``partial``. ``grad_residual``
        (this rank's rows of it) may be ``grad_residual_out`` itself. Both are allocated when not
        given. ``grad_weight`` (sum of ``g * xhat``), ``grad_norm_bias`` (sum of ``g``, layer only)
        and ``grad_bias`` (sum of the rounded ``grad_residual`` rows) are column sums over this
        rank's rows, fp32, rounded once, in a fixed order: each is computed into the ``(H,)`` tensor
        given and skipped when None. The fp32 workspace they need comes from torch's allocator, on
        the stream the call runs on.
        Invalid arguments raise ``ValueError`` before anything is launched.

        Returns ``(grad_partial, grad_residual, grad_weight, grad_norm_bias, grad_bias)``."""
        import torch

        kinds = {"rms": 1, "layer": 2}
        name = "reduce_scatter_residual_norm_backward"
        if norm not in kinds:
            raise ValueError(f"{name}: norm must be 'rms' or 'layer', got {norm!r}")
        if norm != "layer" and grad_norm_bias is not None:
            raise ValueError(f"{name}: grad_norm_bias needs norm='layer'")
        if residual_out.dim() < 2:
            raise ValueError(f"{name}: residual_out must have a token and a hidden dimension")
        shard, H = tuple(residual_out.shape), residual_out.shape[-1]
        full = (self.size * shard[0], *shard[1:])
        if grad_partial is None:
            grad_partial = torch.empty(full, dtype=residual_out.dtype, device=residual_out.device)
        if grad_residual is None:
            grad_residual = torch.empty(shard, dtype=residual_out.dtype, device=residual_out.device)
        named = {"grad_out": grad_out, "residual_out": residual_out, "grad_residual_out": grad_residual_out,
                 "weight": weight, "grad_partial": grad_partial, "grad_residual": grad_residual,
                 "grad_weight": grad_weight, "grad_norm_bias": grad_norm_bias, "grad_bias": grad_bias}
        for key, t in named.items():
            if t is None:
                continue
            if not t.is_cuda or t.dtype != residual_out.dtype or not t.is_contiguous():
                raise ValueError(f"{name}: {key} must be a contiguous CUDA tensor of {residual_out.dtype}, "
                                 f"got {t.dtype} on {t.device}{'' if t.is_contiguous() else ', not contiguous'}")
            if key in ("weight", "grad_weight", "grad_norm_bias", "grad_bias"):
                want = (H,)
            elif key == "grad_partial" or (key == "grad_out" and gather_out):
                want = full
            else:
                want = shard
            if tuple(t.shape) != want:
                raise ValueError(f"{name}: {key} has shape {tuple(t.shape)}, expected {want}")
        _, _, dt, _ = describe(residual_out)
        rows = self.size * (residual_out.numel() // max(H, 1))
        vectors = sum(t is not None for t in (grad_weight, grad_norm_bias, grad_bias))
        plan = _cu.plan_reduce_scatter_norm_backward(self.pc, rows, H, int(dt), kinds[norm], bool(gather_out), vectors)
        launch = _stream(stream)
        ws = self._norm_workspace(plan["workspace_bytes"], residual_out.device, stream, launch)
        ptr = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
        _cu.reduce_scatter_residual_norm_backward(
            self.pc, ptr(grad_out), ptr(residual_out), ptr(grad_residual_out), ptr(grad_residual), ptr(grad_partial),
            ptr(weight), ptr(grad_weight), ptr(grad_norm_bias), ptr(grad_bias), ptr(ws),
            0 if ws is None else ws.numel(), rows, H, int(dt), kinds[norm], float(eps), bool(gather_out), launch)
        return grad_partial, grad_residual, grad_weight, grad_norm_bias, grad_bias

    def allreduce_residual_norm_backward(self, grad_out, residual_out, grad_residual_out=None, weight=None, *,
                                         norm: str, eps: float = 1e-6, grad_partial=None, grad_weight=None,
                                         grad_norm_bias=None, grad_bias=None, algo: str = "auto", stream=None):
        """The backward of :meth:`allreduce_residual_norm` with a norm, in ONE kernel launch per
        chunk: the allreduce of this rank's partial of ``out``'s gradient, the norm's backward and
        the add of ``residual_out``'s gradient.

        ``residual_out`` is the forward's saved output ``(T, ...)``, the same on every rank;
        ``grad_residual_out`` its gradient (None counts as zero), also the same on every rank;
        ``grad_out`` this rank's partial of the gradient of ``out``, ``(T, ...)``. ``norm``, ``eps``
        and ``weight`` are the forward's. Per row, in fp32, with ``g`` the sum over ranks of
        ``grad_out`` (rank order) and the statistics recomputed exactly as the forward computed
        them: ``grad_partial = round(grad_residual_out + the norm's input gradient)``, the gradient
        of both ``partial`` and ``residual``, the same bytes on every rank and for every ``algo``.
        It may be ``grad_residual_out`` itself and is allocated when not given. ``grad_weight`` (sum
        of ``g * xhat``), ``grad_norm_bias`` (sum of ``g``, layer only) and ``grad_bias`` (sum of the
        rounded ``grad_partial`` rows) are column sums over all rows, fp32, rounded once, in a fixed
        order, the same bytes on every rank: each is computed into the ``(H,)`` tensor given and
        skipped when None. The fp32 workspace they need comes from torch's allocator, on the stream
        the call runs on. ``algo``: ``"auto"`` (the forward's choice for these rows, its LL as the
        one-shot), ``"one_shot"`` or ``"two_shot"``. Invalid arguments raise ``ValueError`` before
        anything is launched.

        Returns ``(grad_partial, grad_weight, grad_norm_bias, grad_bias)``."""
        import torch

        kinds = {"rms": 1, "layer": 2}
        name = "allreduce_residual_norm_backward"
        if norm not in kinds:
            raise ValueError(f"{name}: norm must be 'rms' or 'layer', got {norm!r}")
        if algo not in ("auto", "one_shot", "two_shot"):
            raise ValueError(f"{name}: algo must be auto, one_shot or two_shot, got {algo!r}")
        if norm != "layer" and grad_norm_bias is not None:
            raise ValueError(f"{name}: grad_norm_bias needs norm='layer'")
        if residual_out.dim() == 0:
            raise ValueError(f"{name}: residual_out must have a hidden dimension")
        H = residual_out.shape[-1]
        if grad_partial is None:
            grad_partial = torch.empty_like(residual_out, memory_format=torch.contiguous_format)
        named = {"grad_out": grad_out, "residual_out": residual_out, "grad_residual_out": grad_residual_out,
                 "weight": weight, "grad_partial": grad_partial, "grad_weight": grad_weight,
                 "grad_norm_bias": grad_norm_bias, "grad_bias": grad_bias}
        for key, t in named.items():
            if t is None:
                continue
            if not t.is_cuda or t.dtype != residual_out.dtype or not t.is_contiguous():
                raise ValueError(f"{name}: {key} must be a contiguous CUDA tensor of {residual_out.dtype}, "
                                 f"got {t.dtype} on {t.device}{'' if t.is_contiguous() else ', not contiguous'}")
            want = (H,) if key in ("weight", "grad_weight", "grad_norm_bias", "grad_bias") else tuple(residual_out.shape)
            if tuple(t.shape) != want:
                raise ValueError(f"{name}: {key} has shape {tuple(t.shape)}, expected {want}")
        _, _, dt, _ = describe(residual_out)
        rows = residual_out.numel() // max(H, 1)
        vectors = sum(t is not None for t in (grad_weight, grad_norm_bias, grad_bias))
        plan = _cu.plan_residual_norm_backward(self.pc, rows, H, int(dt), kinds[norm], vectors, _algo(algo))
        launch = _stream(stream)
        ws = self._norm_workspace(plan["workspace_bytes"], residual_out.device, stream, launch)
        ptr = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
        _cu.allreduce_residual_norm_backward(
            self.pc, ptr(grad_out), ptr(residual_out), ptr(grad_residual_out), ptr(grad_partial), ptr(weight),
            ptr(grad_weight), ptr(grad_norm_bias), ptr(grad_bias), ptr(ws), 0 if ws is None else ws.numel(), rows, H,
            int(dt), kinds[norm], float(eps), _algo(algo), launch)
        return grad_partial, grad_weight, grad_norm_bias, grad_bias

    @staticmethod
    def _norm_workspace(nbytes, dev, stream, launch):
        """The column sums' fp32 workspace of a norm backward, or None: a temporary of the call,
        allocated on the stream its kernels run on, so that the caching allocator reuses it only for
        work ordered after them."""
        import torch

        if not nbytes:
            return None
        if launch == torch.cuda.current_stream(dev).cuda_stream:
            return torch.empty(nbytes, dtype=torch.uint8, device=dev)
        on = stream if isinstance(stream, torch.cuda.Stream) else torch.cuda.ExternalStream(launch, device=dev)
        with torch.cuda.stream(on):
            return torch.empty(nbytes, dtype=torch.uint8, device=dev)

    # ---- health ---------------------------------------------------------------------------
    def set_timeout(self, ms: int):
        """Device-side waits give up after ``ms`` milliseconds (then the context is poisoned)."""
        self.pc.set_timeout(int(ms))

    def check_health(self):
        """Raise ``IoError`` if a device-side wait timed out (the context is then unusable), or
        ``ValueError`` (``InputError``) once if a kernel found invalid device-side input, such as
        the splits of :meth:`alltoallv_dev`."""
        self.pc.check_health()

    def synchronize(self, stream=None):
        """Wait for the stream and raise ``IoException`` if a peer went missing meanwhile."""
        self.pc.synchronize(_stream(stream))

    # ---- point to point ---------------------------------------------------------------------
    def send(self, tensor, dst: int, stream=None):
        """Stream ``tensor`` to rank ``dst`` over NVLink (matched with its recv in posting order)."""
        _cu.send(self.pc, tensor.data_ptr(), tensor.numel() * tensor.element_size(), dst, _stream(stream))

    def recv(self, tensor, src: int, stream=None):
        _cu.recv(self.pc, tensor.data_ptr(), tensor.numel() * tensor.element_size(), src, _stream(stream))
        return tensor

    def sendrecv(self, send_tensor, dst: int, recv_tensor, src: int, stream=None):
        """Both directions in one kernel: the call for ring / pipeline exchanges."""
        _cu.sendrecv(self.pc, send_tensor.data_ptr(), send_tensor.numel() * send_tensor.element_size(), dst,
                     recv_tensor.data_ptr(), recv_tensor.numel() * recv_tensor.element_size(), src, _stream(stream))
        return recv_tensor

    def exchange(self, send_tensor, dst: int, recv_tensor, src: int, stream=None):
        """Zero-copy sendrecv: ``recv_tensor`` is a registered / symmetric tensor that EVERY rank passes at the
        same offset; my payload is written straight into ``dst``'s copy of it, ``src`` writes into mine.

        One kernel and one pass over the data (sendrecv() stages through a mailbox ring). Falls back to
        sendrecv() when ``recv_tensor`` is not registered."""
        buf, off = self.lookup(recv_tensor)
        if buf is None:
            return self.sendrecv(send_tensor, dst, recv_tensor, src, stream)
        _cu.exchange(self.pc, send_tensor.data_ptr(), send_tensor.numel() * send_tensor.element_size(), dst, buf, off,
                     recv_tensor.numel() * recv_tensor.element_size(), src, _stream(stream))
        return recv_tensor

    def put(self, local, remote, peer: int, remote_offset: int = 0, stream=None):
        """One-sided: copy ``local`` into rank ``peer``'s copy of the registered tensor ``remote``."""
        buf, off = self.lookup(remote)
        assert buf is not None, "put() needs a registered / symmetric remote tensor"
        _cu.put(self.pc, local.data_ptr(), buf, off + remote_offset * remote.element_size(),
                local.numel() * local.element_size(), peer, _stream(stream))

    def get(self, local, remote, peer: int, remote_offset: int = 0, stream=None):
        """One-sided: read rank ``peer``'s copy of the registered tensor ``remote`` into ``local``."""
        buf, off = self.lookup(remote)
        assert buf is not None, "get() needs a registered / symmetric remote tensor"
        _cu.get(self.pc, local.data_ptr(), buf, off + remote_offset * remote.element_size(),
                local.numel() * local.element_size(), peer, _stream(stream))
        return local

    def broadcast(self, tensor, root: int = 0, stream=None):
        ptr, n, dt, _ = describe(tensor)
        nbytes = n * element_size(dt)
        buf, off = self.lookup(tensor)
        if buf is not None:
            _cu.broadcast_reg(self.pc, buf, off, nbytes, root, _stream(stream))
        else:
            _cu.broadcast(self.pc, ptr, nbytes, root, _stream(stream))
        return tensor

    def allgather(self, output, input, stream=None):
        """Every rank's ``input`` (same size on all ranks), concatenated in rank order. Any size:
        a plain ``output`` larger than the staging pool streams through it in one kernel; ``input``
        may be this rank's slice of ``output`` (in place). A float32 ``input`` and a bfloat16 /
        float16 ``output`` take the cast form (see :meth:`allgatherv`)."""
        return self.allgatherv(output, input, [input.numel()] * self.size, stream)

    def allgatherv(self, output, input, counts: Sequence[int], stream=None):
        """Like :meth:`allgather` with ``counts[r]`` elements from rank r (zero allowed); any size.

        When ``output.dtype != input.dtype`` this is the cast form: a float32 ``input`` and a
        bfloat16 / float16 ``output``. Each rank rounds its block once to the output dtype as it
        reads it (round to nearest even, overflow to +-inf, NaN stays NaN: ``input.to(dtype)``),
        so only 16-bit bytes cross NVLink and every rank gets the same bytes, one kernel launch.
        ``input`` must not overlap ``output``. Other pairs raise ``ValueError``."""
        buf, off = self.lookup(output)
        iptr = input.data_ptr() if input is not None else 0
        if input is not None and input.dtype != output.dtype:
            _, _, idt, _ = describe(input)
            _, _, odt, _ = describe(output)
            counts = [int(c) for c in counts]
            if buf is not None:
                _cu.allgatherv_cast_reg(self.pc, iptr, int(idt), buf, off, counts, int(odt), _stream(stream))
            else:
                _cu.allgatherv_cast(self.pc, iptr, int(idt), output.data_ptr(), counts, int(odt), _stream(stream))
            return output
        es = output.element_size()
        sizes = [int(c) * es for c in counts]
        if buf is not None:
            _cu.allgatherv_reg(self.pc, iptr, buf, off, sizes, _stream(stream))
        else:
            _cu.allgatherv(self.pc, iptr, output.data_ptr(), sizes, _stream(stream))
        return output

    def gather(self, output, input, root: int = 0, stream=None):
        """Every rank's ``input`` into the root's ``output``, in rank order; any size. A non-root's
        output is never written. Each rank picks the path from its own ``output``, so the ranks
        must agree: when the root's output is registered / symmetric, every rank passes its copy
        of that registered tensor at the same offset; when it is plain, other ranks pass None or a
        plain tensor. Mixing the two gives a wrong result or leaves the ranks waiting."""
        return self.gatherv(output, input, [input.numel()] * self.size, root, stream)

    def gatherv(self, output, input, counts: Sequence[int], root: int = 0, stream=None):
        """Like :meth:`gather` with ``counts[r]`` elements from rank r; any size. The same rule on
        registered and None outputs applies."""
        es = input.element_size()
        sizes = [int(c) * es for c in counts]
        optr = output.data_ptr() if output is not None else 0
        buf, off = (self.lookup(output) if output is not None else (None, 0))
        if buf is not None:
            _cu.gatherv_reg(self.pc, input.data_ptr(), buf, off, sizes, root, _stream(stream))
        else:
            _cu.gatherv(self.pc, input.data_ptr(), optr, sizes, root, _stream(stream))
        return output

    def alltoall(self, output, input, stream=None):
        """Fixed-size exchange: chunk j of ``input`` goes to rank j (one size for all ranks). Any size;
        a plain ``input`` and ``output`` must not overlap (ValueError beyond the staged path), nor
        may ``input`` overlap a registered / symmetric ``output`` above the LL limit (ValueError:
        the push kernel writes a peer's output while that peer still reads its input there)."""
        per = input.numel() // self.size * input.element_size()
        buf, off = self.lookup(output)
        if buf is not None:
            _cu.alltoall_reg(self.pc, input.data_ptr(), buf, off, per, _stream(stream))
        else:
            _cu.alltoall(self.pc, input.data_ptr(), output.data_ptr(), per, _stream(stream))
        return output

    def alltoallv(self, output, out_counts: Sequence[int], input, in_counts: Sequence[int], stream=None):
        """Block j of ``input`` (``in_counts[j]`` elements) goes to rank j; the block from rank q lands
        in ``output`` after the blocks of ranks < q (``out_counts[q]`` elements). Any size. A plain
        ``input`` and ``output`` must not overlap, at any size (``gloo_b200._C.InputError``, a
        ValueError): the plain alltoallv always runs the pipelined kernel, which writes the output
        while it still reads the input. Earlier versions staged a call that fit the pool, so a small
        in-place call used to work; it now raises. The same holds for a registered / symmetric
        ``output``: its push kernel writes peers' outputs while they still read their inputs."""
        es = input.element_size()
        send = [int(c) * es for c in in_counts]
        recv = [int(c) * es for c in out_counts]
        buf, off = self.lookup(output)
        if buf is not None:
            _cu.alltoallv_reg(self.pc, input.data_ptr(), send, buf, off, recv, _stream(stream))
        else:
            _cu.alltoallv(self.pc, input.data_ptr(), send, output.data_ptr(), recv, _stream(stream))
        return output

    def _dev_rows(self, out, inp) -> int:
        """Bytes of one row (everything but dim 0); ``out`` and ``inp`` must agree on it."""
        _, _, dt, icuda = describe(inp)
        _, _, odt, ocuda = describe(out)
        if not (icuda and ocuda):
            raise ValueError("alltoallv_dev needs CUDA tensors")
        if odt != dt or tuple(out.shape[1:]) != tuple(inp.shape[1:]) or inp.dim() == 0:
            raise ValueError(f"alltoallv_dev: rows of out {tuple(out.shape)} {out.dtype} and input "
                             f"{tuple(inp.shape)} {inp.dtype} differ")
        row = 1
        for d in inp.shape[1:]:
            row *= int(d)
        if row == 0:
            raise ValueError("alltoallv_dev: rows must not be empty")
        return row * element_size(dt)

    def _dev_index(self, t, name: str, n: int) -> int:
        import torch

        if (not isinstance(t, torch.Tensor) or t.dtype != torch.int64 or not t.is_cuda
                or t.device.index != self.device or not t.is_contiguous() or t.numel() != n):
            raise ValueError(f"alltoallv_dev: {name} must be a contiguous int64 tensor of {n} entries on "
                             f"cuda:{self.device}")
        return t.data_ptr()

    def _dev_tensors(self, name: str, tensors, contiguous: bool = True) -> None:
        """Every tensor of ``tensors`` (a name -> tensor mapping) is a CUDA tensor on this context's
        device and, unless ``contiguous`` is False, contiguous."""
        import torch

        for what, t in tensors.items():
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
                raise ValueError(f"{name}: {what} must be a CUDA tensor on cuda:{self.device}")
            if contiguous and not t.is_contiguous():
                raise ValueError(f"{name}: {what} must be contiguous")

    @staticmethod
    def _dev_disjoint(name: str, a, a_name: str, b, b_name: str) -> None:
        """``a`` and ``b`` share no byte."""
        a0, a1 = a.data_ptr(), a.data_ptr() + a.numel() * a.element_size()
        b0, b1 = b.data_ptr(), b.data_ptr() + b.numel() * b.element_size()
        if a0 < b1 and b0 < a1:
            raise ValueError(f"{name}: {a_name} and {b_name} overlap")

    def _fp8_dispatch(self, name: str, in_name: str, inp, out, out_scales):
        """The quantising dispatch's tensors: ``inp`` bfloat16 ``(rows, H)`` with H a multiple of 128,
        ``out`` float8_e4m3fn ``(cap, H)`` and ``out_scales`` float32 ``(cap, H // 128)``, contiguous
        CUDA tensors on this device, ``inp`` and ``out`` 16-byte aligned. Returns H and the binding's
        scales arguments (registration, offset, pointer)."""
        import torch

        form = (f"the quantising {name} takes bfloat16 {in_name} (rows, H) with H a multiple of 128, "
                "float8_e4m3fn out (cap, H) and float32 out_scales (cap, H // 128)")
        if out_scales is None:
            raise ValueError(f"{name}: out_scales missing; {form}")
        if inp.dtype != torch.bfloat16 or out.dtype != torch.float8_e4m3fn:
            raise ValueError(f"{name}: got {inp.dtype} {in_name} and {out.dtype} out; {form}")
        if not isinstance(out_scales, torch.Tensor) or out_scales.dtype != torch.float32:
            raise ValueError(f"{name}: out_scales must be a float32 tensor; {form}")
        tensors = (inp, out, out_scales)
        if not all(t.is_cuda and t.device.index == self.device for t in tensors):
            raise ValueError(f"{name}: {in_name}, out and out_scales must be CUDA tensors on cuda:{self.device}")
        if inp.dim() != 2 or out.dim() != 2 or out_scales.dim() != 2:
            raise ValueError(f"{name}: {in_name} {tuple(inp.shape)}, out {tuple(out.shape)} and out_scales "
                             f"{tuple(out_scales.shape)} must be 2-D; {form}")
        H, cap = int(inp.shape[1]), int(out.shape[0])
        if H == 0 or H % 128 != 0:
            raise ValueError(f"{name}: row length {H} is not a positive multiple of 128; {form}")
        if int(out.shape[1]) != H or tuple(out_scales.shape) != (cap, H // 128):
            raise ValueError(f"{name}: out {tuple(out.shape)} and out_scales {tuple(out_scales.shape)} do not "
                             f"match {in_name} rows of {H}; {form}")
        if not all(t.is_contiguous() for t in tensors):
            raise ValueError(f"{name}: {in_name}, out and out_scales must be contiguous")
        if inp.data_ptr() % 16 != 0 or out.data_ptr() % 16 != 0:
            raise ValueError(f"{name}: {in_name} and out must be 16-byte aligned for the quantising form")
        sbuf, soff = self.lookup(out_scales)
        return H, sbuf, soff, out_scales.data_ptr()

    def alltoallv_dev(self, out, inp, in_splits, out_splits, out_offsets, experts: int = 1, align: int = 1,
                      out_scales=None, stream=None):
        """All-to-all-v whose row counts stay on the device: no host synchronisation, graph-capturable.

        ``in_splits`` (int64 CUDA tensor of ``size * experts`` entries): entry ``j * experts + e`` is
        how many rows of ``inp`` (packed in that order) go to local expert ``e`` of rank ``j``. Each
        rank receives expert-major into ``out``: the segment of expert ``e`` starts at a multiple of
        ``align`` rows and holds the rows of ranks 0, 1, ... in order; ``out_splits[e * size + s]`` and
        ``out_offsets[e * size + s]`` receive the row count and first row of the part from rank ``s``.
        ``out.shape[0]`` is the capacity: a rank that would need more rows receives none. That, or
        invalid splits, is raised as ``ValueError`` on every rank by the first host call on this
        context made after the stream has passed the failed call. Check with ``synchronize()`` (or
        ``check_health()`` after a stream sync) at a point every rank reaches: a rank whose stream
        has not run the call yet does not know about it, and a collective that raises on one rank
        only would leave its peers waiting.
        Registered / symmetric ``out``: zero copy; any other tensor goes through the staging pool.

        Quantising form (FP8 expert dispatch, the 1x128 per-token-group recipe): ``inp`` bf16
        ``(rows, H)`` with H a multiple of 128, ``out`` float8_e4m3fn ``(cap, H)`` and ``out_scales``
        a contiguous float32 ``(cap, H // 128)`` CUDA tensor. The sender quantises while it sends, so
        the link carries FP8. Each row lands at the same index in ``out`` and ``out_scales``, and
        ``x ~= float(code) * scale``. Per block of 128 elements, in fp32 with correct rounding:
        ``amax = max(max |x|, 1e-4)``, ``code = e4m3(x * (448 * (1 / amax)))`` (round to nearest
        even, saturating), ``scale = amax / 448``: what torch computes for
        ``(x.float() * (448.0 / amax)).to(torch.float8_e4m3fn)`` and ``amax / 448.0``, byte for byte.
        NaN and infinite inputs are not supported. ``inp`` and
        ``out`` must be 16-byte aligned, and ``out`` and ``out_scales`` both registered / symmetric
        (zero copy) or both plain (staged; the capacity is then also capped by what fits the pool at
        H + H / 32 bytes a row). Other dtype pairs (other inputs, e5m2) raise ``ValueError``."""
        quant = out_scales is not None or self._is_fp8_dispatch(out, inp)
        sbuf, soff, sptr = None, 0, 0
        if quant:
            rb, sbuf, soff, sptr = self._fp8_dispatch("alltoallv_dev", "input", inp, out, out_scales)
        else:
            rb = self._dev_rows(out, inp)
        k = self.size * int(experts)
        si = self._dev_index(in_splits, "in_splits", k)
        so = self._dev_index(out_splits, "out_splits", k)
        oo = self._dev_index(out_offsets, "out_offsets", k)
        buf, off = self.lookup(out)
        _cu.alltoallv_dev(self.pc, inp.data_ptr(), int(inp.shape[0]), rb, si, 0, buf, off, out.data_ptr(),
                          int(out.shape[0]), so, oo, int(experts), int(align), False, quant, sbuf, soff, sptr,
                          _stream(stream))
        return out

    @staticmethod
    def _is_fp8_dispatch(out, inp) -> bool:
        """A dtype pair that only the quantising form could serve: an FP8 out fed another dtype."""
        import torch

        return (out.dtype in (torch.float8_e4m3fn, torch.float8_e5m2) and inp.dtype != out.dtype)

    def alltoallv_dev_combine(self, out, inp, in_splits, in_offsets, experts: int = 1, stream=None):
        """Inverse of :meth:`alltoallv_dev`: ``inp`` is laid out as a dispatch output, described by
        ``in_splits`` / ``in_offsets`` (that call's ``out_splits`` / ``out_offsets``; gaps allowed).
        Every row goes back to its source, which receives them packed in (rank, expert) order:
        exactly where its dispatch input rows were."""
        rb = self._dev_rows(out, inp)
        k = self.size * int(experts)
        si = self._dev_index(in_splits, "in_splits", k)
        io = self._dev_index(in_offsets, "in_offsets", k)
        buf, off = self.lookup(out)
        _cu.alltoallv_dev(self.pc, inp.data_ptr(), int(inp.shape[0]), rb, si, io, buf, off, out.data_ptr(),
                          int(out.shape[0]), 0, 0, int(experts), 1, True, False, None, 0, 0, _stream(stream))
        return out

    def alltoallv_dev_combine_topk(self, out, expert_out, splits, pos, weights, experts: int = 1, align: int = 1,
                                   stream=None):
        """Top-k MoE combine: the inverse of :meth:`alltoallv_dev` fused with the gate-weighted sum over
        each token's choices. One kernel, no host synchronisation, graph-capturable.

        ``splits`` is the int64 ``(size * experts,)`` tensor this rank passed as ``in_splits`` to the
        dispatch. ``expert_out`` holds, on every rank, the experts' output in that dispatch's output
        layout (``experts`` and ``align`` as there), float32, bfloat16 or float16; ``expert_out.shape[0]``
        is its capacity. ``pos`` is int64 ``(T, k)``: ``pos[t, j]`` is the row of this rank's dispatch
        input that carried token t's choice j, -1 if it was not sent. ``weights`` is float32
        ``(T, k)``; the weight of a -1 entry is ignored. ``out`` is ``(T, *expert_out.shape[1:])`` of
        ``expert_out``'s dtype, written on this rank only. ``weights=None`` gives every routed choice
        weight 1 (the unweighted sum, which is the backward of :meth:`alltoallv_dev_topk`), byte for
        byte what a tensor of ones gives:
        ``out[t] = round(acc)``, ``acc`` starting at +0.0 and, for j = 0..k-1 with ``pos[t, j] >= 0``
        in that order, ``acc = acc + w[t, j] * float(row)``, each a correctly rounded fp32 multiply or
        add (no fused multiply-add), rounded to nearest even into the dtype. That is what torch
        computes on the CPU for ``acc[m] = acc[m] + w[m, j, None] * rows[pos[m, j]].float()``, where
        ``rows`` is what :meth:`alltoallv_dev_combine` would return.

        Each rank pulls its tokens' rows from the ranks holding their experts, so no rank receives
        ``T * k`` rows to reduce itself. Registered / symmetric ``expert_out``: read in place; any
        other tensor is first copied into its rank's staging pool, which also caps the capacity.
        Every rank must pass the same kind. Rows must be a multiple of 16 bytes, ``expert_out`` and
        ``out`` 16-byte aligned, contiguous and disjoint, and 1 <= k <= 32; otherwise ``ValueError``
        before launch. A ``pos`` entry below -1 or at least ``splits.sum()``, invalid splits,
        arguments that differ between ranks, or an ``expert_out`` below the rows its layout needs
        raise ``ValueError`` on every rank at the next host call after the kernel has run (see
        :meth:`alltoallv_dev`), and no rank's ``out`` is written."""
        import torch

        name = "alltoallv_dev_combine_topk"
        dtypes = (torch.float32, torch.bfloat16, torch.float16)
        named = {"out": out, "expert_out": expert_out, "pos": pos}
        if weights is not None:
            named["weights"] = weights
        self._dev_tensors(name, named)
        if expert_out.dtype not in dtypes or out.dtype != expert_out.dtype:
            raise ValueError(f"{name}: expert_out and out must share a dtype of float32, bfloat16 or float16, got "
                             f"{expert_out.dtype} and {out.dtype}")
        if pos.dtype != torch.int64 or pos.dim() != 2 or (weights is not None and (
                weights.dtype != torch.float32 or weights.shape != pos.shape)):
            raise ValueError(f"{name}: pos must be int64 (T, k) and weights float32 of the same shape, got "
                             f"{pos.dtype} {tuple(pos.shape)} and "
                             f"{None if weights is None else (weights.dtype, tuple(weights.shape))}")
        T, k = int(pos.shape[0]), int(pos.shape[1])
        if not 1 <= k <= 32:
            raise ValueError(f"{name}: k = {k} choices per token; 1..32 are supported")
        if expert_out.dim() < 2 or tuple(out.shape) != (T, *expert_out.shape[1:]):
            raise ValueError(f"{name}: out {tuple(out.shape)} must be (T, *expert_out.shape[1:]) with T = {T}, "
                             f"expert_out {tuple(expert_out.shape)} at least 2-D")
        rb = expert_out.element_size()
        for d in expert_out.shape[1:]:
            rb *= int(d)
        if rb == 0 or rb % 16 != 0:
            raise ValueError(f"{name}: rows of {rb} bytes; a positive multiple of 16 is required")
        if expert_out.data_ptr() % 16 != 0 or out.data_ptr() % 16 != 0:
            raise ValueError(f"{name}: expert_out and out must be 16-byte aligned")
        self._dev_disjoint(name, out, "out", expert_out, "expert_out")
        if not 1 <= int(experts) <= 32 or int(align) < 1:
            raise ValueError(f"{name}: experts must be in 1..32 and align at least 1, got {experts} and {align}")
        si = self._dev_index(splits, "splits", self.size * int(experts))
        buf, off = self.lookup(expert_out)
        wp = weights.data_ptr() if weights is not None else 0
        _cu.alltoallv_dev_combine_topk(self.pc, out.data_ptr(), T, k, pos.data_ptr(), wp, si, buf, off,
                                       expert_out.data_ptr(), int(expert_out.shape[0]), rb,
                                       int(_torch_dtype_to_glb(expert_out.dtype)), int(experts), int(align),
                                       _stream(stream))
        return out

    def alltoallv_dev_combine_topk_backward(self, grad_expert_out, grad_weights, grad_out, expert_out, splits, pos,
                                            weights, experts: int = 1, align: int = 1, stream=None):
        """Backward of :meth:`alltoallv_dev_combine_topk` in one kernel, with no host synchronisation
        (graph-capturable). ``expert_out``, ``splits``, ``pos``, ``weights``, ``experts`` and
        ``align`` are the combine's; ``grad_out`` is the gradient of its ``out``, ``(T, *row)`` of
        ``expert_out``'s dtype. For every routed choice ``(t, j)`` (``pos[t, j] >= 0``) this rank
        reads the expert row ``r`` over the link once and writes:

        - ``grad_weights[t, j]`` (float32 ``(T, k)``, this rank) = ``sum_h float(grad_out[t, h]) *
          float(r[h])`` in fp32. The order is fixed, so the bits do not depend on the grid or the
          run: lane ``l`` of the token's warp adds, with one fused multiply-add per element, the
          elements of 16-byte packs ``l, l + 32, l + 64, ...`` of the row in that order, then a
          ``shfl_xor`` butterfly over lane distances 16, 8, 4, 2, 1 sums the 32 lane totals. Where
          ``pos[t, j] = -1`` it is ``+0.0``.
        - the same row of the holder's ``grad_expert_out`` (``expert_out``'s shape, dtype and
          layout, on every rank) = ``(weights[t, j, None] * grad_out[t].float()).to(dtype)``: one
          correctly rounded fp32 multiply, then round to nearest even, byte for byte.

        Every holder writes ``+0`` to each row of its ``grad_expert_out`` outside its receive
        segments (alignment gaps and the rows past the last segment), so experts that run over the
        whole buffer get zero gradient for padded rows. ``pos`` must name each dispatch-input row
        at most once, as :meth:`route <gloo_b200.parallel.strategies.MoEDispatcher.route>` and
        :meth:`alltoallv_dev_topk` produce; with plain tensors a segment row that no choice names is
        left unspecified.

        ``expert_out`` and ``grad_expert_out`` are both registered / symmetric (zero copy: peers
        write ``grad_expert_out`` in place) or both plain (staged: each rank's pool holds its
        ``expert_out`` rows and then its gradient rows, so the capacity is capped at half the
        combine's), else ``ValueError``. Wrong dtypes or shapes, non-contiguous or misaligned
        tensors (``expert_out``, ``grad_expert_out`` and ``grad_out`` 16-byte aligned, rows a
        multiple of 16 bytes), k outside 1..32 and a ``grad_expert_out`` that overlaps
        ``expert_out``, ``grad_out`` or ``grad_weights`` raise ``ValueError`` before launch. Errors
        found on the device (as for the combine, including a peer that runs another form) raise
        ``ValueError`` on every rank at the next host call, and then no rank has written its
        ``grad_expert_out`` or ``grad_weights``."""
        import torch

        name = "alltoallv_dev_combine_topk_backward"
        dtypes = (torch.float32, torch.bfloat16, torch.float16)
        self._dev_tensors(name, {"grad_expert_out": grad_expert_out, "grad_weights": grad_weights,
                                 "grad_out": grad_out, "expert_out": expert_out, "pos": pos, "weights": weights})
        if expert_out.dtype not in dtypes or grad_out.dtype != expert_out.dtype:
            raise ValueError(f"{name}: expert_out and grad_out must share a dtype of float32, bfloat16 or float16, "
                             f"got {expert_out.dtype} and {grad_out.dtype}")
        if grad_expert_out.dtype != expert_out.dtype or grad_expert_out.shape != expert_out.shape:
            raise ValueError(f"{name}: grad_expert_out {grad_expert_out.dtype} {tuple(grad_expert_out.shape)} must "
                             f"match expert_out {expert_out.dtype} {tuple(expert_out.shape)}")
        if pos.dtype != torch.int64 or pos.dim() != 2 or weights.dtype != torch.float32 or weights.shape != pos.shape:
            raise ValueError(f"{name}: pos must be int64 (T, k) and weights float32 of the same shape, got "
                             f"{pos.dtype} {tuple(pos.shape)} and {weights.dtype} {tuple(weights.shape)}")
        if grad_weights.dtype != torch.float32 or grad_weights.shape != pos.shape:
            raise ValueError(f"{name}: grad_weights must be float32 {tuple(pos.shape)}, got {grad_weights.dtype} "
                             f"{tuple(grad_weights.shape)}")
        T, k = int(pos.shape[0]), int(pos.shape[1])
        if not 1 <= k <= 32:
            raise ValueError(f"{name}: k = {k} choices per token; 1..32 are supported")
        if expert_out.dim() < 2 or tuple(grad_out.shape) != (T, *expert_out.shape[1:]):
            raise ValueError(f"{name}: grad_out {tuple(grad_out.shape)} must be (T, *expert_out.shape[1:]) with "
                             f"T = {T}, expert_out {tuple(expert_out.shape)} at least 2-D")
        rb = expert_out.element_size()
        for d in expert_out.shape[1:]:
            rb *= int(d)
        if rb == 0 or rb % 16 != 0:
            raise ValueError(f"{name}: rows of {rb} bytes; a positive multiple of 16 is required")
        if expert_out.data_ptr() % 16 or grad_expert_out.data_ptr() % 16 or grad_out.data_ptr() % 16:
            raise ValueError(f"{name}: expert_out, grad_expert_out and grad_out must be 16-byte aligned")
        for other, what in ((expert_out, "expert_out"), (grad_out, "grad_out"), (grad_weights, "grad_weights")):
            self._dev_disjoint(name, grad_expert_out, "grad_expert_out", other, what)
        if not 1 <= int(experts) <= 32 or int(align) < 1:
            raise ValueError(f"{name}: experts must be in 1..32 and align at least 1, got {experts} and {align}")
        si = self._dev_index(splits, "splits", self.size * int(experts))
        buf, off = self.lookup(expert_out)
        gbuf, goff = self.lookup(grad_expert_out)
        _cu.alltoallv_dev_combine_topk_backward(self.pc, gbuf, goff, grad_expert_out.data_ptr(),
                                                grad_weights.data_ptr(), grad_out.data_ptr(), buf, off,
                                                expert_out.data_ptr(), T, k, pos.data_ptr(), weights.data_ptr(), si,
                                                int(expert_out.shape[0]), rb,
                                                int(_torch_dtype_to_glb(expert_out.dtype)), int(experts),
                                                int(align), _stream(stream))
        return grad_expert_out, grad_weights

    def alltoallv_dev_topk(self, out, x, topk_idx, splits, pos, out_splits, out_offsets, experts: int = 1,
                           align: int = 1, out_scales=None, stream=None):
        """Top-k MoE dispatch: route every token from its gate indices and push its row to each chosen
        expert, in one kernel with no host synchronisation (graph-capturable).

        ``x`` is a contiguous ``(T, *row)`` CUDA tensor, rows a multiple of 16 bytes, 16-byte
        aligned. ``topk_idx`` is int64 ``(T, k)``, 1 <= k <= 32: entry ``j * experts + e`` chooses
        local expert ``e`` of rank ``j``; any entry outside ``0 .. size * experts - 1`` (such as -1)
        is not routed. ``splits`` (int64 ``(size * experts,)``) and ``pos`` (int64 ``(T, k)``) are
        written on this rank, from its own input alone and even when the call fails.

        The result is byte for byte that of ``rows, splits, pos = MoEDispatcher.route(x, topk_idx,
        experts)`` followed by :meth:`alltoallv_dev` ``(out, rows, splits, out_splits, out_offsets,
        experts, align)``: ``splits``, ``pos``, ``out_splits``, ``out_offsets`` and every row of
        ``out`` inside a segment. Within a (rank, expert) group rows go by token, then by choice; a
        token that picks an expert twice sends two rows. Alignment gaps and rows past the last
        segment are not written. No row is read more than once: each token's row goes from ``x`` to
        all its destinations, so nothing of size ``T * k`` is written locally.
        ``combine_dev_topk`` / :meth:`alltoallv_dev_combine_topk` take the returned ``splits`` and
        ``pos`` unchanged.

        ``out``, ``out_splits``, ``out_offsets``, the capacity (``out.shape[0]``), the zero-copy
        (registered / symmetric) and staged (plain) paths and the errors found on the device are those
        of :meth:`alltoallv_dev`; every rank must call this form, with the same row size, ``experts``,
        ``align`` and kind of ``out``, or the call is invalid on every rank. An ``out`` too small on
        one rank leaves it empty, serves the others and raises on every rank at the next host call.

        Quantising form: ``out_scales`` given, ``x`` bfloat16 ``(T, H)`` with H a multiple of 128,
        ``out`` float8_e4m3fn ``(cap, H)``, ``out_scales`` float32 ``(cap, H // 128)``, both registered
        / symmetric or both plain. Each token is quantised once, with :meth:`alltoallv_dev`'s numerics,
        and the same codes and scales are stored to all its destinations.

        Wrong dtypes (int32 ``topk_idx`` included), shapes, non-contiguous or misaligned tensors,
        k outside 1..32, ``T * k`` above 2^31 - 1 and an ``out`` that overlaps ``x`` raise
        ``ValueError`` before launch. Limits: ``size <= 16``, ``1 <= experts <= 32``; T = 0 is allowed."""
        import torch

        name = "alltoallv_dev_topk"
        G = self.size * int(experts)
        if not 1 <= int(experts) <= 32 or int(align) < 1:
            raise ValueError(f"{name}: experts must be in 1..32 and align at least 1, got {experts} and {align}")
        named = {"x": x, "out": out, "topk_idx": topk_idx, "pos": pos}
        # Device first and contiguity after the shape checks, so that the T * k limit is reported
        # for broadcast views of any size.
        self._dev_tensors(name, named, contiguous=False)
        if topk_idx.dtype != torch.int64 or topk_idx.dim() != 2 or x.dim() < 1 or topk_idx.shape[0] != x.shape[0]:
            raise ValueError(f"{name}: topk_idx must be int64 (T, k) with T = x.shape[0], got {topk_idx.dtype} "
                             f"{tuple(topk_idx.shape)} for x {tuple(x.shape)}")
        T, k = int(topk_idx.shape[0]), int(topk_idx.shape[1])
        if not 1 <= k <= 32:
            raise ValueError(f"{name}: k = {k} choices per token; 1..32 are supported")
        if T * k > 2**31 - 1:
            raise ValueError(f"{name}: T * k = {T * k} choices; at most 2^31 - 1 are supported")
        if pos.dtype != torch.int64 or tuple(pos.shape) != (T, k):
            raise ValueError(f"{name}: pos must be int64 {(T, k)}, got {pos.dtype} {tuple(pos.shape)}")
        self._dev_tensors(name, named)
        si = self._dev_index(splits, "splits", G)
        so = self._dev_index(out_splits, "out_splits", G)
        oo = self._dev_index(out_offsets, "out_offsets", G)
        quant = out_scales is not None or self._is_fp8_dispatch(out, x)
        sbuf, soff, sptr = None, 0, 0
        if quant:
            rb, sbuf, soff, sptr = self._fp8_dispatch(name, "x", x, out, out_scales)
        else:
            rb = self._dev_rows(out, x)
            if rb % 16 != 0:
                raise ValueError(f"{name}: rows of {rb} bytes; a positive multiple of 16 is required")
            if x.data_ptr() % 16 != 0 or out.data_ptr() % 16 != 0:
                raise ValueError(f"{name}: x and out must be 16-byte aligned")
        self._dev_disjoint(name, out, "out", x, "x")
        buf, off = self.lookup(out)
        _cu.alltoallv_dev_topk(self.pc, x.data_ptr(), T, rb, k, topk_idx.data_ptr(), si, pos.data_ptr(), buf, off,
                               out.data_ptr(), int(out.shape[0]), so, oo, int(experts), int(align), quant, sbuf, soff,
                               sptr, _stream(stream))
        return out

    # ---- low-latency top-k MoE exchange (decoding) ----------------------------------------------
    def moe_ll_buffer(self, experts: int, max_tokens: int, topk: int, hidden: int, dtype=None, fp8: bool = False):
        """Collective: a :class:`MoELLBuffer` for :meth:`alltoallv_ll_topk` and
        :meth:`alltoallv_ll_combine_topk`. Every rank must pass the same arguments, else ``ValueError``
        on every rank. ``dtype`` (default bfloat16) is the row dtype of ``x``, ``out`` and the combine;
        ``fp8=True`` takes bfloat16 rows and sends e4m3 codes with fp32 scales per 128 elements."""
        import torch

        return MoELLBuffer(self, experts, max_tokens, topk, hidden, torch.bfloat16 if dtype is None else dtype, fp8)

    def alltoallv_ll_topk(self, buf, out, x, topk_idx, out_splits, out_scales=None, stream=None):
        """Low-latency top-k MoE dispatch for decoding: one kernel, one signal round, no barrier, static
        shapes (graph-capturable). ``buf`` is a :class:`MoELLBuffer`; ``x`` is ``(T, hidden)`` of its
        dtype (FP8 form: bfloat16) with ``T <= max_tokens``; ``topk_idx`` int64 ``(T, topk)``, entry
        ``j * experts + e`` = local expert ``e`` of rank ``j``, anything outside ``0 .. size * experts - 1``
        not routed. Each routed choice is pushed to a fixed slot of its expert on rank ``j``, reserved
        for this rank; no layout is agreed first.

        ``out`` ``(experts, size * max_tokens, hidden)`` (FP8: float8_e4m3fn, plus ``out_scales`` float32
        ``(experts, size * max_tokens, hidden // 128)``) receives expert ``e``'s rows in
        ``out[e, :out_splits[e*size:(e+1)*size].sum()]``: source 0's rows, then source 1's, each by token
        and then choice. That is byte for byte expert ``e``'s segment of :meth:`alltoallv_dev_topk` on the
        same inputs (FP8: the same codes and scales). ``out_splits`` (int64 ``(experts * size,)``, entry
        ``e * size + s``) gets the rows from each source. Rows past the count are not written. ``out``
        and ``out_scales`` may be plain tensors: the rows are copied out of the buffer locally.

        A (source, expert) group holds at most ``max_tokens`` rows; only a token that picks one expert
        twice can exceed it. Such a group sends nothing, its choices count as unrouted in the
        combine, the rest of the call is served, and ``ValueError`` naming the source, the expert, the
        rows and ``max_tokens`` is raised on the source and on the holder at the next host call
        (``synchronize()``). Wrong dtypes, shapes, contiguity or alignment, ``T > max_tokens``, a k
        other than the buffer's, overlapping tensors and a dispatch on a buffer whose previous
        dispatch has not been combined raise ``ValueError`` before launch."""
        import torch

        name = "alltoallv_ll_topk"
        if not isinstance(buf, MoELLBuffer) or buf.cc is not self:
            raise ValueError(f"{name}: buf must be a MoELLBuffer of this context")
        if buf._pending is not None:
            raise ValueError(f"{name}: the buffer's previous dispatch has not been combined; dispatch and combine "
                             "must alternate on a buffer")
        named = {"x": x, "topk_idx": topk_idx, "out": out, "out_splits": out_splits}
        if buf.fp8:
            if out_scales is None:
                raise ValueError(f"{name}: the FP8 buffer needs out_scales")
            named["out_scales"] = out_scales
        elif out_scales is not None:
            raise ValueError(f"{name}: out_scales is only for an FP8 buffer")
        self._dev_tensors(name, named)
        E, M, k, H, P = buf.experts, buf.max_tokens, buf.topk, buf.hidden, self.size
        if x.dtype != buf.dtype or x.dim() != 2 or int(x.shape[1]) != H:
            raise ValueError(f"{name}: x must be {buf.dtype} (T, {H}), got {x.dtype} {tuple(x.shape)}")
        T = int(x.shape[0])
        if T > M:
            raise ValueError(f"{name}: {T} tokens; the buffer holds max_tokens = {M}")
        if topk_idx.dtype != torch.int64 or tuple(topk_idx.shape) != (T, k):
            raise ValueError(f"{name}: topk_idx must be int64 {(T, k)} (the buffer's topk), got {topk_idx.dtype} "
                             f"{tuple(topk_idx.shape)}")
        odt = torch.float8_e4m3fn if buf.fp8 else buf.dtype
        if out.dtype != odt or tuple(out.shape) != (E, P * M, H):
            raise ValueError(f"{name}: out must be {odt} {(E, P * M, H)}, got {out.dtype} {tuple(out.shape)}")
        if buf.fp8 and (out_scales.dtype != torch.float32 or tuple(out_scales.shape) != (E, P * M, H // 128)):
            raise ValueError(f"{name}: out_scales must be float32 {(E, P * M, H // 128)}, got {out_scales.dtype} "
                             f"{tuple(out_scales.shape)}")
        if out_splits.dtype != torch.int64 or tuple(out_splits.shape) != (E * P,):
            raise ValueError(f"{name}: out_splits must be int64 ({E * P},), got {out_splits.dtype} "
                             f"{tuple(out_splits.shape)}")
        if x.data_ptr() % 16 or out.data_ptr() % 16:
            raise ValueError(f"{name}: x and out must be 16-byte aligned")
        buf._check_disjoint(name, named)
        _cu.alltoallv_ll_topk(self.pc, buf._pbuf, buf._off, E, M, k, H, buf._elem, buf.fp8, x.data_ptr(), T,
                              topk_idx.data_ptr(), out.data_ptr(), out_scales.data_ptr() if buf.fp8 else 0,
                              out_splits.data_ptr(), _stream(stream))
        buf._pending = T
        return out

    def alltoallv_ll_combine_topk(self, buf, y, expert_out, weights, stream=None):
        """Low-latency top-k MoE combine, after :meth:`alltoallv_ll_topk` on the same ``buf``: every
        row of this rank's experts goes back to its source, one signal round, and each source sums its
        tokens' choices with their gate weights in one kernel (graph-capturable).

        ``expert_out`` is ``(experts, size * max_tokens, hidden)`` of the buffer's dtype (FP8 buffer:
        bfloat16), in the dispatch's ``out`` layout; rows past each expert's count are not read. ``y`` is
        ``(T, hidden)`` of that dtype with the dispatch's T; ``weights`` float32 ``(T, topk)`` or None
        (weight 1). ``y[t] = round(acc)``, ``acc`` from +0.0 adding ``w[t, j] * float(row)`` for
        j = 0..k-1 over the routed choices that were sent, each a correctly rounded fp32 multiply and
        add: byte for byte what :meth:`alltoallv_dev_combine_topk` gives on the same expert rows.
        Combine dtypes are float32, bfloat16 and float16. Wrong dtypes, shapes, contiguity or
        alignment, overlaps and a combine with no dispatch before it raise ``ValueError`` before
        launch."""
        import torch

        name = "alltoallv_ll_combine_topk"
        if not isinstance(buf, MoELLBuffer) or buf.cc is not self:
            raise ValueError(f"{name}: buf must be a MoELLBuffer of this context")
        if buf._pending is None:
            raise ValueError(f"{name}: no dispatch on this buffer to combine")
        named = {"y": y, "expert_out": expert_out}
        if weights is not None:
            named["weights"] = weights
        self._dev_tensors(name, named)
        E, M, k, H, P, T = buf.experts, buf.max_tokens, buf.topk, buf.hidden, self.size, buf._pending
        cdt = torch.bfloat16 if buf.fp8 else buf.dtype
        if cdt not in (torch.float32, torch.bfloat16, torch.float16):
            raise ValueError(f"{name}: a buffer of {buf.dtype} rows cannot combine; float32, bfloat16 and float16 can")
        if expert_out.dtype != cdt or tuple(expert_out.shape) != (E, P * M, H):
            raise ValueError(f"{name}: expert_out must be {cdt} {(E, P * M, H)}, got {expert_out.dtype} "
                             f"{tuple(expert_out.shape)}")
        if y.dtype != cdt or tuple(y.shape) != (T, H):
            raise ValueError(f"{name}: y must be {cdt} {(T, H)} (T of the dispatch), got {y.dtype} {tuple(y.shape)}")
        if weights is not None and (weights.dtype != torch.float32 or tuple(weights.shape) != (T, k)):
            raise ValueError(f"{name}: weights must be float32 {(T, k)}, got {weights.dtype} {tuple(weights.shape)}")
        if y.data_ptr() % 16 or expert_out.data_ptr() % 16:
            raise ValueError(f"{name}: y and expert_out must be 16-byte aligned")
        buf._check_disjoint(name, named)
        _cu.alltoallv_ll_combine_topk(self.pc, buf._pbuf, buf._off, E, M, k, H, buf._elem, buf.fp8, y.data_ptr(), T,
                                      expert_out.data_ptr(), weights.data_ptr() if weights is not None else 0,
                                      int(_torch_dtype_to_glb(cdt)), _stream(stream))
        buf._pending = None
        return y

    def scatter(self, output, input=None, root: int = 0, stream=None):
        """Block ``rank`` of the root's ``input`` -> ``output``. Any size; ``input`` is read on the
        root only (None elsewhere)."""
        nbytes = output.numel() * output.element_size()
        iptr = input.data_ptr() if input is not None else 0
        buf, off = self.lookup(output)
        if buf is not None:
            _cu.scatter_reg(self.pc, iptr, buf, off, nbytes, root, _stream(stream))
        else:
            _cu.scatter(self.pc, iptr, output.data_ptr(), nbytes, root, _stream(stream))
        return output

    def reduce_scatter(self, output, input, counts: Optional[Sequence[int]] = None, op: ReduceOp = ReduceOp.SUM,
                       stream=None, scale: float = 1.0):
        """``output`` := share ``rank`` of the reduction of every rank's ``input`` (``counts[r]``
        elements for rank r, an even split by default), times ``scale`` (floating types), with one
        rounding. Any size: a plain ``input`` larger than the staging pool streams through it in one
        kernel; ``output`` may be this rank's share of ``input`` (in place).

        When ``output.dtype != input.dtype`` this is the cast form: a bfloat16 / float16 ``input``, a
        float32 ``output`` and ``op`` SUM. ``output[i] = fp32(sum over ranks of float(input[off + i]))
        * fp32(scale)``: the sum is accumulated in fp32 and never rounded to 16 bits, so ``output``
        holds exactly what an fp32 reduction of the upcast inputs gives, while only 16-bit bytes
        cross NVLink. One kernel launch; ``output`` must not overlap ``input``. Other pairs or ops
        raise ``ValueError``."""
        ptr, n, dt, _ = describe(input)
        odt = int(describe(output)[2]) if output.dtype != input.dtype else -1
        if counts is None:
            base, rem = divmod(n, self.size)
            counts = [base + (1 if r < rem else 0) for r in range(self.size)]
        buf, off = self.lookup(input)
        if buf is not None:
            _cu.reduce_scatter_reg(self.pc, buf, off, output.data_ptr(), list(counts), int(dt), int(op), _stream(stream), scale,
                                   odt)
        else:
            _cu.reduce_scatter(self.pc, ptr, output.data_ptr(), list(counts), int(dt), int(op), _stream(stream), scale,
                               odt)
        return output

    def reduce(self, output, input, root: int = 0, op: ReduceOp = ReduceOp.SUM, stream=None):
        """``output`` on ``root`` := the reduction of every rank's ``input``. Any size; a non-root's
        ``output`` is never written. Each rank takes the registered path when its own ``input``
        and ``output`` are both registered / symmetric, so the ranks must agree: when the root's
        are, every rank passes registered input and output tensors at the root's offsets; a
        non-root's ``output`` may be None only when the root's input or output is plain."""
        ptr, n, dt, _ = describe(input)
        ibuf, ioff = self.lookup(input)
        obuf, ooff = (self.lookup(output) if output is not None else (None, 0))
        if ibuf is not None and obuf is not None:
            _cu.reduce_reg(self.pc, ibuf, ioff, obuf, ooff, n, int(dt), int(op), root, _stream(stream))
        else:
            optr = output.data_ptr() if output is not None else 0
            _cu.reduce(self.pc, ptr, optr, n, int(dt), int(op), root, _stream(stream))
        return output


class MoELLBuffer:
    """Symmetric memory for the low-latency top-k MoE exchange, made by :meth:`CudaContext.moe_ll_buffer`
    with the same arguments on every rank (checked by an allgather: a mismatch raises ``ValueError``
    on every rank). It holds, per rank, in this order, each part rounded up to 16 bytes:

    - dispatch slots: ``experts * size * max_tokens`` rows of ``row_bytes`` (``hidden`` elements of
      ``dtype``; FP8: ``hidden`` e4m3 codes), then FP8 only their scales, ``hidden / 128 * 4`` bytes a
      row, then an int32 tag a row (``t * topk + j`` of the source's token and choice);
    - ``experts * size`` 64-bit dispatch signal words;
    - combine slots: ``max_tokens * topk`` rows of ``hidden`` elements (FP8: bfloat16);
    - ``size`` 64-bit combine signal words, ``max_tokens * topk`` int32 choice marks and 16 bytes of
      call count and completion ticket.

    So ``bytes ~= E * P * M * (row_bytes + scale_bytes + 4) + M * k * (combine_row_bytes + 4)``: at
    E = 32, P = 8, M = 128, k = 8 and H = 7168 that is 484 MB in bfloat16 (470 MB of slots) and 257 MB
    in FP8 (242 MB of slots and scales). ``layout`` has every offset. Limits: ``size <= 16``,
    ``1 <= experts <= 32``, ``1 <= topk <= 32``, ``max_tokens * topk <= 2^31 - 1``, rows a multiple of
    16 bytes (FP8: ``hidden`` a multiple of 128).

    Dispatch and combine must alternate on a buffer; that is what lets one set of slots serve every
    call. The buffer counts its calls on the device, so a captured dispatch / combine pair can be
    replayed as a CUDA graph."""

    def __init__(self, cc: "CudaContext", experts, max_tokens, topk, hidden, dtype, fp8):
        import torch

        name = "moe_ll_buffer"
        dtypes = [torch.float32, torch.bfloat16, torch.float16, torch.uint8, torch.int8, torch.int16, torch.int32,
                  torch.int64, torch.float64]

        def as_int(v):
            try:
                return int(v) if int(v) == v else -1
            except (TypeError, ValueError):
                return -1

        words = [as_int(experts), as_int(max_tokens), as_int(topk), as_int(hidden),
                 dtypes.index(dtype) if dtype in dtypes else -1, 1 if fp8 else 0]
        if not cc.pc.host_all_same(words):
            raise ValueError(f"{name}: the arguments (experts, max_tokens, topk, hidden, dtype, fp8) differ between "
                             "ranks; every rank must pass the same")
        E, M, k, H = words[:4]
        if not 1 <= E <= 32 or not 1 <= k <= 32 or M < 1 or M * k > 2**31 - 1 or H < 1 or words[4] < 0:
            raise ValueError(f"{name}: need 1 <= experts <= 32, 1 <= topk <= 32, max_tokens >= 1 with max_tokens * "
                             f"topk <= 2^31 - 1, hidden >= 1 and a tensor dtype; got {experts}, {topk}, {max_tokens}, "
                             f"{hidden}, {dtype}")
        es = torch.empty((), dtype=dtype).element_size()
        if fp8 and (dtype != torch.bfloat16 or H % 128):
            raise ValueError(f"{name}: the FP8 form takes bfloat16 rows of a multiple of 128 elements, got {dtype} "
                             f"and {H}")
        if (H * es) % 16:
            raise ValueError(f"{name}: rows of {H * es} bytes; a multiple of 16 is required")
        self.layout = _cu.moe_ll_layout(cc.size, E, M, k, H, es, bool(fp8))
        nbytes = int(self.layout["bytes"])
        free, _ = torch.cuda.mem_get_info(cc.device)
        fits = free >= nbytes * max(1, cc.pc.ranks_on_my_device())
        if not cc.pc.host_all_same([1 if fits else 0]) or not fits:
            raise ValueError(f"{name}: {nbytes} bytes per rank do not fit the free device memory of every rank")
        self.cc, self.experts, self.max_tokens, self.topk, self.hidden = cc, E, M, k, H
        self.dtype, self.fp8, self._elem = dtype, bool(fp8), es
        self.tensor = cc.empty(nbytes, torch.uint8)
        self.tensor.zero_()  # signal words, call count: no call has happened
        torch.cuda.current_stream(cc.device).synchronize()
        cc.pc.host_barrier()  # no peer signals into a buffer that is still being cleared
        self._pbuf, self._off = cc.lookup(self.tensor)
        self._pending = None  # T of a dispatch not yet combined

    @property
    def nbytes(self) -> int:
        return int(self.layout["bytes"])

    def _check_disjoint(self, name, named):
        """No two of ``named`` share a byte, and none lies in the buffer."""
        items = list(named.items()) + [("the buffer", self.tensor)]
        for i, (an, a) in enumerate(items):
            for bn, b in items[i + 1:]:
                if a.numel() and b.numel():
                    CudaContext._dev_disjoint(name, a, an, b, bn)


# ---- old-style class wrappers -----------------------------------------------------------------

def _make_allreduce_class(name: str, algo: str):
    class _Cls:
        __doc__ = f"{name}(ctx, tensors, streams=None, op=SUM, host_workspace=False) — run() is one fused launch."

        def __init__(self, ctx, tensors, streams=None, op: ReduceOp = ReduceOp.SUM, host_workspace: bool = False,
                     literal: bool = False, variant: str = "auto"):
            # literal=True runs the named schedule step by step; otherwise the kernel variant is
            # picked per message size ("auto") or pinned ("one_shot" / "two_shot" / "nvls").
            tensors = list(tensors) if isinstance(tensors, (list, tuple)) else [tensors]
            self.tensors = tensors
            _, n, dt, _ = describe(tensors[0])
            st = [_stream(s) for s in streams] if streams else []
            assert variant in ("auto", "one_shot", "two_shot", "nvls", "ll", "pipelined", "hybrid")
            self._impl = _cu.CudaAllreduce(ctx, [t.data_ptr() for t in tensors], n, int(dt), int(op), st,
                                           ALGOS[algo] if literal else ALGOS[variant], host_workspace)

        def run(self):
            self._impl.run()

        def set_scale(self, scale: float):
            """Fused epilogue: the result is multiplied by ``scale`` inside the collective kernel."""
            self._impl.set_scale(float(scale))

        def set_launch_shape(self, blocks: int = 0, unroll: int = 0, tile: int = 0):
            self._impl.set_launch_shape(blocks, unroll, tile)

        def launches_per_run(self) -> int:
            return self._impl.launches_per_run()

        def resolved_algo(self) -> str:
            return self._impl.resolved_algo()

        def uses_peer_memory(self) -> bool:
            return self._impl.uses_peer_memory()

    _Cls.__name__ = name
    return _Cls


CudaAllreduceRing = _make_allreduce_class("CudaAllreduceRing", "ring")
CudaAllreduceRingChunked = _make_allreduce_class("CudaAllreduceRingChunked", "ring_chunked")
CudaAllreduceHalvingDoubling = _make_allreduce_class("CudaAllreduceHalvingDoubling", "halving_doubling")
CudaAllreduceHalvingDoublingPipelined = _make_allreduce_class("CudaAllreduceHalvingDoublingPipelined",
                                                              "halving_doubling_pipelined")
CudaAllreduceBcube = _make_allreduce_class("CudaAllreduceBcube", "bcube")


class CudaHostAllreduce:
    """Allreduce of pinned *host* buffers through the GPUs, as a three-stage pipeline.

    The reference reaches host-resident data with ``CudaHostWorkspace`` (device <-> pinned host
    staging around a CPU reduction, gloo/cuda_workspace.h:17-40). Here the reduction stays on
    NVLink and the PCIe legs are overlapped with it: the vector is cut into ``chunks`` pieces and
    piece c is copied host->device on one stream while piece c-1 is being reduced across the
    GPUs (one fused kernel per piece, same ``CudaAllreduceRingChunked`` class a user would
    call) and piece c-2 is copied device->host on a third stream. PCIe is full duplex, so a
    step costs about max(H2D, D2H) + one piece instead of H2D + allreduce + D2H.

    ``host_inputs``: one pinned tensor per local input (they are summed first when there are
    several, like the multi-pointer classes); ``host_output``: pinned tensor for the result.
    ``run()`` is asynchronous with respect to the host: the caller's current stream (or
    ``stream``) is made to wait for the last device->host copy, so ``stream.synchronize()``
    or any later work on that stream sees ``host_output`` complete. Collective: construct
    and run in the same order on every rank.
    """

    def __init__(self, ctx, cuda_ctx: "CudaContext", host_inputs, host_output, chunks: int = 16,
                 op: ReduceOp = ReduceOp.SUM, variant: str = "two_shot"):
        import torch

        host_inputs = list(host_inputs) if isinstance(host_inputs, (list, tuple)) else [host_inputs]
        n = host_output.numel()
        for h in host_inputs + [host_output]:
            assert h.is_pinned() and h.is_contiguous() and h.numel() == n and h.dtype == host_output.dtype, \
                "CudaHostAllreduce needs contiguous pinned host tensors of one shape and dtype"
        self.cc = cuda_ctx
        self.hin, self.hout = host_inputs, host_output
        dev = cuda_ctx.device
        with torch.cuda.device(dev):
            self.dev = [cuda_ctx.empty(n, host_output.dtype) for _ in host_inputs]
            self.h2d, self.comp, self.d2h = new_stream(dev), new_stream(dev, True), new_stream(dev)
            # piece boundaries on 4 KiB so every piece keeps the vector alignment of the kernels
            align = max(1, 4096 // host_output.element_size())
            per = -(-n // max(1, chunks))
            per = -(-per // align) * align
            self.bounds = [(lo, min(n, lo + per)) for lo in range(0, n, per)] if n else []
            self.algos = []
            for lo, hi in self.bounds:
                # Pieces are interior ranges of the symmetric buffers. The two-shot kernel is
                # pinned: it is the variant measured on such ranges, and the reduction hides
                # under the PCIe copies either way.
                self.algos.append(CudaAllreduceRingChunked(ctx, [d[lo:hi] for d in self.dev],
                                                           streams=[self.comp] * len(self.dev), op=op,
                                                           variant=variant))
            self.ev_in = [torch.cuda.Event() for _ in self.bounds]
            self.ev_red = [torch.cuda.Event() for _ in self.bounds]
            self.ev_start, self.ev_done = torch.cuda.Event(), torch.cuda.Event()
        self.launches_per_run = len(self.bounds)

    def run(self, stream=None):
        import torch

        caller = torch.cuda.current_stream(self.cc.device) if stream is None else stream
        self.ev_start.record(caller)
        self.h2d.wait_event(self.ev_start)
        self.d2h.wait_event(self.ev_start)
        for c, (lo, hi) in enumerate(self.bounds):
            with torch.cuda.stream(self.h2d):
                for d, h in zip(self.dev, self.hin):
                    d[lo:hi].copy_(h[lo:hi], non_blocking=True)
                self.ev_in[c].record(self.h2d)
            self.comp.wait_event(self.ev_in[c])
            self.algos[c].run()
            self.ev_red[c].record(self.comp)
            self.d2h.wait_event(self.ev_red[c])
            with torch.cuda.stream(self.d2h):
                self.hout[lo:hi].copy_(self.dev[0][lo:hi], non_blocking=True)
        self.ev_done.record(self.d2h)
        caller.wait_event(self.ev_done)
        return self.hout

    def resolved_algo(self) -> str:
        return self.algos[0].resolved_algo() if self.algos else "none"


class CudaBroadcastOneToAll:
    def __init__(self, ctx, tensors, root: int = 0, root_pointer: int = 0, streams=None, host_workspace: bool = False):
        tensors = list(tensors) if isinstance(tensors, (list, tuple)) else [tensors]
        self.tensors = tensors
        _, n, dt, _ = describe(tensors[0])
        st = [_stream(s) for s in streams] if streams else []
        self._impl = _cu.CudaBroadcast(ctx, [t.data_ptr() for t in tensors], n, int(dt), root, root_pointer, st,
                                       host_workspace)

    def run(self):
        self._impl.run()
