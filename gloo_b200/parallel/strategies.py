from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

from .. import _C
from ..ops import host as H
from ..types import ReduceOp


def _is_cuda(t) -> bool:
    return bool(getattr(t, "is_cuda", False))


def _norm_parts(module, dtype):
    """(kind, weight, bias, eps) of a norm module as the fused kernel takes them; kind is None for
    no module and "unsupported" for a module it does not implement."""
    import torch

    if module is None:
        return None, None, None, 0.0
    if isinstance(module, torch.nn.LayerNorm):
        return "layer", module.weight, module.bias, module.eps
    if isinstance(module, getattr(torch.nn, "RMSNorm", ())):
        return "rms", module.weight, None, module.eps if module.eps is not None else torch.finfo(dtype).eps
    return "unsupported", None, None, 0.0


def _norm_fusable(cc, partial, residual, residual_shape, norm_module, kind, vectors) -> bool:
    """Whether a fused residual-norm kernel can run on these tensors: a CUDA context, a
    supported norm and dtype, a hidden size within the kernel's limits, ``residual`` of
    ``residual_shape``, and aligned tensors of one dtype."""
    import torch

    if cc is None or not _is_cuda(partial) or kind == "unsupported" or partial.dim() == 0:
        return False
    H = partial.shape[-1]
    if partial.dtype not in (torch.float32, torch.bfloat16, torch.float16) or tuple(residual.shape) != residual_shape:
        return False
    if H * partial.element_size() % 16 or H > _C.cuda.MAX_NORM_HIDDEN:
        return False
    if norm_module is not None and tuple(norm_module.normalized_shape) != (H,):
        return False
    for t in (partial, residual):
        # a non-contiguous tensor is copied, and the copy is aligned
        if t.dtype != partial.dtype or (t.is_contiguous() and t.data_ptr() % 16):
            return False
    for t in vectors:
        if t is not None and (not t.is_cuda or t.dtype != partial.dtype or not t.is_contiguous() or
                              t.data_ptr() % 16 or tuple(t.shape) != (H,)):
            return False
    return True


def fp8_rows(o):
    """Row-wise FP8 quantisation of ``o`` in torch, the bytes the fused FP8 ``out`` has: ``(codes,
    scales)``, float8_e4m3fn codes of ``o``'s shape and float32 scales ``o.shape[:-1] + (1,)``, with
    ``amax = max(max |o|, 1e-4)`` per row, ``codes = e4m3(o * (448 / amax))`` and ``scales = amax /
    448``. The scale divides by a tensor: on CUDA, torch divides by a Python scalar by multiplying
    with its rounded reciprocal, which is not ``amax / 448`` correctly rounded."""
    import torch

    a = o.float().abs().amax(-1, keepdim=True).clamp_min(1e-4)
    return (o.float() * (448.0 / a)).to(torch.float8_e4m3fn), a / torch.full_like(a, 448.0)


def _check_fp8_call(name, norm_module, tensors):
    """The FP8 form is forward-only and needs a norm."""
    import torch

    if norm_module is None:
        raise ValueError(f"{name}: fp8 needs a norm_module")
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise ValueError(f"{name}: fp8 is forward-only; run it under torch.no_grad() or on tensors that do not "
                         "require grad")


def _aligned_like(s, *grads) -> bool:
    """Whether the gradients (None: absent) have ``s``'s dtype and device and, made contiguous,
    the 16-byte alignment the fused backward needs."""
    for g in grads:
        if g is not None and (g.dtype != s.dtype or g.device != s.device or
                              (g.is_contiguous() and g.data_ptr() % 16)):
            return False
    return True


def _norm_input_grad(kind, H, eps, s, w, nb, grad_out):
    """The norm's gradients, recomputed with torch from its saved input ``s``: ``(grad_s,
    grad_weight, grad_norm_bias)``, None for an absent weight or bias."""
    import torch

    F = torch.nn.functional
    with torch.enable_grad():
        x = s.detach().requires_grad_(True)
        ws = [t.detach().requires_grad_(True) if t is not None else None for t in (w, nb)]
        y = F.rms_norm(x, (H,), ws[0], eps) if kind == "rms" else F.layer_norm(x, (H,), ws[0], ws[1], eps)
        need = [x] + [t for t in ws if t is not None]
        got = list(torch.autograd.grad(y, need, grad_out))
    gs = got.pop(0)
    gw = got.pop(0) if w is not None else None
    gnb = got.pop(0) if nb is not None else None
    return gs, gw, gnb


class _Base:
    def __init__(self, ctx, cuda_ctx=None):
        """ctx: host context (control plane, CPU tensors); cuda_ctx: ops.cuda.CudaContext."""
        self.ctx = ctx
        self.cc = cuda_ctx
        self.rank, self.size = ctx.rank, ctx.size

    def _allreduce(self, t, op=ReduceOp.SUM, average: bool = False):
        """Allreduce, optionally averaged. On CUDA the 1/P is the kernel's fused scale epilogue
        (one launch); on the host it is a second pass."""
        if _is_cuda(t):
            fused = average and t.is_floating_point()
            self.cc.allreduce(t, op=op, average=fused)
            if average and not fused:
                t.div_(self.size)
        else:
            H.allreduce(self.ctx, t, op=op)
            if average:
                t.div_(self.size) if hasattr(t, "div_") else t.__itruediv__(self.size)
        return t


class DataParallel(_Base):
    """Gradient synchronisation for data parallelism.

    Gradients are flattened into buckets of at most ``bucket_bytes`` (sized for launch
    latency and overlap, not link count — NVSwitch gives every peer full bandwidth)
    which live in symmetric memory, so each bucket is one zero-copy fused kernel.
    """

    def __init__(self, ctx, cuda_ctx=None, bucket_bytes: int = 64 << 20):
        super().__init__(ctx, cuda_ctx)
        self.bucket_bytes = bucket_bytes
        self._buckets = {}

    def broadcast_parameters(self, params: Iterable, root: int = 0):
        for p in params:
            t = p.data if hasattr(p, "data") else p
            if _is_cuda(t):
                self.cc.broadcast(t, root=root)
            else:
                H.broadcast(self.ctx, t, root=root)

    def _bucket(self, key, numel, dtype, device):
        b = self._buckets.get(key)
        if b is None or b.numel() < numel:
            if device.type == "cuda":
                b = self.cc.empty(numel, dtype)  # symmetric: zero-copy, NVLS-capable
            else:
                import torch

                b = torch.empty(numel, dtype=dtype)
            self._buckets[key] = b
        return b[:numel]

    def allreduce_gradients(self, params: Iterable, average: bool = True):
        import torch

        grads = [p.grad for p in params if getattr(p, "grad", None) is not None]
        if not grads:
            return
        groups, cur, cur_bytes = [], [], 0
        for g in grads:
            nbytes = g.numel() * g.element_size()
            if cur and (cur_bytes + nbytes > self.bucket_bytes or g.dtype != cur[0].dtype):
                groups.append(cur)
                cur, cur_bytes = [], 0
            cur.append(g)
            cur_bytes += nbytes
        if cur:
            groups.append(cur)
        for i, group in enumerate(groups):
            n = sum(g.numel() for g in group)
            flat = self._bucket((i, group[0].dtype), n, group[0].dtype, group[0].device)
            off = 0
            for g in group:
                flat[off:off + g.numel()].copy_(g.reshape(-1))
                off += g.numel()
            self._allreduce(flat, average=average)
            off = 0
            for g in group:
                g.copy_(flat[off:off + g.numel()].view_as(g))
                off += g.numel()


class GradientBucketer(_Base):
    """Gradient synchronisation that overlaps with the backward pass, without copies.

    Parameters are packed, in reverse order (the last layers finish their backward first), into
    flat buckets of at most ``bucket_bytes``. On CUDA a bucket is SYMMETRIC memory
    (``CudaContext.empty``: peer-mapped and, beyond two GPUs, bound to an NVSwitch multicast
    object) and every ``p.grad`` is a VIEW into its bucket, so autograd accumulates straight into
    the buffer the collective reads: no flatten / unflatten pass, and the allreduce is the zero-copy
    fused kernel (1/P average in its epilogue). A bucket is launched on a side stream as soon as
    the last of its gradients has been accumulated (``register_post_accumulate_grad_hook``), in
    bucket order on every rank; ``finish()`` makes the compute stream wait for the results.
    The reference has no counterpart (its consumers - ProcessGroupGloo + DDP's reducer - copy
    gradients into a bucket, stage it through pinned host memory and reduce on the CPU).

        bucketer = GradientBucketer(ctx, cuda_ctx, model.parameters())
        loss.backward(); bucketer.finish(); optimizer.step(); bucketer.zero_grad()
    """

    def __init__(self, ctx, cuda_ctx, params: Iterable, bucket_bytes: int = 64 << 20, average: bool = True):
        import torch

        super().__init__(ctx, cuda_ctx)
        self.average = average
        self.buckets = []
        self._next = 0
        self._hooks = []
        self._comm_stream = None
        # Ranks that share one GPU (threads-as-ranks tests) rendezvous on the host before every launch
        # (PeerContext::launchGuard) and share the process's single autograd thread: a hook that waits for
        # a peer's hook would wait for itself. There the buckets are launched from finish() instead.
        self._defer = cuda_ctx is not None and cuda_ctx.pc.ranks_on_my_device() > 1
        plist = [p for p in params if p.requires_grad]
        groups, cur, cur_bytes = [], [], 0
        for p in reversed(plist):
            nbytes = p.numel() * p.element_size()
            if cur and (cur_bytes + nbytes > bucket_bytes or p.dtype != cur[0].dtype or p.device != cur[0].device):
                groups.append(cur)
                cur, cur_bytes = [], 0
            cur.append(p)
            cur_bytes += nbytes
        if cur:
            groups.append(cur)
        for group in groups:
            # every view starts on a 16-byte boundary so the kernels stay vectorised
            align = max(1, 16 // group[0].element_size())
            offs, n = [], 0
            for p in group:
                offs.append(n)
                n += (p.numel() + align - 1) // align * align
            cuda = _is_cuda(group[0])
            if cuda:
                flat = self.cc.empty(n, group[0].dtype)
                if self._comm_stream is None:
                    from ..ops.cuda import new_stream  # dedicated: torch.cuda.Stream() comes from a shared pool

                    self._comm_stream = new_stream(group[0].device.index)
            else:
                flat = torch.empty(n, dtype=group[0].dtype)
            flat.zero_()
            b = {"flat": flat, "params": group, "offs": offs, "pending": len(group), "launched": False, "done": None,
                 "cuda": cuda}
            for p, off in zip(group, offs):
                p.grad = flat[off:off + p.numel()].view_as(p)
                self._hooks.append(p.register_post_accumulate_grad_hook(lambda q, b=b: self._ready(b, q)))
            self.buckets.append(b)

    def _view(self, b, p):
        off = b["offs"][[id(x) for x in b["params"]].index(id(p))]
        return b["flat"][off:off + p.numel()].view_as(p)

    def _ready(self, b, p):
        v = self._view(b, p)
        if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
            # somebody replaced the gradient tensor (zero_grad(set_to_none=True), clip utilities that
            # rebind .grad): take the value and point .grad back into the bucket
            v.copy_(p.grad)
            p.grad = v
        b["pending"] -= 1
        if self._defer:
            return
        while self._next < len(self.buckets) and self.buckets[self._next]["pending"] == 0:
            self._launch(self.buckets[self._next])
            self._next += 1

    def _launch(self, b):
        if b["launched"]:
            return
        b["launched"] = True
        if b["cuda"]:
            import torch

            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self._comm_stream.wait_event(ev)
            fused = self.average and b["flat"].is_floating_point()
            self.cc.allreduce(b["flat"], average=fused, stream=self._comm_stream)
            if self.average and not fused:
                with torch.cuda.stream(self._comm_stream):
                    b["flat"].div_(self.size)
            b["done"] = torch.cuda.Event()
            b["done"].record(self._comm_stream)
        else:
            self._allreduce(b["flat"], average=self.average)

    def finish(self):
        """After ``backward()``: launch what has not been launched (buckets with parameters that
        received no gradient this step) in order, and order the compute stream behind the results."""
        for b in self.buckets[self._next:]:
            self._launch(b)
        for b in self.buckets:
            if b["cuda"] and b["done"] is not None:
                import torch

                torch.cuda.current_stream().wait_event(b["done"])
            b["pending"], b["launched"], b["done"] = len(b["params"]), False, None
        self._next = 0

    def zero_grad(self):
        """Zero the buckets in place (keeps every ``p.grad`` a view into symmetric memory)."""
        for b in self.buckets:
            b["flat"].zero_()
            for p, off in zip(b["params"], b["offs"]):
                v = b["flat"][off:off + p.numel()].view_as(p)
                if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                    p.grad = v

    def remove(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []


class ZeroShard(_Base):
    """ZeRO / FSDP building blocks: each rank owns 1/P of a flat parameter vector."""

    def shard_range(self, numel: int):
        base, rem = divmod(numel, self.size)
        counts = [base + (1 if r < rem else 0) for r in range(self.size)]
        start = sum(counts[: self.rank])
        return start, counts[self.rank], counts

    def reduce_scatter_gradients(self, flat_grad, out_shard, average: bool = True):
        """This rank's shard of the sum (or with ``average`` the mean) of every rank's ``flat_grad``.
        A float32 ``out_shard`` of a bfloat16 / float16 ``flat_grad`` is the cast form: the sum is
        accumulated in fp32 and the 1/P applied in fp32, never rounded to 16 bits."""
        _, _, counts = self.shard_range(flat_grad.numel())
        if _is_cuda(flat_grad):
            fused = average and flat_grad.is_floating_point()
            self.cc.reduce_scatter(out_shard, flat_grad, counts, scale=1.0 / self.size if fused else 1.0)
            if average and not fused:
                out_shard.div_(self.size)
        elif out_shard.dtype != flat_grad.dtype:
            # the cast form on host tensors: an fp32 reduction of the upcast gradients, times fp32(1/P)
            H.reduce_scatter(self.ctx, out_shard, flat_grad.to(out_shard.dtype), counts)
            if average:
                out_shard.mul_(1.0 / self.size)
        else:
            H.reduce_scatter(self.ctx, out_shard, flat_grad, counts)
            if average:
                out_shard.div_(self.size) if hasattr(out_shard, "div_") else None
        return out_shard

    def allgather_parameters(self, flat_param, shard):
        """Every rank's ``shard`` into ``flat_param``. A float32 ``shard`` of a bfloat16 / float16
        ``flat_param`` is rounded once to the parameter dtype on its own rank."""
        _, _, counts = self.shard_range(flat_param.numel())
        if _is_cuda(flat_param):
            self.cc.allgatherv(flat_param, shard, counts)
        else:
            H.allgatherv(self.ctx, flat_param, counts, shard.to(flat_param.dtype))
        return flat_param


class ZeroOptimizer(_Base):
    """ZeRO stage 1 on flat buffers: every rank keeps the optimizer state of 1/P of the parameters.

    Parameters and gradients are re-pointed into two flat buffers (symmetric memory on CUDA: the
    collectives read and write them in place). ``step()`` = reduce_scatter of the flat gradient
    (1/P average fused into the kernel) -> the wrapped torch optimizer updates this rank's shard
    only -> allgather of the updated shards back into the flat parameter buffer. Optimizer state
    (Adam moments, ...) exists for the shard only: 1/P of the memory of a replicated optimizer.

        zo = ZeroOptimizer(ctx, cuda_ctx, model.parameters(), torch.optim.AdamW, lr=1e-3)
        loss.backward(); zo.step(); zo.zero_grad()

    ``master_dtype=torch.float32`` with bfloat16 / float16 parameters keeps fp32 master weights: the
    optimizer owns an fp32 copy of this rank's shard (initialised from the parameters), the flat
    buffers stay in the parameter dtype, and ``step()`` runs the cast reduce-scatter of the 16-bit
    gradients into the fp32 shard gradient (fp32 accumulation, the 1/P fused, no 16-bit rounding),
    the optimizer on the fp32 shard, and the cast allgather that rounds each master shard once to
    the parameter dtype. Without it a 16-bit optimizer shard drops every update smaller than half a
    16-bit step of the weight. With float32 parameters, or ``master_dtype=None``, nothing changes.
    """

    def __init__(self, ctx, cuda_ctx, params: Iterable, optimizer_cls, average: bool = True, master_dtype=None,
                 **optimizer_kwargs):
        import torch

        super().__init__(ctx, cuda_ctx)
        if master_dtype not in (None, torch.float32):
            raise ValueError(f"ZeroOptimizer: master_dtype must be None or torch.float32, got {master_dtype}")
        self.average = average
        self.params = [p for p in params if p.requires_grad]
        assert self.params, "no trainable parameters"
        dtype, device = self.params[0].dtype, self.params[0].device
        assert all(p.dtype == dtype and p.device == device for p in self.params), "one dtype / device per ZeroOptimizer"
        # fp32 master weights: only 16-bit parameters have anything to gain
        self.master = master_dtype is not None and dtype in (torch.bfloat16, torch.float16)
        cuda = device.type == "cuda"
        align = max(1, 16 // self.params[0].element_size())
        offs, n = [], 0
        for p in self.params:
            offs.append(n)
            n += (p.numel() + align - 1) // align * align
        unit = align * self.size                       # every shard starts on a 16-byte boundary
        n = (n + unit - 1) // unit * unit
        alloc = (lambda k: self.cc.empty(k, dtype)) if cuda else (lambda k: torch.empty(k, dtype=dtype))
        self.flat_param, self.flat_grad = alloc(n), alloc(n)
        self.flat_param.zero_()
        self.flat_grad.zero_()
        with torch.no_grad():
            for p, off in zip(self.params, offs):
                self.flat_param[off:off + p.numel()].copy_(p.reshape(-1))
                p.data = self.flat_param[off:off + p.numel()].view_as(p)
                p.grad = self.flat_grad[off:off + p.numel()].view_as(p)
        self._offs = offs
        self.counts = [n // self.size] * self.size
        self.start = self.rank * (n // self.size)
        cnt = self.counts[self.rank]
        # the shard the optimizer owns: its own tensors (the collectives' inputs / outputs must not
        # alias the flat buffers they gather into / scatter from); in master mode the fp32 upcast
        mine = self.flat_param[self.start:self.start + cnt].detach()
        self.shard = torch.nn.Parameter(mine.float() if self.master else mine.clone())
        self.shard.grad = torch.zeros_like(self.shard)
        self.optimizer = optimizer_cls([self.shard], **optimizer_kwargs)

    def step(self):
        import torch

        # a gradient tensor that was rebound (zero_grad(set_to_none=True)) is copied back into the flat buffer
        for p, off in zip(self.params, self._offs):
            v = self.flat_grad[off:off + p.numel()].view_as(p)
            if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
                p.grad = v
        ZeroShard(self.ctx, self.cc).reduce_scatter_gradients(self.flat_grad, self.shard.grad, average=self.average)
        self.optimizer.step()
        with torch.no_grad():
            ZeroShard(self.ctx, self.cc).allgather_parameters(self.flat_param, self.shard.data)

    def zero_grad(self):
        self.flat_grad.zero_()
        for p, off in zip(self.params, self._offs):
            v = self.flat_grad[off:off + p.numel()].view_as(p)
            if p.grad is None or p.grad.data_ptr() != v.data_ptr():
                p.grad = v

    def state_bytes(self) -> int:
        """Bytes of optimizer state held by this rank (for the 1/P claim), the fp32 master shard
        included in master mode."""
        import torch

        master = self.shard.numel() * self.shard.element_size() if self.master else 0
        return master + sum(v.numel() * v.element_size() for st in self.optimizer.state.values() for v in st.values()
                            if isinstance(v, torch.Tensor))


class TensorParallel(_Base):
    """Megatron tensor parallelism: row-parallel output is an allreduce of partial sums;
    column-parallel output is an allgather along the feature dimension.

    ``column_linear`` / ``row_linear`` build the two layers of a tensor-parallel MLP block with
    the collectives placed as autograd functions (Megatron's f / g operators): the forward of a
    column -> row pair costs ONE allreduce (after the row-parallel matmul), the backward one
    (before the column-parallel weight gradient)."""

    def row_parallel_output(self, partial):
        return self._allreduce(partial)

    def column_parallel_gather(self, local, out):
        if _is_cuda(local):
            self.cc.allgather(out, local)
        else:
            H.allgather(self.ctx, out, local)
        return out

    # ---- autograd-aware operators --------------------------------------------------------------
    def copy_to_region(self, x):
        """f: identity in the forward pass, allreduce of the gradient in the backward pass."""
        import torch

        tp = self

        class _F(torch.autograd.Function):
            @staticmethod
            def forward(ctx, inp):
                return inp.view_as(inp)

            @staticmethod
            def backward(ctx, grad):
                return tp._allreduce(grad.contiguous().clone())

        return _F.apply(x)

    def reduce_from_region(self, x):
        """g: allreduce in the forward pass, identity in the backward pass."""
        import torch

        tp = self

        class _G(torch.autograd.Function):
            @staticmethod
            def forward(ctx, inp):
                return tp._allreduce(inp.contiguous().clone())

            @staticmethod
            def backward(ctx, grad):
                return grad

        return _G.apply(x)

    def reduce_residual_norm(self, partial, residual, norm_module=None, bias=None, copy_out: bool = False,
                             fp8: bool = False):
        """g fused with what follows a row-parallel matmul: ``s = allreduce(partial) + bias +
        residual`` and the next norm. Returns ``(s, norm_module(s))``, or ``s`` when
        ``norm_module`` is None. ``norm_module`` is an ``nn.LayerNorm``, an ``nn.RMSNorm`` or None.

        CUDA tensors within the fused operation's limits run it as one kernel
        (``CudaContext.allreduce_residual_norm``), into a fresh ``s``. The backward is g's: the
        gradient of ``s`` plus the norm's input gradient (recomputed from the saved ``s``) goes to
        both ``partial`` and ``residual``, its row sum to ``bias``, and the norm's weights get
        theirs from the recompute. Anything else runs ``reduce_from_region``, ``+ bias``,
        ``+ residual`` and the module.

        ``copy_out``: ``out`` is returned inside the tensor-parallel region, as
        ``copy_to_region(norm_module(s))`` (Megatron's f, fused; it needs a norm). The gradient of
        ``out`` that reaches the backward is then this rank's partial, which the backward
        allreduces. After a fused forward that is one fused kernel
        (``CudaContext.allreduce_residual_norm_backward``), which gives every rank the same bytes of
        every gradient and computes only the vector gradients autograd needs; a gradient it cannot
        take (dtype, alignment) is allreduced and the norm recomputed with torch.

        ``fp8``: returns ``(s, (codes, scales))``, the norm's output as float8_e4m3fn codes and
        float32 per-row scales ``(..., 1)`` (``fp8_rows`` of it, byte for byte), for a row-wise scaled
        FP8 GEMM. The fused kernel quantises in the same launch
        (``CudaContext.allreduce_residual_norm(out_scales=)``); where it cannot run (as above, or H
        not a multiple of 16) the composition above runs, then ``fp8_rows``. Forward-only: with
        grad mode on, an input or norm parameter that requires grad raises ``ValueError``."""
        import torch

        if copy_out and norm_module is None:
            raise ValueError("reduce_residual_norm: copy_out needs a norm_module")
        kind, weight, norm_bias, eps = _norm_parts(norm_module, partial.dtype)
        if fp8:
            if copy_out:
                raise ValueError("reduce_residual_norm: fp8 is forward-only and takes no copy_out")
            _check_fp8_call("reduce_residual_norm", norm_module, (partial, residual, bias, weight, norm_bias))
            if not self._fusable(partial, residual, norm_module, kind, (bias, weight, norm_bias)) or \
                    partial.shape[-1] % 16:
                s, out = self.reduce_residual_norm(partial, residual, norm_module, bias)
                return s, fp8_rows(out)
            s = torch.empty_like(residual, memory_format=torch.contiguous_format)
            scales = torch.empty((*partial.shape[:-1], 1), dtype=torch.float32, device=partial.device)
            _, codes = self.cc.allreduce_residual_norm(partial.contiguous(), residual.contiguous(), weight, norm_bias,
                                                       norm=kind, eps=eps, bias=bias, residual_out=s, out_scales=scales)
            return s, (codes, scales)
        if not self._fusable(partial, residual, norm_module, kind, (bias, weight, norm_bias)):
            y = self.reduce_from_region(partial)
            if bias is not None:
                y = y + bias
            s = y + residual
            if norm_module is None:
                return s
            out = norm_module(s)
            return s, (self.copy_to_region(out) if copy_out else out)
        H = partial.shape[-1]
        tp = self

        class _R(torch.autograd.Function):
            @staticmethod
            def forward(ctx, p, res, b, w, nb):
                s = torch.empty_like(res, memory_format=torch.contiguous_format)
                got = tp.cc.allreduce_residual_norm(p.contiguous(), res.contiguous(), w, nb, norm=kind, eps=eps, bias=b,
                                                   residual_out=s)
                ctx.save_for_backward(s, w, nb)
                ctx.has_bias = b is not None
                return got

            @staticmethod
            def backward(ctx, grad_s, grad_out=None):
                s, w, nb = ctx.saved_tensors
                if copy_out and grad_out is not None:
                    if _aligned_like(s, grad_out, grad_s):
                        need_b, need_w, need_nb = ctx.needs_input_grad[2:5]
                        vec = lambda t, need: torch.empty(H, dtype=s.dtype, device=s.device) if t and need else None  # noqa: E731
                        gp, gw, gnb, gb = tp.cc.allreduce_residual_norm_backward(
                            grad_out.contiguous(), s, None if grad_s is None else grad_s.contiguous(), w, norm=kind,
                            eps=eps, grad_weight=vec(w is not None, need_w), grad_norm_bias=vec(nb is not None, need_nb),
                            grad_bias=vec(ctx.has_bias, need_b))
                        return gp, gp, gb, gw, gnb
                    grad_out = tp._allreduce(grad_out.contiguous().clone())
                grad_s = torch.zeros_like(s) if grad_s is None else grad_s
                gw = gnb = None
                if kind is not None and grad_out is not None:
                    gs, gw, gnb = _norm_input_grad(kind, H, eps, s, w, nb, grad_out)
                    grad_s = grad_s + gs
                gb = grad_s.reshape(-1, H).sum(0) if ctx.has_bias else None
                return grad_s, grad_s, gb, gw, gnb

        return _R.apply(partial, residual, bias, weight, norm_bias)

    def _fusable(self, partial, residual, norm_module, kind, vectors) -> bool:
        """Whether reduce_residual_norm can run the fused kernel on these tensors."""
        return _norm_fusable(self.cc, partial, residual, tuple(partial.shape), norm_module, kind, vectors)

    def column_linear(self, in_features: int, out_features: int, bias: bool = True, device=None, dtype=None):
        return ColumnParallelLinear(self, in_features, out_features, bias, device, dtype)

    def row_linear(self, in_features: int, out_features: int, bias: bool = True, device=None, dtype=None):
        return RowParallelLinear(self, in_features, out_features, bias, device, dtype)


def _shard(n: int, size: int, rank: int):
    assert n % size == 0, f"{n} features do not split over {size} ranks"
    return n // size * rank, n // size * (rank + 1)


try:  # the layer classes need torch; everything else in this module does not
    import torch as _torch

    class ColumnParallelLinear(_torch.nn.Module):
        """y_local = x W_r^T + b_r with W split along the OUTPUT features (rank r holds rows
        [r, r+1) * out/P). The input is replicated; its gradient is summed over ranks (f)."""

        def __init__(self, tp: TensorParallel, in_features, out_features, bias=True, device=None, dtype=None):
            super().__init__()
            self.tp = tp
            self.lo, self.hi = _shard(out_features, tp.size, tp.rank)
            self.weight = _torch.nn.Parameter(_torch.empty(self.hi - self.lo, in_features, device=device, dtype=dtype))
            self.bias = _torch.nn.Parameter(_torch.zeros(self.hi - self.lo, device=device, dtype=dtype)) if bias else None
            _torch.nn.init.kaiming_uniform_(self.weight, a=5 ** 0.5)

        def load_full(self, weight, bias=None):
            with _torch.no_grad():
                self.weight.copy_(weight[self.lo:self.hi])
                if self.bias is not None and bias is not None:
                    self.bias.copy_(bias[self.lo:self.hi])

        def forward(self, x):
            return _torch.nn.functional.linear(self.tp.copy_to_region(x), self.weight, self.bias)

    class RowParallelLinear(_torch.nn.Module):
        """y = sum_r x_r W_r^T + b with W split along the INPUT features; the input arrives already
        split (the output of a ColumnParallelLinear); one allreduce of the partial products (g)."""

        def __init__(self, tp: TensorParallel, in_features, out_features, bias=True, device=None, dtype=None):
            super().__init__()
            self.tp = tp
            self.lo, self.hi = _shard(in_features, tp.size, tp.rank)
            self.weight = _torch.nn.Parameter(_torch.empty(out_features, self.hi - self.lo, device=device, dtype=dtype))
            self.bias = _torch.nn.Parameter(_torch.zeros(out_features, device=device, dtype=dtype)) if bias else None
            _torch.nn.init.kaiming_uniform_(self.weight, a=5 ** 0.5)

        def load_full(self, weight, bias=None):
            with _torch.no_grad():
                self.weight.copy_(weight[:, self.lo:self.hi])
                if self.bias is not None and bias is not None:
                    self.bias.copy_(bias)

        def forward(self, x_local):
            y = self.tp.reduce_from_region(_torch.nn.functional.linear(x_local, self.weight))
            return y if self.bias is None else y + self.bias
except ImportError:  # pragma: no cover
    ColumnParallelLinear = RowParallelLinear = None


class SequenceParallel(_Base):
    """Megatron sequence parallelism: reduce_scatter along the sequence going in,
    allgather coming out.

    The autograd operators shard along dim 0 (the sequence, in Megatron's sequence-first layout
    ``[S, B, E]``); rank r holds rows ``[r * S / P, (r + 1) * S / P)``. ``gather_from_sequence``
    feeds a column-parallel layer from the shard, ``reduce_scatter_to_sequence`` brings a
    row-parallel output back to it, and ``reduce_scatter_residual_norm`` fuses the latter with bias,
    residual add and the next norm. Replicated parameters applied to the shard (norm weights and
    biases, row-parallel biases) get gradients from this rank's tokens only:
    ``allreduce_sequence_parallel_grads`` sums them after the backward."""

    def scatter_reduce(self, full, shard):
        return ZeroShard(self.ctx, self.cc).reduce_scatter_gradients(full, shard, average=False)

    def gather(self, shard, full):
        return ZeroShard(self.ctx, self.cc).allgather_parameters(full, shard)

    # ---- autograd-aware operators --------------------------------------------------------------
    def _allgather_rows(self, shard):
        import torch

        shard = shard.contiguous()
        full = torch.empty((self.size * shard.shape[0], *shard.shape[1:]), dtype=shard.dtype, device=shard.device)
        if _is_cuda(shard):
            self.cc.allgather(full, shard)
        else:
            H.allgather(self.ctx, full, shard)
        return full

    def _reduce_scatter_rows(self, full):
        import torch

        if full.shape[0] % self.size:
            raise ValueError(f"{full.shape[0]} rows do not split into {self.size} equal shards")
        full = full.contiguous()
        out = torch.empty((full.shape[0] // self.size, *full.shape[1:]), dtype=full.dtype, device=full.device)
        if _is_cuda(full):
            self.cc.reduce_scatter(out, full)
        else:
            H.reduce_scatter(self.ctx, out, full, [out.numel()] * self.size)
        return out

    def gather_from_sequence(self, x_shard):
        """Allgather of the shards along dim 0 in the forward pass, reduce-scatter of the gradient
        in the backward pass."""
        import torch

        sp = self

        class _Gather(torch.autograd.Function):
            @staticmethod
            def forward(ctx, inp):
                return sp._allgather_rows(inp)

            @staticmethod
            def backward(ctx, grad):
                return sp._reduce_scatter_rows(grad)

        return _Gather.apply(x_shard)

    def reduce_scatter_to_sequence(self, x):
        """Reduce-scatter along dim 0 in the forward pass, allgather of the gradient in the
        backward pass."""
        import torch

        sp = self

        class _Scatter(torch.autograd.Function):
            @staticmethod
            def forward(ctx, inp):
                return sp._reduce_scatter_rows(inp)

            @staticmethod
            def backward(ctx, grad):
                return sp._allgather_rows(grad)

        return _Scatter.apply(x)

    def reduce_scatter_residual_norm(self, partial, residual_shard, norm_module=None, bias=None,
                                     gather_out: bool = True, fp8: bool = False):
        """``reduce_scatter_to_sequence`` fused with what follows a row-parallel matmul: ``s =
        reduce_scatter(partial) + bias + residual_shard`` on this rank's shard and the next norm,
        whose output is allgathered when ``gather_out``. Returns ``(s, out)``, or ``s`` when
        ``norm_module`` (an ``nn.LayerNorm``, an ``nn.RMSNorm`` or None) is None.

        CUDA tensors within the fused operation's limits run it as one kernel
        (``CudaContext.reduce_scatter_residual_norm``), into a fresh ``s``. Its backward
        reduce-scatters the gradient of a gathered ``out``, adds the norm's input gradient
        (recomputed from the saved ``s``) to the gradient of ``s``, and allgathers that sum into the
        gradient of ``partial``; ``residual_shard`` gets the sum, ``bias`` its row sum and the norm's
        weights theirs, all from this rank's tokens. With a norm whose ``out`` got a gradient that is
        one fused kernel too (``CudaContext.reduce_scatter_residual_norm_backward``); otherwise it
        runs the collectives and a torch recompute of the norm. Anything else
        runs ``reduce_scatter_to_sequence``, ``+ bias``, ``+ residual_shard``, the module and
        ``gather_from_sequence``.

        ``fp8``: returns ``(s, (codes, scales))``, ``out`` as float8_e4m3fn codes and float32 per-row
        scales ``(..., 1)`` (``fp8_rows`` of it, byte for byte); a gathered ``out`` travels as codes
        and scales. Where the fused kernel cannot run (as above, or H not a multiple of 16) the
        composition above runs, then ``fp8_rows``. Forward-only, as in
        ``TensorParallel.reduce_residual_norm``."""
        import torch

        kind, weight, norm_bias, eps = _norm_parts(norm_module, partial.dtype)
        if fp8:
            _check_fp8_call("reduce_scatter_residual_norm", norm_module,
                            (partial, residual_shard, bias, weight, norm_bias))
        fused = (partial.dim() > 0 and partial.shape[0] % self.size == 0 and
                 _norm_fusable(self.cc, partial, residual_shard, (partial.shape[0] // self.size, *partial.shape[1:]),
                               norm_module, kind, (bias, weight, norm_bias)) and
                 not (fp8 and partial.shape[-1] % 16))
        if fused:
            from ..types import _torch_map

            try:  # a row too wide for the staging pool is outside the limits too
                _C.cuda.plan_reduce_scatter_norm(self.cc.pc, partial.numel() // partial.shape[-1], partial.shape[-1],
                                                 int(_torch_map()[partial.dtype]), {None: 0, "rms": 1, "layer": 2}[kind],
                                                 gather_out, fp8)
            except ValueError:
                fused = False
        if fp8 and not fused:
            s, out = self.reduce_scatter_residual_norm(partial, residual_shard, norm_module, bias, gather_out)
            return s, fp8_rows(out)
        if fp8:
            s = torch.empty_like(residual_shard, memory_format=torch.contiguous_format)
            rows = partial.shape if gather_out else residual_shard.shape
            scales = torch.empty((*rows[:-1], 1), dtype=torch.float32, device=partial.device)
            _, codes = self.cc.reduce_scatter_residual_norm(partial.contiguous(), residual_shard.contiguous(), weight,
                                                            norm_bias, norm=kind, eps=eps, bias=bias, residual_out=s,
                                                            gather_out=gather_out, out_scales=scales)
            return s, (codes, scales)
        if not fused:
            y = self.reduce_scatter_to_sequence(partial)
            if bias is not None:
                y = y + bias
            s = y + residual_shard
            if norm_module is None:
                return s
            out = norm_module(s)
            return s, (self.gather_from_sequence(out) if gather_out else out)
        H = partial.shape[-1]
        sp = self

        class _RS(torch.autograd.Function):
            @staticmethod
            def forward(ctx, p, res, b, w, nb):
                s = torch.empty_like(res, memory_format=torch.contiguous_format)
                got = sp.cc.reduce_scatter_residual_norm(p.contiguous(), res.contiguous(), w, nb, norm=kind, eps=eps,
                                                         bias=b, residual_out=s, gather_out=gather_out)
                ctx.save_for_backward(s, w, nb)
                ctx.has_bias = b is not None
                return got

            @staticmethod
            def backward(ctx, grad_s, grad_out=None):
                s, w, nb = ctx.saved_tensors
                if kind is not None and grad_out is not None and _aligned_like(s, grad_out, grad_s):
                    need_b, need_w, need_nb = ctx.needs_input_grad[2:5]
                    vec = lambda t, need: torch.empty(H, dtype=s.dtype, device=s.device) if t and need else None  # noqa: E731
                    gp, gr, gw, gnb, gb = sp.cc.reduce_scatter_residual_norm_backward(
                        grad_out.contiguous(), s, None if grad_s is None else grad_s.contiguous(), w, norm=kind,
                        eps=eps, gather_out=gather_out, grad_weight=vec(w is not None, need_w),
                        grad_norm_bias=vec(nb is not None, need_nb), grad_bias=vec(ctx.has_bias, need_b))
                    return gp, gr, gb, gw, gnb
                grad_s = torch.zeros_like(s) if grad_s is None else grad_s
                gw = gnb = None
                if kind is not None and grad_out is not None:
                    if gather_out:
                        grad_out = sp._reduce_scatter_rows(grad_out)
                    gs, gw, gnb = _norm_input_grad(kind, H, eps, s, w, nb, grad_out)
                    grad_s = grad_s + gs
                gb = grad_s.reshape(-1, H).sum(0) if ctx.has_bias else None
                return sp._allgather_rows(grad_s), grad_s, gb, gw, gnb

        return _RS.apply(partial, residual_shard, bias, weight, norm_bias)

    def allreduce_sequence_parallel_grads(self, params: Iterable):
        """Sum over the group, in place, the gradients of replicated parameters that each rank
        applied to its token shard only (norm weights and biases, row-parallel biases): one
        allreduce per dtype and device. Call after the backward, before the optimizer step."""
        import torch

        groups = {}
        for p in params:
            if getattr(p, "grad", None) is not None:
                groups.setdefault((p.grad.dtype, p.grad.device), []).append(p.grad)
        for grads in groups.values():
            flat = torch.cat([g.reshape(-1) for g in grads])
            self._allreduce(flat)
            off = 0
            for g in grads:
                g.copy_(flat[off:off + g.numel()].view_as(g))
                off += g.numel()


class MoEDispatcher(_Base):
    """Expert parallelism: tokens routed to experts living on other ranks.

    dispatch(): rows of ``tokens`` (already sorted by destination rank) are exchanged
    with alltoallv; the per-source receive counts come from a tiny alltoall of the
    send counts. combine() is the inverse exchange.
    """

    def exchange_counts(self, send_counts: Sequence[int]) -> List[int]:
        import numpy as np

        s = np.asarray(send_counts, dtype=np.int64)
        r = np.zeros_like(s)
        H.alltoall(self.ctx, r, s)
        return [int(x) for x in r]

    def dispatch(self, tokens, send_counts: Sequence[int], out, recv_counts: Optional[Sequence[int]] = None):
        if recv_counts is None:
            recv_counts = self.exchange_counts(send_counts)
        width = tokens.shape[-1] if tokens.dim() > 1 else 1
        sc = [c * width for c in send_counts]
        rc = [c * width for c in recv_counts]
        if _is_cuda(tokens):
            self.cc.alltoallv(out, rc, tokens, sc)
        else:
            H.alltoallv(self.ctx, out, rc, tokens, sc)
        return out, list(recv_counts)

    def combine(self, expert_out, recv_counts: Sequence[int], out, send_counts: Sequence[int]):
        # inverse of dispatch: what I received goes back to where it came from
        return self.dispatch(expert_out, recv_counts, out, send_counts)[0]

    def dispatch_dev(self, tokens, splits, out, experts: int = 1, align: int = 1):
        """dispatch() with the counts on the device: no ``.tolist()``, no host count exchange, one
        kernel (CUDA graph capturable). ``splits``: int64 CUDA tensor, entry ``j * experts + e`` =
        rows of ``tokens`` (packed in that order) for local expert ``e`` of rank ``j``. ``out``
        receives expert-major (see ``CudaContext.alltoallv_dev``). Returns
        ``(out, out_splits, out_offsets)``, entry ``e * size + s`` = rows from rank ``s`` for my
        expert ``e`` and where they start. Overflow or invalid splits surface as ``ValueError`` at
        the next ``cc.synchronize()`` (see ``CudaContext.alltoallv_dev``)."""
        import torch

        out_splits = torch.empty(self.size * experts, dtype=torch.int64, device=tokens.device)
        out_offsets = torch.empty_like(out_splits)
        self.cc.alltoallv_dev(out, tokens, splits, out_splits, out_offsets, experts=experts, align=align)
        return out, out_splits, out_offsets

    def dispatch_dev_fp8(self, tokens, splits, out, out_scales, experts: int = 1, align: int = 1):
        """dispatch_dev() that quantises on the way: ``tokens`` bf16 ``(rows, H)``, H a multiple of
        128; ``out`` float8_e4m3fn ``(cap, H)`` receives the codes and ``out_scales`` float32
        ``(cap, H // 128)`` one scale per 1x128 block, row for row (see
        ``CudaContext.alltoallv_dev``). One kernel, no host sync, half the bytes of a bf16 dispatch
        on the link. Returns ``(out, out_scales, out_splits, out_offsets)``. The experts' bf16
        outputs go back with combine_dev(): the row layout is the same."""
        import torch

        out_splits = torch.empty(self.size * experts, dtype=torch.int64, device=tokens.device)
        out_offsets = torch.empty_like(out_splits)
        self.cc.alltoallv_dev(out, tokens, splits, out_splits, out_offsets, experts=experts, align=align,
                              out_scales=out_scales)
        return out, out_scales, out_splits, out_offsets

    dispatch_fp8 = dispatch_dev_fp8

    def combine_dev(self, expert_out, out_splits, out_offsets, out, experts: int = 1):
        """Inverse of dispatch_dev(): the rows of ``expert_out`` (dispatch_dev's layout) go back to
        their sources; ``out`` gets them where the dispatched ``tokens`` rows were."""
        return self.cc.alltoallv_dev_combine(out, expert_out, out_splits, out_offsets, experts=experts)

    def route(self, x, topk_idx, experts: int = 1):
        """Dispatch input for top-k routing, in pure torch with no host synchronisation (CPU tensors
        work too). ``topk_idx`` is ``(T, k)``: entry ``j * experts + e`` sends the token to local
        expert ``e`` of rank ``j``; an entry outside ``0 .. size * experts - 1``, such as -1, is not
        routed. Returns ``(rows, splits, pos)``:
        - ``rows`` holds ``T * k`` rows of ``x``. The first ``splits.sum()`` are the routed
          choices, packed in (rank, expert) order and by token within each, ready for
          ``dispatch_dev``. The rest are unrouted choices and are never sent.
        - ``splits`` is the int64 ``(size * experts,)`` row count per (rank, expert).
        - ``pos`` is int64 ``(T, k)``: the row of ``rows`` that carries each choice, or -1. It is
          what ``combine_dev_topk`` takes."""
        import torch

        T, k = int(topk_idx.shape[0]), int(topk_idx.shape[1])
        G = self.size * int(experts)
        flat = topk_idx.reshape(-1).long()
        routed = (flat >= 0) & (flat < G)
        key = torch.where(routed, flat, torch.full_like(flat, G))  # unrouted choices sort last
        order = torch.argsort(key, stable=True)
        counts = torch.zeros(G + 1, dtype=torch.int64, device=flat.device)
        counts.index_add_(0, key, torch.ones_like(key))
        pos = torch.empty_like(flat).scatter_(0, order, torch.arange(T * k, dtype=torch.int64, device=flat.device))
        pos = torch.where(routed, pos, torch.full_like(pos, -1)).view(T, k)
        return x.index_select(0, order // k), counts[:G], pos

    def dispatch_dev_topk(self, x, topk_idx, out, experts: int = 1, align: int = 1, out_scales=None):
        """route() + dispatch_dev() (or dispatch_dev_fp8() when ``out_scales`` is given) in one kernel:
        ``x (T, H)`` and ``topk_idx (T, k)`` in, each token's row read once and stored to each of its
        k destinations, with no host sync and no ``T * k`` copy of the rows. The results equal route()
        followed by the dispatch byte for byte (see ``CudaContext.alltoallv_dev_topk``). Returns
        ``(out, out_splits, out_offsets, splits, pos)``, with ``out_scales`` after ``out`` in the FP8
        form; ``splits`` and ``pos`` are what combine_dev_topk() takes."""
        import torch

        G = self.size * int(experts)
        dev = x.device
        splits = torch.empty(G, dtype=torch.int64, device=dev)
        out_splits = torch.empty_like(splits)
        out_offsets = torch.empty_like(splits)
        pos = torch.empty(tuple(topk_idx.shape), dtype=torch.int64, device=dev)
        self.cc.alltoallv_dev_topk(out, x, topk_idx, splits, pos, out_splits, out_offsets, experts=experts, align=align,
                                   out_scales=out_scales)
        if out_scales is not None:
            return out, out_scales, out_splits, out_offsets, splits, pos
        return out, out_splits, out_offsets, splits, pos

    def combine_dev_topk(self, expert_out, splits, pos, weights, out, experts: int = 1, align: int = 1):
        """The inverse of dispatch_dev() fused with the gate-weighted sum: ``out[t]`` = sum over
        token t's routed choices j of ``weights[t, j]`` times its expert's output row, in fp32 in
        the order of j, rounded to ``out``'s dtype. ``splits`` and ``pos`` come from route() (or
        describe the dispatch input the same way), ``expert_out`` is in dispatch_dev()'s output
        layout with the same ``experts`` and ``align``. See
        ``CudaContext.alltoallv_dev_combine_topk``."""
        return self.cc.alltoallv_dev_combine_topk(out, expert_out, splits, pos, weights, experts=experts, align=align)

    def combine_dev_topk_backward(self, grad_out, expert_out, splits, pos, weights, grad_expert_out, grad_weights,
                                  experts: int = 1, align: int = 1):
        """The backward of combine_dev_topk() in one kernel: ``grad_weights[t, j]`` = the fp32 dot of
        ``grad_out[t]`` with choice j's expert row, and ``weights[t, j] * grad_out[t]`` written to that
        row of its holder's ``grad_expert_out`` (zero in every row outside the received segments).
        Returns ``(grad_expert_out, grad_weights)``. See
        ``CudaContext.alltoallv_dev_combine_topk_backward``."""
        return self.cc.alltoallv_dev_combine_topk_backward(grad_expert_out, grad_weights, grad_out, expert_out, splits,
                                                           pos, weights, experts=experts, align=align)

    # ---- low-latency form, for decoding ---------------------------------------------------------
    def dispatch_ll(self, x, topk_idx, buf, out, out_scales=None):
        """The low-latency top-k dispatch on ``buf`` (``cc.moe_ll_buffer``): fixed per-expert slots,
        one signal round, static shapes, so a decode step can be captured in a CUDA graph. ``out`` is
        ``(experts, size * max_tokens, hidden)``; expert ``e``'s rows are ``out[e, :count]``, byte for
        byte its segment of dispatch_dev_topk(). Returns ``(out, out_splits)``, or for an FP8 buffer
        ``(out, out_scales, out_splits)``. See ``CudaContext.alltoallv_ll_topk``."""
        import torch

        out_splits = torch.empty(self.size * buf.experts, dtype=torch.int64, device=x.device)
        self.cc.alltoallv_ll_topk(buf, out, x, topk_idx, out_splits, out_scales=out_scales)
        if out_scales is not None:
            return out, out_scales, out_splits
        return out, out_splits

    def combine_ll(self, expert_out, weights, buf, y):
        """The low-latency combine after dispatch_ll() on the same ``buf``: ``y[t]`` = the weighted sum
        of token t's expert rows, byte for byte combine_dev_topk()'s. ``weights`` may be None (weight
        1). See ``CudaContext.alltoallv_ll_combine_topk``."""
        return self.cc.alltoallv_ll_combine_topk(buf, y, expert_out, weights)

    # ---- autograd ------------------------------------------------------------------------------
    # Each backward is a collective: every rank's backward pass must reach it, in the same order. The
    # backward kernels run on the stream current in the backward pass, on plain gradient tensors, so
    # they take the staged path.
    def dispatch_topk_autograd(self, x, topk_idx, out, experts: int = 1, align: int = 1):
        """dispatch_dev_topk() that autograd can differentiate in ``x``. Returns ``(expert_in,
        out_splits, out_offsets, routing)``: ``expert_in`` is a view of ``out``; ``routing`` holds
        ``splits``, ``pos``, ``experts`` and ``align`` for combine_topk_autograd(). The backward
        sums each token's k expert-input gradient rows (the top-k combine with every weight 1)
        into a fresh ``grad_x``. FP8 dispatch is not differentiable."""
        import torch

        moe = self

        class _Dispatch(torch.autograd.Function):
            @staticmethod
            def forward(ctx, inp):
                _, out_splits, out_offsets, splits, pos = moe.dispatch_dev_topk(inp, topk_idx, out, experts=experts,
                                                                               align=align)
                ctx.routing = MoERouting(splits, pos, experts, align)
                ctx.mark_non_differentiable(out_splits, out_offsets, splits, pos)
                return out.view_as(out), out_splits, out_offsets, splits, pos

            @staticmethod
            def backward(ctx, grad, *_):
                r = ctx.routing
                g = grad.contiguous()
                grad_x = torch.empty((r.pos.shape[0], *g.shape[1:]), dtype=g.dtype, device=g.device)
                moe.cc.alltoallv_dev_combine_topk(grad_x, g, r.splits, r.pos, None, experts=r.experts, align=r.align)
                return grad_x

        expert_in, out_splits, out_offsets, splits, pos = _Dispatch.apply(x)
        return expert_in, out_splits, out_offsets, MoERouting(splits, pos, experts, align)

    def combine_topk_autograd(self, expert_out, weights, routing):
        """combine_dev_topk() into a fresh ``y`` that autograd can differentiate in ``expert_out``
        and ``weights`` (float32 ``(T, k)``); ``routing`` comes from dispatch_topk_autograd(). The
        backward is one kernel (combine_dev_topk_backward()): the gradient rows go back to the
        experts' holders and the weight gradients are computed where the weights live. A registered
        or symmetric ``expert_out`` is copied to a plain tensor for the backward, whose gradient
        tensors are plain."""
        import torch

        moe, r = self, routing

        class _Combine(torch.autograd.Function):
            @staticmethod
            def forward(ctx, eo, w):
                eo, w = eo.contiguous(), w.contiguous()
                y = torch.empty((r.pos.shape[0], *eo.shape[1:]), dtype=eo.dtype, device=eo.device)
                moe.cc.alltoallv_dev_combine_topk(y, eo, r.splits, r.pos, w, experts=r.experts, align=r.align)
                ctx.save_for_backward(eo, w)
                return y

            @staticmethod
            def backward(ctx, dy):
                eo, w = ctx.saved_tensors
                if moe.cc.lookup(eo)[0] is not None:
                    eo = eo.clone()
                grad_eo = torch.empty_like(eo)
                grad_w = torch.empty_like(w)
                moe.combine_dev_topk_backward(dy.contiguous(), eo, r.splits, r.pos, w, grad_eo, grad_w,
                                              experts=r.experts, align=r.align)
                return grad_eo, grad_w

        return _Combine.apply(expert_out, weights)


class MoERouting:
    """Where dispatch_topk_autograd() sent each token's choices: the dispatch ``splits`` and ``pos``
    (device tensors) and its ``experts`` and ``align``. Not differentiable."""

    __slots__ = ("splits", "pos", "experts", "align")

    def __init__(self, splits, pos, experts: int, align: int):
        self.splits, self.pos, self.experts, self.align = splits, pos, int(experts), int(align)


class UlyssesAttention(_Base):
    """DeepSpeed-Ulysses: [S/P, H, D] <-> [S, H/P, D] with one alltoall each way."""

    def seq_to_heads(self, x, out):
        if _is_cuda(x):
            self.cc.alltoall(out, x)
        else:
            H.alltoall(self.ctx, out, x)
        return out

    heads_to_seq = seq_to_heads

    def attention(self, q, k, v, causal: bool = False):
        """Full Ulysses attention: q / k / v are this rank's sequence shard [S/P, H, D]; one alltoall
        turns them into all positions of H/P heads ([S, H/P, D]), attention runs locally over the
        whole sequence, one alltoall brings the output back to [S/P, H, D]. On CUDA the exchange
        buffers are symmetric (zero-copy push kernels); three alltoalls in, one out."""
        import torch

        P, r = self.size, self.rank
        s_loc, Hh, D = q.shape
        assert Hh % P == 0, "heads must divide over the ranks"
        hp = Hh // P

        def alloc(n, like):
            return self.cc.empty(n, like.dtype) if _is_cuda(like) else torch.empty(n, dtype=like.dtype)

        def to_heads(x):      # [S/P, H, D] -> [S, H/P, D]
            send = x.view(s_loc, P, hp, D).transpose(0, 1).contiguous()      # block j = my positions of head group j
            out = alloc(send.numel(), x)
            self.seq_to_heads(send.view(-1), out)
            return out.view(P * s_loc, hp, D)                                # block i = rank i's positions, my heads

        def to_seq(y):        # [S, H/P, D] -> [S/P, H, D]
            send = y.contiguous()                                           # block i = positions of rank i
            out = alloc(send.numel(), y)
            self.seq_to_heads(send.view(-1), out)
            return out.view(P, s_loc, hp, D).transpose(0, 1).reshape(s_loc, Hh, D)

        qh, kh, vh = to_heads(q), to_heads(k), to_heads(v)
        o = torch.nn.functional.scaled_dot_product_attention(qh.transpose(0, 1), kh.transpose(0, 1), vh.transpose(0, 1),
                                                             is_causal=causal).transpose(0, 1)
        return to_seq(o)


class RingExchange(_Base):
    """Neighbour exchange for ring attention (KV rotation) and pipeline parallelism.

    CPU tensors go through UnboundBuffer send/recv. CUDA tensors: when ``recv`` is a symmetric /
    registered tensor (``kv_buffers``) the zero-copy kernel writes ``send`` straight into the right
    neighbour's copy of it (``CudaContext.exchange``: one pass, ~link rate); any other tensor goes
    through the fused send+recv kernel and its mailbox ring (``CudaContext.sendrecv``).
    """

    def kv_buffers(self, numel: int, dtype):
        """Two symmetric buffers to rotate between (every rank must call this in the same order)."""
        return self.cc.empty(numel, dtype), self.cc.empty(numel, dtype)

    def rotate(self, send, recv, step: int = 1):
        right, left = (self.rank + step) % self.size, (self.rank - step) % self.size
        if self.size == 1:
            recv.copy_(send)
            return recv
        if _is_cuda(send):
            self.cc.exchange(send, right, recv, left)   # falls back to sendrecv() for unregistered tensors
            return recv
        from ..types import describe

        sp, sn, sdt, _ = describe(send)
        rp, rn, _, _ = describe(recv)
        nbytes = send.numel() * send.element_size() if hasattr(send, "numel") else send.nbytes
        sb = self.ctx.create_unbound_buffer(sp, nbytes)
        rb = self.ctx.create_unbound_buffer(rp, nbytes)
        slot = _C.slot_build(0x7E, step)
        rb.recv(left, slot)
        sb.send(right, slot)
        rb.wait_recv()
        sb.wait_send()
        return recv

    def attention(self, q, k, v, causal: bool = False):
        """Ring attention (forward): rank r holds the queries and the K/V block of sequence shard r
        ([S/P, H, D] each); K/V blocks rotate once around the ring while every rank folds the block
        it currently holds into a running (max, sum, output) with the online-softmax recurrence, so
        no rank ever materialises more than two K/V blocks. The rotation of the NEXT block is
        posted before the current one is consumed (double buffer: on CUDA the two halves of a
        symmetric buffer, written by the neighbour's zero-copy ``exchange`` kernel on a side
        stream while the attention math runs). ``causal``: shard r attends to shards <= r.
        Returns [S/P, H, D] in q's dtype. The math is plain torch (fp32 accumulation)."""
        import torch

        P, r = self.size, self.rank
        scale = q.shape[-1] ** -0.5
        qf = q.float().transpose(0, 1)                                    # [H, Sq, D]
        m = torch.full(qf.shape[:2], float("-inf"), device=q.device)      # running max   [H, Sq]
        l = torch.zeros(qf.shape[:2], device=q.device)                    # running sum   [H, Sq]
        acc = torch.zeros_like(qf)                                        # running out   [H, Sq, D]
        kv = torch.stack([k, v]).contiguous()
        cuda = _is_cuda(kv)
        if cuda and P > 1:
            cur, nxt = self.kv_buffers(kv.numel(), kv.dtype)
            cur = cur.view_as(kv)
            nxt = nxt.view_as(kv)
            cur.copy_(kv)
            side = getattr(self, "_side", None)
            if side is None:
                from ..ops.cuda import new_stream

                side = self._side = new_stream(kv.device.index)
        else:
            cur, nxt = kv, torch.empty_like(kv)
        for step in range(P):
            src = (r - step) % P                                          # whose block `cur` is
            if step + 1 < P:                                              # post the next rotation first
                if cuda:
                    ready = torch.cuda.Event()
                    ready.record(torch.cuda.current_stream())
                    side.wait_event(ready)
                    self.cc.exchange(cur, (r + 1) % P, nxt, (r - 1) % P, stream=side)
                    landed = torch.cuda.Event()
                    landed.record(side)
                else:
                    self.rotate(cur, nxt)
            if not (causal and src > r):
                kf, vf = cur[0].float().transpose(0, 1), cur[1].float().transpose(0, 1)   # [H, Sk, D]
                s = torch.matmul(qf, kf.transpose(1, 2)) * scale                          # [H, Sq, Sk]
                if causal and src == r:
                    sq, sk = s.shape[-2:]
                    s = s.masked_fill(torch.ones(sq, sk, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
                m_new = torch.maximum(m, s.amax(dim=-1))
                p = torch.exp(s - m_new.unsqueeze(-1))
                alpha = torch.exp(m - m_new)
                l = l * alpha + p.sum(dim=-1)
                acc = acc * alpha.unsqueeze(-1) + torch.matmul(p, vf)
                m = m_new
            if step + 1 < P:
                if cuda:
                    torch.cuda.current_stream().wait_event(landed)
                cur, nxt = nxt, cur
        return (acc / l.unsqueeze(-1)).transpose(0, 1).to(q.dtype)


class PipelineParallel(_Base):
    """Pipeline parallelism (GPipe schedule): rank r holds stage r of the model; micro-batches flow
    forward through point-to-point sends of the activations and backward through sends of their
    gradients. All forwards run first, then all backwards in reverse micro-batch order, so every
    stage keeps at most ``len(microbatches)`` activations alive and parameter gradients accumulate
    over the micro-batches exactly as in one big batch.

    CPU tensors move through unbound-buffer send / recv; CUDA tensors through the NVLink
    point-to-point kernels (``CudaContext.send`` / ``recv``: the receiver drains a mailbox ring
    inside its own pool while the sender streams into it, both on the current stream).
    Activation shapes must be the same for every micro-batch (``out_shape`` of the previous stage).
    """

    _TAG_FWD, _TAG_BWD = 0x50, 0x51

    def _send(self, t, dst, tag, seq):
        if _is_cuda(t):
            self.cc.send(t.contiguous(), dst)
            return
        t = t.contiguous()
        b = self.ctx.create_unbound_buffer(t.data_ptr(), t.numel() * t.element_size())
        b.send(dst, _C.slot_build(tag, seq))
        b.wait_send()

    def _recv(self, t, src, tag, seq):
        if _is_cuda(t):
            self.cc.recv(t, src)
            return t
        b = self.ctx.create_unbound_buffer(t.data_ptr(), t.numel() * t.element_size())
        b.recv(src, _C.slot_build(tag, seq))
        b.wait_recv()
        return t

    def run(self, stage, microbatches: Sequence, in_shape=None, loss_fn=None, targets: Optional[Sequence] = None,
            dtype=None, device=None):
        """One training step. ``stage``: this rank's module. ``microbatches``: the inputs (first stage only,
        elsewhere just their count matters). ``in_shape``: shape of the activation this stage receives (all but
        the first stage). ``loss_fn(output, target)`` and ``targets`` on the last stage. Returns the list of
        micro-batch losses on the last stage, ``None`` elsewhere; parameter gradients are left in ``.grad``
        (summed over micro-batches; scale the loss by 1/len(microbatches) for a mean)."""
        import torch

        first, last = self.rank == 0, self.rank == self.size - 1
        n = len(microbatches)
        inputs, outputs, losses = [], [], []
        for i in range(n):
            if first:
                x = microbatches[i]
            else:
                x = self._recv(torch.empty(in_shape, dtype=dtype, device=device), self.rank - 1, self._TAG_FWD, i)
                x.requires_grad_(True)
            y = stage(x)
            inputs.append(x)
            if last:
                loss = loss_fn(y, targets[i])
                losses.append(loss)
                outputs.append(loss)
            else:
                outputs.append(y)
                self._send(y.detach(), self.rank + 1, self._TAG_FWD, i)
        for i in reversed(range(n)):
            if last:
                outputs[i].backward()
            else:
                g = self._recv(torch.empty_like(outputs[i]), self.rank + 1, self._TAG_BWD, i)
                outputs[i].backward(g)
            if not first:
                self._send(inputs[i].grad, self.rank - 1, self._TAG_BWD, i)
        return [float(l.detach()) for l in losses] if last else None
