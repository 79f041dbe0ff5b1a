"""A tensor-parallel transformer block on the library's collectives (Megatron layout).

Attention: the QKV projection is column-parallel (every rank owns H/P heads), attention runs
locally over those heads, the output projection is row-parallel -> ONE allreduce. MLP: column-
parallel up-projection, GELU, row-parallel down-projection -> ONE allreduce. Backward mirrors it
(one allreduce per half). CUDA tensors run the fused NVLink kernels, where each row-parallel
allreduce also adds the bias and the residual and, after the attention, applies ln2
(``TensorParallel.reduce_residual_norm``); CPU tensors run the TCP transport.
With ``sequence_parallel=True`` the residual stream and both norms live on this rank's shard of the
sequence (Megatron sequence parallelism): an allgather feeds each column-parallel half, and each
row-parallel output is reduce-scattered back to the shard instead of allreduced.
``TPBlock.enable_fp8()`` runs the MLP's up-projection as a row-wise scaled FP8 GEMM for inference:
ln2's fused step emits e4m3 codes and per-token scales, the weight is quantised once per output
channel.
``DenseBlock`` is the single-process reference with the same parameters (tests load one into the other).
"""
from __future__ import annotations

import torch
from torch import nn

from ..parallel import SequenceParallel, TensorParallel
from ..parallel.strategies import fp8_rows


class DenseBlock(nn.Module):
    def __init__(self, d_model=64, n_heads=4, d_ff=256):
        super().__init__()
        self.n_heads = n_heads
        self.ln1, self.ln2 = nn.LayerNorm(d_model), nn.LayerNorm(d_model)
        self.qkv, self.proj = nn.Linear(d_model, 3 * d_model), nn.Linear(d_model, d_model)
        self.up, self.down = nn.Linear(d_model, d_ff), nn.Linear(d_ff, d_model)

    def forward(self, x):                                           # x: [B, S, d_model]
        B, S, E = x.shape
        h = self.ln1(x)
        q, k, v = self.qkv(h).view(B, S, 3, self.n_heads, E // self.n_heads).unbind(2)
        a = nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True)
        x = x + self.proj(a.transpose(1, 2).reshape(B, S, E))
        return x + self.down(nn.functional.gelu(self.up(self.ln2(x))))


class TPBlock(nn.Module):
    def __init__(self, tp: TensorParallel, d_model=64, n_heads=4, d_ff=256, device=None, dtype=None,
                 sequence_parallel: bool = False):
        """``sequence_parallel``: ``forward`` takes and returns this rank's shard ``[S / P, B,
        d_model]`` of a sequence-first ``[S, B, d_model]`` input (S divisible by P); after the
        backward, ``SequenceParallel.allreduce_sequence_parallel_grads(block.sequence_parallel_parameters())``
        completes the gradients of the parameters applied to the shard."""
        super().__init__()
        assert n_heads % tp.size == 0 and d_ff % tp.size == 0
        self.tp, self.n_heads, self.d_model = tp, n_heads, d_model
        self.sp = SequenceParallel(tp.ctx, tp.cc) if sequence_parallel else None
        self.local_heads = n_heads // tp.size
        self.ln1, self.ln2 = nn.LayerNorm(d_model, device=device, dtype=dtype), nn.LayerNorm(d_model, device=device, dtype=dtype)
        # q, k and v each column-parallel over heads (one fused parameter per projection kind)
        self.q = tp.column_linear(d_model, d_model, device=device, dtype=dtype)
        self.k = tp.column_linear(d_model, d_model, device=device, dtype=dtype)
        self.v = tp.column_linear(d_model, d_model, device=device, dtype=dtype)
        self.proj = tp.row_linear(d_model, d_model, device=device, dtype=dtype)
        self.up = tp.column_linear(d_model, d_ff, device=device, dtype=dtype)
        self.down = tp.row_linear(d_ff, d_model, device=device, dtype=dtype)
        self._fp8_up = None  # (codes, scales) of up.weight in FP8 inference mode

    def load_dense(self, dense: DenseBlock):
        """Take this rank's shards of a DenseBlock's parameters."""
        E, Hh = self.d_model, self.n_heads
        w = dense.qkv.weight.detach().view(3, Hh, E // Hh, E)       # qkv rows are laid out (kind, head, dim)
        b = dense.qkv.bias.detach().view(3, Hh, E // Hh)
        for i, lin in enumerate((self.q, self.k, self.v)):
            lin.load_full(w[i].reshape(E, E), b[i].reshape(E))
        self.proj.load_full(dense.proj.weight.detach(), dense.proj.bias.detach())
        self.up.load_full(dense.up.weight.detach(), dense.up.bias.detach())
        self.down.load_full(dense.down.weight.detach(), dense.down.bias.detach())
        self.ln1.load_state_dict(dense.ln1.state_dict())
        self.ln2.load_state_dict(dense.ln2.state_dict())

    def sequence_parallel_parameters(self):
        """The replicated parameters that sequence parallelism applies to the token shard: ln1, ln2
        and the row-parallel biases. Their gradients must be summed over the group."""
        return [p for m in (self.ln1, self.ln2) for p in m.parameters()] + \
            [lin.bias for lin in (self.proj, self.down) if lin.bias is not None]

    def enable_fp8(self, enabled: bool = True):
        """FP8 inference (CUDA, bfloat16): the up-projection becomes a row-wise scaled FP8 GEMM
        (``torch._scaled_mm``, bf16 out) of ln2's output, which the fused residual-norm step emits as
        e4m3 codes with one fp32 scale per token, and of ``up.weight``, quantised here once per output
        channel by the same ``amax / 448`` rule (``strategies.fp8_rows``). Everything else stays
        bfloat16. Forward-only: the forward raises ``ValueError`` in grad mode while parameters
        require grad. Call it again after changing ``up.weight``; ``enabled=False`` turns it off."""
        if not enabled:
            self._fp8_up = None
            return self
        w = self.up.weight
        if not w.is_cuda or w.dtype != torch.bfloat16:
            raise ValueError(f"enable_fp8: needs bfloat16 CUDA parameters, got {w.dtype} on {w.device}")
        if self.d_model % 16 or w.shape[0] % 16:
            raise ValueError(f"enable_fp8: the FP8 GEMM needs d_model ({self.d_model}) and d_ff / P ({w.shape[0]}) "
                             "to be multiples of 16")
        with torch.no_grad():
            codes, scales = fp8_rows(w.detach())                   # (d_ff / P, E), (d_ff / P, 1)
        self._fp8_up = (codes, scales.reshape(1, -1).contiguous())
        return self

    def _up_fp8(self, codes, scales):
        """up(ln2(x)) from ln2's FP8 codes (..., E) and per-token scales (..., 1)."""
        wq, ws = self._fp8_up
        lead = codes.shape[:-1]
        h = torch._scaled_mm(codes.reshape(-1, self.d_model), wq.t(), scale_a=scales.reshape(-1, 1), scale_b=ws,
                             out_dtype=torch.bfloat16)
        return (h + self.up.bias).view(*lead, -1)

    def forward(self, x):
        if self._fp8_up is not None and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise ValueError("TPBlock: FP8 mode is for inference; run the forward under torch.no_grad()")
        if self.sp is not None:
            return self._forward_sequence_parallel(x)
        B, S, E = x.shape
        hd = E // self.n_heads
        h = self.ln1(x)
        q, k, v = (lin(h).view(B, S, self.local_heads, hd).transpose(1, 2) for lin in (self.q, self.k, self.v))
        a = nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)
        a = a.transpose(1, 2).reshape(B, S, self.local_heads * hd)
        if x.is_cuda and self._fp8_up is not None:
            # ln2's output as FP8 codes and per-token scales from the fused step, then the FP8 GEMM
            x, (q8, s8) = self.tp.reduce_residual_norm(nn.functional.linear(a, self.proj.weight), x, self.ln2,
                                                       self.proj.bias, fp8=True)
            p = nn.functional.linear(nn.functional.gelu(self._up_fp8(q8, s8)), self.down.weight)
            return self.tp.reduce_residual_norm(p, x, None, self.down.bias)
        if x.is_cuda:
            # each row-parallel output: allreduce + bias + residual add (+ ln2) in one kernel
            # copy_out: h's gradient is allreduced inside the fused backward, so self.up(h)'s
            # copy_to_region would count it P times.
            x, h = self.tp.reduce_residual_norm(nn.functional.linear(a, self.proj.weight), x, self.ln2, self.proj.bias,
                                                copy_out=True)
            h = nn.functional.linear(h, self.up.weight, self.up.bias)
            p = nn.functional.linear(nn.functional.gelu(h), self.down.weight)
            return self.tp.reduce_residual_norm(p, x, None, self.down.bias)
        x = x + self.proj(a)
        return x + self.down(nn.functional.gelu(self.up(self.ln2(x))))

    def _forward_sequence_parallel(self, x):                      # x: [S/P, B, d_model]
        F, sp = nn.functional, self.sp
        # The column-parallel layers take the gathered input directly: gather_from_sequence's
        # backward reduce-scatters its gradient, so copy_to_region's allreduce would count it P times.
        h = sp.gather_from_sequence(self.ln1(x))                 # [S, B, E]
        S, B, _ = h.shape
        hd = self.d_model // self.n_heads
        q, k, v = (F.linear(h, lin.weight, lin.bias).view(S, B, self.local_heads, hd).permute(1, 2, 0, 3)
                   for lin in (self.q, self.k, self.v))
        a = F.scaled_dot_product_attention(q, k, v, is_causal=True).permute(2, 0, 1, 3).reshape(S, B, -1)
        if self._fp8_up is not None:
            x, (q8, s8) = sp.reduce_scatter_residual_norm(F.linear(a, self.proj.weight), x, self.ln2, self.proj.bias,
                                                          fp8=True)
            p = F.linear(F.gelu(self._up_fp8(q8, s8)), self.down.weight)
            return sp.reduce_scatter_residual_norm(p, x, None, self.down.bias, gather_out=False)
        x, h = sp.reduce_scatter_residual_norm(F.linear(a, self.proj.weight), x, self.ln2, self.proj.bias)
        p = F.linear(F.gelu(F.linear(h, self.up.weight, self.up.bias)), self.down.weight)
        return sp.reduce_scatter_residual_norm(p, x, None, self.down.bias, gather_out=False)
