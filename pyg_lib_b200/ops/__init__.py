"""`pyg_lib.ops.segment_matmul` / `grouped_matmul` — same signatures, argument meaning and autograd
behaviour as the reference (pyg_lib/ops/__init__.py:59-172), bound to the sm_90a kernels."""
from typing import List, Optional, Tuple

import torch
import torch.utils._pytree as pytree
from torch import Tensor


def _flatten_apply(fn_cls, tensors: Tuple[Tensor, ...]):
    # autograd.Function cannot take a tuple of tensors as one argument; the reference works around
    # this with a pytree shim (pyg_lib/ops/__init__.py:8-56).  Passing the tensors flat is equivalent.
    return fn_cls.apply(*tensors)


class GroupedMatmul(torch.autograd.Function):
    r"""Reference: pyg_lib/ops/__init__.py:59-96 (forward = one grouped launch; backward = two more
    grouped launches on transposed *views*, which the CUDA kernels read through strides)."""
    @staticmethod
    def forward(ctx, *args: Tensor):
        ctx.save_for_backward(*args)
        n = len(args) // 2
        inputs, others = list(args[:n]), list(args[n:])
        outs = torch.ops.pyg.grouped_matmul(inputs, others)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *outs_grad: Tensor):
        args = ctx.saved_tensors
        n = len(outs_grad)
        inputs, others = list(args[:n]), list(args[n:])
        outs_grad = [g.contiguous() for g in outs_grad]
        if any(ctx.needs_input_grad[:n]):
            inputs_grad = list(torch.ops.pyg.grouped_matmul(outs_grad, [o.t() for o in others]))
        else:
            inputs_grad = [None] * n
        if any(ctx.needs_input_grad[n:]):
            others_grad = list(torch.ops.pyg.grouped_matmul([x.t() for x in inputs], outs_grad))
        else:
            others_grad = [None] * n
        return tuple(inputs_grad + others_grad)


def grouped_matmul(inputs: List[Tensor], others: List[Tensor],
                   biases: Optional[List[Tensor]] = None) -> List[Tensor]:
    r"""Performs dense-dense matrix multiplication according to groups: ``outs[i] = inputs[i] @
    others[i] (+ biases[i])`` for 2-D ``inputs[i]: [N_i, K_i]``, ``others[i]: [K_i, M_i]``.

    Same contract as the reference (pyg_lib/ops/__init__.py:99-134)."""
    outs = list(_flatten_apply(GroupedMatmul, tuple(inputs) + tuple(others)))
    if biases is not None:
        for i in range(len(biases)):
            outs[i] = outs[i] + biases[i]
    return outs


def segment_matmul(inputs: Tensor, ptr: Tensor, other: Tensor, bias: Optional[Tensor] = None) -> Tensor:
    r"""``out[ptr[i]:ptr[i+1]] = inputs[ptr[i]:ptr[i+1]] @ other[i] (+ bias[i])``
    (reference: pyg_lib/ops/__init__.py:137-172).

    ``ptr`` may live on the CPU or on the device (int64); a device ``ptr`` does not cause a sync.
    When no gradient is needed the bias is fused into the GEMM epilogue instead of the reference's
    Python loop over segments (pyg_lib/ops/__init__.py:169-171)."""
    needs_grad = torch.is_grad_enabled() and (inputs.requires_grad or other.requires_grad or
                                              (bias is not None and bias.requires_grad))
    if bias is not None and not needs_grad:
        return torch.ops.pyg.segment_matmul_bias(inputs, ptr, other, bias)
    out = torch.ops.pyg.segment_matmul(inputs, ptr, other)
    if bias is not None:
        sizes = ptr[1:] - ptr[:-1]
        out = out + torch.repeat_interleave(bias, sizes.to(bias.device), dim=0, output_size=inputs.size(0))
    return out


__all__ = ['segment_matmul', 'grouped_matmul', 'GroupedMatmul']
