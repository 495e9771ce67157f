"""One-pass CUDA versions of the elementwise glue in a Llama-shaped block forward
(csrc/block_ops.cu).  Used by llmc_b200.synth modules on CUDA tensors."""
import torch

from ._lib import call, dtype_enum, ptr, stream_ptr
from .prof import TIMER


def rmsnorm(x, weight, eps, out=None):
    assert weight.dtype == x.dtype and weight.numel() == x.shape[-1]
    x2 = x.reshape(-1, x.shape[-1])
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    if out is not None:
        assert out.is_contiguous() and out.shape == x.shape and out.dtype == x.dtype
        y = out.reshape(-1, x.shape[-1])
    else:
        y = torch.empty_like(x2)
    with TIMER.span('rmsnorm', nbytes=2.0 * x2.element_size() * x2.numel()):
        call('llmc_rmsnorm', ptr(x2), ptr(weight.contiguous()), ptr(y), x2.shape[0], x2.shape[1],
             float(eps), dtype_enum(x.dtype), stream_ptr(x.device))
    return y.reshape(x.shape)


def rope_(x, cos, sin, heads, head_dim):
    """In place on x [B, S, heads*head_dim] (contiguous); cos/sin [S, head_dim] in x.dtype."""
    B, S, _ = x.shape
    assert x.is_contiguous() and cos.dtype == x.dtype and sin.dtype == x.dtype
    assert x.shape[-1] == heads * head_dim and cos.shape == sin.shape == (S, head_dim)
    with TIMER.span('rope', nbytes=2.0 * x.element_size() * x.numel()):
        call('llmc_rope', ptr(x), ptr(cos.contiguous()), ptr(sin.contiguous()), B, S, heads, head_dim,
             dtype_enum(x.dtype), stream_ptr(x.device))
    return x


def silu_mul(gate, up, out=None):
    assert gate.is_contiguous() and up.is_contiguous() and gate.shape == up.shape
    assert up.dtype == gate.dtype
    y = torch.empty_like(gate) if out is None else out
    assert y.is_contiguous() and y.shape == gate.shape and y.dtype == gate.dtype
    with TIMER.span('silu_mul', nbytes=3.0 * gate.element_size() * gate.numel()):
        call('llmc_silu_mul', ptr(gate), ptr(up), ptr(y), gate.numel(), dtype_enum(gate.dtype),
             stream_ptr(gate.device))
    return y


def add(a, b, out=None):
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape and b.dtype == a.dtype
    y = torch.empty_like(a) if out is None else out
    assert y.is_contiguous() and y.shape == a.shape and y.dtype == a.dtype
    with TIMER.span('add', nbytes=3.0 * a.element_size() * a.numel()):
        call('llmc_add', ptr(a), ptr(b), ptr(y), a.numel(), dtype_enum(a.dtype), stream_ptr(a.device))
    return y
