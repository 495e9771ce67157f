"""Quantised linear modules — mirror of llmc/compression/quantization/module_utils.py.

FakeQuantLinear (:586-678), EffcientFakeQuantLinear (:681-759), OriginFloatLinear (:396-457),
VllmRealQuantLinear (:762-876) + aliases (:879-933), AutoawqRealQuantLinear (:936-1065) +
MlcllmRealQuantLinear (:1068-1084), and the type maps (:1087-1138).  Same `.new(...)`
factories, buffer names and `buf_*` hand-off; the forward GEMM and the packers run in
libllmc_b200.so.
"""
import ctypes
from collections import namedtuple
from functools import partial

import torch
import torch.nn as nn

from ._lib import MOE_MAX_EXPERTS, call, dtype_enum, ptr, require_cuda, stream_ptr
from .prof import TIMER


def linear_forward(x, weight, bias=None):
    """F.linear on the wgmma GEMM (csrc/gemm.cu) — y = x @ weight.T (+ bias)."""
    require_cuda(x, weight)
    if x.dtype != weight.dtype:
        raise TypeError(f'activation dtype {x.dtype} != weight dtype {weight.dtype}')
    K = x.shape[-1]
    N = weight.shape[0]
    x2 = x.reshape(-1, K)
    if not x2.is_contiguous():
        x2 = x2.contiguous()
    w = weight if weight.is_contiguous() else weight.contiguous()
    y = torch.empty((x2.shape[0], N), dtype=x.dtype, device=x.device)
    b = None
    if bias is not None:
        b = bias.to(x.dtype).contiguous()
    M = x2.shape[0]
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + M * N)):
        call('llmc_gemm_bf16', ptr(x2), ptr(w), ptr(b), ptr(y), M, N, K, dtype_enum(x.dtype),
             stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


# ---- the forward GEMM with the block glue that follows it in its epilogue -------------------------
# Each computes exactly what linear_forward followed by the block_ops kernel computes; the spans are
# 'gemm' spans like linear_forward's, with the GEMM's 2MNK flops.
def _gemm_operands(x, w):
    require_cuda(x, w)
    if x.dtype != w.dtype:
        raise TypeError(f'activation dtype {x.dtype} != weight dtype {w.dtype}')
    x2 = x.reshape(-1, x.shape[-1])
    return (x2 if x2.is_contiguous() else x2.contiguous()), (w if w.is_contiguous() else w.contiguous())


def interleave_gate_up(wg, wu):
    """The weight of llmc_gemm_swiglu: gate and up rows interleaved in blocks of 128
    ([g 0:128, u 0:128, g 128:256, u 128:256, ...])."""
    inter, K = wg.shape
    assert wu.shape == wg.shape and inter % 128 == 0
    return torch.stack([wg.reshape(-1, 128, K), wu.reshape(-1, 128, K)], dim=1).reshape(2 * inter, K)


def gemm_rope_qkv(x, w_qkv, n_q, n_k, cos, sin):
    """q, k, v = x [B, S, K] @ [Wq; Wk; Wv]^T with block_ops.rope_ applied to q and k (head_dim 128,
    cos / sin [S, 128]); three contiguous [B, S, width] tensors."""
    B, S, K = x.shape
    x2, w = _gemm_operands(x, w_qkv)
    n_v = w.shape[0] - n_q - n_k
    M = x2.shape[0]
    q, k, v = (torch.empty((B, S, n), dtype=x.dtype, device=x.device) for n in (n_q, n_k, n_v))
    N = w.shape[0]
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + M * N)):
        call('llmc_gemm_rope_qkv', ptr(x2), ptr(w), ptr(q), ptr(k), ptr(v), ptr(cos.contiguous()),
             ptr(sin.contiguous()), M, n_q, n_k, n_v, K, S, dtype_enum(x.dtype), stream_ptr(x.device))
    return q, k, v


def gemm_mla_qkv(x, w_qkva, heads, kv_lora, cos, sin):
    """MLA's first projections, x [B, S, K] @ [W_q; W_kv_a]^T in one GEMM (llmc_gemm_mla_qkv): q
    [B, S, heads * 192] with each head's pe slice rotated, k [B, S, heads * 192] with the rotated
    k_pe in every head's pe slot (its nope slots are gemm_mla_kv_b's to fill) and the latent
    [B, S, kv_lora].  cos / sin fp32 [S, 32]."""
    B, S, K = x.shape
    x2, w = _gemm_operands(x, w_qkva)
    M, N = x2.shape[0], w.shape[0]
    assert N == heads * 192 + kv_lora + 64 and cos.dtype == sin.dtype == torch.float32
    q, k = (torch.empty((B, S, heads * 192), dtype=x.dtype, device=x.device) for _ in range(2))
    latent = torch.empty((B, S, kv_lora), dtype=x.dtype, device=x.device)
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + M * (N + (heads - 1) * 64))):
        call('llmc_gemm_mla_qkv', ptr(x2), ptr(w), ptr(q), ptr(k), ptr(latent), ptr(cos.contiguous()),
             ptr(sin.contiguous()), M, heads, kv_lora, K, S, dtype_enum(x.dtype), stream_ptr(x.device))
    return q, k, latent


def gemm_mla_kv_b(latent, w_kv_b, k, heads):
    """MLA's kv_b_proj on the normed latent [B, S, kv_lora] (llmc_gemm_mla_kv_b): each head's k_nope
    into the nope slots of gemm_mla_qkv's k, in place; returns v [B, S, heads * 128]."""
    B, S, K = latent.shape
    x2, w = _gemm_operands(latent, w_kv_b)
    M, N = x2.shape[0], w.shape[0]
    assert N == heads * 256 and k.shape == (B, S, heads * 192) and k.is_contiguous() and k.dtype == latent.dtype
    v = torch.empty((B, S, heads * 128), dtype=latent.dtype, device=latent.device)
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + M * N)):
        call('llmc_gemm_mla_kv_b', ptr(x2), ptr(w), ptr(k), ptr(v), M, heads, K, dtype_enum(latent.dtype),
             stream_ptr(latent.device))
    return v


def gemm_swiglu(x, w_gate_up, out=None):
    """block_ops.silu_mul(x @ Wg^T, x @ Wu^T) for w_gate_up = interleave_gate_up(Wg, Wu), into
    `out` (contiguous) when given."""
    K = x.shape[-1]
    x2, w = _gemm_operands(x, w_gate_up)
    N, M = w.shape[0], x2.shape[0]
    y = torch.empty((*x.shape[:-1], N // 2), dtype=x.dtype, device=x.device) if out is None else out
    assert y.is_contiguous() and y.shape == (*x.shape[:-1], N // 2) and y.dtype == x.dtype
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + M * N // 2)):
        call('llmc_gemm_swiglu', ptr(x2), ptr(w), ptr(y), M, N // 2, K, dtype_enum(x.dtype),
             stream_ptr(x.device))
    return y


def linear_forward_residual(x, weight, res, out):
    """out = block_ops.add(res, x @ weight^T); out may be res."""
    K = x.shape[-1]
    x2, w = _gemm_operands(x, weight)
    N, M = w.shape[0], x2.shape[0]
    assert res.is_contiguous() and out.is_contiguous() and res.dtype == out.dtype == x.dtype
    assert res.shape == out.shape == (*x.shape[:-1], N)
    with TIMER.span('gemm', flops=2.0 * M * N * K, nbytes=2.0 * (M * K + N * K + 2 * M * N)):
        call('llmc_gemm_residual', ptr(x2), ptr(w), ptr(res), ptr(out), M, N, K, dtype_enum(x.dtype),
             stream_ptr(x.device))
    return out


def dense_forward_weight(layer, dtype):
    """The dense weight W of `dtype` when `layer`'s forward on a CUDA input of `dtype` is exactly
    linear_forward(x, W) (B200Linear's weight, FakeQuantLinear's cached tmp_weight, which this
    materialises as the first forward would); None for any other forward: activation fake-quant, a
    bias, a weight re-quantised every call, packed / FP8 / W8A8 deploys, hooks, a dtype mismatch."""
    if getattr(layer, 'a_qdq', None) is not None:
        return None
    return _dense_weight(layer, dtype)


def _dense_weight(layer, dtype):
    """dense_forward_weight's weight of a B200Linear or FakeQuantLinear whatever its a_qdq: the
    linear_forward that follows the activation fake-quant."""
    from .synth import B200Linear
    if layer._forward_hooks or layer._forward_pre_hooks:
        return None
    if type(layer) is FakeQuantLinear:
        if layer.bias is not None or layer.dynamic_quant_weight or layer.dynamic_quant_tmp_weight:
            return None
        if not hasattr(layer, 'tmp_weight'):
            layer.register_buffer('tmp_weight', layer.w_qdq(layer), persistent=False)
            layer.tmp_bias = layer.bias
        w = layer.tmp_weight
    elif type(layer) is B200Linear:
        if layer.bias is not None:
            return None
        w = layer.weight
    else:
        return None
    return w if (w.dtype == dtype and w.dim() == 2) else None


PackedOperands = namedtuple('PackedOperands', 'wq scales zeros bits group g_idx transposed')
PackedOperands.__doc__ = """What a packed linear's forward hands to llmc_gemm_w{4,8}a16[_gidx]: codes wq [N, K*bits/32],
scales / zeros as packed_qparams prepares them ([ng, N] when `transposed`, else [N, ng]; zeros None:
symmetric), the group size and g_idx (int32 [K], None for contiguous groups)."""


def packed_forward_operands(layer, dtype):
    """The operands of `layer`'s forward on an input of `dtype` when that forward is exactly
    linear_forward_w4 with 4- or 8-bit integer codes and nothing else, else None: a packed
    EffcientFakeQuantLinear on the integer grid with integer zero-points (not HQQ / SpQR's real
    ones), or a VllmRealQuantLinear weight-only W4A16 / W8A16 export it runs; no activation
    fake-quant, bias or hooks.  The device is the caller's to check."""
    if layer._forward_hooks or layer._forward_pre_hooks or getattr(layer, 'bias', None) is not None:
        return None
    if type(layer) is EffcientFakeQuantLinear:
        return _packed_int_operands(layer, dtype) if layer.a_qdq is None else None
    if isinstance(layer, VllmRealQuantLinear) and 'weight_packed' in layer._buffers:
        if layer.packed_unsupported() is not None:
            return None
        K, wq = layer.in_features, layer.weight_packed
        s, _ = packed_qparams(dtype, layer.weight_scale, None, wq.shape[0], False)
        return PackedOperands(wq.contiguous(), s, None, 32 * wq.shape[1] // K, K // layer.weight_scale.shape[1],
                              None, False)
    return None


def _packed_int_operands(layer, dtype):
    """The PackedOperands of an EffcientFakeQuantLinear on 4- / 8-bit integer codes with integer
    zero-points, whatever its a_qdq; else None."""
    if not layer.packed or layer.q_grid != 'int' or layer.q_rz or layer.q_bits not in (4, 8):
        return None
    N = layer.qweight.shape[0]
    s, z = packed_qparams(dtype, layer.qscales_t, layer.qzeros_t, N, True)
    g = layer.g_idx.contiguous() if layer.g_idx is not None else None
    return PackedOperands(layer.qweight.contiguous(), s, z, layer.q_bits, layer.q_group, g, True)


Fp8Operands = namedtuple('Fp8Operands', 'wq scales zeros bits group g_idx transposed e5m2')
Fp8Operands.__doc__ = """What an FP8-grid EffcientFakeQuantLinear's forward hands to llmc_gemm_fp8a16[_gidx]: its
fp8 bytes [N, K] viewed as int32 wq [N, K/4], scales [ng, N] in the activation dtype or fp32
(`transposed`), the group size, g_idx (None: contiguous groups) and e5m2 (0: e4m3).  zeros (None)
and bits (8) make it read like PackedOperands."""


def fake_quant_forward_operands(layer, dtype):
    """(weight operands, a_qdq) of a fake-quant linear whose forward on an input x of `dtype` is
    exactly a_qdq(x, layer) (when a_qdq is not None) followed by one GEMM on those operands, else
    None: a FakeQuantLinear's dense tmp_weight (_dense_weight), a packed INT4 / INT8
    EffcientFakeQuantLinear's PackedOperands, or an FP8-grid one's Fp8Operands (linear_forward_fp8w);
    no bias or hooks.  The device is the caller's to check."""
    if layer._forward_hooks or layer._forward_pre_hooks or getattr(layer, 'bias', None) is not None:
        return None
    if type(layer) is FakeQuantLinear:
        w = _dense_weight(layer, dtype)
    elif type(layer) is EffcientFakeQuantLinear and layer.packed and not layer.q_rz and layer.q_grid != 'int':
        N = layer.qweight.shape[0]
        qdt = dtype if layer.qscales_t.dtype == dtype else torch.float32
        s = layer.qscales_t.reshape(-1, N).to(qdt).contiguous()
        g = layer.g_idx.contiguous() if layer.g_idx is not None else None
        w = Fp8Operands(layer.qweight.contiguous().view(torch.int32), s, None, 8, layer.q_group, g, True,
                        int(layer.qweight.dtype == torch.float8_e5m2))
    elif type(layer) is EffcientFakeQuantLinear:
        w = _packed_int_operands(layer, dtype)
    else:
        return None
    return None if w is None else (w, layer.a_qdq)


W8A8Operands = namedtuple('W8A8Operands', 'w s_w aq input_scale act_cfg')
W8A8Operands.__doc__ = """What a W8A8 export's forward hands to llmc_gemm_w8a8_*: codes w [N, K] (int8, or e4m3 with
fp8_weight's recovery), weight scales s_w fp32 (N values, or one), the activation quantizer aq, the
static input_scale (None: per-token dynamic) and the act config they come from."""


def w8a8_forward_operands(layer):
    """The operands of `layer`'s forward when that forward is exactly linear_forward_w8a8 and nothing
    else, else None: a VllmRealQuantLinear W8A8 export it runs (w8a8_unsupported() is None) without a
    bias or hooks.  The device is the caller's to check."""
    if (not isinstance(layer, VllmRealQuantLinear) or layer._forward_hooks or layer._forward_pre_hooks
            or layer.bias is not None or layer.w8a8_unsupported() is not None):
        return None
    try:
        w = layer.weight if layer.weight.dtype == torch.int8 else layer.fp8_weight()
    except NotImplementedError:                   # off the e4m3 grid: the forward raises it
        return None
    static = bool(_cfg_get(layer.act_cfg, 'static', False))
    return W8A8Operands(w.contiguous(), layer.weight_scale.reshape(-1).float().contiguous(),
                        layer.activation_quantizer(), layer.input_scale if static else None, layer.act_cfg)


def linear_residual(layer, x, res, out):
    """out = res + layer(x) (block_ops.add), out may be res: in the GEMM's epilogue when the layer
    has a dense forward weight, else the layer's forward and block_ops.add."""
    w = dense_forward_weight(layer, x.dtype)
    if (w is not None and x.is_cuda and w.shape[0] % 8 == 0 and res.is_contiguous()
            and out.is_contiguous() and res.dtype == x.dtype):
        return linear_forward_residual(x, w, res, out)
    from . import block_ops
    return block_ops.add(res, layer(x), out=out)


# ---- sparse-MoE layer as grouped expert GEMMs ------------------------------------------------------
def moe_routing(sel, n_experts):
    """The routing of a top-k MoE layer as device tensors whose shapes do not depend on it, so that
    building them never synchronises with the host.  sel [T, k] holds each token's experts (distinct
    per token).  Returns
      perm [T*k]          the flat (token, slot) indices t*k + s sorted by expert, stably: expert e's
                          tokens in ascending order, as torch.where(sel == e) lists them;
      offsets [E+1]       int32 segment starts: expert e owns positions offsets[e]:offsets[e+1] of perm;
      rows [T, k]         the positions in perm of token t's k pairs, in ascending expert order.
    Counts come from scatter_add_, not torch.bincount, which reads its maximum back to the host."""
    T, k = sel.shape
    flat = sel.reshape(-1)
    perm = torch.sort(flat, stable=True).indices
    counts = torch.zeros(n_experts, dtype=torch.int64, device=sel.device)
    counts.scatter_add_(0, flat, torch.ones_like(flat))
    offsets = torch.cat([counts.new_zeros(1), counts.cumsum(0)]).to(torch.int32)
    pos = torch.empty_like(perm).scatter_(0, perm, torch.arange(T * k, device=sel.device))
    # a token's experts are distinct and perm is sorted by expert, so ascending position is
    # ascending expert
    rows = pos.view(T, k).sort(dim=1).values
    return perm, offsets, rows


def moe_forward(x, sel, w, experts, a_qdq=None, shared=None):
    """A sparse-MoE layer's expert part, out[t] = sum over slots s of
    expert_{sel[t, s]}(x[t]) * w[t, s] with expert(x) = w2(silu(w1 x) * w3 x), as three launches:
    the grouped gate/up GEMM with SiLU-mul in its epilogue, the grouped down GEMM that scales each
    row by its routing weight, and the combine.  x [T, H] and w [T, k] of a 16-bit dtype, sel [T, k]
    int64, experts = one (w1, w3, w2) triple per expert (at most MOE_MAX_EXPERTS): dense weights,
    PackedOperands of one form (packed_forward_operands; the grouped dequant GEMMs of
    csrc/gemm_w4.cu), Fp8Operands of one form (fake_quant_forward_operands; the same GEMMs on fp8
    bytes) or W8A8Operands of one form (w8a8_forward_operands; the grouped W8A8 GEMMs of
    csrc/gemm_8bit.cu, each fed by one activation-quantiser pass).  a_qdq: None, or the activation
    fake-quant of the experts' linears as a pair of routed twins (blockwise.a_qdq_routed), applied
    to the routed rows before gate/up and to act before the down projection.  shared: None, or
    (gate_logit [T, 1], s [T, H]) of a gated shared expert (Qwen2-MoE), added by the combine as
    out[t] + sigmoid(gate_logit[t]) * s[t] (llmc_moe_combine_shared).  fp32 w (DeepSeek-V2): the down
    GEMM runs with unit routing weights of x's dtype (rT(rT(acc) * 1) = rT(acc)), and shared, the
    ungated shared experts' output s [T, H], is required: the combine takes each term as
    rT(y * w) in fp32 and adds s (llmc_moe_combine_weighted).  Bit for bit the eager loop
    (SparseMoe.expert_loop, then the shared expert's add), with no host sync."""
    require_cuda(x, sel, w)
    T, k, E = x.shape[0], sel.shape[1], len(experts)
    weighted = w.dtype == torch.float32
    assert E <= MOE_MAX_EXPERTS and (w.dtype == x.dtype or (weighted and shared is not None))
    o1, o2 = experts[0][0], experts[0][2]
    gemms = (_moe_packed_gemms if isinstance(o1, PackedOperands)
             else _moe_fp8_gemms if isinstance(o1, Fp8Operands)
             else _moe_w8a8_gemms if isinstance(o1, W8A8Operands) else _moe_dense_gemms)
    # one row per output feature: the dense weight, or the codes heading both operand tuples
    inter, N = ((o if isinstance(o, torch.Tensor) else o[0]).shape[0] for o in (o1, o2))
    perm, offsets, rows = moe_routing(sel, E)
    xp = x.index_select(0, perm // k)
    w_route = w.reshape(-1).index_select(0, perm)
    M = T * k
    w_rows = None
    if weighted:
        w_rows, w_route = w_route, torch.ones(M, dtype=x.dtype, device=x.device)
    act = torch.empty((M, inter), dtype=x.dtype, device=x.device)
    y = torch.empty((M, N), dtype=x.dtype, device=x.device)
    out = torch.empty((T, N), dtype=x.dtype, device=x.device)
    qdq_act = None
    if a_qdq is not None and M > 0:
        expert_of_row = sel.reshape(-1).index_select(0, perm)
        xp = a_qdq[0](xp, expert_of_row)
        qdq_act = partial(a_qdq[1], expert_of_row=expert_of_row)
    gemms(xp, experts, sel, perm, offsets, w_route, act, y, qdq_act)
    if weighted:
        moe_combine_weighted(y, rows, w_rows, shared, out)
    elif shared is None:
        with TIMER.span('moe_combine', nbytes=2.0 * (M * N + T * N) + 8.0 * M):
            call('llmc_moe_combine', ptr(y), ptr(rows), ptr(out), T, k, N, dtype_enum(x.dtype), stream_ptr(x.device))
    else:
        moe_combine_shared(y, rows, shared[0], shared[1], out)
    return out


def moe_combine_weighted(y, rows, w, s, out):
    """out [T, N] = rT(acc + s[t]), acc = rT(...rT(rT(y[r0] * w[r0]) + rT(y[r1] * w[r1]))...) over
    r = rows[t, :] in that order: a DeepSeek-V2 layer's routed experts, each scaled by its fp32
    routing weight and rounded once, plus its ungated shared experts.  y [M, N], rows [T, k] int64,
    w fp32 [M] in y's row order, s [T, N] of y's dtype."""
    require_cuda(y, rows, w, s, out)
    T, k = rows.shape
    N = y.shape[1]
    w, s = w.contiguous(), s.contiguous()
    assert w.dtype == torch.float32 and w.numel() == y.shape[0] and s.shape == (T, N) and out.shape == (T, N)
    assert s.dtype == out.dtype == y.dtype and out.is_contiguous()
    with TIMER.span('moe_combine_weighted', nbytes=2.0 * (y.shape[0] * N + 2 * T * N) + 12.0 * T * k):
        call('llmc_moe_combine_weighted', ptr(y), ptr(rows), ptr(w), ptr(s), ptr(out), T, k, N,
             dtype_enum(y.dtype), stream_ptr(y.device))
    return out


def moe_combine_shared(y, rows, gate_logit, s, out):
    """out [T, N] = rT(routed[t] + rT(rT(sigmoid(gate_logit[t])) * s[t])), routed[t] the sum of y's
    rows rows[t, :] in that order (llmc_moe_combine): a Qwen2-MoE layer's routed experts plus its
    gated shared expert.  y [M, N], rows [T, k] int64, gate_logit [T, 1] and s [T, N] of y's dtype."""
    require_cuda(y, rows, gate_logit, s, out)
    T, k = rows.shape
    N = y.shape[1]
    g, s = gate_logit.contiguous(), s.contiguous()
    assert g.numel() == T and s.shape == (T, N) and out.shape == (T, N)
    assert g.dtype == s.dtype == out.dtype == y.dtype and out.is_contiguous()
    with TIMER.span('moe_combine_shared', nbytes=2.0 * (y.shape[0] * N + 2 * T * N + T) + 8.0 * T * k):
        call('llmc_moe_combine_shared', ptr(y), ptr(rows), ptr(g), ptr(s), ptr(out), T, k, N,
             dtype_enum(y.dtype), stream_ptr(y.device))
    return out


def packed_qparams(dtype, scales, zeros, N, qparams_t):
    """scales / zeros as the packed GEMM takes them for activations of `dtype`: qparams already in
    the activation dtype (RTN / AWQ / exported checkpoints) stay so and take the packed half2 / bf16x2
    dequant path; any other (GPTQ's fp32 dynamic groups, an export's fp16 scales under bf16) become
    fp32 and take the fp32 one — same values.  qparams_t: stored [K/group, N] (coalesced loads in the
    kernel), else [N, K/group]; both contiguous in that shape."""
    native = scales.dtype == dtype and (zeros is None or zeros.dtype == dtype)
    qdt = dtype if native else torch.float32
    shape = (-1, N) if qparams_t else (N, -1)
    s = scales.reshape(shape).to(qdt).contiguous()
    z = zeros.reshape(shape).to(qdt).contiguous() if zeros is not None else None
    return s, z


# moe_forward's GEMM pair, one per operand type.  Each takes the routed rows xp [M, K] (expert e's at
# offsets[e]:offsets[e+1]), the experts' (w1, w3, w2) operands, sel [T, k] and perm (moe_routing),
# the routing weights w_route [M] in xp's row order, and fills act [M, inter] and y [M, N].  The
# down projection reads mid(act) when mid (a function of act alone) is given, else act.
def _moe_shapes(xp, experts, act, y):
    """M, K, inter, N, E, the dtype enum and the stream of a GEMM pair's launches."""
    return (*xp.shape, act.shape[1], y.shape[1], len(experts), dtype_enum(xp.dtype), stream_ptr(xp.device))


def _expert_ptrs(experts, i, field=None):
    """A HOST array of the experts' device pointers to operand i (or to its `field`); None when expert
    0's is None (the entry point's "none of them")."""
    ts = [e[i] if field is None else getattr(e[i], field) for e in experts]
    return None if ts[0] is None else (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _down_input(act, mid):
    return act if mid is None else mid(act)


def _moe_dense_gemms(xp, experts, sel, perm, offsets, w_route, act, y, mid=None):
    """Dense weights: llmc_moe_gemm_swiglu and llmc_moe_gemm_down."""
    M, K, inter, N, E, dt, st = _moe_shapes(xp, experts, act, y)
    ws = [[t.contiguous() for t in e] for e in experts]
    w1, w3, w2 = (_expert_ptrs(ws, i) for i in range(3))
    with TIMER.span('moe_gemm_swiglu', flops=2.0 * M * 2 * inter * K,
                    nbytes=2.0 * (M * K + E * 2 * inter * K + M * inter)):
        call('llmc_moe_gemm_swiglu', ptr(xp), w1, w3, ptr(offsets), ptr(act), M, inter, K, E, dt, st)
    a2 = _down_input(act, mid)
    with TIMER.span('moe_gemm_down', flops=2.0 * M * N * inter,
                    nbytes=2.0 * (M * inter + E * N * inter + M * N + M)):
        call('llmc_moe_gemm_down', ptr(a2), w2, ptr(offsets), ptr(w_route), ptr(y), M, N, inter, E, dt, st)


def _moe_packed_gemms(xp, experts, sel, perm, offsets, w_route, act, y, mid=None):
    """PackedOperands: llmc_moe_gemm_packed_swiglu and llmc_moe_gemm_packed_down, one form per launch."""
    M, K, inter, N, E, dt, st = _moe_shapes(xp, experts, act, y)
    arr = partial(_expert_ptrs, experts)

    def weight_bytes(o):                 # codes, qparams and g_idx of one expert linear
        q = o.scales.numel() * o.scales.element_size() * (1 if o.zeros is None else 2)
        return 4.0 * o.wq.numel() + q + (0 if o.g_idx is None else 4.0 * o.g_idx.numel())

    def layout(o):
        ng = o.scales.numel() // o.wq.shape[0]
        return dtype_enum(o.scales.dtype), int(-o.group if o.transposed else o.group), ng

    g1, g2 = experts[0][0], experts[0][2]
    bits = g1.bits
    qd1, grp1, ng1 = layout(g1)
    qd2, grp2, ng2 = layout(g2)
    with TIMER.span('moe_gemm_packed_swiglu', flops=2.0 * M * 2 * inter * K,
                    nbytes=2.0 * (M * K + M * inter) + E * 2 * weight_bytes(g1)):
        call('llmc_moe_gemm_packed_swiglu', ptr(xp), bits, arr(0, 'wq'), arr(1, 'wq'), arr(0, 'scales'),
             arr(1, 'scales'), arr(0, 'zeros'), arr(1, 'zeros'), arr(0, 'g_idx'), arr(1, 'g_idx'), qd1, grp1, ng1,
             ptr(offsets), ptr(act), M, inter, K, E, dt, st)
    a2 = _down_input(act, mid)
    with TIMER.span('moe_gemm_packed_down', flops=2.0 * M * N * inter,
                    nbytes=2.0 * (M * inter + M * N + M) + E * weight_bytes(g2)):
        call('llmc_moe_gemm_packed_down', ptr(a2), bits, arr(2, 'wq'), arr(2, 'scales'), arr(2, 'zeros'),
             arr(2, 'g_idx'), qd2, grp2, ng2, ptr(offsets), ptr(w_route), ptr(y), M, N, inter, E, dt, st)


def _moe_fp8_gemms(xp, experts, sel, perm, offsets, w_route, act, y, mid=None):
    """Fp8Operands: llmc_moe_gemm_fp8a16_swiglu and llmc_moe_gemm_fp8a16_down, one form per launch."""
    M, K, inter, N, E, dt, st = _moe_shapes(xp, experts, act, y)
    arr = partial(_expert_ptrs, experts)

    def weight_bytes(o):                 # bytes, scales and g_idx of one expert linear
        return 4.0 * o.wq.numel() + o.scales.numel() * o.scales.element_size() + (
            0 if o.g_idx is None else 4.0 * o.g_idx.numel())

    def layout(o):
        ng = o.scales.numel() // o.wq.shape[0]
        return dtype_enum(o.scales.dtype), int(-o.group if o.transposed else o.group), ng

    g1, g2 = experts[0][0], experts[0][2]
    qd1, grp1, ng1 = layout(g1)
    qd2, grp2, ng2 = layout(g2)
    with TIMER.span('moe_gemm_fp8a16_swiglu', flops=2.0 * M * 2 * inter * K,
                    nbytes=2.0 * (M * K + M * inter) + E * 2 * weight_bytes(g1)):
        call('llmc_moe_gemm_fp8a16_swiglu', ptr(xp), g1.e5m2, arr(0, 'wq'), arr(1, 'wq'), arr(0, 'scales'),
             arr(1, 'scales'), arr(0, 'g_idx'), arr(1, 'g_idx'), qd1, grp1, ng1, ptr(offsets), ptr(act), M, inter, K,
             E, dt, st)
    a2 = _down_input(act, mid)
    with TIMER.span('moe_gemm_fp8a16_down', flops=2.0 * M * N * inter,
                    nbytes=2.0 * (M * inter + M * N + M) + E * weight_bytes(g2)):
        call('llmc_moe_gemm_fp8a16_down', ptr(a2), g2.e5m2, arr(2, 'wq'), arr(2, 'scales'),
             arr(2, 'g_idx'), qd2, grp2, ng2, ptr(offsets), ptr(w_route), ptr(y), M, N, inter, E, dt, st)


def _moe_w8a8_gemms(xp, experts, sel, perm, offsets, w_route, act, y, mid=None):
    """W8A8Operands: xp quantised once by w1's activation quantizer, llmc_moe_gemm_w8a8_swiglu, act
    quantised once by w2's, llmc_moe_gemm_w8a8_down.  Per-token dynamic activations take the
    quantiser's per-token pass over all rows (each row's codes and scale depend on that row alone);
    static ones its per-tensor pass with one scale per row, the input_scale of the row's expert,
    gathered on the device.  Its activations are quantised here, so mid is None."""
    assert mid is None
    M, K, inter, N, E, dt, st = _moe_shapes(xp, experts, act, y)
    expert_of_row = sel.reshape(-1).index_select(0, perm)
    if M == 0:
        return
    o1 = experts[0][0]
    fp8 = int(o1.w.dtype == torch.float8_e4m3fn)
    stride = int(o1.s_w.numel() != 1)
    arr = partial(_expert_ptrs, experts)

    def quantise(a, i):
        if experts[0][i].input_scale is None:
            return experts[0][i].aq.real_quant_act(a)
        table = torch.cat([e[i].input_scale.reshape(-1) for e in experts])
        return experts[0][i].aq.real_quant_act(a, table.index_select(0, expert_of_row))

    xq, sx = quantise(xp, 0)
    with TIMER.span('moe_gemm_w8a8_swiglu', flops=2.0 * M * 2 * inter * K,
                    nbytes=float(M * K + E * 2 * inter * K) + 2.0 * M * inter):
        call('llmc_moe_gemm_w8a8_swiglu', ptr(xq), ptr(sx), fp8, arr(0, 'w'), arr(1, 'w'), arr(0, 's_w'),
             arr(1, 's_w'), stride, ptr(offsets), ptr(act), M, inter, K, E, dt, st)
    aq, sa = quantise(act, 2)
    with TIMER.span('moe_gemm_w8a8_down', flops=2.0 * M * N * inter,
                    nbytes=float(M * inter + E * N * inter) + 2.0 * (M * N + M)):
        call('llmc_moe_gemm_w8a8_down', ptr(aq), ptr(sa), fp8, arr(2, 'w'), arr(2, 's_w'), stride, ptr(offsets),
             ptr(w_route), ptr(y), M, N, inter, E, dt, st)


def linear_forward_w4(x, wq, scales, zeros, group, bias=None, bits=4, qparams_t=False, g_idx=None):
    """Fake-quant forward on PACKED int4 weights (csrc/gemm_w4.cu): y = x @ dequant(wq).T + bias,
    bit-identical to linear_forward(x, rT((code - zero) * scale)) — the materialised weight of
    FakeQuantLinear (module_utils.py:626-643) — while reading 4.25 instead of 16 bits per weight.

    wq [N, K/8] int32 (unsigned codes, LLMC_OUT_PACK_VLLM layout), scales [N, K/group] in x.dtype
    or fp32, zeros likewise or None (None => 8, the symmetric +2^(bit-1) storage offset).

    bits 2, 8: wq [N, K*bits/32] in the same layout.  bits 3: wq [ceil(N/2), 3K/16], the row-pair
    layout of pack_unsigned_codes; N is then read from the 2-D scales ([N, ng], or [ng, N] with
    qparams_t).

    g_idx: int32 [K] or None.  When given, column k uses the qparams of group g_idx[k] (GPTQ
    act-order: groups are contiguous in the permuted order, g_idx = invperm // group_size), the
    qparams hold ng = scales.numel() // N groups in any order, and `group` is ignored.  Every value
    must lie in [0, ng); the kernel does not check it."""
    require_cuda(x, wq, scales)
    K = x.shape[-1]
    if bits not in (2, 3, 4, 8):
        raise ValueError(f'packed weights are 2, 3, 4 or 8 bits, not {bits}')
    if bits == 3:
        if scales.dim() != 2:
            raise ValueError('3-bit weights need 2-D scales to give N')
        N = scales.shape[1] if qparams_t else scales.shape[0]
        assert wq.dtype == torch.int32 and tuple(wq.shape) == ((N + 1) // 2, 3 * K // 16) and K % 64 == 0, \
            (wq.shape, N, K)
    else:
        N = wq.shape[0]
        assert wq.dtype == torch.int32 and wq.shape[1] * (32 // bits) == K, (wq.shape, K)
    x2 = x.reshape(-1, K)
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    s, z = packed_qparams(x.dtype, scales, zeros, N, qparams_t)
    qdt = s.dtype
    b = bias.to(x.dtype).contiguous() if bias is not None else None
    y = torch.empty((x2.shape[0], N), dtype=x.dtype, device=x.device)
    M = x2.shape[0]
    if g_idx is not None:
        ng = s.numel() // N
        if s.numel() != N * ng or (z is not None and z.numel() != s.numel()) or ng == 0:
            raise ValueError(f'qparams of {s.numel()} elements for N={N} rows')
        if g_idx.dtype != torch.int32 or g_idx.numel() != K or not g_idx.is_cuda:
            raise ValueError(f'g_idx must be a CUDA int32 tensor of K={K} elements')
        gi = g_idx.contiguous()
        with TIMER.span(f'gemm_w{bits}a16_gidx', flops=2.0 * M * N * K,
                        nbytes=2.0 * M * K + bits / 8.0 * N * K + 8.0 * N * ng + 4.0 * K + 2.0 * M * N):
            call(f'llmc_gemm_w{bits}a16_gidx', ptr(x2), ptr(wq.contiguous()), ptr(s), ptr(z), dtype_enum(qdt),
                 ptr(gi), ng, int(bool(qparams_t)), ptr(b), ptr(y), M, N, K, dtype_enum(x.dtype),
                 stream_ptr(x.device))
        return y.reshape(*x.shape[:-1], N)
    with TIMER.span(f'gemm_w{bits}a16', flops=2.0 * M * N * K,
                    nbytes=2.0 * M * K + bits / 8.0 * N * K + 8.0 * N * K / group + 2.0 * M * N):
        call(f'llmc_gemm_w{bits}a16', ptr(x2), ptr(wq.contiguous()), ptr(s), ptr(z), dtype_enum(qdt), ptr(b), ptr(y), M, N, K,
             int(-group if qparams_t else group), dtype_enum(x.dtype), stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


def linear_forward_w4a16_awq(x, qweight, scales, qzeros, group, bias=None):
    """Real-quant forward on the AutoAWQ GEMM export as stored (csrc/gemm_w4.cu, llmc_gemm_w4a16_awq):
    y = x @ W.T (+ bias) with W[n, k] = rT((q - z) * s), bit-identical to linear_forward on that W.

    qweight [K, N/8] int32 and qzeros [K/group, N/8] int32, 8 nibbles per word along N in AutoAWQ's
    order (nibble i = column 8j + (0, 2, 4, 6, 1, 3, 5, 7)[i]); scales [K/group, N] fp16.  q and z are
    the nibbles as stored.  x bf16 or fp16."""
    if x.dtype not in (torch.bfloat16, torch.float16):
        raise ValueError(f'activations must be bf16 or fp16, not {x.dtype}')
    if qweight.dtype != torch.int32 or qzeros.dtype != torch.int32 or scales.dtype != torch.float16:
        raise ValueError(f'AutoAWQ tensors are int32 qweight / qzeros and fp16 scales, not '
                         f'{qweight.dtype} / {qzeros.dtype} / {scales.dtype}')
    K = x.shape[-1]
    if qweight.dim() != 2 or qweight.shape[0] != K:
        raise ValueError(f'qweight {tuple(qweight.shape)} does not match K={K}')
    N = qweight.shape[1] * 8
    if group <= 0 or K % group:
        raise ValueError(f'group {group} does not divide K={K}')
    ng = K // group
    if tuple(scales.shape) != (ng, N) or tuple(qzeros.shape) != (ng, N // 8):
        raise ValueError(f'scales {tuple(scales.shape)} / qzeros {tuple(qzeros.shape)} do not match '
                         f'{ng} groups of N={N} columns')
    if K % 64 or group % 64:
        raise NotImplementedError(f'the AutoAWQ forward steps 64 deep along K: K={K} and group={group} '
                                  'must be multiples of 64')
    if N % 32:
        raise NotImplementedError(f'the AutoAWQ forward needs N % 32 == 0 (a 16-byte qweight row), not N={N}')
    require_cuda(x, qweight, scales, qzeros, bias)
    x2 = x.reshape(-1, K)
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    b = bias.to(x.dtype).contiguous() if bias is not None else None
    M = x2.shape[0]
    y = torch.empty((M, N), dtype=x.dtype, device=x.device)
    with TIMER.span('gemm_w4a16_awq', flops=2.0 * M * N * K,
                    nbytes=2.0 * M * K + 0.5 * N * K + 2.5 * N * ng + 2.0 * M * N):
        call('llmc_gemm_w4a16_awq', ptr(x2), ptr(qweight.contiguous()), ptr(scales.contiguous()),
             ptr(qzeros.contiguous()), ptr(b), ptr(y), M, N, K, int(group), dtype_enum(x.dtype),
             stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


def linear_forward_rz(x, wq, scales, zeros, bits, sym, group_axis, group=None, g_idx=None, outliers=None,
                      bias=None):
    """Fake-quant forward on packed codes with REAL-VALUED zero-points (HQQ, SpQR: round_zp False),
    csrc/gemm_w4.cu: y = x @ dequant(wq).T + bias, dequant = rT((code - zero) * scale) as two fp32
    ops and one rounding — bit-identical to linear_forward on the weight quant.py:710-717 materialises.

    wq: the packed codes of pack_unsigned_codes (bits 2 / 3 / 4 / 8).  scales / zeros: fp32 (zeros
    None => 0); `sym` says that the codes are stored with the +2^(bits-1) offset of a symmetric grid.
    group_axis 0: groups along K, column k in group g_idx[k] (int32 [K], required), qparams [ng, N].
    group_axis 1: groups of `group` rows along N, qparams [K, N/group] (HQQ axis 0).
    outliers: None or (rows int32 [N+1], cols int32 [nnz], vals [nnz] in x.dtype), the CSR of
    outliers_to_csr; each value replaces its dequantised element."""
    require_cuda(x, wq, scales)
    if bits not in (2, 3, 4, 8):
        raise ValueError(f'packed weights are 2, 3, 4 or 8 bits, not {bits}')
    if scales.dim() != 2 or scales.dtype != torch.float32 or (zeros is not None and (
            zeros.dtype != torch.float32 or zeros.shape != scales.shape)):
        raise ValueError('real-zero qparams are 2-D fp32 scales (and zeros of the same shape)')
    K = x.shape[-1]
    if group_axis == 0:
        N = scales.shape[1]
        if g_idx is None or g_idx.dtype != torch.int32 or g_idx.numel() != K or not g_idx.is_cuda:
            raise ValueError(f'group_axis 0 needs g_idx, a CUDA int32 tensor of K={K} elements')
        ng, group = scales.shape[0], 0
    elif group_axis == 1:
        N = scales.shape[1] * group
        if scales.shape[0] != K:
            raise ValueError(f'group_axis 1 qparams are [K={K}, N/group], not {tuple(scales.shape)}')
        ng = 0
    else:
        raise ValueError(f'group_axis must be 0 or 1, not {group_axis}')
    want = ((N + 1) // 2, 3 * K // 16) if bits == 3 else (N, K * bits // 32)
    if wq.dtype != torch.int32 or tuple(wq.shape) != want:
        raise ValueError(f'packed weight {tuple(wq.shape)} does not match N={N}, K={K} at {bits} bits')
    o_rows = o_cols = o_vals = None
    nnz = 0
    if outliers is not None:
        o_rows, o_cols, o_vals = outliers
        if o_rows.numel() != N + 1 or o_vals.dtype != x.dtype or o_cols.numel() != o_vals.numel():
            raise ValueError('outliers must be a CSR (rows [N+1], cols [nnz], vals [nnz] in the activation dtype)')
        nnz = o_cols.numel()
        if nnz == 0:                                  # empty tensors have no storage to point at
            o_rows = o_cols = o_vals = None
    x2 = x.reshape(-1, K)
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    b = bias.to(x.dtype).contiguous() if bias is not None else None
    y = torch.empty((x2.shape[0], N), dtype=x.dtype, device=x.device)
    M = x2.shape[0]
    gi = g_idx.contiguous() if g_idx is not None else None
    with TIMER.span(f'gemm_w{bits}a16_rz', flops=2.0 * M * N * K,
                    nbytes=2.0 * M * K + bits / 8.0 * N * K + 8.0 * scales.numel() + 6.0 * nnz + 2.0 * M * N):
        call(f'llmc_gemm_w{bits}a16_rz', ptr(x2), ptr(wq.contiguous()), ptr(scales.contiguous()),
             ptr(zeros.contiguous() if zeros is not None else None), int(bool(sym)), int(group_axis),
             int(group or 0), ptr(gi), int(ng), ptr(o_rows), ptr(o_cols), ptr(o_vals), ptr(b), ptr(y), M, N, K,
             dtype_enum(x.dtype), stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


def outliers_to_csr(mask, values):
    """A dense outlier mask [R, C] (bool / uint8) and the weight [R, C] -> the CSR of
    linear_forward_rz: rows int32 [R+1], cols int32 [nnz] ascending within a row, values[mask]
    [nnz] in values' dtype.  On the mask's device."""
    m = mask.bool()
    idx = m.nonzero()                                 # row-major: rows, then columns, ascending
    counts = m.sum(dim=1, dtype=torch.int64)
    rows = torch.zeros(m.shape[0] + 1, dtype=torch.int64, device=m.device)
    rows[1:] = counts.cumsum(0)
    return (rows.to(torch.int32), idx[:, 1].to(torch.int32).contiguous(),
            values[idx[:, 0], idx[:, 1]].contiguous())


FP8_GRIDS = {torch.float8_e4m3fn: 'e4m3', torch.float8_e5m2: 'e5m2'}


def linear_forward_fp8w(x, wq, scales, group, bias=None, qparams_t=False, g_idx=None):
    """Fake-quant forward on FP8 weights (csrc/gemm_w4.cu, e4m3 / e5m2 grid): y = x @ dequant(wq).T
    + bias, dequant = rT(fp32(wq) * s) with s = 1 where the scale is 0 — bit-identical to
    linear_forward on the weight FloatQuantizer materialises (llmc_fp8_quant's QDQ output) while
    reading 8 bits plus a scale per group instead of 16 bits per weight.

    wq [N, K] float8_e4m3fn / float8_e5m2; scales [N, K/group] (or [K/group, N] with qparams_t) in
    x.dtype or fp32.  g_idx as in linear_forward_w4."""
    require_cuda(x, wq, scales)
    if wq.dtype not in FP8_GRIDS:
        raise TypeError(f'fp8 weight dtype must be float8_e4m3fn or float8_e5m2, not {wq.dtype}')
    K = x.shape[-1]
    N = wq.shape[0]
    if wq.dim() != 2 or wq.shape[1] != K or K % 4:
        raise ValueError(f'fp8 weight shape {tuple(wq.shape)} does not match K={K}')
    e5m2 = int(wq.dtype == torch.float8_e5m2)
    words = wq.contiguous().view(torch.int32)            # [N, K/4]: byte i of word w = element 4w + i
    x2 = x.reshape(-1, K)
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    qdt = x.dtype if scales.dtype == x.dtype else torch.float32
    shape = (-1, N) if qparams_t else (N, -1)
    s = scales.reshape(shape).to(qdt).contiguous()
    b = bias.to(x.dtype).contiguous() if bias is not None else None
    y = torch.empty((x2.shape[0], N), dtype=x.dtype, device=x.device)
    M = x2.shape[0]
    if g_idx is not None:
        ng = s.numel() // N
        if s.numel() != N * ng or ng == 0:
            raise ValueError(f'scales of {s.numel()} elements for N={N} rows')
        if g_idx.dtype != torch.int32 or g_idx.numel() != K or not g_idx.is_cuda:
            raise ValueError(f'g_idx must be a CUDA int32 tensor of K={K} elements')
        gi = g_idx.contiguous()
        with TIMER.span('gemm_fp8a16_gidx', flops=2.0 * M * N * K,
                        nbytes=2.0 * M * K + 1.0 * N * K + s.element_size() * N * ng + 4.0 * K + 2.0 * M * N):
            call('llmc_gemm_fp8a16_gidx', ptr(x2), ptr(words), ptr(s), None, dtype_enum(qdt), ptr(gi), ng,
                 int(bool(qparams_t)), ptr(b), ptr(y), M, N, K, dtype_enum(x.dtype), e5m2, stream_ptr(x.device))
        return y.reshape(*x.shape[:-1], N)
    with TIMER.span('gemm_fp8a16', flops=2.0 * M * N * K,
                    nbytes=2.0 * M * K + 1.0 * N * K + s.element_size() * N * K / group + 2.0 * M * N):
        call('llmc_gemm_fp8a16', ptr(x2), ptr(words), ptr(s), None, dtype_enum(qdt), ptr(b), ptr(y), M, N, K,
             int(-group if qparams_t else group), dtype_enum(x.dtype), e5m2, stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


def act_quantizer(act_cfg):
    """The activation quantizer of a `quant.act` config section, as the algorithms build it
    (blockwise.set_quant_config): FloatQuantizer for `quant_type: float-quant`, else IntegerQuantizer."""
    from .quant import IntegerQuantizer
    from .quant_float import FloatQuantizer
    kw = dict(act_cfg)
    cls = FloatQuantizer if kw.pop('quant_type', 'int-quant') == 'float-quant' else IntegerQuantizer
    return cls(**kw)


W8A8_ENTRY = {torch.int8: 'llmc_gemm_w8a8_i8', torch.float8_e4m3fn: 'llmc_gemm_w8a8_fp8'}


def linear_forward_w8a8(x, w, s_w, act_cfg, input_scale=None, bias=None):
    """The W8A8 real-quant forward (csrc/gemm_8bit.cu): x is quantised to int8 / e4m3 codes by the
    activation quantizer of `act_cfg` (a `quant.act` section, or the quantizer itself) exactly as the
    fake-quant forward of that config quantises it (real_quant_act), then
        y = rT(fp32(sum_k qx[m, k] * w[n, k]) * s_w[n] * s_x[m] (+ bias[n]))
    on the INT8 or FP8 tensor cores, both operands 8-bit.

    w [N, K] int8 (symmetric per-channel codes) or float8_e4m3fn, the exported `weight`; s_w its
    `weight_scale`, N values (per-channel) or one (per-tensor), any float dtype (widened to fp32);
    input_scale: None for per-token dynamic activations, the exported one-element `input_scale` for
    per-tensor static ones.  x bf16 / fp16, K % 16 == 0."""
    from .quant import BaseQuantizer, IntegerQuantizer
    from .quant_float import FloatQuantizer
    require_cuda(x, w, s_w, input_scale, bias)
    if w.dtype not in W8A8_ENTRY:
        raise NotImplementedError(f'W8A8 weights are int8 or float8_e4m3fn, not {w.dtype}')
    aq = act_cfg if isinstance(act_cfg, BaseQuantizer) else act_quantizer(act_cfg)
    want = IntegerQuantizer if w.dtype == torch.int8 else FloatQuantizer
    if type(aq) is not want:
        raise NotImplementedError(f'{w.dtype} weights need {want.__name__} activations, not {type(aq).__name__}')
    K = x.shape[-1]
    N = w.shape[0]
    if w.dim() != 2 or w.shape[1] != K:
        raise ValueError(f'weight shape {tuple(w.shape)} does not match K={K}')
    sw = s_w.reshape(-1).float().contiguous()
    if sw.numel() not in (1, N):
        raise ValueError(f'weight_scale of {sw.numel()} values for N={N} rows')
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    y = torch.empty((M, N), dtype=x.dtype, device=x.device)
    if M == 0:
        return y.reshape(*x.shape[:-1], N)
    qx, sx = aq.real_quant_act(x2, input_scale)
    b = bias.to(x.dtype).contiguous() if bias is not None else None
    with TIMER.span('gemm_w8a8', flops=2.0 * M * N * K, nbytes=float(M * K + N * K) + 2.0 * M * N):
        call(W8A8_ENTRY[w.dtype], ptr(qx), ptr(sx), int(sx.numel() != 1), ptr(w.contiguous()), ptr(sw),
             int(sw.numel() != 1), ptr(b), ptr(y), M, N, K, dtype_enum(x.dtype), stream_ptr(x.device))
    return y.reshape(*x.shape[:-1], N)


# Counterpart of the reference's USE_FP8GEMM_TRITON_KERNEL (module_utils.py:14-20): when set,
# LlmcFp8Linear keeps its weight in fp8 and runs block_wise_fp8_forward_func on the FP8 tensor cores.
# Off by default: the forward then dequantises once and runs the bf16 GEMM, as it always has here.
USE_FP8GEMM_KERNEL = False


def block_wise_fp8_forward_func(x, w, w_scale, block_size, bias):
    """module_utils.py:40-45: y = bf16(fp8_gemm(act_quant(x))) (+ bias after the rounding), as one
    act_quant pass and one FP8 GEMM whose bf16 epilogue adds the bias (csrc/gemm_8bit.cu)."""
    from .quant_float import act_quant, gemm_fp8_block
    xq, scale = act_quant(x, block_size)
    return gemm_fp8_block(xq, scale, w, w_scale, torch.bfloat16, bias)


def _copy_bufs(dst, ori_module):
    for name, buf in ori_module.named_buffers():
        if name.startswith('buf_'):
            dst.register_buffer(name, buf.data)
    for name, buf in ori_module.named_parameters():
        if name.startswith('buf_'):
            dst.register_buffer(name, buf.data)


def _func_name(any_callable):
    if isinstance(any_callable, partial):
        return any_callable.func.__name__
    return any_callable.__name__


class OriginFloatLinear(nn.Module):
    """module_utils.py:396-457 — plain linear on the (transformed) float weight."""

    def __init__(self, weight, bias, ori_module):
        super().__init__()
        self.register_buffer('weight', weight)
        if bias is not None:
            self.register_buffer('bias', bias)
        else:
            self.bias = None
        _copy_bufs(self, ori_module)
        if getattr(self, 'buf_rotate', False):
            raise NotImplementedError('online rotation (QuaRot) is out of scope (SURVEY §2 #12)')
        self.buf_rotate = False
        # :413-419: a block-FP8 weight (LlmcFp8Linear) keeps its scales and runs the FP8 forward
        if self.weight.data.dtype == torch.float8_e4m3fn:
            self.fp8_forward = True
            self.weight_scale_inv = ori_module.weight_scale_inv
            self.block_size = ori_module.block_size
        else:
            self.fp8_forward = False

    @torch.no_grad()
    def forward(self, x):
        if self.fp8_forward:
            return block_wise_fp8_forward_func(x, self.weight, self.weight_scale_inv, self.block_size,
                                               self.bias)
        return linear_forward(x, self.weight, self.bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module):
        bias = module.bias.data if getattr(module, 'bias', None) is not None else None
        new_module = cls(module.weight.data, bias, module)
        new_module.in_features = module.in_features
        new_module.out_features = module.out_features
        return new_module

    def __repr__(self):
        return (f'OriginFloatLinear(in_features={self.in_features},'
                f'out_features={self.out_features}, bias={self.bias is not None},'
                f'online_rotate={self.buf_rotate},'
                f'fp8_forward={self.fp8_forward})')


class LlmcFp8Linear(nn.Module):
    """module_utils.py:130-191 — holder of a 128x128 block-FP8 checkpoint weight (`weight` fp8 +
    `weight_scale_inv` fp32 [ceil(out/bs), ceil(in/bs)]).  Forward, by default, = the reference's
    non-Hopper branch (:171-178): dequantise ONCE to bf16 (llmc_fp8_block_dequant) and run the wgmma
    GEMM.  With USE_FP8GEMM_KERNEL set (the reference's Hopper branch, :157-166) the weight stays fp8
    and every forward runs block_wise_fp8_forward_func."""

    def __init__(self, in_features, out_features, bias, block_size):
        super().__init__()
        self.block_size, self.in_features, self.out_features = block_size, in_features, out_features
        if bias is not None:
            self.bias = nn.Parameter(torch.empty(out_features))
        else:
            self.register_parameter('bias', None)
        self.weight = nn.Parameter(torch.empty(out_features, in_features, dtype=torch.float8_e4m3fn),
                                   requires_grad=False)
        so, si = -(-out_features // block_size), -(-in_features // block_size)
        self.weight_scale_inv = nn.Parameter(torch.empty(so, si, dtype=torch.float32), requires_grad=False)

    @torch.no_grad()
    def forward(self, x):
        if self.weight.data.dtype == torch.float8_e4m3fn:
            if USE_FP8GEMM_KERNEL:
                return block_wise_fp8_forward_func(x, self.weight.data, self.weight_scale_inv.data,
                                                   self.block_size, self.bias)
            from .quant_float import weight_cast_to_bf16
            self.weight.data = weight_cast_to_bf16(self.weight.data, self.weight_scale_inv.data,
                                                   self.block_size)
        return linear_forward(x, self.weight.data, self.bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module, block_size):
        return cls(module.in_features, module.out_features, module.bias, block_size)

    def __repr__(self):
        return (f'LlmcFp8Linear(in_features={self.in_features}, out_features={self.out_features}, '
                f'bias={self.bias is not None}, weight_shape={self.weight.shape}, '
                f'weight_dtype={self.weight.dtype}, block_size={self.block_size}, '
                f'use_fp8gemm_triton_kernel={USE_FP8GEMM_KERNEL})')


class FakeQuantLinear(nn.Module):
    """module_utils.py:586-678 — calibration-time wrapper; w_qdq is evaluated lazily on the
    first forward and cached in the non-persistent `tmp_weight` buffer (:626-629)."""

    def __init__(self, weight, bias, ori_module, w_qdq, a_qdq):
        super().__init__()
        self.register_buffer('weight', weight)
        if bias is not None:
            self.register_buffer('bias', bias)
        else:
            self.bias = None
        self.a_qdq = a_qdq
        self.w_qdq = w_qdq
        _copy_bufs(self, ori_module)
        if getattr(self, 'buf_rotate', False):
            raise NotImplementedError('online rotation (QuaRot) is out of scope (SURVEY §2 #12)')
        self.buf_rotate = False
        if self.weight.data.dtype == torch.float8_e4m3fn:
            raise NotImplementedError('fp8 checkpoints (LlmcFp8Linear) are a SURVEY §8(f) row')
        self.fp8_forward = False
        self.dynamic_quant_weight = False
        self.dynamic_quant_tmp_weight = False

    def forward(self, x):
        if self.a_qdq is not None:
            x = self.a_qdq(x, self)
        if not hasattr(self, 'tmp_weight'):
            self.register_buffer('tmp_weight', self.w_qdq(self), persistent=False)
            self.tmp_bias = self.bias
        elif self.dynamic_quant_weight:
            self.tmp_weight = self.w_qdq(self)
            self.tmp_bias = self.bias
        elif self.dynamic_quant_tmp_weight:
            self.tmp_weight = self.w_qdq(self)
        return linear_forward(x, self.tmp_weight, self.tmp_bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module, w_qdq, a_qdq):
        bias = module.bias.data if getattr(module, 'bias', None) is not None else None
        new_module = cls(module.weight.data, bias, ori_module=module, w_qdq=w_qdq, a_qdq=a_qdq)
        new_module.in_features = module.in_features
        new_module.out_features = module.out_features
        new_module.w_qdq_name = _func_name(w_qdq)
        new_module.a_qdq_name = _func_name(a_qdq) if a_qdq is not None else 'None'
        return new_module

    def __repr__(self):
        return (f'FakeQuantLinear(in_features={self.in_features},'
                f'out_features={self.out_features}, bias={self.bias is not None},'
                f'weight_quant={self.w_qdq_name},'
                f'act_quant={self.a_qdq_name},'
                f'online_rotate={self.buf_rotate})')


def pack_unsigned_codes(codes, bits, signed):
    """[N, K] integer codes -> [N, K*bits/32] int32 of UNSIGNED codes, little-end first along K
    (the weight layout of llmc_gemm_w2a16 / w4a16 / w8a16).  llmc_pack_vllm_codes adds the
    +2^(bits-1) storage offset of module_utils.py:842-844, so asymmetric (already unsigned) codes are
    shifted down first.

    bits 3: [ceil(N/2), 3K/16] int32 in the row-pair layout of llmc_gemm_w3a16 (llmc_pack_w3_codes;
    include/llmc_b200.h), K a multiple of 64."""
    require_cuda(codes)
    c = codes.to(torch.int32)
    if not signed:
        c = c - (1 << (bits - 1))
    c = c.contiguous()
    rows, cols = c.shape
    if bits == 3:
        out = torch.empty(((rows + 1) // 2, 3 * cols // 16), dtype=torch.int32, device=c.device)
        call('llmc_pack_w3_codes', ptr(c), rows, cols, ptr(out), stream_ptr(c.device))
        return out
    pf = 32 // bits
    out = torch.empty((rows, cols // pf), dtype=torch.int32, device=c.device)
    call('llmc_pack_vllm_codes', ptr(c), 4, rows, cols, int(bits), ptr(out), stream_ptr(c.device))
    return out


def unpack_unsigned_codes(packed, bits, rows):
    """The inverse of pack_unsigned_codes: [rows, K] int32 unsigned codes (elementwise, exact)."""
    if bits == 3:
        P, W = packed.shape
        steps = W // 12
        # [pair, step, row of the pair, word] -> [row, step, word]
        words = packed.reshape(P, steps, 2, 6).permute(0, 2, 1, 3).reshape(2 * P, steps, 6)[:rows]
        i = torch.arange(16, device=packed.device, dtype=torch.int32)
        lo = ((words[..., :4, None] >> (2 * i)) & 3).reshape(rows, steps, 64)
        c = torch.arange(32, device=packed.device, dtype=torch.int32)
        pos = (c & ~24) | ((c & 8) << 1) | ((c & 16) >> 1)      # code 32m + c at bit c with bits 3, 4 swapped
        hi = ((words[..., 4:, None] >> pos) & 1).reshape(rows, steps, 64)
        return (lo | (hi << 2)).reshape(rows, steps * 64)
    pf = 32 // bits
    sh = torch.arange(pf, device=packed.device, dtype=torch.int32) * bits
    return ((packed.unsqueeze(-1) >> sh) & ((1 << bits) - 1)).reshape(packed.shape[0], -1)


class EffcientFakeQuantLinear(nn.Module):
    """module_utils.py:681-759 — eval-time wrapper: w_qdq applied once in `new`.

    Extension (K6): when the weight quantizer is a plain INT2 / INT3 / INT4 / INT8 group or channel
    quantizer, `new` keeps the PACKED codes + group qparams instead of the dequantised weight and
    the forward runs the fused dequant -> wgmma GEMM (csrc/gemm_w4.cu) — bit-identical to F.linear
    on the materialised weight (tests/test_gpu_gemm_w4.py, tests/test_gpu_gemm_w2w3.py), at e.g.
    2.5 (W2 g64) / 3.25 (W3 g128) / 4.25 / 8.25 instead of 16 bits per weight in HBM.  `.weight`
    then dequantises on demand.  LLMC_B200_FUSED_DEQUANT=0 disables it.

    The packed form comes from the algorithm's `w_packed` twin of its `w_qdq` (RTN / AWQ: the base
    one; GPTQ: GPTQ.w_packed).  Its qparams keep the dtype the algorithm stores them in — fp32 for
    GPTQ's dynamic groups, with one rounding of the fp32 product — and `g_idx` (int32 [K], None
    when groups are contiguous) gives each column's group when GPTQ's act-order makes the groups
    contiguous only in the permuted column order.  Packed modules are left alone by
    `convert_dtype`: their codes stay int32 and their qparams keep their dtype.

    FP8 weights (FloatQuantizer on an e4m3 / e5m2 grid) are packed too: `qweight` then holds the
    fp8 bytes [N, K] themselves (`q_grid` 'e4m3' / 'e5m2'; 'int' for codes), with one scale per row
    or group and no zero-point, and the forward runs llmc_gemm_fp8a16 — 8 bits plus the scales per
    weight instead of 16, bit-identical to the materialised forward (tests/test_gpu_gemm_fp8w.py).

    Real-valued zero-points (HQQ.w_packed, SpQR.w_packed; `q_rz`): fp32 qparams in the layout of
    linear_forward_rz — [ng, N] with `g_idx` for groups along K (`q_axis` 0), [K, N/group] for HQQ's
    groups along N (`q_axis` 1) — `q_sym` for codes stored with the symmetric offset, and SpQR's
    outliers as a CSR over rows (`outlier_rows / outlier_cols / outlier_vals`, None without).  The
    forward runs llmc_gemm_w{2,3,4,8}a16_rz (tests/test_gpu_gemm_rz.py)."""

    # the buffers of the packed form; export_state_dict writes the dense `weight` of an FP8, 2- / 3-bit
    # or real-zero module instead
    PACKED_BUFFERS = ('qweight', 'qscales', 'qzeros', 'qscales_t', 'qzeros_t', 'g_idx', 'outlier_rows',
                      'outlier_cols', 'outlier_vals')

    def __init__(self, weight, bias, ori_module, a_qdq, packed=None):
        super().__init__()
        if packed is None:
            self.register_buffer('weight', weight)
        else:
            self.register_buffer('qweight', packed['qweight'])
            self.register_buffer('qscales', packed['scales'])
            if packed['zeros'] is not None:
                self.register_buffer('qzeros', packed['zeros'])
            else:
                self.qzeros = None
            self.q_bits, self.q_group, self.q_dtype = packed['bits'], packed['group'], packed['dtype']
            self.q_grid = FP8_GRIDS.get(packed['qweight'].dtype, 'int')
            self.q_rz = packed.get('rz', False)
            if self.q_rz:
                # the qparams are already in the kernel's layout
                self.q_axis, self.q_sym = packed['group_axis'], packed['sym']
                o = packed.get('outliers')
                for i, leaf in enumerate(('outlier_rows', 'outlier_cols', 'outlier_vals')):
                    self.register_buffer(leaf, o[i] if o is not None else None)
            else:
                # [K/group, N] copies for the GEMM (coalesced qparam loads); tiny next to the codes
                self.register_buffer('qscales_t', packed['scales'].t().contiguous(), persistent=False)
                self.register_buffer('qzeros_t', packed['zeros'].t().contiguous()
                                     if packed['zeros'] is not None else None, persistent=False)
            self.register_buffer('g_idx', packed.get('g_idx'))
        self.packed = packed is not None
        if bias is not None:
            self.register_buffer('bias', bias)
        else:
            self.bias = None
        self.a_qdq = a_qdq
        _copy_bufs(self, ori_module)
        if getattr(self, 'buf_rotate', False):
            raise NotImplementedError('online rotation (QuaRot) is out of scope (SURVEY §2 #12)')
        self.buf_rotate = False

    def __getattr__(self, name):
        if name == 'weight' and self.__dict__.get('packed', False):
            return self.dequantized_weight()
        return super().__getattr__(name)

    @torch.no_grad()
    def dequantized_weight(self):
        """rT((code - zero) * scale): the tensor the reference holds in `.weight` (elementwise, exact).
        FP8 grids: rT(fp32(byte) * scale), a zero scale read as 1, as llmc_fp8_quant's QDQ output."""
        if self.q_rz:
            return self._dequantized_rz()
        if self.q_grid != 'int':
            N, K = self.qweight.shape
            s = self.qscales.float().reshape(N, -1)
            s = s.masked_fill(s == 0, 1.0)
            s = s[:, self.g_idx.long()] if self.g_idx is not None else s.repeat_interleave(self.q_group, dim=1)
            return (self.qweight.float() * s).to(self.q_dtype)
        bits = self.q_bits
        codes = unpack_unsigned_codes(self.qweight, bits, self.qscales.shape[0])
        N, K = codes.shape
        z = self.qzeros if self.qzeros is not None else float(1 << (bits - 1))
        s = self.qscales
        if self.g_idx is not None:
            # column k in group g_idx[k]; (code - zero) * scale in the qparam dtype, one rounding
            gi = self.g_idx.long()
            zz = z.reshape(N, -1)[:, gi] if torch.is_tensor(z) else z
            return ((codes.to(s.dtype) - zz) * s.reshape(N, -1)[:, gi]).to(self.q_dtype)
        c = codes.reshape(N, -1, self.q_group).to(s.dtype)
        zz = z.reshape(N, -1, 1) if torch.is_tensor(z) else z
        return ((c - zz) * s.reshape(N, -1, 1)).reshape(N, K).to(self.q_dtype)

    def _rz_shape(self):
        s = self.qscales
        return (s.shape[1], self.g_idx.numel()) if self.q_axis == 0 else (s.shape[1] * self.q_group, s.shape[0])

    def _dequantized_rz(self):
        """rT((code - zero) * scale) as two fp32 ops, one rounding (quant.py:710-717 then .to(dtype)),
        then the outliers overwrite their elements (SpQR's torch.where)."""
        N, K = self._rz_shape()
        bits = self.q_bits
        code = unpack_unsigned_codes(self.qweight, bits, N)
        if self.q_sym:
            code = code - (1 << (bits - 1))
        code = code.float()
        if self.q_axis == 0:
            gi = self.g_idx.long()
            s = self.qscales[gi].t()
            z = self.qzeros[gi].t() if self.qzeros is not None else 0.0
        else:
            s = self.qscales.repeat_interleave(self.q_group, dim=1).t()
            z = self.qzeros.repeat_interleave(self.q_group, dim=1).t() if self.qzeros is not None else 0.0
        w = ((code - z) * s).to(self.q_dtype)
        if self.outlier_rows is not None:
            counts = (self.outlier_rows[1:] - self.outlier_rows[:-1]).long()
            r = torch.repeat_interleave(torch.arange(N, device=w.device), counts)
            w[r, self.outlier_cols.long()] = self.outlier_vals
        return w

    @torch.no_grad()
    def forward(self, x):
        if self.a_qdq is not None:
            x = self.a_qdq(x, self)
        if self.packed and self.q_rz:
            o = (self.outlier_rows, self.outlier_cols, self.outlier_vals) if self.outlier_rows is not None else None
            return linear_forward_rz(x, self.qweight, self.qscales, self.qzeros, self.q_bits, self.q_sym, self.q_axis,
                                     group=self.q_group, g_idx=self.g_idx, outliers=o, bias=self.bias)
        if self.packed and self.q_grid != 'int':
            return linear_forward_fp8w(x, self.qweight, self.qscales_t, self.q_group, self.bias, qparams_t=True,
                                       g_idx=self.g_idx)
        if self.packed:
            return linear_forward_w4(x, self.qweight, self.qscales_t, self.qzeros_t, self.q_group, self.bias,
                                     bits=self.q_bits, qparams_t=True, g_idx=self.g_idx)
        return linear_forward(x, self.weight, self.bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module, w_qdq, a_qdq, debug_print={}):
        import os
        packer = getattr(w_qdq, 'packed', None)
        packed = None
        if packer is not None and os.environ.get('LLMC_B200_FUSED_DEQUANT', '1') != '0':
            packed = packer(module)
        weight = w_qdq(module) if packed is None else None
        bias = module.bias.data if getattr(module, 'bias', None) is not None else None
        new_module = cls(weight, bias, ori_module=module, a_qdq=a_qdq, packed=packed)
        new_module.in_features = module.in_features
        new_module.out_features = module.out_features
        new_module.w_qdq_name = _func_name(w_qdq)
        new_module.a_qdq_name = _func_name(a_qdq) if a_qdq is not None else 'None'
        new_module.debug_print = debug_print
        return new_module

    def __repr__(self):
        return (f'EffcientFakeQuantLinear(in_features={self.in_features},'
                f'out_features={self.out_features}, bias={self.bias is not None},'
                f'weight_quant={self.w_qdq_name},'
                f'act_quant={self.a_qdq_name},'
                f'online_rotate={self.buf_rotate})')


def _cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


class VllmRealQuantLinear(nn.Module):
    """module_utils.py:762-876 — compressed-tensors layout: `weight_packed` / `weight`,
    `weight_scale` (fp16 when packed) or `weight_scale_inv`, `input_scale`.

    Extension (K7): the W8A8 exports run.  An int8 `weight` with symmetric int8 activations, or an
    e4m3 `weight` with e4m3 activations — per-token dynamic, or per-tensor static from `input_scale`
    — forward through linear_forward_w8a8 on the INT8 / FP8 tensor cores, the activations quantised
    as the fake-quant forward of the same config quantises them.  `act_cfg` (the config's `act`
    section, None for weight-only) is recorded by `new`; it is not a buffer, so the saved tensors are
    those of the export.

    The weight-only packed exports (W4A16 / W8A16: `weight_packed` [N, K*bits/32] of unsigned codes,
    fp16 `weight_scale` [N, K/group]) run on llmc_gemm_w4a16 / llmc_gemm_w8a16, which read that
    layout as stored (zeros NULL: the +2^(bits-1) storage offset).  Every other layout raises
    NotImplementedError saying why."""

    def __init__(self, weight, bias, scales, input_scale, need_pack, scales_name):
        super().__init__()
        self.register_buffer('weight_packed' if need_pack else 'weight', weight)
        if bias is not None:
            self.register_buffer('bias', bias)
        else:
            self.bias = None
        self.register_buffer(scales_name, scales)
        self.register_buffer('input_scale', input_scale)
        self.act_cfg = None
        self._act_quantizer = None

    def packed_unsupported(self):
        """For a `weight_packed` module: None when forward runs it on llmc_gemm_w4a16 / w8a16, else
        the reason it does not."""
        if self.act_cfg is not None:
            return ('packed weights (weight_packed) with quantised activations have no real-quant forward: '
                    'only the weight-only W4A16 / W8A16 exports run')
        if 'weight_scale' not in self._buffers:
            return 'packed weights (weight_packed) need a weight_scale'
        K, words, s = self.in_features, self.weight_packed.shape[1], self.weight_scale
        if (32 * words) % K or (32 * words) // K not in (4, 8):
            return (f'weight_packed holds {words} words per row for in_features={K}: the packed forward '
                    'runs 4- and 8-bit codes')
        if s.dim() != 2 or K % s.shape[1]:
            return f'weight_scale {tuple(s.shape)} does not split in_features={K} into groups'
        group = K // s.shape[1]
        if K % 64 or group % 64:
            return (f'the packed forward steps 64 deep along K: in_features={K} and group={group} must be '
                    'multiples of 64')
        return None

    def w8a8_unsupported(self):
        """None when forward runs on llmc_gemm_w8a8_*, else the reason it does not."""
        if 'weight_packed' in self._buffers:
            return 'packed weights (weight_packed) are W4A16 / W8A16 exports: they run on the packed GEMM'
        if 'weight_scale_inv' in self._buffers:
            return 'per_block FP8 exports (weight_scale_inv) have no real-quant forward'
        if self.act_cfg is None:
            return (f'weight-only {self.weight.dtype} exports have no real-quant forward: the W8A8 GEMM '
                    'needs quantised activations')
        wdt, aqt = self.weight.dtype, _cfg_get(self.act_cfg, 'quant_type', 'int-quant')
        if wdt in (torch.bfloat16, torch.float16) and aqt == 'float-quant':
            wdt = torch.float8_e4m3fn          # GPTQ's e4m3 codes, cast to the model dtype (see fp8_weight)
        if wdt not in W8A8_ENTRY:
            return f'{wdt} weights have no real-quant forward (int8 and float8_e4m3fn do)'
        if (wdt == torch.int8) != (aqt == 'int-quant'):
            return f'{wdt} weights with {aqt} activations have no real-quant forward'
        static = bool(_cfg_get(self.act_cfg, 'static', False))
        gran = _cfg_get(self.act_cfg, 'granularity')
        if gran != ('per_tensor' if static else 'per_token'):
            return (f'{"static" if static else "dynamic"} {gran} activations have no real-quant forward '
                    '(per-token dynamic and per-tensor static do)')
        if static and (self.input_scale is None or self.input_scale.numel() != 1):
            return 'static activations need one input_scale'
        return None

    def activation_quantizer(self):
        if self._act_quantizer is None:
            self._act_quantizer = act_quantizer(self.act_cfg)
        return self._act_quantizer

    def fp8_weight(self):
        """The weight as e4m3 codes.  GPTQ's deploy ends in convert_dtype, which casts an exported e4m3
        weight to the model dtype (its values stay on the e4m3 grid, and the saved checkpoint holds
        them so); the codes are recovered once, exactly, and kept outside the buffers.  A 16-bit weight
        off the grid raises."""
        w = self.weight
        if w.dtype == torch.float8_e4m3fn:
            return w
        key = (w.data_ptr(), w._version)
        if getattr(self, '_w_e4m3_key', None) != key:
            q = w.to(torch.float8_e4m3fn)
            if not torch.equal(q.to(w.dtype), w):
                raise NotImplementedError(f'a {w.dtype} weight with FP8 activations must hold e4m3 grid values')
            self._w_e4m3, self._w_e4m3_key = q, key
        return self._w_e4m3

    @torch.no_grad()
    def forward(self, x):
        if 'weight_packed' in self._buffers:
            reason = self.packed_unsupported()
            if reason is not None:
                raise NotImplementedError(reason)
            K = self.in_features
            return linear_forward_w4(x, self.weight_packed, self.weight_scale, None,
                                     K // self.weight_scale.shape[1], self.bias,
                                     bits=32 * self.weight_packed.shape[1] // K)
        reason = self.w8a8_unsupported()
        if reason is not None:
            raise NotImplementedError(reason)
        static = bool(_cfg_get(self.act_cfg, 'static', False))
        w = self.weight if self.weight.dtype == torch.int8 else self.fp8_weight()
        return linear_forward_w8a8(x, w, self.weight_scale, self.activation_quantizer(),
                                   self.input_scale if static else None, self.bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module, w_q, quant_config):
        weight, scales = cls.quant_pack(module, w_q, quant_config)
        input_scale = getattr(module, 'buf_act_scales_0', None)
        act = _cfg_get(quant_config, 'act')
        if (act is not None and _cfg_get(act, 'static', False)
                and _cfg_get(quant_config, 'quant_type', 'int-quant') == 'int-quant'):
            input_scale = input_scale.unsqueeze(0)
        bias = module.bias.data if module.bias is not None else None
        wcfg = _cfg_get(quant_config, 'weight')
        need_pack = _cfg_get(wcfg, 'need_pack', False)
        scales_name = ('weight_scale_inv' if _cfg_get(wcfg, 'granularity') == 'per_block'
                       else 'weight_scale')
        new_module = cls(weight, bias, scales, input_scale, need_pack, scales_name)
        new_module.in_features = module.in_features
        new_module.out_features = module.out_features
        new_module.weight_shape, new_module.weight_dtype = weight.shape, weight.dtype
        new_module.scales_shape, new_module.scales_dtype = scales.shape, scales.dtype
        new_module.zeros_shape = new_module.zeros_dtype = None
        new_module.act_cfg = dict(act) if act is not None else None
        return new_module

    @classmethod
    @torch.no_grad()
    def quant_pack(cls, module, w_q, quant_config):
        weight, scales, zeros = w_q(module)
        if _cfg_get(_cfg_get(quant_config, 'weight'), 'need_pack', False):
            weight, scales = cls.pack(weight, scales, quant_config)
        return weight, scales

    @classmethod
    @torch.no_grad()
    def pack(cls, weight, scales, quant_config):
        """module_utils.py:836-862 on the device (the reference goes GPU->numpy->GPU)."""
        require_cuda(weight)
        num_bits = _cfg_get(_cfg_get(quant_config, 'weight'), 'bit')
        codes = weight.contiguous()
        if codes.dtype == torch.uint8:
            codes = codes.view(torch.int8)
        assert codes.dtype in (torch.int8, torch.int32), codes.dtype
        rows, cols = codes.shape
        pf = 32 // num_bits
        out = torch.empty((rows, (cols + pf - 1) // pf), dtype=torch.int32, device=codes.device)
        call('llmc_pack_vllm_codes', ptr(codes), codes.element_size(), rows, cols, int(num_bits),
             ptr(out), stream_ptr(codes.device))
        return out, scales.to(torch.float16)

    def __repr__(self):
        return ('VllmRealQuantLinear(' + f'in_features={self.in_features}, '
                + f'out_features={self.out_features}, ' + f'bias={self.bias is not None}, '
                + f'weight_shape={self.weight_shape}, ' + f'weight_dtype={self.weight_dtype}, '
                + f'scales_shape={self.scales_shape}, ' + f'scales_dtype={self.scales_dtype}, '
                + f'zeros_shape={self.zeros_shape}, ' + f'zeros_dtype={self.zeros_dtype})')


class LightllmRealQuantLinear(VllmRealQuantLinear):
    pass


class SglRealQuantLinear(VllmRealQuantLinear):
    pass


class Lightx2vRealQuantLinear(VllmRealQuantLinear):
    pass


class AutoawqRealQuantLinear(nn.Module):
    """module_utils.py:936-1065 — AutoAWQ GEMM layout: qweight [C, R/8], qzeros [ng, R/8],
    scales [ng, R] fp16.

    Extension: forward runs the export as stored on llmc_gemm_w4a16_awq (linear_forward_w4a16_awq);
    the reference's forward is not implemented."""

    def __init__(self, weight, bias, scales, zeros):
        super().__init__()
        self.register_buffer('qweight', weight)
        if bias is not None:
            self.register_buffer('bias', bias)
        else:
            self.bias = None
        self.register_buffer('scales', scales)
        if zeros is not None:
            self.register_buffer('qzeros', zeros)
        else:
            self.qzeros = None

    @torch.no_grad()
    def forward(self, x):
        if self.qzeros is None:
            raise NotImplementedError('an AutoAWQ export without qzeros has no real-quant forward')
        ng = self.scales.shape[0]
        if self.in_features % ng:
            raise ValueError(f'scales of {ng} groups do not split in_features={self.in_features}')
        return linear_forward_w4a16_awq(x, self.qweight, self.scales, self.qzeros, self.in_features // ng,
                                        self.bias)

    @classmethod
    @torch.no_grad()
    def new(cls, module, w_q, quant_config):
        weight, scales, zeros = cls.quant_pack(module, w_q, quant_config)
        bias = module.bias.data if module.bias is not None else None
        new_module = cls(weight, bias, scales, zeros)
        new_module.in_features = module.in_features
        new_module.out_features = module.out_features
        new_module.weight_shape, new_module.weight_dtype = weight.shape, weight.dtype
        new_module.scales_shape, new_module.scales_dtype = scales.shape, scales.dtype
        new_module.zeros_shape = zeros.shape if zeros is not None else None
        new_module.zeros_dtype = zeros.dtype if zeros is not None else None
        return new_module

    @classmethod
    @torch.no_grad()
    def quant_pack(cls, module, w_q, quant_config):
        _, scales, zeros = w_q(module)
        pack_version = _cfg_get(_cfg_get(quant_config, 'weight'), 'pack_version')
        if pack_version != 'gemm_pack':
            raise NotImplementedError(f'Not support {pack_version}.')
        return cls.gemm_pack(module, module.weight.data, scales, zeros, quant_config)

    @classmethod
    @torch.no_grad()
    def gemm_pack(cls, module, weight, scales, zeros, quant_config):
        """module_utils.py:1004-1065 as one tiled kernel (csrc/pack_awq.cu)."""
        assert scales is not None and zeros is not None
        wcfg = _cfg_get(quant_config, 'weight')
        bit, group_size = _cfg_get(wcfg, 'bit'), _cfg_get(wcfg, 'group_size')
        if bit != 4:
            raise NotImplementedError('Only 4-bit are supported for now.')
        require_cuda(weight, scales, zeros)
        w = weight.contiguous()
        R, C = w.shape
        ng = C // group_size
        s = scales.contiguous()
        z = zeros.to(torch.int32).contiguous()
        qweight = torch.empty((C, R // 32 * bit), dtype=torch.int32, device=w.device)
        qzeros = torch.empty((ng, R // 32 * bit), dtype=torch.int32, device=w.device)
        scales_out = torch.empty((ng, R), dtype=torch.float16, device=w.device)
        call('llmc_pack_awq', ptr(w), R, C, dtype_enum(w.dtype), ptr(s), dtype_enum(s.dtype),
             ptr(z), int(group_size), ptr(qweight), ptr(qzeros), ptr(scales_out),
             stream_ptr(w.device))
        return qweight, scales_out, qzeros

    def __repr__(self):
        return (f'{type(self).__name__}(' + f'in_features={self.in_features}, '
                + f'out_features={self.out_features}, ' + f'bias={self.bias is not None}, '
                + f'weight_shape={self.weight_shape}, ' + f'weight_dtype={self.weight_dtype}, '
                + f'scales_shape={self.scales_shape}, ' + f'scales_dtype={self.scales_dtype}, '
                + f'zeros_shape={self.zeros_shape}, ' + f'zeros_dtype={self.zeros_dtype})')


class MlcllmRealQuantLinear(AutoawqRealQuantLinear):
    pass


_TRANSFORMERS_LINEAR_TYPES_ = [nn.Linear]

_LLMC_LINEAR_TYPES_ = [
    LlmcFp8Linear, OriginFloatLinear, FakeQuantLinear, EffcientFakeQuantLinear, VllmRealQuantLinear,
    SglRealQuantLinear, AutoawqRealQuantLinear, MlcllmRealQuantLinear, LightllmRealQuantLinear,
    Lightx2vRealQuantLinear,
]

_REALQUANT_LINEAR_MAP_ = {
    'vllm_quant': VllmRealQuantLinear,
    'lightllm_quant': LightllmRealQuantLinear,
    'sgl_quant': SglRealQuantLinear,
    'autoawq_quant': AutoawqRealQuantLinear,
    'mlcllm_quant': MlcllmRealQuantLinear,
    'lightx2v_quant': Lightx2vRealQuantLinear,
}
