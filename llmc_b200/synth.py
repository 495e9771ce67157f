"""Shape-faithful synthetic models for the BASELINE.json configs (random-init weights, synthetic
tokens; there is no network for checkpoints).

The reference reaches decoder blocks through llmc/models/*.py wrappers around HF models
(base_model.py:22-481, llama.py:52-91, opt.py:60-100).  Those wrappers are out of scope
(SURVEY.md §2 #15); what the hot path needs from them is restated here: where the blocks are,
which linears form a subset and share an input, how a block is called, and module replacement.
Module / subset names follow the HF naming the reference uses, so `ignored_layers`, buffers
and exported state-dict keys line up.
"""
import math
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn
import torch.nn.functional as F

from ._lib import MOE_MAX_EXPERTS
from .module_utils import (_LLMC_LINEAR_TYPES_, _TRANSFORMERS_LINEAR_TYPES_, dense_forward_weight,
                           gemm_mla_kv_b, gemm_mla_qkv, gemm_rope_qkv, gemm_swiglu, interleave_gate_up,
                           linear_forward,
                           Fp8Operands, fake_quant_forward_operands, moe_forward, packed_forward_operands,
                           w8a8_forward_operands)

SHAPES = {
    # name: hidden, intermediate, layers, heads, kv_heads, vocab, kind, dtype
    'opt-125m': dict(hidden=768, inter=3072, layers=12, heads=12, kv_heads=12, vocab=50272,
                     kind='opt', dtype=torch.float16),
    'llama-2-7b': dict(hidden=4096, inter=11008, layers=32, heads=32, kv_heads=32, vocab=32000,
                       kind='llama', dtype=torch.float16),
    'llama-3-8b': dict(hidden=4096, inter=14336, layers=32, heads=32, kv_heads=8, vocab=128256,
                       kind='llama', dtype=torch.bfloat16),
    'llama-3-70b': dict(hidden=8192, inter=28672, layers=80, heads=64, kv_heads=8, vocab=128256,
                        kind='llama', dtype=torch.bfloat16),
    'mixtral-8x7b': dict(hidden=4096, inter=14336, layers=32, heads=32, kv_heads=8, vocab=32000,
                         kind='mixtral', dtype=torch.bfloat16, experts=8, top_k=2),
    'tiny-mixtral': dict(hidden=256, inter=512, layers=2, heads=4, kv_heads=2, vocab=512,
                         kind='mixtral', dtype=torch.bfloat16, experts=4, top_k=2),
    # Qwen1.5-MoE-A2.7B: transformers' Qwen2MoeConfig defaults (every layer sparse, q/k/v with bias);
    # inter is the dense intermediate size the config states, moe_inter / shared_inter the experts'
    'qwen1.5-moe-a2.7b': dict(hidden=2048, inter=5632, layers=24, heads=16, kv_heads=16, vocab=151936,
                              kind='qwen2moe', dtype=torch.bfloat16, experts=60, top_k=4, moe_inter=1408,
                              shared_inter=5632, rope_theta=1000000.0, rms_eps=1e-6),
    'tiny-qwen-moe': dict(hidden=256, inter=512, layers=2, heads=4, kv_heads=4, vocab=512,
                          kind='qwen2moe', dtype=torch.bfloat16, experts=12, top_k=4, moe_inter=128,
                          shared_inter=256, rope_theta=1000000.0, rms_eps=1e-6),
    # DeepSeek-V2-Lite (the published config.json; its yarn rope scaling is not built: default rope):
    # MLA without q LoRA, layer 0 dense (inter), the others 64 routed experts top-6 + 2 shared
    'deepseek-v2-lite': dict(hidden=2048, inter=10944, layers=27, heads=16, kv_heads=16, vocab=102400,
                             kind='deepseek_v2', dtype=torch.bfloat16, experts=64, top_k=6, moe_inter=1408,
                             shared_experts=2, first_k_dense=1, kv_lora=512, rope_dim=64, nope_dim=128,
                             v_dim=128, rope_theta=10000.0, routed_scale=1.0, rms_eps=1e-6),
    'tiny-deepseek-v2': dict(hidden=256, inter=512, layers=2, heads=4, kv_heads=4, vocab=512,
                             kind='deepseek_v2', dtype=torch.bfloat16, experts=12, top_k=6, moe_inter=128,
                             shared_experts=2, first_k_dense=1, kv_lora=128, rope_dim=64, nope_dim=128,
                             v_dim=128, rope_theta=10000.0, routed_scale=1.5, rms_eps=1e-6),
    'tiny-llama': dict(hidden=256, inter=512, layers=2, heads=4, kv_heads=2, vocab=512,
                       kind='llama', dtype=torch.bfloat16),
    'tiny-opt': dict(hidden=128, inter=512, layers=2, heads=4, kv_heads=4, vocab=512,
                     kind='opt', dtype=torch.float16),
}


class B200Linear(nn.Linear):
    """nn.Linear whose forward is the wgmma GEMM (csrc/gemm.cu) on CUDA tensors."""

    def forward(self, x):
        if x.is_cuda:
            return linear_forward(x, self.weight, self.bias)
        return F.linear(x, self.weight, self.bias)


class RMSNorm(nn.Module):
    def __init__(self, hidden, eps=1e-5):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden))
        self.variance_epsilon = eps

    def forward(self, x):
        if x.is_cuda and x.shape[-1] % 8 == 0 and self.weight.dtype == x.dtype:
            from . import block_ops
            return block_ops.rmsnorm(x, self.weight.data, self.variance_epsilon)
        dt = x.dtype
        x = x.float()
        x = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.variance_epsilon)
        return self.weight * x.to(dt)


def rope_cos_sin(seq_len, head_dim, device, dtype, theta=500000.0):
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, device=device).float() / head_dim))
    t = torch.arange(seq_len, device=device).float()
    freqs = torch.outer(t, inv)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def _rot_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


class LlamaAttention(nn.Module):
    """qkv_bias (Qwen2): q / k / v carry a bias, added in the GEMM's bias epilogue (B200Linear)."""

    def __init__(self, hidden, heads, kv_heads, qkv_bias=False):
        super().__init__()
        self.heads, self.kv_heads, self.head_dim = heads, kv_heads, hidden // heads
        self.q_proj = B200Linear(hidden, heads * self.head_dim, bias=qkv_bias)
        self.k_proj = B200Linear(hidden, kv_heads * self.head_dim, bias=qkv_bias)
        self.v_proj = B200Linear(hidden, kv_heads * self.head_dim, bias=qkv_bias)
        self.o_proj = B200Linear(heads * self.head_dim, hidden, bias=False)

    def fused_qkv_weight(self, dtype):
        """[Wq; Wk; Wv], the weight of qkv_rope's single GEMM with RoPE in its epilogue, or None
        when the projections cannot run that way: a projection without a dense forward weight of
        `dtype` (module_utils.dense_forward_weight), head_dim != 128, or q / k widths that are not
        multiples of 256 (the GEMM's n-tile)."""
        if self.head_dim != 128:
            return None
        ws = [dense_forward_weight(m, dtype) for m in (self.q_proj, self.k_proj, self.v_proj)]
        if (any(w is None for w in ws) or ws[0].shape[0] % 256 or ws[1].shape[0] % 256
                or ws[2].shape[0] % 8 or len({w.shape[1] for w in ws}) != 1):
            return None
        return torch.cat(ws)

    def qkv_rope(self, x, position_embeddings, w_qkv=None):
        """q, k, v of x [B, S, hidden] with RoPE applied to q and k, as the [B, heads, S, head_dim]
        views sdpa takes.  One GEMM with RoPE in its epilogue when w_qkv = fused_qkv_weight() is
        given or can be built here (once per call; callers that project many chunks build it once),
        else the three projections and `attend`'s rotary path."""
        if w_qkv is None and x.is_cuda:
            w_qkv = self.fused_qkv_weight(x.dtype)
        if w_qkv is not None and x.is_cuda and position_embeddings is not None:
            B, S, _ = x.shape
            cos, sin = position_embeddings
            if cos.dtype == x.dtype and sin.dtype == x.dtype and cos.shape[0] >= S:
                q, k, v = gemm_rope_qkv(x, w_qkv, self.heads * self.head_dim,
                                        self.kv_heads * self.head_dim, cos[:S], sin[:S])
                return self._heads(q, k, v)
        return self._rope(self.q_proj(x), self.k_proj(x), self.v_proj(x), position_embeddings)

    def _heads(self, q, k, v):
        B, S, _ = q.shape
        return (q.view(B, S, self.heads, self.head_dim).transpose(1, 2),
                k.view(B, S, self.kv_heads, self.head_dim).transpose(1, 2),
                v.view(B, S, self.kv_heads, self.head_dim).transpose(1, 2))

    def attend(self, q, k, v, position_embeddings):
        return self.sdpa(*self._rope(q, k, v, position_embeddings))

    def _rope(self, q, k, v, position_embeddings):
        B, S, _ = q.shape
        cos, sin = position_embeddings
        fused = (q.is_cuda and self.head_dim % 16 == 0 and q.is_contiguous() and k.is_contiguous()
                 and cos.dtype == q.dtype and cos.shape[0] >= S)
        if fused:                        # rotary in place on the fresh projection outputs
            from . import block_ops
            block_ops.rope_(q, cos[:S], sin[:S], self.heads, self.head_dim)
            block_ops.rope_(k, cos[:S], sin[:S], self.kv_heads, self.head_dim)
        q, k, v = self._heads(q, k, v)
        if not fused:
            cos, sin = cos[None, None, :S], sin[None, None, :S]
            q = q * cos + _rot_half(q) * sin
            k = k * cos + _rot_half(k) * sin
        return q, k, v

    def sdpa(self, q, k, v):
        """Causal attention over [B, heads, S, head_dim] q, k, v; [B, S, heads * head_dim]."""
        B, _, S, _ = q.shape
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True,
                                           enable_gqa=self.kv_heads != self.heads)
        return o.transpose(1, 2).reshape(B, S, self.heads * self.head_dim)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        return self.o_proj(self.sdpa(*self.qkv_rope(hidden_states, position_embeddings)))


class LlamaMLP(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.gate_proj = B200Linear(hidden, inter, bias=False)
        self.up_proj = B200Linear(hidden, inter, bias=False)
        self.down_proj = B200Linear(inter, hidden, bias=False)

    def act(self, g, u, out=None):
        if (g.is_cuda and g.is_contiguous() and u.is_contiguous() and u.dtype == g.dtype
                and g.numel() % 8 == 0):
            from . import block_ops
            return block_ops.silu_mul(g, u, out=out)
        y = F.silu(g) * u
        if out is not None:
            out.copy_(y)
            return out
        return y

    def fused_gate_up_weight(self, dtype):
        """Gate and up interleaved in 128-row blocks, the weight of gate_up_act's single GEMM with
        SiLU-mul in its epilogue, or None when the projections cannot run that way: a projection
        without a dense forward weight of `dtype` (module_utils.dense_forward_weight), or an
        intermediate size that is not a multiple of 128."""
        wg = dense_forward_weight(self.gate_proj, dtype)
        wu = dense_forward_weight(self.up_proj, dtype)
        if wg is None or wu is None or wg.shape != wu.shape or wg.shape[0] % 128:
            return None
        return interleave_gate_up(wg, wu)

    def gate_up_act(self, x, out=None, w_gate_up=None):
        """act(gate_proj(x), up_proj(x)), into `out` when given.  One GEMM with SiLU-mul in its
        epilogue when w_gate_up = fused_gate_up_weight() is given or can be built here (once per
        call; callers that run many chunks build it once), else the two projections and `act`."""
        if w_gate_up is None and x.is_cuda:
            w_gate_up = self.fused_gate_up_weight(x.dtype)
        if w_gate_up is not None and x.is_cuda and (out is None or out.is_contiguous()):
            return gemm_swiglu(x, w_gate_up, out=out)
        return self.act(self.gate_proj(x), self.up_proj(x), out=out)

    def forward(self, x):
        return self.down_proj(self.gate_up_act(x))


class LlamaBlock(nn.Module):
    def __init__(self, hidden, inter, heads, kv_heads):
        super().__init__()
        self.self_attn = LlamaAttention(hidden, heads, kv_heads)
        self.mlp = LlamaMLP(hidden, inter)
        self.input_layernorm = RMSNorm(hidden)
        self.post_attention_layernorm = RMSNorm(hidden)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        h = hidden_states + self.self_attn(self.input_layernorm(hidden_states),
                                           position_embeddings=position_embeddings)
        return h + self.mlp(self.post_attention_layernorm(h))


class MixtralExpert(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.w1 = B200Linear(hidden, inter, bias=False)
        self.w2 = B200Linear(inter, hidden, bias=False)
        self.w3 = B200Linear(hidden, inter, bias=False)

    def forward(self, x):
        return self.w2(F.silu(self.w1(x)) * self.w3(x))


# the largest K of llmc_gemm_w8a8_i8 (csrc/gemm_8bit.cu kMaxKInt8): its int32 sum is exact below it
W8A8_MAX_K_INT8 = ((1 << 17) - 1) // 16 * 16


def _same_input_scale(a, b):
    """Whether the static input scales of linears a and b hold one value.  Read once per pair of
    buffer versions and cached on a, keyed by both buffers' (data_ptr, _version) as fp8_weight keys
    its codes, so that later forwards do not synchronise."""
    sa, sb = a.input_scale, b.input_scale
    key = (sa.data_ptr(), sa._version, sb.data_ptr(), sb._version)
    cached = getattr(a, '_same_input_scale', None)
    if cached is None or cached[0] != key:
        cached = (key, sa.numel() == sb.numel() and torch.equal(sa.reshape(-1).float(), sb.reshape(-1).float()))
        a._same_input_scale = cached
    return cached[1]


def _dense_triple_form(ws, hidden):
    """The form (inter) of one expert's dense (w1, w3, w2) forward weights when the grouped bf16
    GEMMs take them for hidden size `hidden`, else None: none missing, 16-byte aligned, inter a
    multiple of 128, shapes [inter, hidden] / [inter, hidden] / [hidden, inter]."""
    if any(t is None or t.data_ptr() % 16 for t in ws):
        return None
    inter = ws[0].shape[0]
    ok = inter % 128 == 0 and (ws[0].shape, ws[1].shape, ws[2].shape) == (
        (inter, hidden), (inter, hidden), (hidden, inter))
    return inter if ok else None


def _packed_triple_form(triple, hidden):
    """The form of one expert's (w1, w3, w2) PackedOperands / Fp8Operands when the grouped dequant
    GEMMs take it for hidden size `hidden`, else None: codes of the right shape, 16-byte aligned,
    inter and the groups multiples of 64, CUDA tensors, int32 g_idx of K entries, and w1 / w3 of one
    form, w2 the same but its groups.  The form is per linear: (grid, bits, qparam dtype, zeros or
    not, g_idx or not, layout, group, groups per row), then inter."""
    inter = triple[0].wq.shape[0]
    for o, (n, k) in zip(triple, ((inter, hidden), (inter, hidden), (hidden, inter))):
        ng = o.scales.numel() // n
        if (tuple(o.wq.shape) != (n, k * o.bits // 32) or o.wq.data_ptr() % 16
                or inter % 64 or o.group % 64 or k % o.group or o.scales.numel() != n * ng):
            return None
        if not all(t.is_cuda for t in (o.wq, o.scales, o.zeros, o.g_idx) if t is not None):
            return None
        if o.g_idx is not None and (o.g_idx.dtype != torch.int32 or o.g_idx.numel() != k
                                    or o.g_idx.data_ptr() % 16):
            return None
    f = tuple((getattr(o, 'e5m2', None), o.bits, o.scales.dtype, o.zeros is None, o.g_idx is None, o.transposed,
               o.group, o.scales.numel() // o.wq.shape[0]) for o in triple)
    if f[0] != f[1] or f[0][:6] != f[2][:6]:          # w1 / w3 one form, w2 the same but its groups
        return None
    return f + (inter,)


class SparseMoe(nn.Module):
    """A sparse-MoE layer with per-expert nn.Linear experts, as the reference's wrappers expect them;
    the installed transformers 5.x fuses the experts, so the shape models are restated here (SURVEY.md
    §7.3 item 8).  A subclass names its expert class and the attribute names of an expert's (gate,
    up, down) linears; the router, the per-expert loop and the grouped-path selectors are written
    once here.  Hooks on an expert only ever see the tokens routed to it (Appendix E-11)."""

    expert_cls = None
    linear_names = None                       # an expert's (gate, up, down) linears
    norm_topk_prob = True

    def __init__(self, hidden, experts, top_k, make_expert):
        super().__init__()
        self.top_k = top_k
        self.gate = nn.Linear(hidden, experts, bias=False)
        self.experts = nn.ModuleList([make_expert() for _ in range(experts)])

    def expert_linears(self, ex):
        """Expert ex's (gate, up, down) linears: Mixtral's (w1, w3, w2)."""
        return tuple(getattr(ex, n) for n in self.linear_names)

    def _plain(self, ex):
        return type(ex) is self.expert_cls and not ex._forward_hooks and not ex._forward_pre_hooks

    def route(self, x):
        """The router on x [T, H]: each token's top_k experts sel [T, k] and weights w [T, k] of x's
        dtype: softmax in fp32, top-k, renormalised when norm_topk_prob."""
        logits = self.gate(x)                      # module call: hooks / FakeQuantLinear see it
        w = F.softmax(logits, dim=1, dtype=torch.float)
        w, sel = torch.topk(w, self.top_k, dim=-1)
        if self.norm_topk_prob:
            w = w / w.sum(dim=-1, keepdim=True)
        return sel, w.to(x.dtype)

    def expert_loop(self, x, sel, w):
        """The experts one by one, each module called on exactly its routed tokens: the path for
        experts the grouped GEMMs cannot run, and the definition moe_forward reproduces bit for bit.
        Synchronises with the host once per expert (torch.where)."""
        out = torch.zeros_like(x)
        for e, expert in enumerate(self.experts):
            tok, slot = torch.where(sel == e)
            if tok.numel() == 0:
                continue
            out.index_add_(0, tok, expert(x[tok]) * w[tok, slot, None])
        return out

    def grouped_weights(self, x):
        """One (gate, up, down) triple of dense forward weights per expert when
        module_utils.moe_forward computes exactly what expert_loop computes on x, else None: every
        expert a plain expert_cls without hooks whose linears have a dense forward weight of x's
        16-bit dtype (module_utils.dense_forward_weight: no hooks, activation fake-quant, bias or
        packing), shapes the grouped GEMMs take (inter a multiple of 128, hidden of 8), at most
        MOE_MAX_EXPERTS."""
        if (not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16)
                or len(self.experts) > MOE_MAX_EXPERTS or x.shape[1] % 8):
            return None
        weights, form = [], None
        for ex in self.experts:
            if not self._plain(ex):
                return None
            ws = tuple(dense_forward_weight(m, x.dtype) for m in self.expert_linears(ex))
            f = _dense_triple_form(ws, x.shape[1])
            if f is None or (form is not None and f != form):
                return None
            form = f
            weights.append(ws)
        return weights

    def grouped_packed_operands(self, x):
        """One (gate, up, down) triple of module_utils.PackedOperands per expert when moe_forward on
        them computes exactly what expert_loop computes on x, else None: the checks of
        grouped_weights, every expert linear packed_forward_operands' (4- / 8-bit integer codes, no
        hooks, activation fake-quant or bias), all of one form (bits, qparam dtype and layout, zeros
        or not, g_idx or not, groups per row), and the shapes the grouped dequant GEMMs take (hidden,
        inter and the groups multiples of 64)."""
        if (not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16)
                or len(self.experts) > MOE_MAX_EXPERTS or x.shape[1] % 64):
            return None
        hidden = x.shape[1]
        ops, form = [], None
        for ex in self.experts:
            if not self._plain(ex):
                return None
            triple = tuple(packed_forward_operands(m, x.dtype) for m in self.expert_linears(ex))
            if any(o is None for o in triple):
                return None
            f = _packed_triple_form(triple, hidden)
            if f is None or (form is not None and f != form):
                return None
            form = f
            ops.append(triple)
        return ops

    def grouped_w8a8_operands(self, x):
        """One (gate, up, down) triple of module_utils.W8A8Operands per expert when moe_forward on
        them computes exactly what expert_loop computes on x, else None: every expert a plain
        expert_cls without hooks, every linear w8a8_forward_operands' (a W8A8 export without bias or
        hooks), all of one form (int8 or e4m3 codes, dynamic or static activations of one act config,
        per-channel or per-tensor weight scales), the shapes the grouped W8A8 GEMMs take (hidden and
        inter multiples of 16, inter of 64), at most MOE_MAX_EXPERTS.  Static activations also need
        gate.input_scale == up.input_scale in every expert: the gate/up launch quantises each row
        once, where the loop quantises it for gate and for up apart."""
        if (not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16)
                or len(self.experts) > MOE_MAX_EXPERTS or x.shape[1] % 16):
            return None
        hidden = x.shape[1]
        ops, form = [], None
        for ex in self.experts:
            if not self._plain(ex):
                return None
            lin = self.expert_linears(ex)
            triple = tuple(w8a8_forward_operands(m) for m in lin)
            if any(o is None for o in triple):
                return None
            inter = triple[0].w.shape[0]
            if inter % 64 or (triple[0].w.dtype == torch.int8 and max(hidden, inter) > W8A8_MAX_K_INT8):
                return None
            for o, (n, k) in zip(triple, ((inter, hidden), (inter, hidden), (hidden, inter))):
                if (tuple(o.w.shape) != (n, k) or o.w.data_ptr() % 16 or o.s_w.numel() not in (1, n)
                        or not (o.w.is_cuda and o.s_w.is_cuda)
                        or (o.input_scale is not None and not o.input_scale.is_cuda)):
                    return None
            f = [(o.w.dtype, o.input_scale is None, o.s_w.numel() == 1, o.act_cfg) for o in triple]
            if f[0] != f[1] or f[0] != f[2] or (form is not None and f[0] != form):
                return None
            form = f[0]
            if triple[0].input_scale is not None and not _same_input_scale(lin[0], lin[1]):
                return None
            ops.append(triple)
        return ops

    def grouped_fake_quant_operands(self, x):
        """(experts, a_qdq) for module_utils.moe_forward when it computes exactly what expert_loop
        computes on x, else None: the fake-quant forms the other selectors leave to the loop.  Every
        expert a plain expert_cls without hooks; every linear's forward a_qdq then one GEMM
        (module_utils.fake_quant_forward_operands: FakeQuantLinear's dense tmp_weight, packed INT4 /
        INT8 or FP8-grid EffcientFakeQuantLinear, no bias or hooks), of one weight form with the
        shapes its grouped GEMMs take, at most MOE_MAX_EXPERTS; and either
          no activation fake-quant on any linear (FP8 weights only: the other two have their own
          selectors), or
          one a_qdq on all of them, the same bound method and arguments, whose class gives it a
          routed twin (`a_qdq.routed`, blockwise.a_qdq_routed) that accepts the layer: one pass
          over the routed rows before gate/up for every expert's gate and up linears, one over act
          before the down projection for every down linear.
        a_qdq is then None, or the pair of those passes."""
        if (not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16)
                or len(self.experts) > MOE_MAX_EXPERTS or x.shape[1] % 8):
            return None
        hidden = x.shape[1]
        ops, qdqs, form = [], [], None
        for ex in self.experts:
            if not self._plain(ex):
                return None
            got = tuple(fake_quant_forward_operands(m, x.dtype) for m in self.expert_linears(ex))
            if any(g is None for g in got):
                return None
            triple = tuple(g[0] for g in got)
            kind = torch.Tensor if isinstance(triple[0], torch.Tensor) else type(triple[0])
            if any(not isinstance(o, kind) for o in triple) or (kind is not torch.Tensor and hidden % 64):
                return None
            f = _dense_triple_form(triple, hidden) if kind is torch.Tensor else _packed_triple_form(triple, hidden)
            if f is None or (form is not None and (kind, f) != form):
                return None
            form = (kind, f)
            ops.append(triple)
            qdqs.extend(g[1] for g in got)
        a0 = qdqs[0]
        if a0 is None:
            return (ops, None) if form[0] is Fp8Operands and all(a is None for a in qdqs) else None
        routed = getattr(a0, 'routed', None)
        if routed is None or not all(isinstance(a, partial) and a.func == a0.func and a.args == a0.args
                                     and a.keywords == a0.keywords for a in qdqs):
            return None
        lins = [self.expert_linears(ex) for ex in self.experts]
        qdq_in = routed([lin[:2] for lin in lins])
        qdq_act = routed([lin[2:] for lin in lins])
        if qdq_in is None or qdq_act is None:
            return None
        return ops, (qdq_in, qdq_act)

    def grouped_operands(self, x):
        """(experts, a_qdq) of the first selector that accepts x, else (None, None): the grouped
        path's operands, or the per-expert loop."""
        experts, a_qdq = self.grouped_weights(x), None
        if experts is None:
            experts = self.grouped_packed_operands(x)
        if experts is None:
            experts = self.grouped_w8a8_operands(x)
        if experts is None:
            experts, a_qdq = self.grouped_fake_quant_operands(x) or (None, None)
        return experts, a_qdq


class MixtralSparseMoe(SparseMoe):
    """Mixtral's block_sparse_moe: gate / experts[i].w1|w2|w3 (models/mixtral.py:43-86), top-k
    weights renormalised."""

    expert_cls = MixtralExpert
    linear_names = ('w1', 'w3', 'w2')

    def __init__(self, hidden, inter, experts, top_k):
        super().__init__(hidden, experts, top_k, partial(MixtralExpert, hidden, inter))

    def forward(self, hidden_states):
        B, S, H = hidden_states.shape
        x = hidden_states.reshape(-1, H)
        sel, w = self.route(x)
        experts, a_qdq = self.grouped_operands(x)
        if experts is None:
            out = self.expert_loop(x, sel, w)
        elif a_qdq is None:
            out = moe_forward(x, sel, w, experts)
        else:
            out = moe_forward(x, sel, w, experts, a_qdq)
        return out.reshape(B, S, H)


class Qwen2MoeSparseMoe(SparseMoe):
    """Qwen2-MoE's mlp (models/qwen2moe.py:51-116): gate / experts[i].gate_proj|up_proj|down_proj,
    a shared expert (shared_expert.gate_proj|up_proj|down_proj) and its gate shared_expert_gate
    (Linear(hidden, 1)).  Top-k weights are not renormalised (norm_topk_prob False).  The block's
    output is transformers' Qwen2MoeSparseMoeBlock.forward (modeling_qwen2_moe.py):
      routed = index_add_ of each expert's rows * weight into zeros, expert by expert;
      shared = F.sigmoid(shared_expert_gate(x)) * shared_expert(x);
      out = routed + shared,
    each op rounding to the activation dtype once (shared_loop restates it)."""

    expert_cls = LlamaMLP
    linear_names = ('gate_proj', 'up_proj', 'down_proj')
    norm_topk_prob = False

    def __init__(self, hidden, inter, shared_inter, experts, top_k):
        super().__init__(hidden, experts, top_k, partial(LlamaMLP, hidden, inter))
        self.shared_expert = LlamaMLP(hidden, shared_inter)
        self.shared_expert_gate = B200Linear(hidden, 1, bias=False)

    def shared(self, x):
        """(shared_expert_gate(x) [T, 1], shared_expert(x) [T, H]) through the modules' own forwards:
        the shared expert's gate/up on the fused SwiGLU GEMM when its weights allow."""
        return self.shared_expert_gate(x), self.shared_expert(x)

    def shared_loop(self, x, sel, w):
        """The definition: expert_loop's routed sum plus F.sigmoid(gate logit) * shared expert."""
        g, s = self.shared(x)
        return self.expert_loop(x, sel, w) + F.sigmoid(g) * s

    def forward(self, hidden_states):
        B, S, H = hidden_states.shape
        x = hidden_states.reshape(-1, H)
        sel, w = self.route(x)
        experts, a_qdq = self.grouped_operands(x)
        if experts is None:
            out = self.shared_loop(x, sel, w)
        else:
            out = moe_forward(x, sel, w, experts, a_qdq, self.shared(x))
        return out.reshape(B, S, H)


class MixtralBlock(nn.Module):
    def __init__(self, hidden, inter, heads, kv_heads, experts, top_k):
        super().__init__()
        self.self_attn = LlamaAttention(hidden, heads, kv_heads)
        self.block_sparse_moe = MixtralSparseMoe(hidden, inter, experts, top_k)
        self.input_layernorm = RMSNorm(hidden)
        self.post_attention_layernorm = RMSNorm(hidden)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        h = hidden_states + self.self_attn(self.input_layernorm(hidden_states),
                                           position_embeddings=position_embeddings)
        return h + self.block_sparse_moe(self.post_attention_layernorm(h))


class Qwen2MoeBlock(nn.Module):
    """transformers' Qwen2MoeDecoderLayer with every layer sparse: attention with q/k/v bias, then
    the sparse-MoE mlp with its shared expert."""

    def __init__(self, hidden, heads, kv_heads, moe_inter, shared_inter, experts, top_k, eps):
        super().__init__()
        self.self_attn = LlamaAttention(hidden, heads, kv_heads, qkv_bias=True)
        self.mlp = Qwen2MoeSparseMoe(hidden, moe_inter, shared_inter, experts, top_k)
        self.input_layernorm = RMSNorm(hidden, eps)
        self.post_attention_layernorm = RMSNorm(hidden, eps)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        h = hidden_states + self.self_attn(self.input_layernorm(hidden_states),
                                           position_embeddings=position_embeddings)
        return h + self.mlp(self.post_attention_layernorm(h))


def mla_rope_cos_sin(seq_len, rope_dim, device, theta):
    """DeepSeek-V2's default rotary tables as fp32 (cos, sin) [seq_len, rope_dim / 2]: the real and
    imaginary parts of transformers' freqs_cis (torch.polar of position * inv_freq), computed on the
    CPU so that every device sees the same bits."""
    inv = 1.0 / (theta ** (torch.arange(0, rope_dim, 2, dtype=torch.int64).float() / rope_dim))
    freqs = torch.outer(torch.arange(seq_len).float(), inv)
    fc = torch.polar(torch.ones_like(freqs), freqs)
    return fc.real.contiguous().to(device), fc.imag.contiguous().to(device)


def mla_rotate(t, cos, sin):
    """apply_rotary_emb of modeling_deepseek_v2 on t [..., S, (H,) 64] (the position axis is the one
    cos [S, 32] lines up with): interleaved pairs (a, b) become (a c - b s, a s + b c) in fp32, one
    rounding per operation as torch's complex64 product takes them, then t's dtype."""
    a, b = t[..., 0::2].float(), t[..., 1::2].float()
    if t.dim() == 4:                                     # [B, S, H, 64]: one table row per S
        cos, sin = cos[:, None], sin[:, None]
    return torch.stack((a * cos - b * sin, a * sin + b * cos), dim=-1).flatten(-2).to(t.dtype)


class DeepseekV2Attention(nn.Module):
    """transformers' DeepseekV2Attention without q LoRA (DeepSeek-V2-Lite): q_proj, then MLA's
    compressed kv (kv_a_proj_with_mqa -> latent | k_pe, kv_a_layernorm, kv_b_proj -> k_nope | v),
    rotary on q's and k's pe slices (mla_rotate), k_pe shared by every head, causal SDPA at scale
    qk_head_dim ** -0.5, o_proj.  q, k and v are built in buffers [B, S, H * 192], [B, S, H * 192] and
    [B, S, H * 128] that SDPA reads as [B, S, H, D] views.  No qkv_rope: MLA blocks take GPTQ's
    generic hook schedule, not the Llama staged pass."""

    def __init__(self, hidden, heads, kv_lora, rope_dim=64, nope_dim=128, v_dim=128, eps=1e-6,
                 q_lora_rank=None):
        super().__init__()
        if q_lora_rank is not None:
            raise NotImplementedError(
                'DeepseekV2Attention: q_lora_rank models (q_a_proj / q_b_proj, DeepSeek-V2 236B) are not '
                'built; only DeepSeek-V2-Lite\'s q_proj form is')
        self.heads, self.kv_lora = heads, kv_lora
        self.rope_dim, self.nope_dim, self.v_dim = rope_dim, nope_dim, v_dim
        self.qk_dim = nope_dim + rope_dim
        self.q_proj = B200Linear(hidden, heads * self.qk_dim, bias=False)
        self.kv_a_proj_with_mqa = B200Linear(hidden, kv_lora + rope_dim, bias=False)
        self.kv_a_layernorm = RMSNorm(kv_lora, eps)
        self.kv_b_proj = B200Linear(kv_lora, heads * (nope_dim + v_dim), bias=False)
        self.o_proj = B200Linear(heads * v_dim, hidden, bias=False)
        self.scaling = self.qk_dim ** (-0.5)

    def fused_weights(self, dtype):
        """([W_q; W_kv_a], W_kv_b) for the two MLA GEMMs (llmc_gemm_mla_qkv / _kv_b), or None when
        the projections cannot run that way: a projection without a dense forward weight of `dtype`
        (module_utils.dense_forward_weight: no hooks, fake-quant activations, bias or packing), head
        dims other than 128 / 64 / 128, heads not a multiple of 4 or kv_lora not of 64."""
        if ((self.nope_dim, self.rope_dim, self.v_dim) != (128, 64, 128) or self.heads % 4
                or self.kv_lora % 64):
            return None
        ws = [dense_forward_weight(m, dtype) for m in (self.q_proj, self.kv_a_proj_with_mqa, self.kv_b_proj)]
        if any(w is None for w in ws) or ws[0].shape[1] != ws[1].shape[1]:
            return None
        return torch.cat(ws[:2]), ws[2]

    def qkv(self, x, position_embeddings):
        """The q, k, v buffers of x [B, S, hidden]: the two fused GEMMs when fused_weights allows,
        else the module calls (hooks and fake-quant linears see their inputs) and the torch glue."""
        B, S, _ = x.shape
        cos, sin = position_embeddings
        cos, sin = cos[:S], sin[:S]
        w = self.fused_weights(x.dtype) if x.is_cuda else None
        if w is not None and cos.dtype == torch.float32 and sin.dtype == torch.float32 and cos.is_cuda:
            q, k, latent = gemm_mla_qkv(x, w[0], self.heads, self.kv_lora, cos, sin)
            v = gemm_mla_kv_b(self.kv_a_layernorm(latent), w[1], k, self.heads)
            return q, k, v
        H, dn = self.heads, self.nope_dim
        q = self.q_proj(x).contiguous()
        qh = q.view(B, S, H, self.qk_dim)
        qh[..., dn:] = mla_rotate(qh[..., dn:], cos, sin)
        ckv = self.kv_a_proj_with_mqa(x)
        latent = ckv[..., :self.kv_lora].contiguous()
        kv = self.kv_b_proj(self.kv_a_layernorm(latent)).view(B, S, H, dn + self.v_dim)
        k = torch.empty_like(q)
        kh = k.view(B, S, H, self.qk_dim)
        kh[..., :dn] = kv[..., :dn]
        kh[..., dn:] = mla_rotate(ckv[..., self.kv_lora:], cos, sin)[:, :, None, :]
        v = kv[..., dn:].reshape(B, S, H * self.v_dim)
        return q, k, v

    def sdpa(self, q, k, v):
        """Causal attention of the q, k, v buffers; [B, S, H * v_dim]."""
        B, S, _ = q.shape
        H = self.heads
        o = F.scaled_dot_product_attention(q.view(B, S, H, -1).transpose(1, 2), k.view(B, S, H, -1).transpose(1, 2),
                                           v.view(B, S, H, -1).transpose(1, 2), is_causal=True, scale=self.scaling)
        return o.transpose(1, 2).reshape(B, S, H * self.v_dim)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        return self.o_proj(self.sdpa(*self.qkv(hidden_states, position_embeddings)))


class DeepseekV2Gate(nn.Module):
    """The remote-code MoEGate as the reference's DeepseekV2 wrapper meets it: its own module with a
    weight [experts, hidden] and no nn.Linear base, so it is a member of the MoE subset (AWQ scales
    it and searches over it) but not a block linear (no deploy replaces it, GPTQ skips it).  Called
    as a module, so hooks see x; the logits are F.linear in fp32."""

    def __init__(self, hidden, experts):
        super().__init__()
        self.in_features, self.out_features = hidden, experts
        self.weight = nn.Parameter(torch.empty(experts, hidden))

    def forward(self, x):
        return F.linear(x.float(), self.weight.float())


class DeepseekV2SparseMoe(SparseMoe):
    """DeepSeek-V2's mlp (models/deepseekv2.py): gate (DeepseekV2Gate) / experts[i].gate_proj|up_proj|
    down_proj and shared_experts (one SwiGLU MLP of n_shared * moe_inter).  The router is greedy
    top-k of the fp32 softmax, not renormalised, times routed_scaling_factor, all in fp32; the
    weights stay fp32.  The output is transformers' DeepseekV2Moe.forward (shared_loop restates it):
      routed = zeros, then per expert in ascending order index_add_(tok, (expert(x[tok]) * w).to(dtype)),
               the product bf16 x fp32 computed in fp32 and rounded once;
      out = routed + shared_experts(x)."""

    expert_cls = LlamaMLP
    linear_names = ('gate_proj', 'up_proj', 'down_proj')

    def __init__(self, hidden, inter, experts, top_k, n_shared, routed_scale, topk_method='greedy'):
        if topk_method != 'greedy':
            raise NotImplementedError(
                f'DeepseekV2SparseMoe: topk_method {topk_method!r} (DeepSeek-V2 236B\'s group-limited '
                'routing) is not built; only greedy top-k is')
        super().__init__(hidden, experts, top_k, partial(LlamaMLP, hidden, inter))
        self.gate = DeepseekV2Gate(hidden, experts)
        self.shared_experts = LlamaMLP(hidden, inter * n_shared)
        self.routed_scaling_factor = routed_scale

    def route(self, x):
        """sel [T, k] and fp32 weights w [T, k]: softmax of the fp32 logits, greedy top-k (unsorted),
        times routed_scaling_factor."""
        scores = self.gate(x).softmax(dim=-1, dtype=torch.float32)
        w, sel = torch.topk(scores, self.top_k, dim=-1, sorted=False)
        return sel, w * self.routed_scaling_factor

    def expert_loop(self, x, sel, w):
        """DeepseekV2Experts.forward on per-expert modules: one rounding of expert(x) * w (fp32)."""
        out = torch.zeros_like(x)
        for e, expert in enumerate(self.experts):
            tok, slot = torch.where(sel == e)
            if tok.numel() == 0:
                continue
            out.index_add_(0, tok, (expert(x[tok]) * w[tok, slot, None]).to(x.dtype))
        return out

    def shared_loop(self, x, sel, w):
        """The definition: expert_loop's routed sum plus the shared experts."""
        return self.expert_loop(x, sel, w) + self.shared_experts(x)

    def forward(self, hidden_states):
        B, S, H = hidden_states.shape
        x = hidden_states.reshape(-1, H)
        sel, w = self.route(x)
        experts, a_qdq = self.grouped_operands(x)
        if experts is None:
            out = self.shared_loop(x, sel, w)
        else:
            out = moe_forward(x, sel, w, experts, a_qdq, self.shared_experts(x))
        return out.reshape(B, S, H)


class DeepseekV2Block(nn.Module):
    """transformers' DeepseekV2DecoderLayer: MLA attention, then a dense SwiGLU MLP (layers before
    first_k_dense_replace) or the sparse MoE with its shared experts."""

    def __init__(self, s, layer_idx):
        super().__init__()
        self.self_attn = DeepseekV2Attention(s['hidden'], s['heads'], s['kv_lora'], s['rope_dim'], s['nope_dim'],
                                             s['v_dim'], s['rms_eps'], s.get('q_lora_rank'))
        if layer_idx >= s['first_k_dense']:
            self.mlp = DeepseekV2SparseMoe(s['hidden'], s['moe_inter'], s['experts'], s['top_k'],
                                           s['shared_experts'], s['routed_scale'], s.get('topk_method', 'greedy'))
        else:
            self.mlp = LlamaMLP(s['hidden'], s['inter'])
        self.input_layernorm = RMSNorm(s['hidden'], s['rms_eps'])
        self.post_attention_layernorm = RMSNorm(s['hidden'], s['rms_eps'])

    def forward(self, hidden_states, position_embeddings=None, **kw):
        h = hidden_states + self.self_attn(self.input_layernorm(hidden_states),
                                           position_embeddings=position_embeddings)
        return h + self.mlp(self.post_attention_layernorm(h))


class OPTAttention(nn.Module):
    def __init__(self, hidden, heads):
        super().__init__()
        self.heads, self.head_dim = heads, hidden // heads
        self.q_proj = B200Linear(hidden, hidden)
        self.k_proj = B200Linear(hidden, hidden)
        self.v_proj = B200Linear(hidden, hidden)
        self.out_proj = B200Linear(hidden, hidden)

    def forward(self, hidden_states, **kw):
        B, S, H = hidden_states.shape
        q = self.q_proj(hidden_states).view(B, S, self.heads, self.head_dim).transpose(1, 2)
        k = self.k_proj(hidden_states).view(B, S, self.heads, self.head_dim).transpose(1, 2)
        v = self.v_proj(hidden_states).view(B, S, self.heads, self.head_dim).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        return self.out_proj(o.transpose(1, 2).reshape(B, S, H))


class OPTBlock(nn.Module):
    def __init__(self, hidden, inter, heads):
        super().__init__()
        self.self_attn = OPTAttention(hidden, heads)
        self.self_attn_layer_norm = nn.LayerNorm(hidden)
        self.fc1 = B200Linear(hidden, inter)
        self.fc2 = B200Linear(inter, hidden)
        self.final_layer_norm = nn.LayerNorm(hidden)

    def forward(self, hidden_states, **kw):
        h = hidden_states + self.self_attn(self.self_attn_layer_norm(hidden_states))
        return h + self.fc2(F.relu(self.fc1(self.final_layer_norm(h))))


class _Decoder(nn.Module):
    def __init__(self, shape, n_layers):
        super().__init__()
        s = shape
        self.embed_tokens = nn.Embedding(s['vocab'], s['hidden'])
        if s['kind'] == 'llama':
            blocks = [LlamaBlock(s['hidden'], s['inter'], s['heads'], s['kv_heads'])
                      for _ in range(n_layers)]
            self.norm = RMSNorm(s['hidden'])
        elif s['kind'] == 'mixtral':
            blocks = [MixtralBlock(s['hidden'], s['inter'], s['heads'], s['kv_heads'], s['experts'],
                                   s['top_k']) for _ in range(n_layers)]
            self.norm = RMSNorm(s['hidden'])
        elif s['kind'] == 'qwen2moe':
            blocks = [Qwen2MoeBlock(s['hidden'], s['heads'], s['kv_heads'], s['moe_inter'], s['shared_inter'],
                                    s['experts'], s['top_k'], s['rms_eps']) for _ in range(n_layers)]
            self.norm = RMSNorm(s['hidden'], s['rms_eps'])
        elif s['kind'] == 'deepseek_v2':
            blocks = [DeepseekV2Block(s, i) for i in range(n_layers)]
            self.norm = RMSNorm(s['hidden'], s['rms_eps'])
        else:
            blocks = [OPTBlock(s['hidden'], s['inter'], s['heads']) for _ in range(n_layers)]
            self.norm = nn.LayerNorm(s['hidden'])
        self.layers = nn.ModuleList(blocks)
        self.lm_head = nn.Linear(s['hidden'], s['vocab'], bias=False)


class SynthModel:
    """What the block-wise framework needs from llmc's BaseModel (base_model.py), for the
    synthetic shapes.  `n_layers` lets a test/bench instantiate a prefix of the stack."""

    def __init__(self, name, n_layers=None, seed=0, device='cpu', outlier_seed=None,
                 with_head=True, init='cpu'):
        self.shape = dict(SHAPES[name])
        self.name = name
        self.kind = self.shape['kind']
        self.torch_dtype = self.shape['dtype']
        n_layers = n_layers or self.shape['layers']
        g = torch.Generator().manual_seed(seed)
        with torch.device('meta'):
            self.model = _Decoder(self.shape, n_layers)
        self.model = self.model.to(self.torch_dtype).to_empty(device=device)
        if not with_head:
            self.model.lm_head = None
        # HF default init N(0, 0.02^2), generated on CPU so CPU and GPU runs see identical bits
        gd = None
        if init == 'device':      # bench-sized models: draw on the GPU (seeded), no 8B-element CPU RNG
            gd = torch.Generator(device=device).manual_seed(seed)
        for n, p in self.model.named_parameters():
            if p.dim() >= 2:
                if gd is not None:
                    p.data.normal_(0, 0.02, generator=gd)
                    continue
                w = torch.empty(p.shape, dtype=torch.float32).normal_(0, 0.02, generator=g)
                p.data.copy_(w.to(device))
            elif 'norm' in n and n.endswith('weight'):
                p.data.fill_(1.0)
            else:
                p.data.zero_()
        if outlier_seed is not None:   # SURVEY §8(d) config 2: x8 on 0.5 % of input channels
            go = torch.Generator().manual_seed(outlier_seed)
            for m in self.model.layers.modules():
                if isinstance(m, nn.Linear):
                    C = m.in_features
                    idx = torch.randperm(C, generator=go)[: max(1, C // 200)]
                    m.weight.data[:, idx.to(m.weight.device)] *= 8
        self.model = self.model.to(self.torch_dtype)
        self.block_name_prefix = 'model.decoder.layers' if self.kind == 'opt' else 'model.layers'
        self.mm_model = None
        self.tokenizer = None

    @torch.no_grad()
    def load_hf_state_dict(self, sd):
        """Load a HuggingFace-named state dict (`model.embed_tokens.weight`, `model.layers.N...`,
        `model.norm.weight`, `lm_head.weight`) — the names the reference's wrappers operate on —
        into the shape model.  Used by the end-to-end parity tests, whose fixtures hold the
        random-init weights the reference was run on."""
        own = dict(self.model.named_parameters())
        used = set()
        for k, v in sd.items():
            n = k[len('model.'):] if k.startswith('model.') else k
            if n.startswith('decoder.'):
                n = n[len('decoder.'):]
            if n not in own:
                continue
            assert own[n].shape == v.shape, (k, own[n].shape, v.shape)
            own[n].data.copy_(v.to(own[n].dtype))
            used.add(n)
        missing = [n for n in own if n not in used]
        if missing:
            raise KeyError(f'state dict lacks {missing[:4]}... ({len(missing)} tensors)')

    # ---- export hooks (base_model.py:334-344; llama.py:40-41 / opt.py:41-42 / mixtral.py:26-27) -----
    def get_model(self):
        return self.model

    def get_num_attention_heads(self):
        return self.shape['heads']

    def skip_layer_name(self):
        return ['lm_head']

    def hf_config_dict(self):
        """The architecture part of the config.json `save_pretrained` would write for this shape."""
        s = self.shape
        arch = {'llama': ('LlamaForCausalLM', 'llama'), 'mixtral': ('MixtralForCausalLM', 'mixtral'),
                'qwen2moe': ('Qwen2MoeForCausalLM', 'qwen2_moe'), 'opt': ('OPTForCausalLM', 'opt'),
                'deepseek_v2': ('DeepseekV2ForCausalLM', 'deepseek_v2')}[self.kind]
        doc = {'architectures': [arch[0]], 'model_type': arch[1], 'hidden_size': s['hidden'],
               'num_hidden_layers': len(self.model.layers), 'num_attention_heads': s['heads'],
               'vocab_size': s['vocab'], 'torch_dtype': str(self.torch_dtype).replace('torch.', '')}
        if self.kind == 'opt':
            doc['ffn_dim'] = s['inter']
        else:
            doc.update({'intermediate_size': s['inter'], 'num_key_value_heads': s['kv_heads']})
        if self.kind == 'mixtral':
            doc.update({'num_local_experts': s['experts'], 'num_experts_per_tok': s['top_k']})
        if self.kind == 'qwen2moe':
            doc.update({'num_experts': s['experts'], 'num_experts_per_tok': s['top_k'],
                        'moe_intermediate_size': s['moe_inter'], 'shared_expert_intermediate_size': s['shared_inter'],
                        'norm_topk_prob': False, 'qkv_bias': True, 'rms_norm_eps': s['rms_eps'],
                        'rope_theta': s['rope_theta']})
        if self.kind == 'deepseek_v2':
            doc.update({'n_routed_experts': s['experts'], 'num_experts_per_tok': s['top_k'],
                        'moe_intermediate_size': s['moe_inter'], 'n_shared_experts': s['shared_experts'],
                        'first_k_dense_replace': s['first_k_dense'], 'kv_lora_rank': s['kv_lora'],
                        'q_lora_rank': None, 'qk_rope_head_dim': s['rope_dim'], 'qk_nope_head_dim': s['nope_dim'],
                        'v_head_dim': s['v_dim'], 'routed_scaling_factor': s['routed_scale'],
                        'topk_method': 'greedy', 'norm_topk_prob': False, 'rms_norm_eps': s['rms_eps'],
                        'rope_theta': s['rope_theta']})
        return doc

    # ---- structure (base_model.py:346-351, llama.py:52-91, opt.py:60-100) -----------------------
    def get_blocks(self):
        return self.model.layers

    def get_block_linears(self, block):
        return OrderedDict(
            (n, m) for n, m in block.named_modules()
            if isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)))

    def get_extra_modules(self, block):
        if self.kind == 'mixtral':                         # models/mixtral.py:38-41
            return {'block_sparse_moe': block.block_sparse_moe}
        if self.kind in ('qwen2moe', 'deepseek_v2'):       # models/qwen2moe.py:28-31, deepseekv2.py:26-29
            return {'mlp': block.mlp}
        return {}

    def get_subsets_in_block(self, block):
        if self.kind == 'mixtral':                         # models/mixtral.py:43-86
            a, moe = block.self_attn, block.block_sparse_moe
            ne = len(moe.experts)
            first = OrderedDict([(f'block_sparse_moe.experts.{i}.w1', moe.experts[i].w1) for i in range(ne)])
            first.update((f'block_sparse_moe.experts.{i}.w3', moe.experts[i].w3) for i in range(ne))
            first['block_sparse_moe.gate'] = moe.gate
            return [
                dict(layers=OrderedDict([('self_attn.q_proj', a.q_proj), ('self_attn.k_proj', a.k_proj),
                                         ('self_attn.v_proj', a.v_proj)]),
                     prev_op=[block.input_layernorm], input=['self_attn.q_proj'], inspect=a,
                     has_kwargs=True),
                dict(layers=OrderedDict([('self_attn.o_proj', a.o_proj)]), prev_op=[a.v_proj],
                     input=['self_attn.o_proj'], inspect=a.o_proj, has_kwargs=False),
                dict(layers=first, prev_op=[block.post_attention_layernorm], input=['block_sparse_moe'],
                     inspect=moe, has_kwargs=False, is_mlp=True),
                *[dict(layers=OrderedDict([(f'block_sparse_moe.experts.{i}.w2', moe.experts[i].w2)]),
                       prev_op=[moe.experts[i].w3], input=[f'block_sparse_moe.experts.{i}.w2'],
                       inspect=moe.experts[i].w2, has_kwargs=False, is_mlp=True) for i in range(ne)],
            ]
        if self.kind == 'qwen2moe':
            return self._qwen2moe_subsets(block)
        if self.kind == 'deepseek_v2':
            return self._deepseek_v2_subsets(block)
        if self.kind == 'llama':
            a, m = block.self_attn, block.mlp
            return [
                dict(layers=OrderedDict([('self_attn.q_proj', a.q_proj), ('self_attn.k_proj', a.k_proj),
                                         ('self_attn.v_proj', a.v_proj)]),
                     prev_op=[block.input_layernorm], input=['self_attn.q_proj'], inspect=a,
                     has_kwargs=True),
                dict(layers=OrderedDict([('self_attn.o_proj', a.o_proj)]), prev_op=[a.v_proj],
                     input=['self_attn.o_proj'], inspect=a.o_proj, has_kwargs=False),
                dict(layers=OrderedDict([('mlp.gate_proj', m.gate_proj), ('mlp.up_proj', m.up_proj)]),
                     prev_op=[block.post_attention_layernorm], input=['mlp.gate_proj'], inspect=m,
                     has_kwargs=False, is_mlp=True),
                dict(layers=OrderedDict([('mlp.down_proj', m.down_proj)]), prev_op=[m.up_proj],
                     input=['mlp.down_proj'], inspect=m.down_proj, has_kwargs=False, is_mlp=True),
            ]
        a = block.self_attn
        return [
            dict(layers=OrderedDict([('self_attn.q_proj', a.q_proj), ('self_attn.k_proj', a.k_proj),
                                     ('self_attn.v_proj', a.v_proj)]),
                 prev_op=[block.self_attn_layer_norm], input=['self_attn.q_proj'], inspect=a,
                 has_kwargs=True),
            dict(layers=OrderedDict([('self_attn.out_proj', a.out_proj)]), prev_op=[a.v_proj],
                 input=['self_attn.out_proj'], inspect=a.out_proj, has_kwargs=False),
            dict(layers=OrderedDict([('fc1', block.fc1)]), prev_op=[block.final_layer_norm],
                 input=['fc1'], inspect=block.fc1, has_kwargs=False, is_mlp=True),
            dict(layers=OrderedDict([('fc2', block.fc2)]), prev_op=[block.fc1], input=['fc2'],
                 inspect=block.fc2, has_kwargs=False, is_mlp=True),
        ]

    @staticmethod
    def _qwen2moe_subsets(block):
        """models/qwen2moe.py:51-116, its sparse branch (every layer here is sparse)."""
        a, moe = block.self_attn, block.mlp
        ne = len(moe.experts)
        first = OrderedDict([(f'mlp.experts.{i}.gate_proj', moe.experts[i].gate_proj) for i in range(ne)])  # :81-82
        first.update((f'mlp.experts.{i}.up_proj', moe.experts[i].up_proj) for i in range(ne))              # :83-84
        first['mlp.shared_expert.gate_proj'] = moe.shared_expert.gate_proj                                 # :85
        first['mlp.shared_expert.up_proj'] = moe.shared_expert.up_proj                                     # :86
        first['mlp.gate'] = moe.gate                                                                       # :87
        first['mlp.shared_expert_gate'] = moe.shared_expert_gate                                           # :88
        return [
            dict(layers=OrderedDict([('self_attn.q_proj', a.q_proj), ('self_attn.k_proj', a.k_proj),   # :53-65
                                     ('self_attn.v_proj', a.v_proj)]),
                 prev_op=[block.input_layernorm], input=['self_attn.q_proj'], inspect=a, has_kwargs=True),
            dict(layers=OrderedDict([('self_attn.o_proj', a.o_proj)]), prev_op=[a.v_proj],            # :67-75
                 input=['self_attn.o_proj'], inspect=a.o_proj, has_kwargs=False),
            dict(layers=first, prev_op=[block.post_attention_layernorm], input=['mlp'], inspect=moe,  # :78-96
                 has_kwargs=False, is_mlp=True),
            *[dict(layers=OrderedDict([(f'mlp.experts.{i}.down_proj', moe.experts[i].down_proj)]),   # :97-107
                   prev_op=[moe.experts[i].up_proj], input=[f'mlp.experts.{i}.down_proj'],
                   inspect=moe.experts[i].down_proj, has_kwargs=False, is_mlp=True) for i in range(ne)],
            dict(layers=OrderedDict([('mlp.shared_expert.down_proj', moe.shared_expert.down_proj)]),  # :108-116
                 prev_op=[moe.shared_expert.up_proj], input=['mlp.shared_expert.down_proj'],
                 inspect=moe.shared_expert.down_proj, has_kwargs=False),
        ]

    @staticmethod
    def _deepseek_v2_subsets(block):
        """models/deepseekv2.py:67-190: the q_proj branch (no q LoRA), then the MoE or the dense
        branch by whether the mlp has a router."""
        a, m = block.self_attn, block.mlp
        subsets = [
            dict(layers=OrderedDict([('self_attn.q_proj', a.q_proj),                                  # :69-81
                                     ('self_attn.kv_a_proj_with_mqa', a.kv_a_proj_with_mqa)]),
                 prev_op=[block.input_layernorm], input=['self_attn.q_proj'], inspect=a, has_kwargs=True),
            dict(layers=OrderedDict([('self_attn.o_proj', a.o_proj)]), prev_op=[None],               # :106-114
                 input=['self_attn.o_proj'], inspect=a.o_proj, has_kwargs=False),
            dict(layers=OrderedDict([('self_attn.kv_b_proj', a.kv_b_proj)]), prev_op=[a.kv_a_layernorm],  # :115-124
                 input=['self_attn.kv_b_proj'], inspect=a.kv_b_proj, has_kwargs=False, skip_rotate=True),
        ]
        if hasattr(m, 'gate'):
            ne = len(m.experts)
            first = OrderedDict([(f'mlp.experts.{i}.gate_proj', m.experts[i].gate_proj) for i in range(ne)])  # :130-131
            first.update((f'mlp.experts.{i}.up_proj', m.experts[i].up_proj) for i in range(ne))              # :132-133
            first['mlp.shared_experts.gate_proj'] = m.shared_experts.gate_proj                                # :134
            first['mlp.shared_experts.up_proj'] = m.shared_experts.up_proj                                    # :135
            first['mlp.gate'] = m.gate                                                                        # :136
            subsets += [
                dict(layers=first, prev_op=[block.post_attention_layernorm], input=['mlp'], inspect=m,   # :126-144
                     has_kwargs=False, is_mlp=True),
                *[dict(layers=OrderedDict([(f'mlp.experts.{i}.down_proj', m.experts[i].down_proj)]),      # :145-155
                       prev_op=[m.experts[i].up_proj], input=[f'mlp.experts.{i}.down_proj'],
                       inspect=m.experts[i].down_proj, has_kwargs=False, is_mlp=True) for i in range(ne)],
                dict(layers=OrderedDict([('mlp.shared_experts.down_proj', m.shared_experts.down_proj)]),  # :157-165
                     prev_op=[m.shared_experts.up_proj], input=['mlp.shared_experts.down_proj'],
                     inspect=m.shared_experts.down_proj, has_kwargs=False),
            ]
        else:
            subsets += [
                dict(layers=OrderedDict([('mlp.gate_proj', m.gate_proj), ('mlp.up_proj', m.up_proj)]),   # :167-178
                     prev_op=[block.post_attention_layernorm], input=['mlp.gate_proj'], inspect=m,
                     has_kwargs=False),
                dict(layers=OrderedDict([('mlp.down_proj', m.down_proj)]), prev_op=[m.up_proj],          # :180-188
                     input=['mlp.down_proj'], inspect=m.down_proj, has_kwargs=False),
            ]
        return subsets

    def _rope(self, seq_len, device):
        if self.kind == 'deepseek_v2':
            return mla_rope_cos_sin(seq_len, self.shape['rope_dim'], device, self.shape['rope_theta'])
        hd = self.shape['hidden'] // self.shape['heads']
        return rope_cos_sin(seq_len, hd, device, self.torch_dtype, theta=self.shape.get('rope_theta', 500000.0))

    # ---- first block input (base_model.py:264-321 Catcher), synthetic tokens ----------------------
    @torch.no_grad()
    def first_block_input(self, n_samples, seq_len, bs=1, seed=1, device='cuda', ids=None):
        """`ids` [n_samples, seq_len]: calibration token ids (default: uniform random, `seed`)."""
        if ids is None:
            g = torch.Generator().manual_seed(seed)
            ids = torch.randint(0, self.shape['vocab'], (n_samples, seq_len), generator=g)
        n_samples, seq_len = ids.shape
        emb = self.model.embed_tokens
        data, kwargs = [], []
        step = n_samples if bs == -1 else bs
        kw = {}
        if self.kind in ('llama', 'mixtral', 'qwen2moe', 'deepseek_v2'):
            kw['position_embeddings'] = self._rope(seq_len, device)
        for i in range(0, n_samples, step):
            x = emb(ids[i:i + step].to(emb.weight.device)).to(device)
            if self.kind == 'opt':
                pos = torch.arange(seq_len, device=device)
                # learned positions replaced by a fixed sinusoid of the same scale (synthetic)
                x = x + 0.02 * torch.sin(pos[None, :, None] * 0.01 +
                                         torch.arange(x.shape[-1], device=device)[None, None, :]).to(x.dtype)
            data.append(x)
            kwargs.append(dict(kw))
        return {'data': data, 'kwargs': kwargs}

    # ---- module replacement (base_model.py:386-455) -------------------------------------------------
    @staticmethod
    def _set(block, name, new):
        parent = block
        parts = name.split('.')
        for p in parts[:-1]:
            parent = getattr(parent, p)
        setattr(parent, parts[-1], new)

    def replace_module_subset(self, module_cls, block, subset, block_idx, params_dict):
        for name, m in list(subset['layers'].items()):
            if getattr(m, 'no_quant', False):
                continue
            if not isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                continue                                   # DeepseekV2Gate: a subset member, not a linear
            if isinstance(m, module_cls):
                continue
            new = module_cls.new(m, **params_dict)
            self._set(block, name, new)
            subset['layers'][name] = new

    def replace_module_block(self, module_cls, block, block_idx, params_dict):
        for name, m in list(self.get_block_linears(block).items()):
            if getattr(m, 'no_quant', False):
                continue
            self._set(block, name, module_cls.new(m, **params_dict))

    def replace_language_module_all(self, module_cls, params_dict, keep_device=False):
        for i, block in enumerate(self.get_blocks()):
            self.replace_module_block(module_cls, block, i, params_dict)

    def convert_dtype(self, dtype):
        for b in self.get_blocks():
            for m in b.modules():
                if getattr(m, 'packed', False):
                    # EffcientFakeQuantLinear on packed codes: `.weight` is computed from the codes
                    # in the model dtype already, and its qparams (fp32 for GPTQ's dynamic groups)
                    # must keep their dtype
                    continue
                if isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                    if getattr(m, 'weight', None) is not None and m.weight.is_floating_point():
                        m.weight.data = m.weight.data.to(dtype)

    # ---- PPL (eval/eval_ppl.py:15-58) ---------------------------------------------------------------
    @torch.no_grad()
    def logits(self, ids, device='cuda'):
        m = self.model
        x = m.embed_tokens(ids.to(m.embed_tokens.weight.device)).to(device)
        kw = {}
        if self.kind in ('llama', 'mixtral', 'qwen2moe', 'deepseek_v2'):
            kw['position_embeddings'] = self._rope(ids.shape[1], device)
        for b in m.layers:
            x = b(x, **kw)
        x = m.norm(x)
        return F.linear(x, m.lm_head.weight.to(device))


@torch.no_grad()
def perplexity(model, tokens, seq_len, bs=1, device='cuda', ce_dtype=None):
    """eval/eval_ppl.py:15-58: mean-CE per batch x seq_len*(j-i); exp(sum / (nsamples*seq_len)).
    Like the reference, the cross entropy is taken on the logits in the MODEL dtype (`:38-43`; for a
    bf16 model each batch loss is therefore a bf16 number and the PPL moves in steps of ~0.4 %);
    ce_dtype=torch.float32 evaluates it in fp32 instead."""
    nsamples = tokens.numel() // seq_len
    tokens = tokens[:, : nsamples * seq_len]
    nlls = []
    for i in range(0, nsamples, bs):
        j = min(i + bs, nsamples)
        inputs = tokens[:, i * seq_len: j * seq_len].view(j - i, seq_len)
        lg = model.logits(inputs, device=device)
        if ce_dtype is not None:
            lg = lg.to(ce_dtype)
        shift_logits = lg[:, :-1, :].contiguous()
        shift_labels = inputs[:, 1:].to(device)
        loss = F.cross_entropy(shift_logits.view(-1, shift_logits.size(-1)), shift_labels.reshape(-1))
        nlls.append(loss.float() * seq_len * (j - i))
    return math.exp(torch.stack(nlls).sum().item() / (nsamples * seq_len))
