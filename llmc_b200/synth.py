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

import torch
import torch.nn as nn
import torch.nn.functional as F

from .module_utils import _LLMC_LINEAR_TYPES_, _TRANSFORMERS_LINEAR_TYPES_, linear_forward

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
    def __init__(self, hidden, heads, kv_heads):
        super().__init__()
        self.heads, self.kv_heads, self.head_dim = heads, kv_heads, hidden // heads
        self.q_proj = B200Linear(hidden, heads * self.head_dim, bias=False)
        self.k_proj = B200Linear(hidden, kv_heads * self.head_dim, bias=False)
        self.v_proj = B200Linear(hidden, kv_heads * self.head_dim, bias=False)
        self.o_proj = B200Linear(heads * self.head_dim, hidden, bias=False)

    def attend(self, q, k, v, position_embeddings):
        B, S, _ = q.shape
        cos, sin = position_embeddings
        fused = (q.is_cuda and self.head_dim % 16 == 0 and q.is_contiguous() and k.is_contiguous()
                 and cos.dtype == q.dtype and cos.shape[0] >= S)
        if fused:                        # rotary in place on the fresh projection outputs
            from . import block_ops
            block_ops.rope_(q, cos[:S], sin[:S], self.heads, self.head_dim)
            block_ops.rope_(k, cos[:S], sin[:S], self.kv_heads, self.head_dim)
        q = q.view(B, S, self.heads, self.head_dim).transpose(1, 2)
        k = k.view(B, S, self.kv_heads, self.head_dim).transpose(1, 2)
        v = v.view(B, S, self.kv_heads, self.head_dim).transpose(1, 2)
        if not fused:
            cos, sin = cos[None, None, :S], sin[None, None, :S]
            q = q * cos + _rot_half(q) * sin
            k = k * cos + _rot_half(k) * sin
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True,
                                           enable_gqa=self.kv_heads != self.heads)
        return o.transpose(1, 2).reshape(B, S, self.heads * self.head_dim)

    def forward(self, hidden_states, position_embeddings=None, **kw):
        q, k, v = self.q_proj(hidden_states), self.k_proj(hidden_states), self.v_proj(hidden_states)
        return self.o_proj(self.attend(q, k, v, position_embeddings))


class LlamaMLP(nn.Module):
    def __init__(self, hidden, inter):
        super().__init__()
        self.gate_proj = B200Linear(hidden, inter, bias=False)
        self.up_proj = B200Linear(hidden, inter, bias=False)
        self.down_proj = B200Linear(inter, hidden, bias=False)

    def act(self, g, u, out=None):
        if g.is_cuda and g.is_contiguous() and u.is_contiguous() and g.numel() % 8 == 0:
            from . import block_ops
            return block_ops.silu_mul(g, u, out=out)
        y = F.silu(g) * u
        if out is not None:
            out.copy_(y)
            return out
        return y

    def forward(self, x):
        return self.down_proj(self.act(self.gate_proj(x), self.up_proj(x)))


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


class MixtralSparseMoe(nn.Module):
    """Per-expert nn.Linear layout the reference's wrapper expects (models/mixtral.py:43-86:
    block_sparse_moe.gate / experts[i].w1|w2|w3); the installed transformers 5.x fuses the experts,
    so the shape model is restated here (SURVEY.md §7.3 item 8).  Hooks on an expert only ever see
    the tokens routed to it (Appendix E-11)."""

    def __init__(self, hidden, inter, experts, top_k):
        super().__init__()
        self.top_k = top_k
        self.gate = nn.Linear(hidden, experts, bias=False)
        self.experts = nn.ModuleList([MixtralExpert(hidden, inter) for _ in range(experts)])

    def forward(self, hidden_states):
        B, S, H = hidden_states.shape
        x = hidden_states.reshape(-1, H)
        logits = self.gate(x)                      # module call: hooks / FakeQuantLinear see it
        w = F.softmax(logits, dim=1, dtype=torch.float)
        w, sel = torch.topk(w, self.top_k, dim=-1)
        w = (w / w.sum(dim=-1, keepdim=True)).to(x.dtype)
        out = torch.zeros_like(x)
        for e, expert in enumerate(self.experts):
            tok, slot = torch.where(sel == e)
            if tok.numel() == 0:
                continue
            out.index_add_(0, tok, expert(x[tok]) * w[tok, slot, None])
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
                'opt': ('OPTForCausalLM', 'opt')}[self.kind]
        doc = {'architectures': [arch[0]], 'model_type': arch[1], 'hidden_size': s['hidden'],
               'num_hidden_layers': len(self.model.layers), 'num_attention_heads': s['heads'],
               'vocab_size': s['vocab'], 'torch_dtype': str(self.torch_dtype).replace('torch.', '')}
        if self.kind == 'opt':
            doc['ffn_dim'] = s['inter']
        else:
            doc.update({'intermediate_size': s['inter'], 'num_key_value_heads': s['kv_heads']})
        if self.kind == 'mixtral':
            doc.update({'num_local_experts': s['experts'], 'num_experts_per_tok': s['top_k']})
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
        if self.kind in ('llama', 'mixtral'):
            hd = self.shape['hidden'] // self.shape['heads']
            kw['position_embeddings'] = rope_cos_sin(seq_len, hd, device, self.torch_dtype)
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
                if isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                    if getattr(m, 'weight', None) is not None and m.weight.is_floating_point():
                        m.weight.data = m.weight.data.to(dtype)

    # ---- PPL (eval/eval_ppl.py:15-58) ---------------------------------------------------------------
    @torch.no_grad()
    def logits(self, ids, device='cuda'):
        m = self.model
        x = m.embed_tokens(ids.to(m.embed_tokens.weight.device)).to(device)
        kw = {}
        if self.kind in ('llama', 'mixtral'):
            hd = self.shape['hidden'] // self.shape['heads']
            kw['position_embeddings'] = rope_cos_sin(ids.shape[1], hd, device, self.torch_dtype)
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
