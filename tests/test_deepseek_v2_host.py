"""CPU: the DeepSeek-V2 shape model against transformers' modules (the golden fixture written by
oracle/gen_deepseek_v2_golden.py), its wrapper surface (subsets as the reference's
models/deepseekv2.py declares them, the router a subset member but not a block linear, one GPTQ
Hessian per expert linear), the refusals of what is not built, and what the MLA GEMMs and
llmc_moe_combine_weighted refuse before any CUDA call."""
import ctypes
import os

import pytest
import torch

from llmc_b200 import _lib, synth
from llmc_b200.synth import (DeepseekV2Attention, DeepseekV2Block, DeepseekV2Gate, DeepseekV2SparseMoe,
                             LlamaMLP, mla_rope_cos_sin)

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'deepseek_v2_kat.pt')


def _model(n_layers=None):
    return synth.SynthModel('tiny-deepseek-v2', n_layers=n_layers, seed=0)


@pytest.fixture(scope='module')
def golden():
    g = torch.load(GOLDEN)
    m = _model()
    digest = {n: float(p.detach().double().sum()) for n, p in m.model.layers.named_parameters()}
    assert digest == g['weights'], 'the seeded shape-model weights differ from the fixture\'s'
    return g, m


def test_shapes():
    s = synth.SHAPES['deepseek-v2-lite']
    assert (s['hidden'], s['inter'], s['moe_inter'], s['layers'], s['heads'], s['vocab'], s['dtype']) == (
        2048, 10944, 1408, 27, 16, 102400, torch.bfloat16)
    assert (s['kv_lora'], s['rope_dim'], s['nope_dim'], s['v_dim']) == (512, 64, 128, 128)
    assert (s['experts'], s['top_k'], s['shared_experts'], s['first_k_dense']) == (64, 6, 2, 1)
    assert (s['rope_theta'], s['routed_scale'], s['rms_eps']) == (10000.0, 1.0, 1e-6)
    assert s['experts'] <= _lib.MOE_MAX_EXPERTS
    t = synth.SHAPES['tiny-deepseek-v2']
    assert t['kind'] == 'deepseek_v2' and t['layers'] == 2 and t['first_k_dense'] == 1
    assert (t['hidden'], t['heads'], t['kv_lora'], t['experts'], t['top_k'], t['moe_inter']) == (
        256, 4, 128, 12, 6, 128)
    assert t['routed_scale'] != 1.0


def test_block_structure():
    m = _model()
    dense, sparse = m.get_blocks()
    assert isinstance(dense, DeepseekV2Block) and type(dense.mlp) is LlamaMLP
    assert dense.mlp.gate_proj.out_features == 512
    moe = sparse.mlp
    assert isinstance(moe, DeepseekV2SparseMoe) and len(moe.experts) == 12 and moe.top_k == 6
    assert all(type(e) is LlamaMLP and e.gate_proj.out_features == 128 for e in moe.experts)
    assert type(moe.shared_experts) is LlamaMLP and moe.shared_experts.gate_proj.out_features == 256
    assert type(moe.gate) is DeepseekV2Gate and not isinstance(moe.gate, torch.nn.Linear)
    assert tuple(moe.gate.weight.shape) == (12, 256)
    a = sparse.self_attn
    assert isinstance(a, DeepseekV2Attention) and not hasattr(a, 'qkv_rope')
    assert (a.q_proj.out_features, a.kv_a_proj_with_mqa.out_features, a.kv_b_proj.out_features,
            a.o_proj.in_features) == (4 * 192, 128 + 64, 4 * 256, 4 * 128)
    assert a.kv_a_layernorm.variance_epsilon == 1e-6 and sparse.input_layernorm.variance_epsilon == 1e-6
    assert all(lin.bias is None for lin in (a.q_proj, a.kv_a_proj_with_mqa, a.kv_b_proj, a.o_proj))
    assert m.get_extra_modules(sparse) == {'mlp': moe} and m.get_extra_modules(dense) == {'mlp': dense.mlp}
    cfg = m.hf_config_dict()
    assert cfg['model_type'] == 'deepseek_v2' and cfg['architectures'] == ['DeepseekV2ForCausalLM']
    assert (cfg['n_routed_experts'], cfg['n_shared_experts'], cfg['num_experts_per_tok']) == (12, 2, 6)
    assert (cfg['kv_lora_rank'], cfg['q_lora_rank'], cfg['qk_rope_head_dim'], cfg['qk_nope_head_dim'],
            cfg['v_head_dim']) == (128, None, 64, 128, 128)
    assert cfg['first_k_dense_replace'] == 1 and cfg['routed_scaling_factor'] == 1.5
    assert cfg['topk_method'] == 'greedy' and cfg['moe_intermediate_size'] == 128
    inp = m.first_block_input(1, 16, device='cpu')
    cos, sin = inp['kwargs'][0]['position_embeddings']
    assert cos.dtype == sin.dtype == torch.float32 and tuple(cos.shape) == (16, 32)


def _check_attn_subsets(subs, blk):
    a = blk.self_attn
    q, o, kvb = subs[:3]
    assert list(q['layers']) == ['self_attn.q_proj', 'self_attn.kv_a_proj_with_mqa']
    assert q['prev_op'] == [blk.input_layernorm] and q['input'] == ['self_attn.q_proj']
    assert q['inspect'] is a and q['has_kwargs'] is True and 'is_mlp' not in q
    assert list(o['layers']) == ['self_attn.o_proj'] and o['prev_op'] == [None]
    assert o['input'] == ['self_attn.o_proj'] and o['inspect'] is a.o_proj and o['has_kwargs'] is False
    assert list(kvb['layers']) == ['self_attn.kv_b_proj'] and kvb['prev_op'] == [a.kv_a_layernorm]
    assert kvb['input'] == ['self_attn.kv_b_proj'] and kvb['inspect'] is a.kv_b_proj
    assert kvb['has_kwargs'] is False and kvb['skip_rotate'] is True


def test_subsets_match_the_reference_wrapper():
    """models/deepseekv2.py:67-190: the q_proj branch, then the MoE branch or the dense one."""
    m = _model()
    dense, blk = m.get_blocks()
    moe = blk.mlp
    ne = len(moe.experts)
    subs = m.get_subsets_in_block(blk)
    assert len(subs) == 3 + 1 + ne + 1
    _check_attn_subsets(subs, blk)
    first, *downs, shared_down = subs[3:]
    want = ([f'mlp.experts.{i}.gate_proj' for i in range(ne)] + [f'mlp.experts.{i}.up_proj' for i in range(ne)]
            + ['mlp.shared_experts.gate_proj', 'mlp.shared_experts.up_proj', 'mlp.gate'])
    assert list(first['layers']) == want
    assert first['layers']['mlp.gate'] is moe.gate
    assert first['layers']['mlp.experts.5.up_proj'] is moe.experts[5].up_proj
    assert first['prev_op'] == [blk.post_attention_layernorm] and first['input'] == ['mlp']
    assert first['inspect'] is moe and first['has_kwargs'] is False and first['is_mlp'] is True
    for i, d in enumerate(downs):
        assert list(d['layers']) == [f'mlp.experts.{i}.down_proj']
        assert d['prev_op'] == [moe.experts[i].up_proj] and d['input'] == [f'mlp.experts.{i}.down_proj']
        assert d['inspect'] is moe.experts[i].down_proj and d['has_kwargs'] is False and d['is_mlp'] is True
    assert list(shared_down['layers']) == ['mlp.shared_experts.down_proj']
    assert shared_down['prev_op'] == [moe.shared_experts.up_proj]
    assert shared_down['input'] == ['mlp.shared_experts.down_proj']
    assert shared_down['inspect'] is moe.shared_experts.down_proj and 'is_mlp' not in shared_down
    # the dense branch
    dsubs = m.get_subsets_in_block(dense)
    assert len(dsubs) == 5
    _check_attn_subsets(dsubs, dense)
    gu, down = dsubs[3:]
    assert list(gu['layers']) == ['mlp.gate_proj', 'mlp.up_proj'] and gu['input'] == ['mlp.gate_proj']
    assert gu['prev_op'] == [dense.post_attention_layernorm] and gu['inspect'] is dense.mlp
    assert 'is_mlp' not in gu and gu['has_kwargs'] is False
    assert list(down['layers']) == ['mlp.down_proj'] and down['prev_op'] == [dense.mlp.up_proj]
    assert down['inspect'] is dense.mlp.down_proj and 'is_mlp' not in down


def test_router_is_a_subset_member_but_not_a_block_linear():
    m = _model()
    blk = m.get_blocks()[1]
    linears = m.get_block_linears(blk)
    assert 'mlp.gate' not in linears
    for s in m.get_subsets_in_block(blk):
        for n, lin in s['layers'].items():
            assert n == 'mlp.gate' or linears[n] is lin
    # no deploy replaces it: neither the block replacement nor the subset replacement
    from llmc_b200.module_utils import OriginFloatLinear
    first = m.get_subsets_in_block(blk)[3]
    m.replace_module_subset(OriginFloatLinear, blk, first, 1, {})
    assert type(blk.mlp.gate) is DeepseekV2Gate and first['layers']['mlp.gate'] is blk.mlp.gate
    assert type(blk.mlp.experts[0].gate_proj) is OriginFloatLinear
    m.replace_module_block(OriginFloatLinear, blk, 1, {})
    assert type(blk.mlp.gate) is DeepseekV2Gate


def test_gptq_hessians_are_per_expert_and_skip_the_router():
    from llmc_b200.gptq import GPTQ
    m = _model()
    blk = m.get_blocks()[1]
    subs = m.get_subsets_in_block(blk)
    linears = m.get_block_linears(blk)
    algo = object.__new__(GPTQ)
    algo.layers_cache, algo.dev = {}, torch.device('cpu')
    algo._init_layers(linears, subs)
    share = {n: c['share'] for n, c in algo.layers_cache.items()}
    assert share['self_attn.kv_a_proj_with_mqa'] == 'self_attn.q_proj'
    experts = [n for n in subs[3]['layers'] if n != 'mlp.gate']
    for n in experts:
        assert share[n] == n and algo.layers_cache[n]['H'].shape[0] == linears[n].in_features
    hs = [algo.layers_cache[n]['H'] for n in experts]
    assert len({h.data_ptr() for h in hs}) == len(hs)
    # a subset's own initialisation (true_sequential) gives the router no Hessian
    algo.layers_cache = {}
    algo.subset_init(subs[3])
    assert 'mlp.gate' not in algo.layers_cache and set(algo.layers_cache) == set(experts)


def test_attention_equals_transformers(golden):
    g, m = golden
    a = m.get_blocks()[1].self_attn
    with torch.no_grad():
        out = a(g['x'], position_embeddings=(g['cos'], g['sin']))
    assert torch.equal(out, g['attn'])


def test_rope_tables_equal_freqs_cis(golden):
    g, _ = golden
    cos, sin = mla_rope_cos_sin(g['x'].shape[1], 64, 'cpu', 10000.0)
    assert torch.equal(cos, g['cos']) and torch.equal(sin, g['sin'])


def test_router_equals_transformers(golden):
    g, m = golden
    moe = m.get_blocks()[1].mlp
    x = g['x'].reshape(-1, g['x'].shape[-1])
    with torch.no_grad():
        sel, w = moe.route(x)
    assert w.dtype == torch.float32
    # greedy unsorted top-k: the same set per token with the same weight per expert
    o, og = sel.argsort(1), g['sel'].argsort(1)
    assert torch.equal(sel.gather(1, o), g['sel'].gather(1, og))
    assert torch.equal(w.gather(1, o), g['w'].gather(1, og))


def test_moe_loop_equals_transformers(golden):
    g, m = golden
    moe = m.get_blocks()[1].mlp
    with torch.no_grad():
        assert torch.equal(moe(g['x']), g['moe'])


@pytest.mark.parametrize('layer', [0, 1])
def test_decoder_layer_equals_transformers(golden, layer):
    """Every op of the layer is bit for bit on this fixture, including apply_rotary_emb: torch's
    complex64 product on the CPU equals mla_rotate's real restatement on its vectorised path."""
    g, m = golden
    blk = m.get_blocks()[layer]
    with torch.no_grad():
        out = blk(g['x'], position_embeddings=(g['cos'], g['sin']))
    assert torch.equal(out, g[f'layer{layer}'])


def test_refusals_of_what_is_not_built():
    with pytest.raises(NotImplementedError, match='q_lora_rank'):
        DeepseekV2Attention(256, 4, 128, q_lora_rank=1536)
    with pytest.raises(NotImplementedError, match='group_limited_greedy'):
        DeepseekV2SparseMoe(256, 128, 12, 6, 2, 1.0, topk_method='group_limited_greedy')
    s = dict(synth.SHAPES['tiny-deepseek-v2'], q_lora_rank=1536)
    with pytest.raises(NotImplementedError):
        DeepseekV2Block(s, 0)


def _last(lib):
    return lib.llmc_b200_last_error().decode()


def test_combine_weighted_refusals_without_gpu():
    lib = _lib.load()
    fn = lib.llmc_moe_combine_weighted
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    BF16 = _lib.BF16
    # scalars first, refused even when there are no tokens
    assert fn(p, p, p, p, p, -1, 6, 256, BF16, null) == -1
    assert fn(p, p, p, p, p, 16, 0, 256, BF16, null) == -1
    assert fn(p, p, p, p, p, 16, 6, 0, BF16, null) == -1
    assert 'bad shape' in _last(lib)
    assert fn(null, null, null, null, null, 0, 6, 256, _lib.F32, null) == -1
    assert 'dtype must be bf16 or fp16' in _last(lib)
    assert fn(null, null, null, null, null, 0, 6, 100, BF16, null) == -4
    assert 'N=100' in _last(lib)
    # no tokens: a no-op that touches no pointer
    assert fn(null, null, null, null, null, 0, 6, 256, BF16, null) == 0
    assert fn(null, null, null, null, null, 0, 6, 256, _lib.F16, null) == 0
    # then the pointers: nulls (the shared output is required), 16-byte alignment
    for i in range(5):
        args = [p] * 5
        args[i] = null
        assert fn(*args, 16, 6, 256, BF16, null) == -1
        assert 'null pointer' in _last(lib)
    for i in (0, 3, 4):                      # y, shared, out; w is read per row
        args = [p] * 5
        args[i] = ctypes.c_void_p(258)
        assert fn(*args, 16, 6, 256, BF16, null) == -4
        assert '16-byte aligned' in _last(lib)


def test_down_entry_points_refuse_a_null_route_weight():
    """The weighted path feeds the four down launches unit weights; none accepts a missing one."""
    lib = _lib.load()
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    arr = (ctypes.c_void_p * 1)(256)
    BF16 = _lib.BF16
    assert lib.llmc_moe_gemm_down(p, arr, p, null, p, 128, 256, 128, 1, BF16, null) == -1
    assert lib.llmc_moe_gemm_packed_down(p, 4, arr, arr, None, None, BF16, 64, 2, p, null, p, 128, 256, 128, 1,
                                         BF16, null) == -1
    assert lib.llmc_moe_gemm_fp8a16_down(p, 0, arr, arr, None, BF16, 64, 2, p, null, p, 128, 256, 128, 1,
                                         BF16, null) == -1
    assert lib.llmc_moe_gemm_w8a8_down(p, p, 0, arr, arr, 1, p, null, p, 128, 256, 128, 1, BF16, null) == -1


def test_mla_qkv_refusals_without_gpu():
    lib = _lib.load()
    fn = lib.llmc_gemm_mla_qkv
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    BF16 = _lib.BF16
    # (x, w, q, k, latent, cos, sin, M, heads, kv_lora, K, seq)
    assert fn(p, p, p, p, p, p, p, 128, 6, 128, 256, 64, BF16, null) == -1
    assert 'heads=6' in _last(lib)
    assert fn(p, p, p, p, p, p, p, 128, 0, 128, 256, 64, BF16, null) == -1
    assert fn(p, p, p, p, p, p, p, 128, 4, 100, 256, 64, BF16, null) == -1
    assert 'kv_lora=100' in _last(lib)
    assert fn(p, p, p, p, p, p, p, 128, 4, 128, 256, 0, BF16, null) == -1
    assert fn(p, p, p, p, p, p, p, 100, 4, 128, 256, 64, BF16, null) == -1
    assert 'multiple of seq' in _last(lib)
    for i in (3, 4, 5, 6):                           # k, latent, cos, sin
        args = [p] * 7
        args[i] = null
        assert fn(*args, 128, 4, 128, 256, 64, BF16, null) == -1
        assert 'null pointer' in _last(lib)
        args[i] = ctypes.c_void_p(260)
        assert fn(*args, 128, 4, 128, 256, 64, BF16, null) == -4
        assert '16-byte aligned' in _last(lib)
    # then the GEMM's own checks: no rows is a no-op, nulls, dtype, K and alignment
    assert fn(null, null, null, p, p, p, p, 0, 4, 128, 256, 64, BF16, null) == 0
    assert fn(null, p, p, p, p, p, p, 128, 4, 128, 256, 64, BF16, null) == -1
    assert fn(p, p, p, p, p, p, p, 128, 4, 128, 256, 64, _lib.F32, null) == -1
    assert fn(p, p, p, p, p, p, p, 128, 4, 128, 250, 64, BF16, null) == -4


def test_mla_kv_b_refusals_without_gpu():
    lib = _lib.load()
    fn = lib.llmc_gemm_mla_kv_b
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    BF16 = _lib.BF16
    # (x, w, k, v, M, heads, K)
    assert fn(p, p, p, p, 128, 0, 128, BF16, null) == -1
    assert 'heads=0' in _last(lib)
    assert fn(p, p, p, null, 128, 4, 128, BF16, null) == -1
    assert 'null pointer' in _last(lib)
    assert fn(p, p, p, ctypes.c_void_p(260), 128, 4, 128, BF16, null) == -4
    assert fn(null, null, null, p, 0, 4, 128, BF16, null) == 0
    assert fn(p, p, null, p, 128, 4, 128, BF16, null) == -1
    assert fn(p, p, p, p, 128, 4, 128, _lib.F32, null) == -1
    assert fn(p, p, p, p, 128, 4, 100, BF16, null) == -4


@pytest.mark.parametrize('name', ['deepseek-v2-lite', 'tiny-deepseek-v2'])
def test_main_accepts_the_shapes(name):
    from llmc_b200.__main__ import adapt_reference_config
    cfg = adapt_reference_config({'model': {'type': 'DeepseekV2'}, 'quant': {'method': 'RTN'}}, name)
    assert cfg['model'] == {'type': 'DeepseekV2', 'path': f'synthetic:{name}'}
