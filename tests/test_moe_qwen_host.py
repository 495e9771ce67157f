"""CPU: the Qwen2-MoE shape model's wrapper surface (subsets as the reference's models/qwen2moe.py
declares them, one GPTQ Hessian per expert linear) and what llmc_moe_combine_shared refuses before
any CUDA call."""
import ctypes

import pytest
import torch

from llmc_b200 import _lib, synth
from llmc_b200.synth import LlamaMLP, Qwen2MoeBlock, Qwen2MoeSparseMoe


def _model(name='tiny-qwen-moe'):
    return synth.SynthModel(name, n_layers=1)


def test_shapes():
    s = synth.SHAPES['qwen1.5-moe-a2.7b']
    assert (s['hidden'], s['layers'], s['heads'], s['kv_heads'], s['vocab'], s['dtype']) == (
        2048, 24, 16, 16, 151936, torch.bfloat16)
    assert (s['experts'], s['top_k'], s['moe_inter'], s['shared_inter']) == (60, 4, 1408, 5632)
    t = synth.SHAPES['tiny-qwen-moe']
    assert t['experts'] > 8 and t['kind'] == 'qwen2moe'


def test_block_structure():
    m = _model()
    blk = m.get_blocks()[0]
    assert isinstance(blk, Qwen2MoeBlock) and isinstance(blk.mlp, Qwen2MoeSparseMoe)
    moe = blk.mlp
    assert len(moe.experts) == 12 and moe.top_k == 4 and not moe.norm_topk_prob
    assert all(type(e) is LlamaMLP for e in moe.experts) and type(moe.shared_expert) is LlamaMLP
    assert moe.shared_expert_gate.out_features == 1 and moe.shared_expert_gate.bias is None
    assert moe.gate.out_features == 12 and moe.gate.bias is None
    a = blk.self_attn
    assert all(lin.bias is not None for lin in (a.q_proj, a.k_proj, a.v_proj)) and a.o_proj.bias is None
    assert m.get_extra_modules(blk) == {'mlp': moe}
    cfg = m.hf_config_dict()
    assert cfg['model_type'] == 'qwen2_moe' and cfg['num_experts'] == 12 and cfg['norm_topk_prob'] is False


def test_subsets_match_the_reference_wrapper():
    """models/qwen2moe.py:51-116 (sparse branch)."""
    m = _model()
    blk = m.get_blocks()[0]
    a, moe = blk.self_attn, blk.mlp
    ne = len(moe.experts)
    subs = m.get_subsets_in_block(blk)
    assert len(subs) == 3 + ne + 1
    qkv, o, first, *downs, shared_down = subs
    assert list(qkv['layers']) == ['self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj']
    assert qkv['prev_op'] == [blk.input_layernorm] and qkv['input'] == ['self_attn.q_proj']
    assert qkv['inspect'] is a and qkv['has_kwargs'] is True and 'is_mlp' not in qkv
    assert list(o['layers']) == ['self_attn.o_proj'] and o['prev_op'] == [a.v_proj]
    assert o['input'] == ['self_attn.o_proj'] and o['inspect'] is a.o_proj and o['has_kwargs'] is False
    want = ([f'mlp.experts.{i}.gate_proj' for i in range(ne)] + [f'mlp.experts.{i}.up_proj' for i in range(ne)]
            + ['mlp.shared_expert.gate_proj', 'mlp.shared_expert.up_proj', 'mlp.gate', 'mlp.shared_expert_gate'])
    assert list(first['layers']) == want
    assert first['layers']['mlp.gate'] is moe.gate
    assert first['layers']['mlp.shared_expert_gate'] is moe.shared_expert_gate
    assert first['layers']['mlp.experts.3.up_proj'] is moe.experts[3].up_proj
    assert first['prev_op'] == [blk.post_attention_layernorm] and first['input'] == ['mlp']
    assert first['inspect'] is moe and first['has_kwargs'] is False and first['is_mlp'] is True
    for i, d in enumerate(downs):
        assert list(d['layers']) == [f'mlp.experts.{i}.down_proj']
        assert d['prev_op'] == [moe.experts[i].up_proj] and d['input'] == [f'mlp.experts.{i}.down_proj']
        assert d['inspect'] is moe.experts[i].down_proj and d['has_kwargs'] is False and d['is_mlp'] is True
    assert list(shared_down['layers']) == ['mlp.shared_expert.down_proj']
    assert shared_down['prev_op'] == [moe.shared_expert.up_proj]
    assert shared_down['input'] == ['mlp.shared_expert.down_proj']
    assert shared_down['inspect'] is moe.shared_expert.down_proj and shared_down['has_kwargs'] is False
    assert 'is_mlp' not in shared_down
    # every subset linear is a block linear under the same name
    linears = m.get_block_linears(blk)
    for s in subs:
        for n, lin in s['layers'].items():
            assert linears[n] is lin


def test_gptq_hessians_are_not_shared_across_experts():
    from llmc_b200.gptq import GPTQ
    m = _model()
    blk = m.get_blocks()[0]
    subs = m.get_subsets_in_block(blk)
    linears = m.get_block_linears(blk)
    algo = object.__new__(GPTQ)
    algo.layers_cache, algo.dev = {}, torch.device('cpu')
    algo._init_layers(linears, subs)
    share = {n: c['share'] for n, c in algo.layers_cache.items()}
    assert share['self_attn.k_proj'] == share['self_attn.v_proj'] == 'self_attn.q_proj'
    for n in subs[2]['layers']:
        assert share[n] == n and algo.layers_cache[n]['H'].shape[0] == linears[n].in_features
    for s in subs[3:]:
        (n,) = s['layers']
        assert share[n] == n
    hs = [algo.layers_cache[n]['H'] for n in subs[2]['layers']]
    assert len({h.data_ptr() for h in hs}) == len(hs)


def test_router_does_not_renormalise():
    torch.manual_seed(0)
    moe = Qwen2MoeSparseMoe(64, 128, 128, 12, 4)
    x = torch.randn(10, 64)
    sel, w = moe.route(x)
    p = torch.softmax(moe.gate(x).float(), dim=1)
    assert torch.equal(w, torch.gather(p, 1, sel).to(x.dtype))
    assert (w.sum(dim=1) < 1).all()


def test_combine_shared_refusals_without_gpu():
    lib = _lib.load()
    fn = lib.llmc_moe_combine_shared
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    BF16 = _lib.BF16

    def last():
        return lib.llmc_b200_last_error().decode()

    # scalars first, refused even when there are no tokens
    assert fn(p, p, p, p, p, -1, 4, 256, BF16, null) == -1
    assert fn(p, p, p, p, p, 16, 0, 256, BF16, null) == -1
    assert fn(p, p, p, p, p, 16, 4, 0, BF16, null) == -1
    assert 'bad shape' in last()
    assert fn(null, null, null, null, null, 0, 4, 256, _lib.F32, null) == -1
    assert 'dtype must be bf16 or fp16' in last()
    assert fn(null, null, null, null, null, 0, 4, 100, BF16, null) == -4
    assert 'N=100' in last()
    # no tokens: a no-op that touches no pointer
    assert fn(null, null, null, null, null, 0, 4, 256, BF16, null) == 0
    assert fn(null, null, null, null, null, 0, 4, 256, _lib.F16, null) == 0
    # then the pointers: nulls, 16-byte alignment
    for i in range(5):
        args = [p] * 5
        args[i] = null
        assert fn(*args, 16, 4, 256, BF16, null) == -1
        assert 'null pointer' in last()
    for i in (0, 3, 4):                      # y, shared, out; the gate logit is read per element
        args = [p] * 5
        args[i] = ctypes.c_void_p(258)
        assert fn(*args, 16, 4, 256, BF16, null) == -4
        assert '16-byte aligned' in last()


@pytest.mark.parametrize('name', ['qwen1.5-moe-a2.7b', 'tiny-qwen-moe'])
def test_main_accepts_the_shapes(name):
    from llmc_b200.__main__ import adapt_reference_config
    from llmc_b200.blockwise import AttrDict
    cfg = adapt_reference_config({'model': {'type': 'Qwen2Moe'}, 'quant': {'method': 'RTN'}}, name)
    assert cfg['model'] == {'type': 'Qwen2Moe', 'path': f'synthetic:{name}'}
    cfg = AttrDict.wrap(cfg)
    assert str(cfg.model.path).split(':', 1)[1] in synth.SHAPES
