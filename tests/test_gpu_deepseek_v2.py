"""GPU: DeepSeek-V2 layers.  The fused MLA projection pair (llmc_gemm_mla_qkv / llmc_gemm_mla_kv_b)
gives the bits of the unfused module path; llmc_moe_combine_weighted gives the bits of a torch
restatement; synth.DeepseekV2SparseMoe (fp32 routing weights, ungated shared experts) on the grouped
expert GEMMs gives the bits of its per-expert loop in every expert form the grouped path serves,
with no host sync; RTN, AWQ and GPTQ block loops and the fake-quant perplexity give the same results
either way, and the router is never quantised or replaced."""
import copy
import json
import os

import pytest
import torch

from llmc_b200 import module_utils, synth
from llmc_b200.module_utils import moe_forward
from llmc_b200.synth import DeepseekV2Attention, DeepseekV2Block, DeepseekV2Gate, DeepseekV2SparseMoe
from test_gpu_moe_fake_quant import ACTS, WEIGHTS, _algo, _set_static
from test_gpu_moe_packed import _packed_linear
from test_gpu_moe_qwen import FORMS, _bits, _init, _sel_random, _x
from test_gpu_moe_w8a8 import FORMS as W8A8_FORMS
from test_gpu_moe_w8a8 import _w8a8_linear

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HIDDEN, INTER, TOP_K, SCALE = 256, 128, 6, 1.5


def deepseek_moe(E, dtype=torch.bfloat16, form='dense', k=TOP_K, seed=0):
    """A DeepseekV2SparseMoe on cuda whose routed expert linears have `form` (the forms of
    test_gpu_moe_qwen.qwen_moe).  The shared experts stay dense."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = DeepseekV2SparseMoe(HIDDEN, INTER, E, k, 2, SCALE)
    moe = moe.to(dtype).to_empty(device='cuda')
    _init(moe, g)
    if form == 'dense':
        return moe
    if form.startswith('fq:'):
        _, wform, aform = form.split(':')
        cls, wq = WEIGHTS[wform]
        static, aq = ACTS[aform]
        aq = aq() if aq is not None else None
        params = _algo(wq(), aq, static).get_replacement_params('fake_quant', w_only=aq is None)
    for ex in moe.experts:
        if form.startswith('w8a8:'):
            kind, static, per_channel = W8A8_FORMS[form[5:]]
            ex.gate_proj = _w8a8_linear(INTER, HIDDEN, kind, static, per_channel, g)
            ex.up_proj = _w8a8_linear(INTER, HIDDEN, kind, static, per_channel, g,
                                      input_scale=ex.gate_proj.input_scale.clone() if static else None)
            ex.down_proj = _w8a8_linear(HIDDEN, INTER, kind, static, per_channel, g)
        elif form.startswith('fq:'):
            s_in = torch.rand((), generator=g, device='cuda') * 0.02 + 0.01
            for n in ('gate_proj', 'up_proj', 'down_proj'):
                m = cls.new(getattr(ex, n), params['w_qdq'], params['a_qdq'])
                if static:
                    _set_static(m, s_in if n != 'down_proj'
                                else torch.rand((), generator=g, device='cuda') * 0.004 + 1e-3, aq)
                setattr(ex, n, m)
        else:
            for n in ('gate_proj', 'up_proj', 'down_proj'):
                setattr(ex, n, _packed_linear(getattr(ex, n), form, dtype, g))
    return moe


def _check(moe, x, sel, w):
    experts, a_qdq = moe.grouped_operands(x)
    assert experts is not None
    got = moe_forward(x, sel, w, experts, a_qdq, moe.shared_experts(x))
    assert torch.equal(_bits(got), _bits(moe.shared_loop(x, sel, w)))


def _weights_f32(T, k, seed=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand(T, k, device='cuda', generator=g) * 1.7


@pytest.mark.parametrize('E', [12, 64])
@pytest.mark.parametrize('form', FORMS)
def test_grouped_equals_loop(form, E):
    moe = deepseek_moe(E, torch.bfloat16, form)
    T = 300
    x = _x(T, torch.bfloat16)
    sel, w = moe.route(x)
    assert w.dtype == torch.float32
    _check(moe, x, sel, w)
    # segment edges: experts 0, 7 and the last one empty, expert 3 holding slot 0 of every token
    others = [e for e in range(E) if e not in (0, 3, 7, E - 1)]
    pick = torch.tensor(others)[_sel_random(T, len(others), TOP_K - 1).cpu()]
    sel = torch.cat([torch.full((T, 1), 3, dtype=torch.int64), pick], dim=1).cuda()
    _check(moe, x, sel, _weights_f32(T, TOP_K))


def test_fp16_and_top1():
    moe = deepseek_moe(64, torch.float16, 'dense', k=1)
    x = _x(200, torch.float16)
    sel = torch.full((200, 1), 63, dtype=torch.int64, device='cuda')
    _check(moe, x, sel, _weights_f32(200, 1))
    sel, w = moe.route(x)
    _check(moe, x, sel, w)


@pytest.mark.parametrize('form', ['dense', 'w4_g128_gidx_f32', 'w8a8:e4m3-static', 'fq:e4m3_channel:int8_static'])
def test_module_forward_no_host_sync(form, monkeypatch):
    moe = deepseek_moe(64, torch.bfloat16, form)
    hs = _x(256, torch.bfloat16).view(2, 128, -1)
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(len(a)) or real(*a))
    ref = moe(hs)                                  # warm-up: library load, cached checks
    torch.cuda.synchronize()
    x = hs.view(-1, HIDDEN)
    sel, w = moe.route(x)
    assert torch.equal(_bits(ref.view(-1, HIDDEN)), _bits(moe.shared_loop(x, sel, w)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = moe(hs)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert calls == [6, 6]
    assert torch.equal(out, ref)


# ---- the weighted combine ---------------------------------------------------------------------------
def _combine_weighted_ref(y, rows, w, s):
    """DeepseekV2Moe.forward's roundings: (y * w).to(dtype) per term in fp32, index_add_ into zeros
    per expert (rows ascending expert), then + shared."""
    out = torch.zeros(rows.shape[0], y.shape[1], dtype=y.dtype, device=y.device)
    for j in range(rows.shape[1]):
        r = rows[:, j]
        out = out + (y[r] * w[r, None]).to(y.dtype)
    return out + s


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('k', range(1, 9))
def test_combine_weighted_against_torch(k, dtype):
    gen = torch.Generator(device='cuda').manual_seed(k)
    for T, N in ((0, 64), (1, 8), (333, 2048), (1000, 264)):
        M = T * k + 5
        y = torch.randn(M, N, generator=gen, device='cuda').to(dtype)
        w = torch.rand(M, generator=gen, device='cuda') * 2.5
        rows = torch.randperm(M, generator=torch.Generator().manual_seed(k))[:T * k].view(T, k).cuda()
        s = torch.randn(T, N, generator=gen, device='cuda').to(dtype)
        out = torch.full((T, N), float('nan'), dtype=dtype, device='cuda')
        module_utils.moe_combine_weighted(y, rows, w, s, out)
        assert torch.equal(_bits(out), _bits(_combine_weighted_ref(y, rows, w, s))), (T, N)


# ---- MLA ----------------------------------------------------------------------------------------------
def _attn(shape):
    s = synth.SHAPES[shape]
    g = torch.Generator(device='cuda').manual_seed(11)
    with torch.device('meta'):
        a = DeepseekV2Attention(s['hidden'], s['heads'], s['kv_lora'], eps=s['rms_eps'])
    a = a.to(torch.bfloat16).to_empty(device='cuda')
    _init(a, g)
    a.kv_a_layernorm.weight.data.uniform_(0.5, 1.5, generator=g)
    return a, s


@pytest.mark.parametrize('shape', ['tiny-deepseek-v2', 'deepseek-v2-lite'])
@pytest.mark.parametrize('B,S', [(1, 37), (3, 100), (2, 128), (5, 64)])
def test_mla_fused_equals_unfused(shape, B, S, monkeypatch):
    a, s = _attn(shape)
    assert a.fused_weights(torch.bfloat16) is not None
    g = torch.Generator(device='cuda').manual_seed(B * 1000 + S)
    x = (torch.randn(B, S, s['hidden'], device='cuda', generator=g)).to(torch.bfloat16)
    pos = synth.mla_rope_cos_sin(S + 3, 64, 'cuda', s['rope_theta'])    # longer tables: sliced to S
    calls = []
    real = synth.gemm_mla_qkv
    monkeypatch.setattr(synth, 'gemm_mla_qkv', lambda *a_: calls.append(1) or real(*a_))
    q, k, v = a.qkv(x, pos)
    out = a(x, position_embeddings=pos)
    assert calls == [1, 1]
    monkeypatch.setattr(DeepseekV2Attention, 'fused_weights', lambda self, dtype: None)
    q0, k0, v0 = a.qkv(x, pos)
    for t, t0 in ((q, q0), (k, k0), (v, v0)):
        assert t.shape == t0.shape and t.is_contiguous() and t0.is_contiguous()
        assert torch.equal(_bits(t), _bits(t0))
    assert torch.equal(_bits(out), _bits(a(x, position_embeddings=pos)))


def test_mla_hooked_projection_takes_the_module_path():
    a, s = _attn('tiny-deepseek-v2')
    x = torch.randn(2, 40, s['hidden'], device='cuda').to(torch.bfloat16)
    pos = synth.mla_rope_cos_sin(40, 64, 'cuda', s['rope_theta'])
    ref = a(x, position_embeddings=pos)
    seen = []
    h = a.kv_b_proj.register_forward_hook(lambda m, i, o: seen.append(tuple(i[0].shape)))
    try:
        assert a.fused_weights(torch.bfloat16) is None
        out = a(x, position_embeddings=pos)
    finally:
        h.remove()
    assert seen == [(2, 40, s['kv_lora'])]
    assert torch.equal(_bits(out), _bits(ref))


# ---- the block ----------------------------------------------------------------------------------------
def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.shared_loop(x, sel, w).reshape(B, S, H)


@pytest.mark.parametrize('shape', ['tiny-deepseek-v2', 'deepseek-v2-lite'])
def test_block_forward_grouped_equals_loop(shape, monkeypatch):
    model = synth.SynthModel(shape, n_layers=2, seed=0, device='cuda', with_head=False, init='device')
    dense, blk = model.get_blocks()
    assert isinstance(blk, DeepseekV2Block) and isinstance(blk.mlp, DeepseekV2SparseMoe)
    inp = model.first_block_input(2, 100, device='cuda')
    x, kw = inp['data'][0], inp['kwargs'][0]
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    h = dense(x, **kw)
    got = blk(h, **kw)
    assert calls == [1]
    monkeypatch.setattr(DeepseekV2SparseMoe, 'forward', _loop_forward)
    monkeypatch.setattr(DeepseekV2Attention, 'fused_weights', lambda self, dtype: None)
    ref = blk(dense(x, **kw), **kw)
    assert torch.equal(_bits(got), _bits(ref))
    del model, blk, dense
    torch.cuda.empty_cache()


# ---- block loops and end to end ------------------------------------------------------------------------
def _state(model):
    m = model.get_model()
    return {n: t.detach().clone() for n, t in list(m.named_parameters()) + list(m.named_buffers())}


def _run(monkeypatch, method, loop):
    from llmc_b200 import awq, gptq, rtn  # noqa: F401  (importing registers the algorithms)
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.registry import ALGO_REGISTRY
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    if loop:
        monkeypatch.setattr(DeepseekV2SparseMoe, 'forward', _loop_forward)
    weight = {'bit': 4, 'symmetric': method != 'GPTQ', 'granularity': 'per_group', 'group_size': 128}
    special = {'RTN': {},
               'Awq': {'trans': True, 'trans_version': 'v2', 'weight_clip': True, 'clip_sym': True},
               'GPTQ': {'actorder': True, 'static_groups': False, 'percdamp': 0.01, 'blocksize': 128,
                        'true_sequential': True}}[method]
    quant = {'method': method, 'weight': weight, 'special': special}
    if method == 'GPTQ':
        quant['quant_out'] = True
    if method == 'RTN':       # static activations: the block loop runs the observers
        quant['act'] = {'bit': 8, 'symmetric': True, 'granularity': 'per_tensor', 'static': True,
                        'calib_algo': 'static_minmax'}
    cfg = AttrDict.wrap({'base': {'seed': 0}, 'calib': {'seq_len': 64}, 'quant': quant})
    model = synth.SynthModel('tiny-deepseek-v2', seed=0, device='cuda', outlier_seed=3, with_head=False)
    gate0 = model.get_blocks()[1].mlp.gate.weight.detach().clone()
    bs = -1 if method == 'Awq' else 2
    inp = model.first_block_input(8, 64, bs=bs, seed=1, device='cuda')
    algo = ALGO_REGISTRY[method](model, cfg.quant, inp, None, cfg)
    algo.run_block_loop()
    if method == 'GPTQ':
        algo.check_factorizations(wait=True)
    torch.cuda.synchronize()
    out = algo.input.get('stacked')
    out = [t.clone() for t in algo.input['data']] if out is None else [out.clone()]
    algo.deploy('fake_quant')
    gate = model.get_blocks()[1].mlp.gate
    # the router: never replaced; only AWQ touches its weight (the scales it folds in)
    assert type(gate) is DeepseekV2Gate
    assert method == 'Awq' or torch.equal(gate.weight, gate0)
    fresh = model.first_block_input(8, 64, bs=bs, seed=1, device='cuda')
    for x, kw in zip(fresh['data'], fresh['kwargs']):
        for blk in model.get_blocks():
            x = blk(x, **kw)
        out.append(x)
    torch.cuda.synchronize()
    monkeypatch.undo()
    return _state(model), out, len(calls)


@pytest.mark.parametrize('method', ['RTN', 'Awq', 'GPTQ'])
def test_block_loop_grouped_equals_loop(method, monkeypatch):
    s1, out1, n1 = _run(monkeypatch, method, loop=False)
    s0, out0, n0 = _run(monkeypatch, method, loop=True)
    assert n1 > 0 and n0 == 0
    assert set(s1) == set(s0)
    for n in s1:
        assert torch.equal(s1[n], s0[n]), n
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        assert torch.equal(a, b)


def test_fake_quant_perplexity_end_to_end_grouped_equals_loop(monkeypatch):
    from llmc_b200.__main__ import adapt_reference_config, main
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        doc = json.load(fh)['methods/RTN/rtn_w_only.yml']
    cfg = adapt_reference_config(copy.deepcopy(doc), 'tiny-deepseek-v2', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['model']['type'] = 'DeepseekV2'
    cfg.pop('save', None)
    cfg['eval']['eval_pos'] = ['fake_quant']
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    _, model, report = main(cfg, quiet=True)
    assert calls and report['ppl_fake_quant'] == report['ppl_fake_quant']
    assert type(model.get_blocks()[1].mlp.gate) is DeepseekV2Gate
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(5))
    ppl_grouped = synth.perplexity(model, tokens, 128)
    monkeypatch.setattr(DeepseekV2SparseMoe, 'forward', _loop_forward)
    assert synth.perplexity(model, tokens, 128) == ppl_grouped
