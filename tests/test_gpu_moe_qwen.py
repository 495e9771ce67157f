"""GPU: Qwen2-MoE layers (synth.Qwen2MoeSparseMoe: up to 64 routed experts, top-4 without
renormalisation, a gated shared expert) on the grouped expert GEMMs and llmc_moe_combine_shared give
the bits of the per-expert loop plus the shared expert's add, in every expert form the grouped path
serves, with no host sync; RTN, AWQ and GPTQ block loops and the fake-quant perplexity give the same
results either way."""
import copy
import ctypes
import json
import os

import pytest
import torch
import torch.nn.functional as F

from llmc_b200 import module_utils, synth
from llmc_b200._lib import MOE_MAX_EXPERTS, call, dtype_enum, load, stream_ptr
from llmc_b200.module_utils import moe_forward, moe_routing
from llmc_b200.synth import Qwen2MoeBlock, Qwen2MoeSparseMoe
from test_gpu_moe_fake_quant import ACTS, WEIGHTS, _algo, _set_static
from test_gpu_moe_packed import _packed_linear
from test_gpu_moe_w8a8 import FORMS as W8A8_FORMS
from test_gpu_moe_w8a8 import _w8a8_linear

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HIDDEN, INTER, SHARED_INTER, TOP_K = 256, 128, 256, 4


def _init(mod, g):
    for p in mod.parameters():
        p.data.normal_(0, 0.02, generator=g)


def qwen_moe(E, dtype=torch.bfloat16, form='dense', k=TOP_K, seed=0, hidden=HIDDEN, inter=INTER):
    """A Qwen2MoeSparseMoe on cuda whose routed expert linears have `form`: 'dense', a packed form of
    test_gpu_moe_packed, 'w8a8:<test_gpu_moe_w8a8 form>' or 'fq:<weight>:<act>' (a fake-quant deploy
    of test_gpu_moe_fake_quant's WEIGHTS / ACTS).  The shared expert stays dense."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = Qwen2MoeSparseMoe(hidden, inter, SHARED_INTER, E, k)
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
            ex.gate_proj = _w8a8_linear(inter, hidden, kind, static, per_channel, g)
            ex.up_proj = _w8a8_linear(inter, hidden, kind, static, per_channel, g,
                                      input_scale=ex.gate_proj.input_scale.clone() if static else None)
            ex.down_proj = _w8a8_linear(hidden, inter, kind, static, per_channel, g)
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


def _x(T, dtype, seed=1, hidden=HIDDEN):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(T, hidden, device='cuda', generator=g).to(dtype)


def _bits(t):
    return t.view(torch.int16)


def _grouped(moe, x):
    experts, a_qdq = moe.grouped_operands(x)
    assert experts is not None
    return experts, a_qdq


def _check_routed(moe, x, sel, w):
    """moe_forward on the routed experts equals expert_loop, and with the shared expert the module's
    definition (shared_loop)."""
    experts, a_qdq = _grouped(moe, x)
    got = moe_forward(x, sel, w, experts, a_qdq)
    assert torch.equal(_bits(got), _bits(moe.expert_loop(x, sel, w)))
    got = moe_forward(x, sel, w, experts, a_qdq, moe.shared(x))
    assert torch.equal(_bits(got), _bits(moe.shared_loop(x, sel, w)))


def _sel_random(T, E, k, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, E, generator=g).argsort(dim=1)[:, :k].cuda()


def _weights(T, k, dtype, seed=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.rand(T, k, device='cuda', generator=g) * 0.5).to(dtype)


FORMS = ['dense', 'w4_g128_native', 'w4_g128_gidx_f32', 'w8_channel', 'w8a8:int8-dynamic', 'w8a8:int8-static',
         'w8a8:e4m3-dynamic', 'w8a8:e4m3-static', 'fq:e4m3_channel:e4m3_token', 'fq:e4m3_channel:int8_static',
         'fq:e4m3_channel:none']


def test_cap_is_64():
    assert MOE_MAX_EXPERTS == 64


@pytest.mark.parametrize('E', [12, 60, 64])
@pytest.mark.parametrize('form', FORMS)
def test_grouped_equals_loop(form, E):
    dtype = torch.bfloat16
    moe = qwen_moe(E, dtype, form)
    T = 300
    x = _x(T, dtype)
    sel, w = moe.route(x)
    _check_routed(moe, x, sel, w)
    # segment edges: experts 0, 7 and the last one empty, expert 3 holding slot 0 of every token
    others = [e for e in range(E) if e not in (0, 3, 7, E - 1)]
    pick = torch.tensor(others)[_sel_random(T, len(others), TOP_K - 1).cpu()]
    sel = torch.cat([torch.full((T, 1), 3, dtype=torch.int64), pick], dim=1).cuda()
    _check_routed(moe, x, sel, _weights(T, TOP_K, dtype))


@pytest.mark.parametrize('form', ['dense', 'w4_g128_native'])
def test_fp16_and_top1(form):
    moe = qwen_moe(60, torch.float16, form, k=1)
    x = _x(200, torch.float16)
    sel = torch.full((200, 1), 59, dtype=torch.int64, device='cuda')           # one expert holds every row
    _check_routed(moe, x, sel, _weights(200, 1, torch.float16))
    sel, w = moe.route(x)
    _check_routed(moe, x, sel, w)


@pytest.mark.parametrize('form', ['dense', 'w8a8:int8-dynamic'])
def test_zero_tokens(form):
    moe = qwen_moe(64, torch.bfloat16, form)
    x = torch.empty(0, HIDDEN, dtype=torch.bfloat16, device='cuda')
    sel = torch.empty(0, TOP_K, dtype=torch.int64, device='cuda')
    w = torch.empty(0, TOP_K, dtype=torch.bfloat16, device='cuda')
    experts, a_qdq = _grouped(moe, x)
    out = moe_forward(x, sel, w, experts, a_qdq, moe.shared(x))
    assert out.shape == (0, HIDDEN) and out.dtype == torch.bfloat16
    out = moe(x.view(1, 0, HIDDEN))
    assert out.shape == (1, 0, HIDDEN)


@pytest.mark.parametrize('form', ['dense', 'w4_g128_gidx_f32', 'w8a8:e4m3-static', 'fq:e4m3_channel:int8_static'])
def test_module_forward_no_host_sync(form, monkeypatch):
    moe = qwen_moe(60, torch.bfloat16, form)
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


def test_hooked_expert_takes_the_loop():
    moe = qwen_moe(12)
    x = _x(300, torch.bfloat16)
    sel, w = moe.route(x)
    ref = moe(x.view(1, 300, -1))
    seen = []
    h = moe.experts[1].down_proj.register_forward_hook(lambda m, i, o: seen.append(i[0].shape[0]))
    try:
        assert moe.grouped_operands(x) == (None, None)
        out = moe(x.view(1, 300, -1))
    finally:
        h.remove()
    assert seen == [int((sel == 1).sum())]
    assert torch.equal(out, ref)


# ---- the combine with the gated shared expert ----------------------------------------------------
def _combine_shared_ref(y, rows, g, s):
    """Qwen2MoeSparseMoeBlock.forward's roundings: index_add_ into zeros per expert (rows ascending
    expert), then F.sigmoid(gate) * shared, then the add."""
    out = torch.zeros(rows.shape[0], y.shape[1], dtype=y.dtype, device=y.device)
    for j in range(rows.shape[1]):
        out = out + y[rows[:, j]]
    return out + F.sigmoid(g) * s


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('k', range(1, 9))
def test_combine_shared_against_torch(k, dtype):
    gen = torch.Generator(device='cuda').manual_seed(k)
    for T, N in ((0, 64), (1, 8), (333, 2048), (1000, 264)):
        M = T * k + 5
        y = torch.randn(M, N, generator=gen, device='cuda').to(dtype)
        rows = torch.randperm(M, generator=torch.Generator().manual_seed(k))[:T * k].view(T, k).cuda()
        g = (torch.randn(T, 1, generator=gen, device='cuda') * 4).to(dtype)
        s = torch.randn(T, N, generator=gen, device='cuda').to(dtype)
        out = torch.full((T, N), float('nan'), dtype=dtype, device='cuda')
        module_utils.moe_combine_shared(y, rows, g, s, out)
        assert torch.equal(_bits(out), _bits(_combine_shared_ref(y, rows, g, s))), (T, N)


def test_combine_shared_zero_tokens_launch_nothing():
    torch.cuda.synchronize()
    before = load().llmc_b200_launch_count()
    null = ctypes.c_void_p(0)
    call('llmc_moe_combine_shared', null, null, null, null, null, 0, 4, 256, dtype_enum(torch.bfloat16),
         stream_ptr())
    torch.cuda.synchronize()
    assert load().llmc_b200_launch_count() == before


# ---- the block --------------------------------------------------------------------------------------
def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.shared_loop(x, sel, w).reshape(B, S, H)


@pytest.mark.parametrize('shape', ['tiny-qwen-moe', 'qwen1.5-moe-a2.7b'])
def test_block_forward_grouped_equals_loop(shape, monkeypatch):
    model = synth.SynthModel(shape, n_layers=1, seed=0, device='cuda', with_head=False, init='device')
    blk = model.get_blocks()[0]
    assert isinstance(blk, Qwen2MoeBlock)
    g = torch.Generator(device='cuda').manual_seed(3)
    for lin in (blk.self_attn.q_proj, blk.self_attn.k_proj, blk.self_attn.v_proj):
        lin.bias.data.normal_(0, 0.5, generator=g)
    inp = model.first_block_input(2, 128, device='cuda')
    x, kw = inp['data'][0], inp['kwargs'][0]
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    got = blk(x, **kw)
    assert calls == [1]
    monkeypatch.setattr(Qwen2MoeSparseMoe, 'forward', _loop_forward)
    ref = blk(x, **kw)
    assert torch.equal(_bits(got), _bits(ref))
    del model, blk
    torch.cuda.empty_cache()


# ---- block loops and end to end ------------------------------------------------------------------------
def _state(model):
    m = model.get_model()
    return {n: t.detach().clone() for n, t in list(m.named_parameters()) + list(m.named_buffers())}


def _assert_same(a, b):
    assert set(a) == set(b)
    for n in a:
        assert torch.equal(a[n], b[n]), n


def _run(monkeypatch, method, loop):
    from llmc_b200 import awq, gptq, rtn  # noqa: F401  (importing registers the algorithms)
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.registry import ALGO_REGISTRY
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    if loop:
        monkeypatch.setattr(Qwen2MoeSparseMoe, 'forward', _loop_forward)
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
    model = synth.SynthModel('tiny-qwen-moe', n_layers=1, seed=0, device='cuda', outlier_seed=3, with_head=False)
    bs = -1 if method == 'Awq' else 2
    inp = model.first_block_input(8, 64, bs=bs, seed=1, device='cuda')
    algo = ALGO_REGISTRY[method](model, cfg.quant, inp, None, cfg)
    algo.run_block_loop()
    if method == 'GPTQ':
        algo.check_factorizations(wait=True)
    torch.cuda.synchronize()
    out = algo.input.get('stacked')
    out = [t.clone() for t in algo.input['data']] if out is None else [out.clone()]
    # the deployed fake-quant block on the calibration input
    algo.deploy('fake_quant')
    fresh = model.first_block_input(8, 64, bs=bs, seed=1, device='cuda')
    blk = model.get_blocks()[0]
    out += [blk(x, **kw) for x, kw in zip(fresh['data'], fresh['kwargs'])]
    torch.cuda.synchronize()
    monkeypatch.undo()
    return _state(model), out, len(calls)


@pytest.mark.parametrize('method', ['RTN', 'Awq', 'GPTQ'])
def test_block_loop_grouped_equals_loop(method, monkeypatch):
    s1, out1, n1 = _run(monkeypatch, method, loop=False)
    s0, out0, n0 = _run(monkeypatch, method, loop=True)
    assert n1 > 0 and n0 == 0
    _assert_same(s1, s0)
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        assert torch.equal(a, b)


def test_fake_quant_perplexity_end_to_end_grouped_equals_loop(monkeypatch):
    from llmc_b200.__main__ import adapt_reference_config, main
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        doc = json.load(fh)['methods/RTN/rtn_w_only.yml']
    cfg = adapt_reference_config(copy.deepcopy(doc), 'tiny-qwen-moe', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['model']['type'] = 'Qwen2Moe'
    cfg.pop('save', None)
    cfg['eval']['eval_pos'] = ['fake_quant']
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    _, model, report = main(cfg, quiet=True)
    assert calls and report['ppl_fake_quant'] == report['ppl_fake_quant']
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(5))
    ppl_grouped = synth.perplexity(model, tokens, 128)
    monkeypatch.setattr(Qwen2MoeSparseMoe, 'forward', _loop_forward)
    assert synth.perplexity(model, tokens, 128) == ppl_grouped
