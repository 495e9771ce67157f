"""GPU: fake-quant Mixtral experts under activation fake-quant, and FP8-grid experts, on the grouped
GEMMs.  The FP8 grouped entry points give the bits of the per-expert llmc_gemm_fp8a16[_gidx] with
SiLU-mul / the routing weight at every segment edge; MixtralSparseMoe gives the bits of its
per-expert loop in every accepted weight x activation form, with no host sync after the first call;
refused forms take the loop; end to end, W8A8 and FP8 recipes give the same fake-quant perplexity,
and a quant_out recipe the same weights, either way."""
import copy
import ctypes
import functools
import json
import os

import pytest
import torch
import torch.nn.functional as F

from llmc_b200 import _lib, module_utils, synth
from llmc_b200.blockwise import BaseBlockwiseQuantization
from llmc_b200.module_utils import (EffcientFakeQuantLinear, FakeQuantLinear, Fp8Operands, linear_forward_fp8w,
                                    moe_forward)
from llmc_b200.quant import IntegerQuantizer
from llmc_b200.quant_float import FloatQuantizer
from llmc_b200.synth import MixtralSparseMoe

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP8 = {0: torch.float8_e4m3fn, 1: torch.float8_e5m2}


# ---- the entry points against the per-expert definition ------------------------------------------
def _scales(form, N, K, dtype, g):
    """(scales [ng, N] as the GEMM takes them, group, g_idx) of `form`, some scales zero.  Groups
    are 128 columns, or 64 where K is no multiple of 128."""
    grp = 128 if K % 128 == 0 else 64
    if form == 'f32_row':
        s, group, gi = torch.rand(1, N, generator=g, device='cuda') * 0.02, K, None
    elif form == 'native_channel':
        s, group, gi = (torch.rand(1, N, generator=g, device='cuda') * 0.02).to(dtype), K, None
    elif form == 'groups':
        s, group, gi = (torch.rand(K // grp, N, generator=g, device='cuda') * 0.02).to(dtype), grp, None
    else:                                               # g_idx: groups in a random column order
        s, group = torch.rand(K // grp, N, generator=g, device='cuda') * 0.02, grp
        gi = (torch.randperm(K, generator=g, device='cuda') // grp).to(torch.int32)
    s.view(-1)[::7] = 0                                 # read as 1
    return s.contiguous(), group, gi


def _linear(N, K, e5m2, form, dtype, g):
    wq = (torch.randn(N, K, generator=g, device='cuda') * 4).to(FP8[e5m2])
    s, group, gi = _scales(form, N, K, dtype, g)
    return wq, s, group, gi


def _arr(ts):
    return None if ts[0] is None else (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _ref(x, lin):
    wq, s, group, gi = lin
    return linear_forward_fp8w(x, wq, s, group, qparams_t=True, g_idx=gi)


# (E, rows per expert, K = hidden, inter), each run over both grids, dtypes and every scale form
CASES = [
    (1, [129], 256, 128),                               # one expert, a partial second m-tile
    (2, [0, 300], 256, 64),                             # an empty leading expert, one n-tile of gate/up
    (3, [127, 0, 129], 384, 128),                       # an empty middle expert, down N not of 256
    (5, [128, 1, 0, 128, 129], 256, 192),               # one-row and full-tile segments
    (8, [1, 127, 128, 129, 0, 5, 300, 0], 256, 128),    # every segment edge, a trailing empty expert
]


@pytest.mark.parametrize('form', ['f32_row', 'native_channel', 'groups', 'g_idx'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('e5m2', [0, 1])
@pytest.mark.parametrize('case', range(len(CASES)))
def test_entry_points_equal_per_expert_definition(case, e5m2, dtype, form):
    E, counts, K, inter = CASES[case]
    N = K
    g = torch.Generator(device='cuda').manual_seed(case * 16 + e5m2 * 8 + (dtype == torch.float16) * 4)
    M = sum(counts)
    offsets = torch.tensor([0] + list(torch.tensor(counts).cumsum(0)), dtype=torch.int32, device='cuda')
    xp = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    a_in = (torch.randn(M, inter, generator=g, device='cuda') * 2).to(dtype)
    w_route = torch.rand(M, generator=g, device='cuda').to(dtype)
    w_route[::11] = 0
    lins = [[_linear(inter, K, e5m2, form, dtype, g), _linear(inter, K, e5m2, form, dtype, g),
             _linear(N, inter, e5m2, form, dtype, g)] for _ in range(E)]
    act = torch.full((M + 8, inter), float('nan'), dtype=dtype, device='cuda')
    y = torch.full((M + 8, N), float('nan'), dtype=dtype, device='cuda')

    def ops(i, j):
        return [lins[e][i][j] for e in range(E)]
    words = [[t.view(torch.int32) for t in ops(i, 0)] for i in range(3)]
    qd = _lib.dtype_enum(lins[0][0][1].dtype)
    dt, st = _lib.dtype_enum(dtype), _lib.stream_ptr(xp.device)
    for i, (Kl, out, src) in ((0, (K, act, xp)), (2, (inter, y, a_in))):
        grp = lins[0][i][2]
        ng = lins[0][i][1].shape[0]
        if i == 0:
            _lib.call('llmc_moe_gemm_fp8a16_swiglu', _lib.ptr(src), e5m2, _arr(words[0]), _arr(words[1]),
                      _arr(ops(0, 1)), _arr(ops(1, 1)), _arr(ops(0, 3)), _arr(ops(1, 3)), qd, -grp, ng,
                      _lib.ptr(offsets), _lib.ptr(out), M, inter, K, E, dt, st)
        else:
            _lib.call('llmc_moe_gemm_fp8a16_down', _lib.ptr(src), e5m2, _arr(words[2]), _arr(ops(2, 1)),
                      _arr(ops(2, 3)), qd, -grp, ng, _lib.ptr(offsets), _lib.ptr(w_route), _lib.ptr(out), M, N,
                      inter, E, dt, st)
    torch.cuda.synchronize()
    want_act = torch.empty(M, inter, dtype=dtype, device='cuda')
    want_y = torch.empty(M, N, dtype=dtype, device='cuda')
    for e in range(E):
        a, b = int(offsets[e]), int(offsets[e + 1])
        if a == b:
            continue
        want_act[a:b] = F.silu(_ref(xp[a:b], lins[e][0])) * _ref(xp[a:b], lins[e][1])
        want_y[a:b] = _ref(a_in[a:b], lins[e][2]) * w_route[a:b, None]
    assert torch.equal(act[:M].view(torch.int16), want_act.view(torch.int16))
    assert torch.equal(y[:M].view(torch.int16), want_y.view(torch.int16))
    assert act[M:].isnan().all() and y[M:].isnan().all()       # nothing past the last row


# ---- the module forward --------------------------------------------------------------------------
WEIGHTS = {                                             # (module class, weight quantizer)
    'dense_int8': (FakeQuantLinear, lambda: IntegerQuantizer(8, True, 'per_channel')),
    'int8': (EffcientFakeQuantLinear, lambda: IntegerQuantizer(8, True, 'per_channel')),
    'int4_g128': (EffcientFakeQuantLinear, lambda: IntegerQuantizer(4, False, 'per_group', group_size=128)),
    'e4m3_tensor': (EffcientFakeQuantLinear, lambda: FloatQuantizer('e4m3', True, 'per_tensor', use_qtorch=True)),
    'e4m3_channel': (EffcientFakeQuantLinear,
                     lambda: FloatQuantizer('e4m3', True, 'per_channel', use_qtorch=True)),
}
ACTS = {                                                # (static, activation quantizer)
    'none': (False, None),
    'int8_token': (False, lambda: IntegerQuantizer(8, True, 'per_token')),
    'e4m3_token': (False, lambda: FloatQuantizer('e4m3', True, 'per_token', use_qtorch=True)),
    'int8_static': (True, lambda: IntegerQuantizer(8, True, 'per_tensor', calib_algo='static_minmax')),
    'e4m3_static': (True, lambda: FloatQuantizer('e4m3', True, 'per_tensor', use_qtorch=True,
                                                 calib_algo='static_minmax')),
    # refused: the scale of a per-tensor dynamic pass depends on the whole expert segment
    'int8_tensor_dynamic': (False, lambda: IntegerQuantizer(8, True, 'per_tensor')),
    'int8_static_asym': (True, lambda: IntegerQuantizer(8, False, 'per_tensor', calib_algo='static_minmax')),
}


def _algo(wq, aq, static):
    """A BaseBlockwiseQuantization holding just what get_replacement_params reads."""
    algo = object.__new__(BaseBlockwiseQuantization)
    algo.wquantizer, algo.aquantizer, algo.act_static = wq, aq, static
    return algo


def _set_static(m, scale, q):
    dev = 'cuda'
    m.register_buffer('buf_act_scales_0', scale)
    zero = torch.tensor(0.0, device=dev) if q.sym else torch.round(torch.rand((), device=dev) * 10)
    m.register_buffer('buf_act_zeros_0', zero)
    m.register_buffer('buf_act_qmin_0', q.qmin.to(dev))
    m.register_buffer('buf_act_qmax_0', q.qmax.to(dev))


def fake_quant_moe(shape, wform, aform, dtype=torch.bfloat16, top_k=None, seed=0):
    """A MixtralSparseMoe of synth.SHAPES[shape] whose expert linears are replaced as a fake-quant
    deploy replaces them: weights quantised by WEIGHTS[wform], activations by ACTS[aform] (static
    scales differ per expert, w1's and w3's one tensor, as register_act_qparams stores them)."""
    s = synth.SHAPES[shape]
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = MixtralSparseMoe(s['hidden'], s['inter'], s['experts'], top_k or s['top_k'])
    moe = moe.to(dtype).to_empty(device='cuda')
    for p in moe.parameters():
        p.data.normal_(0, 0.02, generator=g)
    cls, wq = WEIGHTS[wform]
    static, aq = ACTS[aform]
    aq = aq() if aq is not None else None
    params = _algo(wq(), aq, static).get_replacement_params('fake_quant', w_only=aq is None)
    for ex in moe.experts:
        s_in = torch.rand((), generator=g, device='cuda') * 0.02 + 0.01
        for n in ('w1', 'w3', 'w2'):
            m = cls.new(getattr(ex, n), params['w_qdq'], params['a_qdq'])
            if static:
                _set_static(m, s_in if n != 'w2' else torch.rand((), generator=g, device='cuda') * 0.004 + 1e-3, aq)
            setattr(ex, n, m)
    return moe


def _x(T, H, dtype, seed=1):
    return torch.randn(T, H, generator=torch.Generator(device='cuda').manual_seed(seed), device='cuda').to(dtype)


def _grouped_equals_loop(moe, x, monkeypatch):
    sel, w = moe.route(x)
    calls = []
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(len(a)) or moe_forward(*a))
    out = moe(x.view(1, *x.shape)).view(x.shape)
    ref = moe.expert_loop(x, sel, w)
    assert calls == [5] or (calls == [4] and isinstance(moe.grouped_fake_quant_operands(x)[0][0][0], Fp8Operands))
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')                     # cached checks: no sync any more
    try:
        again = moe(x.view(1, *x.shape)).view(x.shape)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert torch.equal(again.view(torch.int16), ref.view(torch.int16))


ACCEPTED = ([(w, a) for w in WEIGHTS for a in ('int8_token', 'e4m3_token', 'int8_static', 'e4m3_static')]
            + [('e4m3_tensor', 'none'), ('e4m3_channel', 'none')])


@pytest.mark.parametrize('wform,aform', ACCEPTED)
def test_tiny_mixtral_grouped_equals_loop(wform, aform, monkeypatch):
    moe = fake_quant_moe('tiny-mixtral', wform, aform)
    _grouped_equals_loop(moe, _x(300, 256, torch.bfloat16), monkeypatch)


@pytest.mark.parametrize('wform,aform', [('int8', 'e4m3_static'), ('e4m3_channel', 'int8_token'),
                                         ('dense_int8', 'int8_static')])
def test_fp16_and_top1(wform, aform, monkeypatch):
    moe = fake_quant_moe('tiny-mixtral', wform, aform, dtype=torch.float16)
    _grouped_equals_loop(moe, _x(257, 256, torch.float16), monkeypatch)
    moe = fake_quant_moe('tiny-mixtral', wform, aform, top_k=1, seed=3)
    _grouped_equals_loop(moe, _x(129, 256, torch.bfloat16), monkeypatch)


@pytest.mark.parametrize('wform,aform', [('e4m3_tensor', 'e4m3_static'), ('e4m3_channel', 'e4m3_token'),
                                         ('int8', 'int8_token'), ('dense_int8', 'int8_static'),
                                         ('int4_g128', 'e4m3_token')])
def test_mixtral_8x7b_layer_grouped_equals_loop(wform, aform, monkeypatch):
    moe = fake_quant_moe('mixtral-8x7b', wform, aform)
    _grouped_equals_loop(moe, _x(2048, 4096, torch.bfloat16), monkeypatch)
    del moe
    torch.cuda.empty_cache()


# ---- refusals take the loop ------------------------------------------------------------------------
class _Override(BaseBlockwiseQuantization):
    def a_qdq(self, act, module, aquantizer, input_index=0):      # no routed twin of its own
        return super().a_qdq(act, module, aquantizer, input_index)


REFUSED = ['tensor_dynamic', 'static_asym', 'w1_w3_scales_differ', 'two_quantizers', 'some_without_a_qdq',
           'override_without_twin', 'lambda', 'int_weights_without_a_qdq', 'mixed_weight_forms']


@pytest.mark.parametrize('case', REFUSED)
def test_refused_forms_take_the_loop(case, monkeypatch):
    aform = {'tensor_dynamic': 'int8_tensor_dynamic', 'static_asym': 'int8_static_asym',
             'w1_w3_scales_differ': 'int8_static', 'int_weights_without_a_qdq': 'none'}.get(case, 'int8_token')
    wform = 'int8' if case != 'mixed_weight_forms' else 'e4m3_channel'
    moe = fake_quant_moe('tiny-mixtral', wform, aform)
    ex = moe.experts[1]
    if case == 'w1_w3_scales_differ':
        ex.w3.register_buffer('buf_act_scales_0', ex.w3.buf_act_scales_0 * 2)
    elif case == 'two_quantizers':
        ex.w2.a_qdq = functools.partial(ex.w2.a_qdq.func, aquantizer=IntegerQuantizer(8, True, 'per_token'))
        ex.w2.a_qdq.routed = moe.experts[0].w2.a_qdq.routed
    elif case == 'some_without_a_qdq':
        ex.w2.a_qdq = None
    elif case == 'override_without_twin':
        aq = IntegerQuantizer(8, True, 'per_token')
        algo = object.__new__(_Override)
        algo.wquantizer, algo.aquantizer, algo.act_static = IntegerQuantizer(8, True, 'per_channel'), aq, False
        a = algo.get_replacement_params('fake_quant')['a_qdq']
        assert not hasattr(a, 'routed')
        for e in moe.experts:
            for n in ('w1', 'w3', 'w2'):
                getattr(e, n).a_qdq = a
    elif case == 'lambda':
        ex.w1.a_qdq = lambda x, layer: x
    elif case == 'mixed_weight_forms':
        other = fake_quant_moe('tiny-mixtral', 'int8', 'int8_token')
        moe.experts[1] = other.experts[1]
    x = _x(300, 256, torch.bfloat16)
    sel, w = moe.route(x)
    assert moe.grouped_fake_quant_operands(x) is None
    calls = []
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or moe_forward(*a))
    out = moe(x.view(1, 300, -1)).view(300, -1)
    if case == 'int_weights_without_a_qdq':
        assert calls == [1]                             # the packed selector's, not this one's
    else:
        assert not calls
    assert torch.equal(out.view(torch.int16), moe.expert_loop(x, sel, w).view(torch.int16))


# ---- end to end ----------------------------------------------------------------------------------
def _recipe(name):
    import yaml
    if name == 'rtn_fp8_static_mixtral':
        with open(os.path.join(ROOT, 'configs', 'rtn_fp8_static_mixtral.yml')) as fh:
            return yaml.safe_load(fh)
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[name]


def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.expert_loop(x, sel, w).reshape(B, S, H)


def _run_main(monkeypatch, name, loop):
    from llmc_b200.__main__ import adapt_reference_config, main
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    if loop:
        monkeypatch.setattr(MixtralSparseMoe, 'forward', _loop_forward)
    cfg = adapt_reference_config(copy.deepcopy(_recipe(name)), 'tiny-mixtral', n_samples=8, seq_len=128,
                                 eval_seq_len=128)
    cfg['model']['type'] = 'Mixtral'
    cfg.pop('save', None)
    cfg['eval'] = dict(cfg.get('eval') or {}, eval_pos=['fake_quant'], seq_len=128)
    if cfg['quant']['method'] == 'Awq':                 # auto-clip under activation fake-quant is not built
        cfg['quant']['special']['weight_clip'] = False
    _, model, report = main(cfg, quiet=True)
    monkeypatch.undo()
    state = {n: t.detach().clone() for n, t in model.get_model().state_dict().items()}
    return report['ppl_fake_quant'], len(calls), state


# the last two calibrate with quant_out: each block's output runs through linears under a_qdq
@pytest.mark.parametrize('name', ['rtn_fp8_static_mixtral', 'backend/vllm/fp8/rtn_fp8.yml',
                                  'backend/vllm/rtn_w8a8.yml', 'backend/sglang/awq_w8a8.yml',
                                  'backend/vllm/fp8/gptq_fp8.yml'])
def test_end_to_end_grouped_equals_loop(name, monkeypatch):
    ppl1, n1, s1 = _run_main(monkeypatch, name, loop=False)
    ppl0, n0, s0 = _run_main(monkeypatch, name, loop=True)
    assert n1 > 0 and n0 == 0
    assert ppl1 == ppl0 and ppl1 == ppl1
    assert set(s1) == set(s0)
    for n in s1:
        assert torch.equal(s1[n], s0[n]), n
