"""GPU: Mixtral sparse-MoE layers with PACKED experts (deployed fake-quant W4 / W8 linears, vLLM W4A16
exports) on the grouped dequant GEMMs give the bits of the per-expert loop
(MixtralSparseMoe.expert_loop) on the same module, with no host sync; out-of-scope, hooked and
mixed-form experts take the loop; end to end, a GPTQ and an RTN Mixtral give the same fake-quant
perplexity either way."""
import copy
import os

import pytest
import torch
import yaml

from llmc_b200 import module_utils, synth
from llmc_b200.module_utils import (EffcientFakeQuantLinear, PackedOperands, VllmRealQuantLinear,
                                    moe_forward, pack_unsigned_codes)
from llmc_b200.synth import MixtralSparseMoe

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMS = ['w4_g128_native', 'w4_g128_gidx_f32', 'w8_channel', 'vllm_w4_sym']


def _packed_linear(lin, form, dtype, g, group=128):
    """A packed stand-in of B200Linear `lin` ([N, K]) with random codes and qparams of `form` (groups
    of `group` columns but W8's one per row)."""
    N, K = lin.out_features, lin.in_features
    dev = 'cuda'
    if form == 'vllm_w4_sym':
        words = torch.randint(-2**31, 2**31 - 1, (N, K // 8), generator=g, device=dev, dtype=torch.int32)
        s = (torch.rand(N, K // group, generator=g, device=dev) * 0.01 + 1e-3).to(torch.float16)
        m = VllmRealQuantLinear(words, None, s, None, True, 'weight_scale')
        m.in_features, m.out_features = K, N
        return m
    bits, group = (8, K) if form == 'w8_channel' else (4, group)
    ng = K // group
    qdt = torch.float32 if form == 'w4_g128_gidx_f32' else dtype
    codes = torch.randint(0, 2**bits, (N, K), generator=g, device=dev, dtype=torch.int32)
    packed = dict(qweight=pack_unsigned_codes(codes, bits, signed=False),
                  scales=(torch.rand(N, ng, generator=g, device=dev) * 0.01 + 1e-3).to(qdt),
                  zeros=None if form == 'w8_channel'
                  else torch.randint(0, 2**bits, (N, ng), generator=g, device=dev).to(qdt),
                  bits=bits, group=group, dtype=dtype)
    if form == 'w8_channel':                           # symmetric: the +128 storage offset
        packed['qweight'] = pack_unsigned_codes(codes - 128, bits, signed=True)
    if form == 'w4_g128_gidx_f32':                     # act-order: a different g_idx per linear
        packed['g_idx'] = (torch.randperm(K, generator=g, device=dev) // group).to(torch.int32)
    m = EffcientFakeQuantLinear(None, None, lin, None, packed=packed)
    m.in_features, m.out_features = K, N
    return m


def _moe(hidden, inter, E, k, dtype, form, seed=0, group=128):
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = MixtralSparseMoe(hidden, inter, E, k)
    moe.gate = moe.gate.to_empty(device='cuda').to(dtype)
    moe.gate.weight.data.normal_(0, 0.02, generator=g)
    forms = form if isinstance(form, list) else [form] * E
    for ex, f in zip(moe.experts, forms):
        for n in ('w1', 'w3', 'w2'):
            setattr(ex, n, _packed_linear(getattr(ex, n), f, dtype, g, group))
    return moe


def _x(T, hidden, dtype, seed=1):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(T, hidden, device='cuda', generator=g).to(dtype)


def _weights(T, k, dtype, seed=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    w = torch.rand(T, k, device='cuda', generator=g) + 0.05
    return (w / w.sum(dim=1, keepdim=True)).to(dtype)


def _sel_from_sizes(sizes, k_other, seed=3):
    sel0 = torch.cat([torch.full((n,), e, dtype=torch.int64) for e, n in enumerate(sizes)])
    sel0 = sel0[torch.randperm(sel0.numel(), generator=torch.Generator().manual_seed(seed))]
    return torch.stack([sel0, torch.full_like(sel0, k_other)], dim=1).cuda()


def _check(moe, x, sel, w):
    assert moe.grouped_weights(x) is None
    ops = moe.grouped_packed_operands(x)
    assert ops is not None and all(isinstance(o, PackedOperands) for t in ops for o in t)
    got = moe_forward(x, sel, w, ops)
    ref = moe.expert_loop(x, sel, w)
    assert got.dtype == ref.dtype and got.shape == ref.shape
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    return got


@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_tiny_mixtral_forms(dtype, form):
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype, form)
    T = 300
    hs = _x(T, s['hidden'], dtype).view(1, T, -1)
    sel, w = moe.route(hs.view(T, -1))
    _check(moe, hs.view(T, -1), sel, w)
    out = moe(hs)                                       # the module forward takes the grouped path
    assert torch.equal(out.view(T, -1).view(torch.int16),
                       moe.expert_loop(hs.view(T, -1), sel, w).view(torch.int16))


@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_mixtral_8x7b_layer_2048_tokens(dtype, form):
    s = synth.SHAPES['mixtral-8x7b']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype, form)
    x = _x(2048, s['hidden'], dtype)
    sel, w = moe.route(x)
    _check(moe, x, sel, w)
    del moe
    torch.cuda.empty_cache()


@pytest.mark.parametrize('form', FORMS)
def test_segment_sizes_one_expert_and_top1(form):
    dtype, E, hidden, inter = torch.bfloat16, 8, 256, 512
    moe = _moe(hidden, inter, E, 2, dtype, form)
    sizes = [0, 1, 63, 64, 127, 128, 129]             # expert 7 takes slot 1 of every token
    sel = _sel_from_sizes(sizes, 7)
    T = sel.shape[0]
    _check(moe, _x(T, hidden, dtype), sel, _weights(T, 2, dtype))
    T = 1000                                           # every token on expert 3 (slot 0)
    other = torch.randint(0, E - 1, (T,), generator=torch.Generator().manual_seed(4))
    sel = torch.stack([torch.full((T,), 3), other + (other >= 3).long()], dim=1).cuda()
    _check(moe, _x(T, hidden, dtype), sel, _weights(T, 2, dtype))
    moe1 = _moe(hidden, inter, E, 1, dtype, form)      # top-1, every token on one expert
    sel = torch.full((T, 1), 5, dtype=torch.int64, device='cuda')
    _check(moe1, _x(T, hidden, dtype), sel, torch.ones(T, 1, dtype=dtype, device='cuda'))


@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_partial_tiles(dtype, form):
    """hidden 320 and inter 576 with groups of 64: the down projection's last 128-row n-tile holds
    64 rows of w2 (TMA rows past N, zero qparams, the column guard of the routed store), and
    gate/up takes nine 64-row n-tiles."""
    hidden, inter, E = 320, 576, 8
    moe = _moe(hidden, inter, E, 2, dtype, form, group=64)
    T = 700
    x = _x(T, hidden, dtype)
    sel, w = moe.route(x)
    _check(moe, x, sel, w)
    sel = _sel_from_sizes([0, 1, 63, 64, 127, 128, 129], 7)
    T = sel.shape[0]
    _check(moe, _x(T, hidden, dtype), sel, _weights(T, 2, dtype))


# expert counts below 8 and top_k up to E, at widths with a partial 128-column n-tile of the down
# projection (320) and inter 64: one gate/up n-tile, one k-step in the down projection
EXPERTS_TOP_K = [(1, 1), (2, 1), (2, 2), (3, 2), (3, 3), (5, 3), (5, 5), (8, 3), (8, 8)]


def _sel_random(T, E, k, seed=5):
    """Each token's k distinct experts, in random order."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, E, generator=g).argsort(dim=1)[:, :k].cuda()


@pytest.mark.parametrize('hidden,inter', [(320, 64), (320, 128), (4096, 384)])
@pytest.mark.parametrize('E,k', EXPERTS_TOP_K)
@pytest.mark.parametrize('form', FORMS)
def test_expert_counts_top_k_and_widths(form, E, k, hidden, inter):
    dtype = torch.bfloat16 if (E + k) % 2 else torch.float16
    moe = _moe(hidden, inter, E, k, dtype, form, group=64)
    T = 200
    _check(moe, _x(T, hidden, dtype), _sel_random(T, E, k), _weights(T, k, dtype))


@pytest.mark.parametrize('form', FORMS)
def test_zero_tokens_launch_nothing(form):
    from llmc_b200._lib import load
    dtype, hidden = torch.bfloat16, 320
    moe = _moe(hidden, 64, 3, 2, dtype, form, group=64)
    x = torch.empty(0, hidden, dtype=dtype, device='cuda')
    sel = torch.empty(0, 2, dtype=torch.int64, device='cuda')
    ops = moe.grouped_packed_operands(x)
    assert ops is not None
    torch.cuda.synchronize()
    before = load().llmc_b200_launch_count()
    out = moe_forward(x, sel, torch.empty(0, 2, dtype=dtype, device='cuda'), ops)
    torch.cuda.synchronize()
    assert load().llmc_b200_launch_count() == before
    assert out.shape == (0, hidden) and out.dtype == dtype


@pytest.mark.parametrize('form', ['w4_g128_gidx_f32', 'vllm_w4_sym'])
def test_no_host_sync_on_the_grouped_packed_path(form):
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16, form)
    hs = _x(256, s['hidden'], torch.bfloat16).view(2, 128, -1)
    ref = moe(hs)                                      # warm-up: library load, kernel attributes
    torch.cuda.synchronize()
    assert not module_utils.TIMER.enabled
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = moe(hs)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert torch.equal(out, ref)


def _w3_linear(lin, g):
    N, K = lin.out_features, lin.in_features
    codes = torch.randint(0, 8, (N, K), generator=g, device='cuda', dtype=torch.int32)
    packed = dict(qweight=pack_unsigned_codes(codes, 3, signed=False),
                  scales=(torch.rand(N, K // 128, generator=g, device='cuda') * 0.01).to(torch.bfloat16),
                  zeros=torch.randint(0, 8, (N, K // 128), generator=g, device='cuda').to(torch.bfloat16),
                  bits=3, group=128, dtype=torch.bfloat16)
    m = EffcientFakeQuantLinear(None, None, lin, None, packed=packed)
    m.in_features, m.out_features = K, N
    return m


def _fp8_linear(lin, g):
    N, K = lin.out_features, lin.in_features
    packed = dict(qweight=torch.randn(N, K, generator=g, device='cuda').to(torch.float8_e4m3fn),
                  scales=(torch.rand(N, 1, generator=g, device='cuda') * 0.01).to(torch.bfloat16), zeros=None,
                  bits=8, group=K, dtype=torch.bfloat16)
    m = EffcientFakeQuantLinear(None, None, lin, None, packed=packed)
    m.in_features, m.out_features = K, N
    return m


@pytest.mark.parametrize('case', ['w3', 'fp8', 'a_qdq', 'hooked', 'mixed'])
def test_fallbacks_take_the_loop(case, monkeypatch):
    s = synth.SHAPES['tiny-mixtral']
    dtype = torch.bfloat16
    form = ['w8_channel'] + ['w4_g128_native'] * (s['experts'] - 1) if case == 'mixed' else 'w4_g128_native'
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype, form)
    g = torch.Generator(device='cuda').manual_seed(9)
    ex = moe.experts[1]
    seen = []
    if case == 'w3':
        ex.w3 = _w3_linear(ex.w3, g)
    elif case == 'fp8':
        ex.w2 = _fp8_linear(ex.w2, g)
    elif case == 'a_qdq':
        ex.w1.a_qdq = lambda x, layer: x
    elif case == 'hooked':
        ex.register_forward_hook(lambda m, i, o: seen.append(i[0].clone()))
    T = 300
    x = _x(T, s['hidden'], dtype)
    sel, w = moe.route(x)
    assert moe.grouped_packed_operands(x) is None
    calls = []
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or moe_forward(*a))
    out = moe(x.view(1, T, -1)).view(T, -1)
    assert not calls
    assert torch.equal(out.view(torch.int16), moe.expert_loop(x, sel, w).view(torch.int16))
    if case == 'hooked':
        assert torch.equal(seen[0], x[torch.where(sel == 1)[0]])


def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.expert_loop(x, sel, w).reshape(B, S, H)


def _run_main(monkeypatch, doc, loop):
    from llmc_b200.__main__ import adapt_reference_config, main
    packed_calls = []
    real = module_utils.moe_forward

    def counting(x, sel, w, experts):
        packed_calls.append(isinstance(experts[0][0], PackedOperands))
        return real(x, sel, w, experts)
    monkeypatch.setattr(synth, 'moe_forward', counting)
    if loop:
        monkeypatch.setattr(MixtralSparseMoe, 'forward', _loop_forward)
    cfg = adapt_reference_config(copy.deepcopy(doc), 'tiny-mixtral', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['model']['type'] = 'Mixtral'
    cfg.pop('save', None)
    _, model, report = main(cfg, quiet=True)
    monkeypatch.undo()
    experts = [m for m in model.get_model().modules() if isinstance(m, synth.MixtralExpert)]
    assert experts and all(type(ex.w1) is EffcientFakeQuantLinear and ex.w1.packed for ex in experts)
    return report['ppl_fake_quant'], sum(packed_calls)


@pytest.mark.parametrize('cfg_name', ['gptq_w_only.yml', 'rtn_w8a16_per_channel.yml'])
def test_end_to_end_fake_quant_perplexity(cfg_name, monkeypatch):
    with open(os.path.join(ROOT, 'configs', cfg_name)) as fh:
        doc = yaml.safe_load(fh)
    ppl1, n1 = _run_main(monkeypatch, doc, loop=False)
    ppl0, n0 = _run_main(monkeypatch, doc, loop=True)
    assert n1 > 0 and n0 == 0                          # the grouped packed path ran, and only there
    assert ppl1 == ppl0
