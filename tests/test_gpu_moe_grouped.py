"""GPU: the Mixtral sparse-MoE layer on the grouped expert GEMMs (module_utils.moe_forward) gives the
bits of the per-expert loop (MixtralSparseMoe.expert_loop), issues no host sync, and leaves hooked
experts to the loop; AWQ and GPTQ block loops give the same results either way."""
import copy

import pytest
import torch

from llmc_b200 import module_utils, synth
from llmc_b200.module_utils import FakeQuantLinear, moe_forward
from llmc_b200.synth import MixtralSparseMoe

pytestmark = pytest.mark.gpu


def _moe(hidden, inter, E, k, dtype, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = MixtralSparseMoe(hidden, inter, E, k)
    moe = moe.to(dtype).to_empty(device='cuda')
    for p in moe.parameters():
        p.data.normal_(0, 0.02, generator=g)
    return moe


def _x(T, hidden, dtype, seed=1):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(T, hidden, device='cuda', generator=g).to(dtype)


def _weights(T, k, dtype, seed=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    w = torch.rand(T, k, device='cuda', generator=g) + 0.05
    return (w / w.sum(dim=1, keepdim=True)).to(dtype)


def _sel_from_sizes(sizes, k_other, seed=3):
    """k = 2 routing whose slot 0 gives expert e exactly sizes[e] tokens and whose slot 1 is expert
    k_other for every token (the tokens shuffled)."""
    sel0 = torch.cat([torch.full((n,), e, dtype=torch.int64) for e, n in enumerate(sizes)])
    sel0 = sel0[torch.randperm(sel0.numel(), generator=torch.Generator().manual_seed(seed))]
    return torch.stack([sel0, torch.full_like(sel0, k_other)], dim=1).cuda()


def _check(moe, x, sel, w):
    weights = moe.grouped_weights(x)
    assert weights is not None
    got = moe_forward(x, sel, w, weights)
    ref = moe.expert_loop(x, sel, w)
    assert got.dtype == ref.dtype and got.shape == ref.shape
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
    return got


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_segment_sizes_and_one_expert(dtype):
    E, hidden, inter = 8, 256, 512
    moe = _moe(hidden, inter, E, 2, dtype)
    sizes = [0, 1, 63, 64, 127, 128, 129]       # expert 7 takes slot 1 of every token
    sel = _sel_from_sizes(sizes, 7)
    T = sel.shape[0]
    _check(moe, _x(T, hidden, dtype), sel, _weights(T, 2, dtype))
    # every token on expert 3 (slot 0), the rest of the experts on slot 1; T not a multiple of 128
    T = 1000
    other = torch.randint(0, E - 1, (T,), generator=torch.Generator().manual_seed(4))
    sel = torch.stack([torch.full((T,), 3), other + (other >= 3).long()], dim=1).cuda()
    _check(moe, _x(T, hidden, dtype), sel, _weights(T, 2, dtype))
    # top-1: every token on one expert
    moe1 = _moe(hidden, inter, E, 1, dtype)
    sel = torch.full((T, 1), 5, dtype=torch.int64, device='cuda')
    _check(moe1, _x(T, hidden, dtype), sel, torch.ones(T, 1, dtype=dtype, device='cuda'))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('T', [1, 77, 300])
def test_tiny_mixtral_module_forward(dtype, T):
    """The module forward (router included) on tiny-mixtral, grouped path against the loop."""
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype)
    hs = _x(T, s['hidden'], dtype).view(1, T, -1)
    sel, w = moe.route(hs.view(T, -1))
    _check(moe, hs.view(T, -1), sel, w)
    out = moe(hs)
    assert torch.equal(out.view(T, -1).view(torch.int16),
                       moe.expert_loop(hs.view(T, -1), sel, w).view(torch.int16))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_mixtral_8x7b_layer_2048_tokens(dtype):
    s = synth.SHAPES['mixtral-8x7b']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype)
    T = 2048
    x = _x(T, s['hidden'], dtype)
    sel, w = moe.route(x)
    _check(moe, x, sel, w)
    # the same layer with a skewed routing: segments 0, 1, 63, 64, 127, 128, 129 and the rest
    sizes = [0, 1, 63, 64, 127, 128, 129]
    sel = _sel_from_sizes(sizes + [0], 7)
    sel = torch.cat([sel, torch.stack([torch.full((T - sel.shape[0],), 2, device='cuda'),
                                       torch.full((T - sel.shape[0],), 7, device='cuda')], 1)])
    _check(moe, x, sel, w)
    del moe
    torch.cuda.empty_cache()


# expert counts below 8 and top_k up to E, at widths with a K tail (264), a partial 256-column
# n-tile of the down projection (264, 320) and one gate/up n-tile (inter 128)
EXPERTS_TOP_K = [(1, 1), (2, 1), (2, 2), (3, 2), (3, 3), (5, 3), (5, 5), (8, 3), (8, 8)]


def _sel_random(T, E, k, seed=5):
    """Each token's k distinct experts, in random order."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, E, generator=g).argsort(dim=1)[:, :k].cuda()


@pytest.mark.parametrize('hidden,inter', [(264, 128), (320, 384), (4096, 128)])
@pytest.mark.parametrize('E,k', EXPERTS_TOP_K)
def test_expert_counts_top_k_and_widths(E, k, hidden, inter):
    dtype = torch.bfloat16 if (E + k) % 2 else torch.float16
    moe = _moe(hidden, inter, E, k, dtype)
    T = 200
    _check(moe, _x(T, hidden, dtype), _sel_random(T, E, k), _weights(T, k, dtype))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_zero_tokens_launch_nothing(dtype):
    from llmc_b200._lib import load
    hidden = 264
    moe = _moe(hidden, 128, 3, 2, dtype)
    x = torch.empty(0, hidden, dtype=dtype, device='cuda')
    sel = torch.empty(0, 2, dtype=torch.int64, device='cuda')
    torch.cuda.synchronize()
    before = load().llmc_b200_launch_count()
    out = moe_forward(x, sel, torch.empty(0, 2, dtype=dtype, device='cuda'), moe.grouped_weights(x))
    torch.cuda.synchronize()
    assert load().llmc_b200_launch_count() == before
    assert out.shape == (0, hidden) and out.dtype == dtype


def test_no_host_sync_on_the_grouped_path():
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16)
    hs = _x(256, s['hidden'], torch.bfloat16).view(2, 128, -1)
    ref = moe(hs)                                  # warm-up: library load, kernel attributes
    torch.cuda.synchronize()
    assert not module_utils.TIMER.enabled
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = moe(hs)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert torch.equal(out, ref)


def test_fake_quant_experts():
    """FakeQuantLinear experts (dense tmp_weight) take the grouped path with the same bits."""
    from llmc_b200.quant import IntegerQuantizer
    q = IntegerQuantizer(4, True, 'per_group', group_size=128)

    def w_qdq(layer):
        return q.fake_quant_weight_dynamic(layer.weight)
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16)
    for ex in moe.experts:
        for n in ('w1', 'w2', 'w3'):
            setattr(ex, n, FakeQuantLinear.new(getattr(ex, n), w_qdq, None))
    x = _x(500, s['hidden'], torch.bfloat16)
    sel, w = moe.route(x)
    weights = moe.grouped_weights(x)
    assert weights is not None and weights[0][0] is moe.experts[0].w1.tmp_weight
    assert not torch.equal(moe.experts[0].w1.tmp_weight, moe.experts[0].w1.weight)
    _check(moe, x, sel, w)


def test_hooked_expert_takes_the_loop_and_sees_its_tokens():
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16)
    T = 300
    x = _x(T, s['hidden'], torch.bfloat16)
    sel, w = moe.route(x)
    ref = moe_forward(x, sel, w, moe.grouped_weights(x))
    for target in ('w1', None):
        seen = []
        mod = moe.experts[1] if target is None else moe.experts[1].w1
        h = mod.register_forward_hook(lambda m, i, o: seen.append(i[0].clone()))
        try:
            assert moe.grouped_weights(x) is None
            out = moe(x.view(1, T, -1)).view(T, -1)
        finally:
            h.remove()
        tok = torch.where(sel == 1)[0]
        assert len(seen) == 1 and torch.equal(seen[0], x[tok])
        assert torch.equal(out, ref)
    assert moe.grouped_weights(x) is not None


def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.expert_loop(x, sel, w).reshape(B, S, H)


def _state(model):
    m = model.get_model()
    return {n: t.detach().clone() for n, t in list(m.named_parameters()) + list(m.named_buffers())}


def _assert_same(a, b):
    assert set(a) == set(b)
    for n in a:
        assert torch.equal(a[n], b[n]), n


def _run_awq(monkeypatch, loop):
    from llmc_b200.awq import Awq
    from llmc_b200.blockwise import AttrDict
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    if loop:
        monkeypatch.setattr(MixtralSparseMoe, 'forward', _loop_forward)
    cfg = {'calib': {'seq_len': 64},
           'quant': {'method': 'Awq',
                     'weight': {'bit': 4, 'symmetric': True, 'granularity': 'per_group', 'group_size': 128},
                     'special': {'trans': True, 'trans_version': 'v2', 'weight_clip': True,
                                 'clip_sym': True}}}
    model = synth.SynthModel('tiny-mixtral', n_layers=1, seed=0, device='cuda', outlier_seed=3,
                             with_head=False)
    inp = model.first_block_input(8, 64, bs=-1, seed=1, device='cuda')
    c = AttrDict.wrap(copy.deepcopy(cfg))
    algo = Awq(model, c.quant, inp, None, c)
    algo.run_block_loop()
    torch.cuda.synchronize()
    monkeypatch.undo()
    out = [t.clone() for t in algo.input['data']]
    return _state(model), {k: v.clone() for k, v in algo.search_log.items()}, out, len(calls)


def test_awq_block_loop_grouped_equals_loop(monkeypatch):
    s1, log1, out1, n1 = _run_awq(monkeypatch, loop=False)
    s0, log0, out0, n0 = _run_awq(monkeypatch, loop=True)
    assert n1 > 0 and n0 == 0
    _assert_same(s1, s0)
    assert set(log1) == set(log0)
    for k in log1:
        assert torch.equal(log1[k], log0[k]), k
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        assert torch.equal(a, b)


def _run_gptq(monkeypatch, loop):
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.gptq import GPTQ
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or real(*a))
    if loop:
        monkeypatch.setattr(MixtralSparseMoe, 'forward', _loop_forward)
    cfg = AttrDict.wrap({'base': {'seed': 0},
                         'quant': {'method': 'GPTQ', 'quant_out': True,
                                   'weight': {'bit': 4, 'symmetric': False, 'granularity': 'per_group',
                                              'group_size': 128},
                                   'special': {'actorder': True, 'static_groups': False, 'percdamp': 0.01,
                                               'blocksize': 128, 'true_sequential': True}}})
    model = synth.SynthModel('tiny-mixtral', n_layers=1, seed=0, device='cuda', with_head=False)
    inp = model.first_block_input(6, 96, bs=2, device='cuda')
    algo = GPTQ(model, cfg.quant, inp, None, cfg)
    algo.run_block_loop()
    algo.check_factorizations(wait=True)
    torch.cuda.synchronize()
    monkeypatch.undo()
    out = algo.input.get('stacked')
    out = [t.clone() for t in algo.input['data']] if out is None else [out.clone()]
    return _state(model), out, len(calls)


def test_gptq_block_loop_grouped_equals_loop(monkeypatch):
    s1, out1, n1 = _run_gptq(monkeypatch, loop=False)
    s0, out0, n0 = _run_gptq(monkeypatch, loop=True)
    assert n1 > 0 and n0 == 0
    _assert_same(s1, s0)
    assert len(out1) == len(out0)
    for a, b in zip(out1, out0):
        assert torch.equal(a, b)
