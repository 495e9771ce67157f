"""GPU: the forward GEMM with the block glue in its epilogue (llmc_gemm_rope_qkv, llmc_gemm_swiglu,
llmc_gemm_residual) bit for bit against the unfused composition — llmc_gemm_bf16 followed by
llmc_rope / llmc_silu_mul / llmc_add — at M tails, several samples per chunk, fp16 overflow and in
place; and one progressive GPTQ block at a shape the fused path accepts against the same block with
the fused path disabled."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

DT16 = [torch.bfloat16, torch.float16]


def _bits(a, b, what=''):
    """The same bits, or both NaN."""
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape)
    ok = (a.view(torch.int16) == b.view(torch.int16)) | (torch.isnan(a) & torch.isnan(b))
    assert bool(ok.all()), f'{what}: {int((~ok).sum())}/{ok.numel()} elements differ'


def _rand(shape, scale, seed, dtype):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(shape, generator=g, device='cuda') * scale).to(dtype)


@pytest.mark.parametrize('dtype', DT16)
@pytest.mark.parametrize('B,S,K,n_q,n_k,n_v', [
    (3, 200, 512, 512, 256, 256),      # 600 rows: an M tail, three samples per chunk
    (1, 64, 136, 256, 512, 136),       # one partial m-tile, v narrower than a tile
    (2, 384, 4096, 1024, 256, 264),    # k wider than q's tile, a v column tail
])
def test_rope_qkv_matches_gemm_then_rope(dtype, B, S, K, n_q, n_k, n_v):
    from llmc_b200 import block_ops
    from llmc_b200.module_utils import gemm_rope_qkv, linear_forward
    from llmc_b200.synth import rope_cos_sin
    x = _rand((B, S, K), 1.0, 0, dtype)
    w = _rand((n_q + n_k + n_v, K), 0.05, 1, dtype)
    cos, sin = rope_cos_sin(S + 7, 128, 'cuda', dtype)          # longer tables, sliced as attend does
    q, k, v = gemm_rope_qkv(x, w, n_q, n_k, cos[:S], sin[:S])
    y = linear_forward(x, w)
    rq, rk = y[..., :n_q].contiguous(), y[..., n_q:n_q + n_k].contiguous()
    block_ops.rope_(rq, cos[:S], sin[:S], n_q // 128, 128)
    block_ops.rope_(rk, cos[:S], sin[:S], n_k // 128, 128)
    _bits(q, rq, 'q')
    _bits(k, rk, 'k')
    _bits(v, y[..., n_q + n_k:].contiguous(), 'v')


@pytest.mark.parametrize('dtype', DT16)
@pytest.mark.parametrize('M,K,inter,scale', [
    (700, 512, 1024, 1.0),            # an M tail
    (128, 264, 128, 1.0),             # one tile
    (300, 512, 384, 40.0),            # fp16: gate / up near and past overflow (inf; silu(-inf) NaN)
])
def test_swiglu_matches_gemm_then_silu_mul(dtype, M, K, inter, scale):
    from llmc_b200 import block_ops
    from llmc_b200.module_utils import gemm_swiglu, interleave_gate_up, linear_forward
    x = _rand((M, K), scale, 2, dtype)
    ws = 0.05 * scale ** 2
    wg, wu = _rand((inter, K), ws, 3, dtype), _rand((inter, K), ws, 4, dtype)
    g, u = linear_forward(x, wg), linear_forward(x, wu)
    if scale > 1 and dtype == torch.float16:
        big = (g.abs() > 30000) & torch.isfinite(g)
        assert bool(torch.isinf(g).any()) and bool(big.any())
        assert bool(torch.isnan(block_ops.silu_mul(g, u)).any())
    ref = block_ops.silu_mul(g, u)
    out = torch.full((M, inter), float('nan'), dtype=dtype, device='cuda')
    got = gemm_swiglu(x, interleave_gate_up(wg, wu), out=out)
    assert got is out
    _bits(got, ref, 'act')


@pytest.mark.parametrize('dtype', DT16)
@pytest.mark.parametrize('M,K,N', [(600, 512, 512), (64, 136, 264), (1000, 1024, 4096)])
@pytest.mark.parametrize('in_place', [False, True])
def test_residual_matches_gemm_then_add(dtype, M, K, N, in_place):
    from llmc_b200 import block_ops
    from llmc_b200.module_utils import linear_forward, linear_forward_residual
    x, w = _rand((M, K), 1.0, 5, dtype), _rand((N, K), 0.05, 6, dtype)
    res = _rand((M, N), 1.0, 7, dtype)
    ref = block_ops.add(res, linear_forward(x, w))
    out = res if in_place else torch.empty_like(res)
    assert linear_forward_residual(x, w, res, out) is out
    _bits(out, ref, 'h')


def test_entry_points_refuse_what_they_cannot_fuse():
    from llmc_b200 import _lib
    from llmc_b200.module_utils import gemm_rope_qkv, gemm_swiglu, linear_forward_residual
    from llmc_b200.synth import rope_cos_sin
    dt = torch.bfloat16
    x = _rand((1, 64, 128), 1.0, 8, dt)
    cos, sin = rope_cos_sin(64, 128, 'cuda', dt)
    with pytest.raises(_lib.LlmcB200Error, match='multiples of 256'):
        gemm_rope_qkv(x, _rand((128 + 256 + 128, 128), 1.0, 9, dt), 128, 256, cos, sin)
    with pytest.raises(_lib.LlmcB200Error, match='multiple of 128'):
        gemm_swiglu(x, _rand((2 * 200, 128), 1.0, 9, dt))
    with pytest.raises(_lib.LlmcB200Error, match='multiple of 8'):
        w = _rand((12, 128), 1.0, 9, dt)
        r = torch.zeros((1, 64, 12), dtype=dt, device='cuda')
        linear_forward_residual(x, w, r, r)


FUSED_SHAPE = dict(hidden=512, inter=1024, layers=2, heads=4, kv_heads=2, vocab=512, kind='llama',
                   dtype=torch.bfloat16)
GPTQ_CFG = {
    'base': {'seed': 0},
    'quant': {'method': 'GPTQ',
              'weight': {'bit': 4, 'symmetric': False, 'granularity': 'per_group', 'group_size': 128},
              'special': {'actorder': True, 'static_groups': False, 'percdamp': 0.01,
                          'blocksize': 128, 'true_sequential': True},
              'quant_out': True},
}


def _progressive_block(monkeypatch, fused):
    """Calibrate block 0 of the FUSED_SHAPE model on 20 samples of 128 tokens (two chunks, the second
    partial) with the progressive schedule; returns what it left and every Hessian it accumulated."""
    from llmc_b200 import gptq, module_utils, synth
    from llmc_b200.blockwise import AttrDict
    monkeypatch.setitem(synth.SHAPES, 'fused-llama', FUSED_SHAPE)
    calls = {'rope_qkv': 0, 'swiglu': 0, 'residual': 0}

    def spy(name, fn):
        def wrapped(*a, **kw):
            calls[name] += 1
            return fn(*a, **kw)
        return wrapped
    monkeypatch.setattr(synth, 'gemm_rope_qkv', spy('rope_qkv', synth.gemm_rope_qkv))
    monkeypatch.setattr(synth, 'gemm_swiglu', spy('swiglu', synth.gemm_swiglu))
    monkeypatch.setattr(module_utils, 'linear_forward_residual',
                        spy('residual', module_utils.linear_forward_residual))
    if not fused:
        monkeypatch.setattr(synth.LlamaAttention, 'fused_qkv_weight', lambda self, dtype: None)
        monkeypatch.setattr(synth.LlamaMLP, 'fused_gate_up_weight', lambda self, dtype: None)
        monkeypatch.setattr(module_utils, 'dense_forward_weight', lambda layer, dtype: None)
    hessians = []
    add_batch = gptq.ops.hessian_add_batch

    def record(H, n, x):
        out = add_batch(H, n, x)
        hessians.append(H.clone())
        return out
    monkeypatch.setattr(gptq.ops, 'hessian_add_batch', record)
    model = synth.SynthModel('fused-llama', n_layers=1, seed=0, device='cuda', outlier_seed=3,
                             with_head=False)
    inp = model.first_block_input(20, 128, bs=1, seed=1, device='cuda')
    c = AttrDict.wrap(copy.deepcopy(GPTQ_CFG))
    algo = gptq.GPTQ(model, c.quant, inp, None, c)
    block = model.get_blocks()[0]
    assert algo.progressive_ok(block)
    algo.block_idx = 0
    algo.block_opt(block)
    algo.check_factorizations(wait=True)
    monkeypatch.undo()
    return block, algo, hessians, calls


def test_progressive_block_fused_equals_unfused(monkeypatch):
    b1, a1, h1, calls1 = _progressive_block(monkeypatch, fused=True)
    b0, a0, h0, calls0 = _progressive_block(monkeypatch, fused=False)
    assert calls1 == {'rope_qkv': 2, 'swiglu': 2, 'residual': 4}, calls1
    assert calls0 == {'rope_qkv': 0, 'swiglu': 0, 'residual': 0}, calls0
    assert len(h1) == len(h0) == 4
    for i, (x, y) in enumerate(zip(h1, h0)):
        assert torch.equal(x, y), f'Hessian of subset {i}'
    _bits(a1.input['stacked'], a0.input['stacked'], 'block output')
    t1 = dict(list(b1.named_parameters()) + list(b1.named_buffers()))
    t0 = dict(list(b0.named_parameters()) + list(b0.named_buffers()))
    assert set(t1) == set(t0)
    for n, t in t1.items():
        assert torch.equal(t, t0[n]), n
    assert set(a1.losses) == set(a0.losses)
    for k in a1.losses:
        assert torch.equal(a1.losses[k], a0.losses[k]), k
