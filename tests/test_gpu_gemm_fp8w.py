"""The FP8-weight form of the packed GEMM (`llmc_gemm_fp8a16`, `llmc_gemm_fp8a16_gidx`) and the FP8
recipes' fake-quant deploy on it.

Kernel: the weight is the e4m3 / e5m2 bytes [N, K] with one scale per row or group.  Every output
must equal `llmc_gemm_bf16` on the weight `llmc_fp8_quant` materialises from the same input, bit for
bit, with the bytes from the same pass's byte mode.  In the group-index form a random group
permutation must equal the materialised weight (W[:, perm] quantised in groups, gathered back with
[:, invperm]), and an identity map the contiguous call.  On an exact grid (power-of-two scales,
small integer activations, bytes that include the saturating values, subnormals and -0) every sum
is exact, so a wrong decode or a wrong group lookup shows as a wrong integer.

End to end: the shipped FP8 YAMLs run through `python -m llmc_b200`'s main() on the tiny models and
are deployed with FP8 linears kept in fp8 and with materialised ones (LLMC_B200_FUSED_DEQUANT=0);
weights, logits, fp32-CE perplexity and the `save_fake` tensors must agree bit for bit.

The argument checks at the top run without a GPU."""
import ctypes
import json
import os
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
GRIDS = ['e4m3', 'e5m2']
FP8 = {'e4m3': torch.float8_e4m3fn, 'e5m2': torch.float8_e5m2}
FMAX = {'e4m3': 448.0, 'e5m2': 57344.0}


# ---- argument checks (CPU) ------------------------------------------------------------------------
def test_fp8_arguments_are_checked_before_launch():
    from llmc_b200 import _lib
    lib = _lib.load()
    f, fg = lib.llmc_gemm_fp8a16, lib.llmc_gemm_fp8a16_gidx
    null, p = ctypes.c_void_p(0), ctypes.c_void_p(256)

    def last():
        return lib.llmc_b200_last_error().decode()

    # x, wq, scales, zeros, qdt, bias, y, M, N, K, group, dtype, e5m2, stream
    assert f(p, p, p, p, 0, null, p, 128, 256, 256, 128, 2, 0, null) == -1
    assert 'zero-point' in last()
    assert f(null, null, null, p, 0, null, null, 0, 256, 256, 128, 2, 0, null) == -1      # before M == 0
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, 128, 2, 2, null) == -1
    assert 'e5m2 must be' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, 96, 2, 1, null) == -1
    assert 'group 96' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, 0, 2, 1, null) == -1
    assert f(p, p, p, null, 0, null, p, 128, 256, 100, 100, 2, 0, null) == -1             # group % 64
    assert f(p, p, p, null, 1, null, p, 128, 256, 256, 128, 2, 0, null) == -1
    assert 'qparam_dtype' in last()
    assert f(ctypes.c_void_p(258), p, p, null, 0, null, p, 128, 256, 256, 128, 2, 0, null) == -4
    assert '16-byte aligned' in last()
    assert f(null, null, null, null, 0, null, null, 0, 256, 256, 128, 2, 0, null) == 0    # M == 0
    # x, wq, scales, zeros, qdt, g_idx, ng, q_t, bias, y, M, N, K, dtype, e5m2, stream
    assert fg(p, p, p, null, 0, null, 2, 1, null, p, 128, 256, 256, 2, 0, null) == -1
    assert 'g_idx is NULL' in last()
    assert fg(p, p, p, p, 0, p, 2, 1, null, p, 128, 256, 256, 2, 0, null) == -1
    assert 'zero-point' in last()
    assert fg(p, p, p, null, 0, p, 2, 1, null, p, 128, 256, 100, 2, 1, null) == -4
    assert 'multiple of 64' in last()
    assert fg(p, p, p, null, 0, p, 0, 1, null, p, 128, 256, 256, 2, 1, null) == -1
    assert 'ng=0' in last()
    assert fg(p, p, p, null, 0, p, 257, 1, null, p, 128, 256, 256, 2, 1, null) == -1
    assert 'ng=257' in last()
    assert fg(p, p, p, null, 0, ctypes.c_void_p(260), 2, 1, null, p, 128, 256, 256, 2, 1, null) == -4
    assert fg(null, null, null, null, 0, p, 2, 1, null, null, 0, 256, 256, 2, 0, null) == 0  # M == 0


@pytest.mark.gpu
def test_fp8_packer_declines_what_the_gemm_does_not_cover():
    """The base w_packed returns None (the layer is materialised as before) for per_block weights,
    clipped layers, K or groups not a multiple of 64 and fp32 weights."""
    from llmc_b200.blockwise import BaseBlockwiseQuantization
    from llmc_b200.quant_float import FloatQuantizer

    class Lin:
        def __init__(self, shape, dtype=torch.bfloat16, **bufs):
            self.weight = torch.nn.Parameter(torch.randn(shape, device='cuda').to(dtype), requires_grad=False)
            for k, v in bufs.items():
                setattr(self, k, v)

    def q(**kw):
        return FloatQuantizer(**dict(dict(bit='e4m3', symmetric=True, granularity='per_channel',
                                          use_qtorch=True), **kw))
    pk = BaseBlockwiseQuantization._fp8_packed
    assert pk(Lin((128, 256)), q(granularity='per_block', block_size=128)) is None
    assert pk(Lin((128, 256), buf_upbound_factor=torch.ones(1)), q()) is None
    assert pk(Lin((128, 96)), q()) is None
    assert pk(Lin((128, 256)), q(granularity='per_group', group_size=32)) is None
    assert pk(Lin((128, 256), dtype=torch.float32), q()) is None
    p = pk(Lin((128, 256)), q(granularity='per_group', group_size=128))
    assert p['qweight'].dtype == torch.float8_e4m3fn and p['scales'].shape == (128, 2) and p['group'] == 128
    p = pk(Lin((128, 256)), q(bit='e5m2', granularity='per_tensor'))
    assert p['qweight'].dtype == torch.float8_e5m2 and p['scales'].dtype == torch.float32
    assert p['scales'].shape == (128, 1) and p['group'] == 256


# ---- kernel, bit for bit (GPU) --------------------------------------------------------------------
def _gen(*key):
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    bad = a.view(torch.int16) != b.view(torch.int16)
    assert not bool(bad.any()), (what, bad.nonzero()[:4].tolist(), int(bad.sum()))


def _quantizer(grid):
    from llmc_b200.quant_float import FloatQuantizer
    return FloatQuantizer(bit=grid, symmetric=True, granularity='per_channel', use_qtorch=True)


def _materialise(w, scales, group, grid, dtype):
    """llmc_fp8_quant's static pass on w [N, K] with scales [N, K/group] (w's dtype, or fp32 on the
    fp32 weight): (fp8 bytes, the QDQ weight in `dtype`) of one and the same pass."""
    q = _quantizer(grid)
    ng = w.shape[1] // group
    s = scales.reshape(-1).contiguous()
    wq = q._run(w, group, 0, s, 2, ng)
    qdq = q._run(w, group, 0, s, 1, ng)
    return wq, qdq.to(dtype)


def _weights(N, K, g):
    """Rows of very different magnitudes, so that some groups saturate the grid relative to others."""
    row = torch.exp(torch.randn(N, 1, generator=g, device='cuda') * 2)
    return torch.randn(N, K, generator=g, device='cuda') * row * 0.02


def _case_from(grid, dtype, native, w32, group, per_tensor=False):
    """-> (bytes, scales [N, ng], group, materialised weight) for one qparam flavour: native scales
    in `dtype` on the `dtype` weight (RTN / SmoothQuant), fp32 scales on the fp32 weight followed by
    the cast to `dtype` (GPTQ).  per_tensor: one absmax, expanded to a scale per row."""
    N, K = w32.shape
    amax = w32.abs().reshape(N, K // group, group).amax(-1).clamp(min=1e-5)
    if per_tensor:
        amax = amax.amax().expand(N, 1).contiguous()
    s32 = amax / FMAX[grid]
    if native:
        wq, ref = _materialise(w32.to(dtype), s32.to(dtype), group, grid, dtype)
        return wq, s32.to(dtype), group, ref
    wq, ref = _materialise(w32, s32, group, grid, dtype)
    return wq, s32, group, ref


def _case(grid, dtype, gran, native, N, K, g):
    group = {'per_tensor': K, 'per_channel': K, 'g64': 64, 'g128': 128}[gran]
    return _case_from(grid, dtype, native, _weights(N, K, g), group, per_tensor=gran == 'per_tensor')


GRANS = ['per_tensor', 'per_channel', 'g64', 'g128']
SHAPES = [(M, K) for K in (64, 4096, 14336) for M in (1, 127, 129, 2048 + 17)]


@pytest.mark.gpu
@pytest.mark.parametrize('transposed', [False, True], ids=['plain', 'transposed'])
@pytest.mark.parametrize('native', [True, False], ids=['q-native', 'q-fp32'])
@pytest.mark.parametrize('gran', GRANS)
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('grid', GRIDS)
def test_fp8w_gemm_equals_the_materialised_weight(grid, dtype, gran, native, transposed):
    """M in {1, 127, 129, 2065} x K in {64, 4096, 14336}, N = 300 (a partial n-tile), with and without
    a bias: llmc_gemm_fp8a16 against llmc_gemm_bf16 on llmc_fp8_quant's QDQ weight."""
    from llmc_b200.module_utils import linear_forward, linear_forward_fp8w
    N = 300
    for i, (M, K) in enumerate(SHAPES):
        if gran == 'g128' and K % 128:
            continue
        g = _gen('fp8w', grid, str(dtype), gran, native, transposed, M, K)
        wq, s, group, ref_w = _case(grid, dtype, gran, native, N, K, g)
        assert wq.dtype == FP8[grid] and s.dtype == (dtype if native else torch.float32)
        x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
        bias = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if i % 2 else None
        ss = s.t().contiguous() if transposed else s
        y = linear_forward_fp8w(x, wq, ss, group, bias=bias, qparams_t=transposed)
        _same(y, linear_forward(x, ref_w, bias), f'{M}x{N}x{K}')


def _perm_case(grid, dtype, native, N, K, group, g):
    """GPTQ's act-order flow: W[:, perm] quantised in contiguous groups, gathered back with
    [:, invperm]; g_idx = invperm // group."""
    perm = torch.randperm(K, generator=g, device='cuda')
    invperm = torch.argsort(perm)
    wp_bytes, s, _, ref_p = _case_from(grid, dtype, native, _weights(N, K, g)[:, perm], group)
    wq = wp_bytes.view(torch.uint8)[:, invperm].view(FP8[grid]).contiguous()
    return wq, s, ref_p[:, invperm].contiguous(), (invperm // group).to(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize('group', [64, 128, 0], ids=['g64', 'g128', 'channel'])
@pytest.mark.parametrize('transposed', [False, True], ids=['plain', 'transposed'])
@pytest.mark.parametrize('native', [True, False], ids=['q-native', 'q-fp32'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('grid', GRIDS)
def test_fp8w_gidx_gemm(grid, dtype, native, transposed, group):
    """A random group permutation equals the materialised weight; an identity map equals the
    contiguous call (M = 200 and N = 300: partial tiles; and a long K)."""
    from llmc_b200.module_utils import linear_forward, linear_forward_fp8w
    for M, N, K in ((200, 300, 512), (129, 129, 4096)):
        group_ = group or K
        g = _gen('fp8w-gidx', grid, str(dtype), native, transposed, group_, M, K)
        wq, s, ref_w, gi = _perm_case(grid, dtype, native, N, K, group_, g)
        x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
        bias = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if native else None
        ss = s.t().contiguous() if transposed else s
        y = linear_forward_fp8w(x, wq, ss, group_, bias=bias, qparams_t=transposed, g_idx=gi)
        _same(y, linear_forward(x, ref_w, bias), f'perm {M}x{N}x{K}')
        wq, s, _, ref_w = _case_from(grid, dtype, native, _weights(N, K, g), group_)
        ident = (torch.arange(K, device='cuda') // group_).to(torch.int32)
        ss = s.t().contiguous() if transposed else s
        y = linear_forward_fp8w(x, wq, ss, group_, bias=bias, qparams_t=transposed, g_idx=ident)
        _same(y, linear_forward_fp8w(x, wq, s, group_, bias=bias), f'identity {M}x{N}x{K}')
        _same(y, linear_forward(x, ref_w, bias), f'identity vs materialised {M}x{N}x{K}')


def _window_bytes(grid, large, shape, g):
    """Random bytes of one magnitude window: 'small' = exponent fields 0..2 (subnormals, +-0, -0 and
    the smallest normals), 'large' = the top three exponent fields up to the saturating value."""
    mbits = 3 if grid == 'e4m3' else 2
    top = 15 if grid == 'e4m3' else 30
    exps = list(range(top - 2, top + 1)) if large else [0, 1, 2]
    vals = []
    for e in exps:
        for m in range(1 << mbits):
            b = (e << mbits) | m
            if grid == 'e4m3' and b == 0x7F:           # NaN
                continue
            vals += [b, 0x80 | b]
    vals = torch.tensor(vals, dtype=torch.int32, device='cuda')
    out = vals[torch.randint(0, len(vals), shape, generator=g, device='cuda')].to(torch.uint8)
    sat = 0x7E if grid == 'e4m3' else 0x7B                 # +448 / +57344
    if large:
        out[:, 0], out[:, 1] = sat, 0x80 | sat
    else:
        out[:, 0], out[:, 1], out[:, 2] = 0x80, 0x01, 0x81      # -0 and the smallest subnormals
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('native', [True, False], ids=['q-native', 'q-fp32'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('grid', GRIDS)
def test_fp8w_gemm_on_an_exact_grid(grid, dtype, native):
    """Rows alternate between a small-magnitude and a large-magnitude byte window (each spans at most
    6 significant bits), scales are powers of two per (row, group), activations integers in [-8, 8]:
    every dequantised weight is exact in the 16-bit dtype and every partial sum below 2^21 units, so
    the output is one rounding of the exact fp64 product (compared by value: an exact zero may come
    out of the tensor cores as -0).  Both the contiguous and the group-index form."""
    from llmc_b200.module_utils import linear_forward_fp8w
    M, N, K, group = 200, 300, 512, 64
    ng = K // group
    g = _gen('fp8w-exact', grid, str(dtype), native)
    large = torch.arange(N, device='cuda') % 2 == 1
    b = torch.where(large[:, None], _window_bytes(grid, True, (N, K), g), _window_bytes(grid, False, (N, K), g))
    wq = b.view(FP8[grid])
    e = torch.randint(-2, 2, (N, ng), generator=g, device='cuda')
    if dtype == torch.float16:                       # large weights and their sums stay finite in fp16
        e = torch.where(large[:, None], e - (6 if grid == 'e4m3' else 12), e)
    s = ((e + 1023) << 52).view(torch.float64)                  # 2^e from its bits: exact
    x = torch.randint(-8, 9, (M, K), generator=g, device='cuda').double()
    qdt = dtype if native else torch.float32
    for kind in ('contiguous', 'perm'):
        if kind == 'perm':
            gi = (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
        else:
            gi = (torch.arange(K, device='cuda') // group).to(torch.int32)
        # the reference on the host: fp64 products and sums, then the two roundings
        w = wq.cpu().double() * s.cpu()[:, gi.long().cpu()]
        assert torch.equal(w.to(dtype).double(), w)               # exact in the 16-bit dtype
        exact = (x.cpu() @ w.t()).to(torch.float32).to(dtype).cuda()
        y = linear_forward_fp8w(x.to(dtype), wq, s.to(qdt), group, g_idx=gi if kind == 'perm' else None)
        bad = y != exact
        assert not bool(bad.any()), (kind, [(i, y[tuple(i)].item(), exact[tuple(i)].item())
                                            for i in bad.nonzero()[:4].tolist()])
    # a wrong lookup would show: the same data with contiguous groups gives other integers
    assert not torch.equal(linear_forward_fp8w(x.to(dtype), wq, s.to(qdt), group), exact)


@pytest.mark.gpu
def test_fp8w_zero_scale_dequantises_with_one():
    """A scale of 0 (an fp16 scale that underflowed) is read as 1, like llmc_fp8_quant's QDQ."""
    from llmc_b200.module_utils import linear_forward, linear_forward_fp8w
    N, K = 256, 256
    g = _gen('fp8w-zero')
    w = (torch.randn(N, K, generator=g, device='cuda') * 1e-6).half()
    s = (w.float().abs().amax(-1, keepdim=True) / 448).half()
    s[::3] = 0
    wq, ref = _materialise(w, s, K, 'e4m3', torch.float16)
    x = torch.randn(64, K, generator=g, device='cuda').half()
    _same(linear_forward_fp8w(x, wq, s, K), linear_forward(x, ref), 'zero scales')


# ---- FP8 recipes end to end (GPU) -------------------------------------------------------------------
def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


def _gptq_e5m2_g128_actorder():
    doc = _yaml('backend/vllm/fp8/gptq_fp8.yml')
    doc['quant']['weight'] = dict(doc['quant']['weight'], bit='e5m2', granularity='per_group', group_size=128)
    doc['quant'].pop('act')
    return doc


def _rtn_static_mixtral():
    import yaml
    with open(os.path.join(ROOT, 'configs', 'rtn_fp8_static_mixtral.yml')) as fh:
        return yaml.safe_load(fh)


E2E = {f'{be}/{algo}': (lambda be=be, algo=algo: _yaml(f'backend/{be}/fp8/{algo}_fp8.yml'), 'tiny-llama')
       for be in ('vllm', 'sglang') for algo in ('rtn', 'smoothquant', 'gptq')}
E2E['gptq_e5m2_g128_actorder'] = (_gptq_e5m2_g128_actorder, 'tiny-llama')
E2E['rtn_fp8_static_mixtral'] = (_rtn_static_mixtral, 'tiny-mixtral')


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(E2E))
def test_fp8_recipes_deploy_fp8_linears(name, tmp_path):
    from safetensors.torch import load_file
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.export import save_model
    from llmc_b200.module_utils import EffcientFakeQuantLinear
    from llmc_b200.synth import SynthModel, perplexity
    make, shape = E2E[name]
    doc = make()
    doc.pop('save', None)
    cfg = adapt_reference_config(doc, shape, n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['eval']['eval_pos'] = []                       # calibrate only; deployed twice below
    algo, model, _ = main(cfg, quiet=True)
    wq = algo.wquantizer
    assert type(wq).__name__ == 'FloatQuantizer'
    blocks = model.get_blocks()
    calibrated = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    w_qdq = {k: algo.w_qdq(m, wq) for k, m in calibrated.items()}
    dtype = next(iter(w_qdq.values())).dtype
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(4))

    def deploy(fused):
        for (i, n), m in calibrated.items():
            SynthModel._set(blocks[i], n, m)
        os.environ['LLMC_B200_FUSED_DEQUANT'] = fused
        try:
            algo.deploy('fake_quant')
        finally:
            os.environ.pop('LLMC_B200_FUSED_DEQUANT', None)
        mods = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
        logits = model.logits(tokens[:, :128 * 2].view(2, 128))
        ppl = perplexity(model, tokens, 128, ce_dtype=torch.float32)
        path = os.path.join(str(tmp_path), f'fused{fused}')
        save_model(model, path)
        return mods, logits, ppl, load_file(os.path.join(path, 'model.safetensors'))

    mods, logits, ppl, saved = deploy('1')
    bits = n_weights = 0
    for k, m in mods.items():
        assert isinstance(m, EffcientFakeQuantLinear) and m.packed, k
        assert 'weight' not in m._buffers, k                       # no dense weight kept
        assert m.qweight.dtype == FP8[wq.bit] and m.q_grid == wq.bit and m.qzeros is None, k
        assert (m.g_idx is not None) == bool(getattr(algo, 'need_perm', False)), k
        _same(m.weight, w_qdq[k], f'{k} .weight vs w_qdq')
        R, K = m.out_features, m.in_features
        ng = m.qscales.numel() // R
        assert m.qweight.numel() == R * K
        bits += 8 * R * K + 8 * m.qscales.element_size() * R * ng
        n_weights += R * K
    bpw = bits / n_weights
    print(f'\n{name}: fp8 bytes + scales = {bpw:.4f} bits per weight ({dtype} weight: 16)')
    mods0, logits0, ppl0, saved0 = deploy('0')
    for k, m in mods0.items():
        assert not m.packed and m.weight.dtype == dtype, k
        _same(m.weight, w_qdq[k], f'{k} materialised .weight vs w_qdq')
    _same(logits, logits0, 'logits')
    assert ppl == ppl0, (ppl, ppl0)
    assert sorted(saved) == sorted(saved0)
    for n in saved0:
        assert saved[n].dtype == saved0[n].dtype and torch.equal(saved[n], saved0[n]), n
