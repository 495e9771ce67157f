"""The group-index form of the packed W4/W8 GEMM (`llmc_gemm_w4a16_gidx`, `llmc_gemm_w8a16_gidx`) and
GPTQ's fake-quant deploy on it.

Kernel: column k dequantises with the qparams of group g_idx[k].  Every output must equal
`llmc_gemm_bf16` on the weight materialised from the same codes, qparams and g_idx, bit for bit; an
identity map must also equal the contiguous `llmc_gemm_w4a16` / `w8a16` call.  On the exact integer
grid (small codes, power-of-two scales that differ per group, integer activations) every sum is
exact, so a wrong group lookup shows as a wrong integer.

GPTQ end to end: the tiny Llama calibrated through `python -m llmc_b200`'s main() is deployed with
packed linears and with materialised ones (LLMC_B200_FUSED_DEQUANT=0); the weights, logits and
fp32-CE perplexity must agree bit for bit, and each deployed `.weight` must equal GPTQ.w_qdq of the
calibrated layer.

The argument checks at the top run without a GPU."""
import ctypes
import json
import os
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]


# ---- argument checks (CPU) ------------------------------------------------------------------------
@pytest.mark.parametrize('bits', [4, 8])
def test_gidx_arguments_are_checked_before_launch(bits):
    from llmc_b200 import _lib
    lib = _lib.load()
    f = getattr(lib, f'llmc_gemm_w{bits}a16_gidx')
    null, p = ctypes.c_void_p(0), ctypes.c_void_p(256)

    def last():
        return lib.llmc_b200_last_error().decode()

    # x, wq, scales, zeros, qdt, g_idx, ng, q_t, bias, y, M, N, K, dtype, stream
    assert f(p, p, p, null, 0, null, 2, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'g_idx is NULL' in last()
    assert f(p, p, p, null, 0, p, 2, 1, null, p, 128, 256, 100, 2, null) == -4
    assert 'multiple of 64' in last()
    assert f(p, p, p, null, 0, p, 0, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=0' in last()
    assert f(p, p, p, null, 0, p, 257, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=257' in last()
    assert f(p, p, p, null, 1, p, 2, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'qparam_dtype' in last()
    assert f(null, null, null, null, 0, null, 2, 1, null, null, 0, 256, 256, 2, null) == -1   # g_idx first
    assert f(null, null, null, null, 0, p, 2, 1, null, null, 0, 256, 256, 2, null) == 0       # M == 0


# ---- kernel, bit for bit (GPU) --------------------------------------------------------------------
def _gen(*key):
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def _gidx(kind, K, group, g):
    ng = K // group
    if kind == 'perm':                      # GPTQ act-order: invperm // group
        return (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
    if kind == 'one-group':
        return torch.full((K,), ng - 1, dtype=torch.int32, device='cuda')
    return (torch.arange(K, device='cuda') // group).to(torch.int32)


def _materialise(codes, s, z, gi, bits, dtype):
    """rT((code - zero) * scale) in the qparam dtype's arithmetic (fp32 products), as GPTQ.w_qdq."""
    gl = gi.long()
    zz = z.float()[:, gl] if z is not None else float(1 << (bits - 1))
    return ((codes.float() - zz) * s.float()[:, gl]).to(dtype)


def _pack(codes, bits):
    from llmc_b200.module_utils import pack_unsigned_codes
    return pack_unsigned_codes(codes, bits, signed=False)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    iv = torch.int16
    bad = a.view(iv) != b.view(iv)
    assert not bool(bad.any()), (what, bad.nonzero()[:4].tolist(), int(bad.sum()))


GROUPS = [64, 128, 0]       # 0: per-channel (group = K)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['perm', 'one-group', 'identity'])
@pytest.mark.parametrize('group', GROUPS, ids=['g64', 'g128', 'channel'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('sym', [False, True], ids=['asym', 'sym'])
@pytest.mark.parametrize('bits', [4, 8])
def test_gidx_gemm_equals_the_materialised_weight(bits, sym, native, dtype, group, kind):
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    M, N, K = 200, 300, 512                 # partial M and N tiles
    group = group or K
    ng = K // group
    g = _gen('gidx', bits, sym, native, str(dtype), group, kind)
    qdt = dtype if native else torch.float32
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s = (torch.rand(N, ng, generator=g, device='cuda') * 0.004 + 0.001).to(qdt)
    z = None if sym else torch.randint(0, 1 << bits, (N, ng), generator=g, device='cuda').to(qdt)
    gi = _gidx(kind, K, group, g)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    bias = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if sym == native else None
    transposed = group == 128               # both qparam layouts
    ss = s.t().contiguous() if transposed else s
    zz = (z.t().contiguous() if transposed else z) if z is not None else None
    packed = _pack(codes, bits)
    y = linear_forward_w4(x, packed, ss, zz, group, bias=bias, bits=bits, qparams_t=transposed, g_idx=gi)
    ref = linear_forward(x, _materialise(codes, s, z, gi, bits, dtype), bias)
    _same(y, ref, 'gidx vs materialised')
    if kind == 'identity':
        _same(y, linear_forward_w4(x, packed, s, z, group, bias=bias, bits=bits), 'gidx vs contiguous')


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K', [(1, 128, 256), (1, 300, 1024), (1100, 2100, 256), (129, 129, 4096)],
                         ids=['one-row', 'one-row-partial-n', 'persistent-loop', 'long-k'])
@pytest.mark.parametrize('bits', [4, 8])
def test_gidx_gemm_shapes(bits, M, N, K):
    """A single row, more tiles than CTAs (153 tiles on 132 SMs), and a long K with 32 groups."""
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    group = 128
    ng = K // group
    g = _gen('gidx-shape', bits, M, N, K)
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s = torch.rand(N, ng, generator=g, device='cuda') * 0.004 + 0.001
    z = torch.randint(0, 1 << bits, (N, ng), generator=g, device='cuda').float()
    gi = _gidx('perm', K, group, g)
    x = torch.randn(M, K, generator=g, device='cuda').bfloat16()
    y = linear_forward_w4(x, _pack(codes, bits), s.t().contiguous(), z.t().contiguous(), group, bits=bits,
                          qparams_t=True, g_idx=gi)
    _same(y, linear_forward(x, _materialise(codes, s, z, gi, bits, torch.bfloat16)), f'{M}x{N}x{K}')


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('bits', [4, 8])
def test_gidx_gemm_on_the_exact_integer_grid(bits, native, dtype):
    """The integer grid of test_gpu_gemm_paths.py: codes and zero-points in [0, 2^bits), scales
    2^-3 .. 2^1 chosen per (row, group), integer activations small enough that every partial sum is
    below 2^24 units of 2^-3.  Every dequantised weight is exact in the 16-bit dtype and every sum
    exact in fp32, so the output is one rounding of the exact fp64 product (compared by value: an
    exact zero may come out of the tensor cores as -0)."""
    from llmc_b200.module_utils import linear_forward_w4
    M, N, K, group = 200, 300, 512, 64
    ng = K // group
    qmax = (1 << bits) - 1
    g = _gen('gidx-exact', bits, native, str(dtype))
    qdt = dtype if native else torch.float32
    codes = torch.randint(0, qmax + 1, (N, K), generator=g, device='cuda')
    z = torch.randint(0, qmax + 1, (N, ng), generator=g, device='cuda')
    s = torch.pow(2.0, torch.randint(-3, 2, (N, ng), generator=g, device='cuda').double())
    r = min(64, ((1 << 21) - 256) // (K * qmax * 2))
    if dtype == torch.float16:
        r = min(r, 65504 // (K * qmax * 2) or 1)     # keep the outputs finite in fp16
    gi = _gidx('perm', K, group, g)
    x = torch.randint(-r, r + 1, (M, K), generator=g, device='cuda').double()
    w = (codes.double() - z.double()[:, gi.long()]) * s[:, gi.long()]
    exact = (x @ w.t()).to(torch.float32).to(dtype)
    y = linear_forward_w4(x.to(dtype), _pack(codes, bits), s.to(qdt), z.to(qdt), group, bits=bits, g_idx=gi)
    bad = y != exact
    assert not bool(bad.any()), [(i, y[tuple(i)].item(), exact[tuple(i)].item()) for i in bad.nonzero()[:4].tolist()]
    # a wrong lookup would show: the same data with contiguous groups gives other integers
    y_contig = linear_forward_w4(x.to(dtype), _pack(codes, bits), s.to(qdt), z.to(qdt), group, bits=bits)
    assert not torch.equal(y_contig, exact)


# ---- GPTQ end to end (GPU) ------------------------------------------------------------------------
def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


def _w8_per_channel():
    """The W8 per-channel weight of the shipped w8a8_combin GPTQ step, weight-only."""
    doc = _yaml('backend/vllm/w8a8_combin/step_2_gptq.yml')
    doc['quant'] = {k: v for k, v in doc['quant'].items() if k != 'act'}
    return doc


E2E = {'gptq_w_only': lambda: _yaml('methods/GPTQ/gptq_w_only.yml'),
       'vllm_gptq_w4a16': lambda: _yaml('backend/vllm/gptq_w4a16.yml'),
       'gptq_w8_per_channel': _w8_per_channel}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(E2E))
def test_gptq_deploys_packed_linears(name, tmp_path):
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.module_utils import EffcientFakeQuantLinear
    from llmc_b200.synth import SynthModel, perplexity
    doc = E2E[name]()
    doc.pop('save', None)
    cfg = adapt_reference_config(doc, 'tiny-llama', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['eval']['eval_pos'] = []                       # calibrate only; deployed twice below
    algo, model, _ = main(cfg, quiet=True)
    wq = algo.wquantizer
    blocks = model.get_blocks()
    calibrated = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    w_qdq = {k: algo.w_qdq(m, wq) for k, m in calibrated.items()}
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
        return mods, logits, ppl

    mods, logits, ppl = deploy('1')
    storages = {}
    codes_qparams = n_weights = 0
    for k, m in mods.items():
        assert isinstance(m, EffcientFakeQuantLinear) and m.packed, k
        assert 'weight' not in m._buffers, k                       # no dense weight kept
        assert m.qweight.dtype == torch.int32, k
        assert (m.g_idx is not None) == algo.need_perm, k
        if wq.granularity == 'per_group' and not algo.static_groups:
            assert m.qscales.dtype == torch.float32 and m.qscales_t.dtype == torch.float32, k
            assert m.qzeros is None or m.qzeros_t.dtype == torch.float32, k
        _same(m.weight, w_qdq[k], f'{k} .weight vs GPTQ.w_qdq')
        tensors = [m.qweight, m.qscales] + ([m.qzeros] if m.qzeros is not None else [])
        codes_qparams += sum(t.numel() * t.element_size() for t in tensors)
        for b in m.buffers():
            storages[b.untyped_storage().data_ptr()] = b.untyped_storage().nbytes()
        n_weights += m.in_features * m.out_features
        R, K = m.out_features, m.in_features
        ng = m.qscales.numel() // R
        per_group = m.qscales.element_size() * (2 if m.qzeros is not None else 1)
        assert sum(t.numel() * t.element_size() for t in tensors) == R * K * wq.bit // 8 + R * ng * per_group
    bpw = 8.0 * codes_qparams / n_weights
    held = sum(storages.values())
    print(f'\n{name}: codes + qparams {codes_qparams} B = {bpw:.3f} bits per weight; all buffers of the '
          f'deployed linears {held} B ({8.0 * held / n_weights:.3f} bits per weight, bf16: 16)')
    if name == 'gptq_w_only':                           # W4 g128, fp32 scale + zero
        assert bpw == 4.5
    mods0, logits0, ppl0 = deploy('0')
    for k, m in mods0.items():
        assert not m.packed and m.weight.dtype == algo.model_dtype, k
        _same(m.weight, w_qdq[k], f'{k} materialised .weight vs GPTQ.w_qdq')
    _same(logits, logits0, 'logits')
    assert ppl == ppl0, (ppl, ppl0)
