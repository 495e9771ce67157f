"""The packed GEMM on 2- and 3-bit weights (`llmc_gemm_w2a16`, `llmc_gemm_w3a16` and their `_gidx`
forms), the W3 packer (`llmc_pack_w3_codes`), and the 2- / 3-bit fake-quant deploys of AWQ and GPTQ.

Kernel: every output must equal `llmc_gemm_bf16` on the weight materialised from the same codes and
qparams, rT((code - zero) * scale), bit for bit.  On the exact integer grid (small codes,
power-of-two scales, integer activations) every sum is exact in fp32, so the output must also be
one rounding of the exact fp64 product, at every tile edge.  An identity `g_idx` must give the
contiguous call's bits.

W3 layout (include/llmc_b200.h): rows 2r and 2r+1 share a packed row; per 64-column step, six words
per row: four of low two bits (code 16l + i in bits 2i..2i+1 of word l) and two of third bits (code
32m + c at bit c of word 4 + m, with bits 3 and 4 of c swapped).  `_encode_w3` restates it in plain
torch; the packer must write exactly those words and the unpacker must read the codes back.

End to end: the shipped W2A16 g64 / W3A16 g128 AWQ steps and GPTQ at 3 and 2 bits on the tiny
Llama, deployed with packed linears and with materialised ones (LLMC_B200_FUSED_DEQUANT=0): weights,
logits, fp32-CE perplexity and the saved tensors must agree bit for bit.

The argument checks and the layout round trip at the top run without a GPU."""
import ctypes
import json
import os
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
EXACT_LIMIT = 1 << 24


# ---- the W3 layout in plain torch ------------------------------------------------------------------
def _swap34(c):
    return (c & ~24) | ((c & 8) << 1) | ((c & 16) >> 1)


def _encode_w3(codes):
    """Unsigned codes [N, K] (0..7) -> the W3 words [ceil(N/2), 12 K/64] int32, per the header."""
    N, K = codes.shape
    c = codes.to(torch.int64).cpu()
    if N % 2:
        c = torch.cat([c, torch.zeros(1, K, dtype=torch.int64)])
    S = K // 64
    c = c.reshape(-1, S, 64)                                   # [row, step, code]
    words = torch.zeros(c.shape[0], S, 6, dtype=torch.int64)
    for l in range(4):
        for i in range(16):
            words[:, :, l] |= (c[:, :, 16 * l + i] & 3) << (2 * i)
    for m in range(2):
        for b in range(32):
            words[:, :, 4 + m] |= ((c[:, :, 32 * m + _swap34(b)] >> 2) & 1) << b
    # [row pair, row of the pair, step, word] -> [pair, step, row of the pair, word]
    words = words.reshape(-1, 2, S, 6).permute(0, 2, 1, 3).reshape(-1, 12 * S)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def _encode_w2(codes):
    """Unsigned codes [N, K] (0..3) -> LLMC_OUT_PACK_VLLM words [N, K/16] int32."""
    N, K = codes.shape
    c = codes.to(torch.int64).cpu().reshape(N, K // 16, 16)
    w = (c << (torch.arange(16, dtype=torch.int64) * 2)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


# ---- CPU -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_arguments_are_checked_before_launch(bits):
    from llmc_b200 import _lib
    lib = _lib.load()
    f = getattr(lib, f'llmc_gemm_w{bits}a16')
    fg = getattr(lib, f'llmc_gemm_w{bits}a16_gidx')
    null, p, odd = ctypes.c_void_p(0), ctypes.c_void_p(256), ctypes.c_void_p(264)

    def last():
        return lib.llmc_b200_last_error().decode()

    # x, wq, scales, zeros, qdt, bias, y, M, N, K, group, dtype, stream
    assert f(p, null, p, null, 0, null, p, 128, 256, 256, 128, 2, null) == -1
    assert 'null pointer' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 100, 100, 2, null) == -1
    assert 'multiple of 64' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, 96, 2, null) == -1
    assert 'must divide K=256' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 384, 256, 2, null) == -1
    assert 'must divide K=384' in last()
    assert f(p, p, p, null, 1, null, p, 128, 256, 256, 128, 2, null) == -1
    assert 'qparam_dtype' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, 128, 0, null) == -1
    assert 'dtype must be bf16 or fp16' in last()
    assert f(p, odd, p, null, 0, null, p, 128, 256, 256, 128, 2, null) == -4
    assert 'aligned' in last()
    assert f(p, p, p, null, 0, null, p, 128, 256, 256, -96, 2, null) == -1      # transposed qparams
    assert 'group 96 must divide K=256' in last()
    assert f(null, null, null, null, 0, null, null, 0, 256, 256, 128, 2, null) == 0     # M == 0

    # x, wq, scales, zeros, qdt, g_idx, ng, q_t, bias, y, M, N, K, dtype, stream
    assert fg(p, p, p, null, 0, null, 2, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'g_idx is NULL' in last()
    assert fg(p, p, p, null, 0, p, 2, 1, null, p, 128, 256, 100, 2, null) == -4
    assert 'multiple of 64' in last()
    assert fg(p, p, p, null, 0, p, 0, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=0' in last()
    assert fg(p, p, p, null, 0, p, 257, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=257' in last()
    assert fg(p, p, p, null, 1, p, 2, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'qparam_dtype' in last()
    assert fg(p, p, p, null, 0, odd, 2, 1, null, p, 128, 256, 256, 2, null) == -4
    assert fg(p, null, p, null, 0, p, 2, 1, null, p, 128, 256, 256, 2, null) == -1
    assert 'null pointer' in last()
    assert fg(null, null, null, null, 0, p, 2, 1, null, null, 0, 256, 256, 2, null) == 0    # M == 0


def test_w3_packer_arguments_are_checked_before_launch():
    from llmc_b200 import _lib
    lib = _lib.load()
    null, p = ctypes.c_void_p(0), ctypes.c_void_p(256)
    assert lib.llmc_pack_w3_codes(p, 4, 100, p, null) == -1
    assert 'multiple of 64' in lib.llmc_b200_last_error().decode()
    assert lib.llmc_pack_w3_codes(p, -1, 64, p, null) == -1
    assert lib.llmc_pack_w3_codes(null, 4, 64, p, null) == -1
    assert 'null pointer' in lib.llmc_b200_last_error().decode()
    assert lib.llmc_pack_w3_codes(p, 4, 64, null, null) == -1
    assert lib.llmc_pack_w3_codes(null, 0, 64, null, null) == 0


@pytest.mark.parametrize('N', [1, 2, 7, 130])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_layout_round_trip(bits, N):
    """unpack_unsigned_codes reads every code back from the plain-torch encoding, odd N included;
    each code changes exactly its own 2 or 3 bits."""
    from llmc_b200.module_utils import unpack_unsigned_codes
    K = 192
    codes = torch.randint(0, 1 << bits, (N, K), generator=torch.Generator().manual_seed(N))
    enc = _encode_w3 if bits == 3 else _encode_w2
    words = enc(codes)
    assert tuple(words.shape) == (((N + 1) // 2, 3 * K // 16) if bits == 3 else (N, K // 16))
    assert torch.equal(unpack_unsigned_codes(words, bits, N), codes.to(torch.int32))
    # one code at its maximum flips exactly `bits` bits of the encoding
    one = torch.zeros(N, K, dtype=torch.int64)
    one[N - 1, K - 1] = (1 << bits) - 1
    pop = sum(bin(int(w) & 0xFFFFFFFF).count('1') for w in enc(one).flatten())
    assert pop == bits


# ---- GPU helpers -----------------------------------------------------------------------------------
def _gen(*key):
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def _pack(codes, bits):
    from llmc_b200.module_utils import pack_unsigned_codes
    return pack_unsigned_codes(codes, bits, signed=False)


def _materialise(codes, s, z, gi, bits, dtype):
    """rT((code - zero) * scale) in fp32 products (exact for 16-bit qparams), per column group."""
    gl = gi.long()
    zz = z.float()[:, gl] if z is not None else float(1 << (bits - 1))
    return ((codes.float() - zz) * s.float()[:, gl]).to(dtype)


def _contig_gidx(K, group):
    return (torch.arange(K, device='cuda') // group).to(torch.int32)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    bad = a.view(torch.int16) != b.view(torch.int16)
    assert not bool(bad.any()), (what, bad.nonzero()[:4].tolist(), int(bad.sum()))


def _case(bits, M, N, K, group, sym, native, dtype, bias, transposed, key=()):
    """Random codes / qparams; returns (packed forward, materialised forward)."""
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    g = _gen('lowbit', bits, M, N, K, group, sym, native, str(dtype), bias, transposed, key)
    ng = K // group
    qdt = dtype if native else torch.float32
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s = (torch.rand(N, ng, generator=g, device='cuda') * 0.02 + 0.002).to(qdt)
    z = None if sym else torch.randint(0, 1 << bits, (N, ng), generator=g, device='cuda').to(qdt)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    b = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if bias else None
    ss = s.t().contiguous() if transposed else s
    zz = (z.t().contiguous() if transposed else z) if z is not None else None
    y = linear_forward_w4(x, _pack(codes, bits), ss, zz, group, bias=b, bits=bits, qparams_t=transposed)
    ref = linear_forward(x, _materialise(codes, s, z, _contig_gidx(K, group), bits, dtype), b)
    return y, ref


# ---- kernel, bit for bit (GPU) ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('transposed', [False, True], ids=['nk', 'kn'])
@pytest.mark.parametrize('group', [64, 128, 0], ids=['g64', 'g128', 'channel'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('sym', [False, True], ids=['asym', 'sym'])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_gemm_equals_the_materialised_weight(bits, sym, native, dtype, group, transposed):
    M, N, K = 200, 301, 512                 # partial M tile, odd N (W3: a padded row pair)
    group = group or K
    y, ref = _case(bits, M, N, K, group, sym, native, dtype, sym != native, transposed)
    _same(y, ref, 'packed vs materialised')


SHAPES = [
    # M, N, K: one row / one column / odd N / full-width N; K from one step to 14336; the persistent
    # loop (more tiles than the 132 CTAs)
    (1, 1, 64), (127, 1, 640), (1, 28672, 4096), (127, 301, 14336), (2048, 28672, 4096),
    (2048, 4095, 14336), (1100, 2100, 256),
]


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K', SHAPES, ids=[f'{m}x{n}x{k}' for m, n, k in SHAPES])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_gemm_shapes(bits, M, N, K):
    for i, (group, native, dtype) in enumerate([(64, True, torch.bfloat16), (128, False, torch.float16)]):
        group = group if K % group == 0 else K
        y, ref = _case(bits, M, N, K, group, i == 0, native, dtype, i == 1, i == 1)
        _same(y, ref, f'{M}x{N}x{K} group={group}')


def _exact_case(bits, M, N, K, group, sym, native, dtype, bias, gidx_kind=None):
    """The integer grid: codes and zero-points in [0, 2^bits), scales 2^-3 .. 2^1 per (row, group),
    integer activations: every dequantised weight is exact in the dtype and every partial sum exact
    in fp32, so the output is one rounding of the exact fp64 product."""
    from llmc_b200.module_utils import linear_forward_w4
    g = _gen('lowbit-exact', bits, M, N, K, group, sym, native, str(dtype), bias, gidx_kind)
    qmax = (1 << bits) - 1
    ng = K // group
    codes = torch.randint(0, qmax + 1, (N, K), generator=g, device='cuda')
    z = None if sym else torch.randint(0, qmax + 1, (N, ng), generator=g, device='cuda')
    s = torch.pow(2.0, torch.randint(-3, 2, (N, ng), generator=g, device='cuda').double())
    r = min(64, (EXACT_LIMIT // 8 - 256) // (K * qmax * 2))
    if dtype == torch.float16:
        r = min(r, max(65504 // (K * qmax * 2), 1))
    gi = _contig_gidx(K, group)
    if gidx_kind == 'perm':
        gi = (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
    x = torch.randint(-r, r + 1, (M, K), generator=g, device='cuda').double()
    zz = z.double()[:, gi.long()] if z is not None else float(1 << (bits - 1))
    w = (codes.double() - zz) * s[:, gi.long()]
    exact = x @ w.t()
    b = None
    if bias:
        bb = torch.randint(-255, 256, (N,), generator=g, device='cuda').double()
        exact += bb
        b = bb.to(dtype)
    exact = exact.to(torch.float32).to(dtype)
    qdt = dtype if native else torch.float32
    y = linear_forward_w4(x.to(dtype), _pack(codes, bits), s.to(qdt), z.to(qdt) if z is not None else None, group,
                          bias=b, bits=bits, g_idx=gi if gidx_kind else None)
    bad = y != exact
    assert not bool(bad.any()), [(i, y[tuple(i)].item(), exact[tuple(i)].item()) for i in bad.nonzero()[:4].tolist()]
    return y, exact


EDGES = [
    # M, N, K, group: M and N on both sides of the 128 x 128 tile, W3 row pairs split by a tile edge
    (1, 1, 64, 64), (127, 127, 128, 64), (128, 128, 192, 64), (129, 129, 512, 128), (255, 257, 256, 256),
    (65, 519, 1024, 1024), (300, 14336, 4096, 128), (257, 14335, 512, 64),
]


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_gemm_on_the_exact_integer_grid(bits, native, dtype):
    for i, (M, N, K, group) in enumerate(EDGES):
        _exact_case(bits, M, N, K, group, i % 2 == 0, native, dtype, i % 3 == 0)


@pytest.mark.gpu
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_gidx_on_the_exact_integer_grid(bits, native):
    y, exact = _exact_case(bits, 200, 301, 512, 64, False, native, torch.bfloat16, True, 'perm')
    assert not torch.equal(_exact_case(bits, 200, 301, 512, 64, False, native, torch.bfloat16, True)[0], y)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['perm', 'one-group', 'identity'])
@pytest.mark.parametrize('group', [64, 128, 0], ids=['g64', 'g128', 'channel'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('sym', [False, True], ids=['asym', 'sym'])
@pytest.mark.parametrize('bits', [2, 3])
def test_lowbit_gidx_gemm_equals_the_materialised_weight(bits, sym, native, dtype, group, kind):
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    M, N, K = 200, 301, 512
    group = group or K
    ng = K // group
    g = _gen('lowbit-gidx', bits, sym, native, str(dtype), group, kind)
    qdt = dtype if native else torch.float32
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s = (torch.rand(N, ng, generator=g, device='cuda') * 0.02 + 0.002).to(qdt)
    z = None if sym else torch.randint(0, 1 << bits, (N, ng), generator=g, device='cuda').to(qdt)
    if kind == 'perm':
        gi = (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
    elif kind == 'one-group':
        gi = torch.full((K,), ng - 1, dtype=torch.int32, device='cuda')
    else:
        gi = _contig_gidx(K, group)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    bias = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if sym == native else None
    transposed = group == 128
    ss = s.t().contiguous() if transposed else s
    zz = (z.t().contiguous() if transposed else z) if z is not None else None
    packed = _pack(codes, bits)
    y = linear_forward_w4(x, packed, ss, zz, group, bias=bias, bits=bits, qparams_t=transposed, g_idx=gi)
    _same(y, linear_forward(x, _materialise(codes, s, z, gi, bits, dtype), bias), 'gidx vs materialised')
    if kind == 'identity':
        _same(y, linear_forward_w4(x, packed, s, z, group, bias=bias, bits=bits), 'gidx vs contiguous')


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 2, 301, 4096])
@pytest.mark.parametrize('bits', [2, 3])
def test_packer_writes_the_documented_layout(bits, N):
    """pack_unsigned_codes (llmc_pack_w3_codes at 3 bits) equals the plain-torch encoding, from
    unsigned and from signed codes, and unpacks to the codes, odd N included."""
    from llmc_b200.module_utils import pack_unsigned_codes, unpack_unsigned_codes
    K = 1024
    g = _gen('lowbit-pack', bits, N)
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    enc = (_encode_w3 if bits == 3 else _encode_w2)(codes)
    packed = pack_unsigned_codes(codes, bits, signed=False)
    assert torch.equal(packed.cpu(), enc)
    signed = codes.to(torch.int8) - (1 << (bits - 1))
    assert torch.equal(pack_unsigned_codes(signed, bits, signed=True).cpu(), enc)
    assert torch.equal(unpack_unsigned_codes(packed, bits, N), codes.to(torch.int32))


# ---- AWQ and GPTQ end to end (GPU) -----------------------------------------------------------------
def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


def _gptq(bit, group, static_groups):
    doc = _yaml('methods/GPTQ/gptq_w_only.yml')
    doc['quant']['weight'] = dict(doc['quant']['weight'], bit=bit, group_size=group)
    doc['quant']['special'] = dict(doc['quant']['special'], static_groups=static_groups)
    return doc


E2E = {
    'awq_w2a16g64': (lambda: _yaml('combination/awq_comb_omni/w2a16g64/step_1_awq.yml'), 2.5),
    'awq_w3a16g128': (lambda: _yaml('combination/awq_comb_omni/w3a16g128/step_1_awq.yml'), 3.25),
    'gptq_w3_actorder': (lambda: _gptq(3, 128, False), None),
    'gptq_w2g64_static_groups': (lambda: _gptq(2, 64, True), None),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(E2E))
def test_lowbit_recipes_deploy_packed_linears(name, tmp_path):
    from safetensors.torch import load_file
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.export import save_model
    from llmc_b200.module_utils import EffcientFakeQuantLinear
    from llmc_b200.synth import SynthModel, perplexity
    make, want_bpw = E2E[name]
    doc = make()
    doc.pop('save', None)
    cfg = adapt_reference_config(doc, 'tiny-llama', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['eval']['eval_pos'] = []                       # calibrate only; deployed twice below
    algo, model, _ = main(cfg, quiet=True)
    wq = algo.wquantizer
    assert wq.bit == doc['quant']['weight']['bit']
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
        path = os.path.join(str(tmp_path), f'fused{fused}')
        save_model(model, path)
        return mods, logits, ppl, load_file(os.path.join(path, 'model.safetensors'))

    mods, logits, ppl, saved = deploy('1')
    bits = n_weights = 0
    for k, m in mods.items():
        assert isinstance(m, EffcientFakeQuantLinear) and m.packed, k
        assert 'weight' not in m._buffers, k                       # no dense weight kept
        assert m.qweight.dtype == torch.int32 and m.q_bits == wq.bit, k
        _same(m.weight, w_qdq[k], f'{k} .weight vs w_qdq')
        R, K = m.out_features, m.in_features
        rows = (R + 1) // 2 * 2 if wq.bit == 3 else R
        assert m.qweight.numel() * 32 == rows * K * wq.bit, k
        tensors = [m.qweight, m.qscales] + ([m.qzeros] if m.qzeros is not None else [])
        bits += 8 * sum(t.numel() * t.element_size() for t in tensors)
        n_weights += R * K
    bpw = bits / n_weights
    print(f'\n{name}: codes + qparams = {bpw:.4f} bits per weight (16-bit weight: 16)')
    if want_bpw is not None:
        assert bpw == want_bpw, bpw
    mods0, logits0, ppl0, saved0 = deploy('0')
    for k, m in mods0.items():
        assert not m.packed, k
        _same(m.weight, w_qdq[k], f'{k} materialised .weight vs w_qdq')
    _same(logits, logits0, 'logits')
    assert ppl == ppl0, (ppl, ppl0)
    assert sorted(saved) == sorted(saved0)
    for n in saved0:
        assert saved[n].dtype == saved0[n].dtype and torch.equal(saved[n], saved0[n]), n
