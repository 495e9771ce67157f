"""The packed GEMM with real-valued zero-points (`llmc_gemm_w{2,3,4,8}a16_rz`), its outlier patch, and
the packed HQQ / SpQR fake-quant deploys.

Kernel: every output must equal `llmc_gemm_bf16` on the weight materialised in torch from the same
codes and qparams, rT((code - zero) * scale) as two fp32 ops and one rounding, with the outliers
written over their elements — bit for bit.  Zero-points carry fractional parts; on those inputs the
2^23 formula of the integer forms gives a different weight, so the tests tell the two apart.
Integer zero-points through `_rz` must give the `_gidx` call's bits.

End to end: the shipped HQQ (axis 0) and SpQR YAMLs and their variants on the tiny Llama, deployed
with packed linears and with materialised ones (LLMC_B200_FUSED_DEQUANT=0): weights, logits,
fp32-CE perplexity and the saved tensors must agree bit for bit.

The argument checks and the mask -> CSR round trip at the top run without a GPU."""
import ctypes
import json
import os
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]


# ---- CPU -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_rz_arguments_are_checked_before_launch(bits):
    from llmc_b200 import _lib
    lib = _lib.load()
    f = getattr(lib, f'llmc_gemm_w{bits}a16_rz')
    null, p, odd = ctypes.c_void_p(0), ctypes.c_void_p(256), ctypes.c_void_p(264)

    def last():
        return lib.llmc_b200_last_error().decode()

    # x, wq, scales, zeros, sym, axis, group, g_idx, ng, o_rows, o_cols, o_vals, bias, y, M, N, K, dtype, stream
    assert f(p, null, p, null, 0, 0, 0, p, 4, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'null pointer' in last()
    assert f(p, p, p, null, 0, 0, 0, p, 4, null, null, null, null, p, 128, 256, 256, 0, null) == -1
    assert 'dtype must be bf16 or fp16' in last()
    assert f(p, p, p, null, 2, 0, 0, p, 4, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'sym must be 0 or 1' in last()
    assert f(p, p, p, null, 0, 2, 0, p, 4, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'group_axis' in last()
    assert f(p, p, p, null, 0, 0, 0, null, 4, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'needs g_idx' in last()
    assert f(p, p, p, null, 0, 0, 0, p, 0, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=0' in last()
    assert f(p, p, p, null, 0, 0, 0, p, 257, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'ng=257' in last()
    assert f(p, p, p, null, 0, 1, 96, null, 0, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'must divide N=256' in last()
    assert f(p, p, p, null, 0, 1, 0, null, 0, null, null, null, null, p, 128, 256, 256, 2, null) == -1
    assert 'must divide N=256' in last()
    for o in [(p, null, null), (null, p, null), (null, null, p), (p, p, null), (null, p, p)]:
        assert f(p, p, p, null, 0, 1, 128, null, 0, *o, null, p, 128, 256, 256, 2, null) == -1
        assert 'outlier rows, cols and vals' in last()
    assert f(p, p, p, null, 0, 1, 128, null, 0, null, null, null, null, p, 128, 256, 100, 2, null) == -4
    assert 'multiple of 64' in last()
    assert f(p, odd, p, null, 0, 1, 128, null, 0, null, null, null, null, p, 128, 256, 256, 2, null) == -4
    assert f(p, p, p, null, 0, 0, 0, odd, 4, null, null, null, null, p, 128, 256, 256, 2, null) == -4
    assert 'aligned' in last()
    assert f(null, null, null, null, 0, 0, 0, null, 0, null, null, null, null, null, 0, 256, 256, 2, null) == 0


@pytest.mark.parametrize('R,C,frac', [(1, 64, 0.0), (7, 64, 0.3), (130, 192, 0.01), (5, 64, 1.0)])
def test_outlier_csr_round_trips(R, C, frac):
    """outliers_to_csr: rows / cols / vals rebuild exactly the masked weights, columns ascending."""
    from llmc_b200.module_utils import outliers_to_csr
    g = torch.Generator().manual_seed(R * C)
    mask = (torch.rand(R, C, generator=g) < frac).to(torch.uint8)
    if frac == 0.3:
        mask[R - 1] = 1                                   # a full row
        mask[:, C - 1] = 1                                # a full column
    w = torch.randn(R, C, generator=g).to(torch.bfloat16)
    rows, cols, vals = outliers_to_csr(mask, w)
    assert rows.dtype == cols.dtype == torch.int32 and vals.dtype == torch.bfloat16
    assert rows.numel() == R + 1 and int(rows[0]) == 0 and int(rows[-1]) == int(mask.sum()) == cols.numel()
    dense = torch.zeros(R, C, dtype=torch.bfloat16)
    back = torch.zeros(R, C, dtype=torch.bool)
    for r in range(R):
        cs = cols[rows[r]:rows[r + 1]].long()
        assert bool((cs[1:] > cs[:-1]).all())
        dense[r, cs] = vals[rows[r]:rows[r + 1]]
        back[r, cs] = True
    assert torch.equal(back, mask.bool())
    assert torch.equal(dense, torch.where(mask.bool(), w, torch.zeros_like(w)))


# ---- GPU helpers -----------------------------------------------------------------------------------
def _gen(*key):
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    bad = a.view(torch.int16) != b.view(torch.int16)
    assert not bool(bad.any()), (what, bad.nonzero()[:4].tolist(), int(bad.sum()))


def _expand(q, axis, group, gi, N):
    """[N, K] view of the qparams: axis 0 [ng, N] by g_idx, axis 1 [K, N/group] by n // group."""
    if axis == 0:
        return q[gi.long()].t()
    return q.repeat_interleave(group, dim=1).t()


def _materialise(codes, s, z, bits, sym, axis, group, gi, dtype, outliers=None):
    """rT((code - zero) * scale): two fp32 ops, one rounding; then the outliers overwrite."""
    N, K = codes.shape
    code = codes.float() - (float(1 << (bits - 1)) if sym else 0.0)
    ss = _expand(s, axis, group, gi, N)
    zz = _expand(z, axis, group, gi, N) if z is not None else 0.0
    w = ((code - zz) * ss).to(dtype)
    if outliers is not None:
        mask, vals = outliers
        w = torch.where(mask, vals, w)
    return w


def _qparams(g, rows, cols, bits, asym):
    s = torch.rand(rows, cols, generator=g, device='cuda') * 0.02 + 0.002
    # fractional zero-points, inside and just outside the grid
    z = (torch.rand(rows, cols, generator=g, device='cuda') * ((1 << bits) + 1) - 0.5) if asym else None
    return s, z


def _case(bits, M, N, K, group, sym, zeros, axis, dtype, bias, mask=None, gi=None, key=()):
    """Random codes / qparams (fp32, fractional zero-points); returns (packed forward, materialised
    forward)."""
    from llmc_b200.module_utils import linear_forward, linear_forward_rz, outliers_to_csr, pack_unsigned_codes
    g = _gen('rz', bits, M, N, K, group, sym, zeros, axis, str(dtype), bias, key)
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    if axis == 0:
        gi = gi if gi is not None else (torch.arange(K, device='cuda') // group).to(torch.int32)
        s, z = _qparams(g, K // group, N, bits, zeros)
    else:
        s, z = _qparams(g, K, N // group, bits, zeros)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    b = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype) if bias else None
    o = None
    dense = None
    if mask is not None:
        wo = (torch.randn(N, K, generator=g, device='cuda') * 0.5).to(dtype)
        o = outliers_to_csr(mask, wo)
        dense = (mask.bool(), wo)
    wq = pack_unsigned_codes(codes, bits, signed=False)
    y = linear_forward_rz(x, wq, s, z, bits, sym, axis, group=group, g_idx=gi, outliers=o, bias=b)
    ref = linear_forward(x, _materialise(codes, s, z, bits, sym, axis, group, gi, dtype, dense), b)
    return y, ref


# ---- kernel, bit for bit (GPU) ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('axis', [0, 1], ids=['groups-k', 'groups-n'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('zeros', [True, False], ids=['zeros', 'no-zeros'])
@pytest.mark.parametrize('sym', [False, True], ids=['asym', 'sym'])
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_rz_gemm_equals_the_materialised_weight(bits, sym, zeros, dtype, axis):
    M, N, K = 200, 192, 512                # partial M tile, N not a multiple of 128 (g = 64)
    y, ref = _case(bits, M, N, K, 64, sym, zeros, axis, dtype, sym == zeros)
    _same(y, ref, 'rz vs materialised')


SHAPES = [
    # M, N, K, group: one row; N not a multiple of 128; K from one step to 14336; the persistent
    # loop (more tiles than the 132 CTAs); M above 2048
    (1, 128, 64, 32), (127, 192, 640, 64), (1, 4096, 14336, 128), (2048, 6144, 4096, 128),
    (2100, 1280, 1024, 128), (257, 384, 14336, 16),
]


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,K,group', SHAPES, ids=[f'{m}x{n}x{k}g{g}' for m, n, k, g in SHAPES])
@pytest.mark.parametrize('axis', [0, 1], ids=['groups-k', 'groups-n'])
@pytest.mark.parametrize('bits', [3, 4])
def test_rz_gemm_shapes(bits, axis, M, N, K, group):
    dtype = torch.bfloat16 if bits == 4 else torch.float16
    y, ref = _case(bits, M, N, K, group, bits == 3, True, axis, dtype, axis == 1)
    _same(y, ref, f'{M}x{N}x{K} group={group}')


@pytest.mark.gpu
@pytest.mark.parametrize('bits', [2, 4, 8])
def test_fractional_zero_points_tell_the_two_formulas_apart(bits):
    """On fractional zero-points the 2^23 formula of the integer forms, fmul((2^23 + q) - (2^23 + z), s),
    rounds z and gives another weight; the kernel must give the (q - z) * s one."""
    from llmc_b200.module_utils import linear_forward, linear_forward_rz, pack_unsigned_codes
    M, N, K, group = 64, 256, 256, 64
    g = _gen('rz-formulas', bits)
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s, z = _qparams(g, K // group, N, bits, True)
    gi = (torch.arange(K, device='cuda') // group).to(torch.int32)
    magic = torch.tensor(8388608.0, device='cuda')
    zz = _expand(z, 0, group, gi, N)
    old = (((codes.float() + magic) - (zz + magic)) * _expand(s, 0, group, gi, N)).to(torch.bfloat16)
    new = _materialise(codes, s, z, bits, False, 0, group, gi, torch.bfloat16)
    assert int((old != new).sum()) > N * K // 100
    x = torch.randn(M, K, generator=g, device='cuda').to(torch.bfloat16)
    y = linear_forward_rz(x, pack_unsigned_codes(codes, bits, signed=False), s, z, bits, False, 0, g_idx=gi)
    _same(y, linear_forward(x, new, None), 'rz vs (q - z) * s')
    assert not torch.equal(y, linear_forward(x, old, None))


@pytest.mark.gpu
@pytest.mark.parametrize('sym', [False, True], ids=['asym', 'sym'])
@pytest.mark.parametrize('bits', [2, 3, 4, 8])
def test_integer_zero_points_equal_the_gidx_call(bits, sym):
    """Integer zero-points (and no zero-points on a symmetric grid) through `_rz` give the bits of
    llmc_gemm_w{bits}a16_gidx with fp32 qparams, permuted g_idx included."""
    from llmc_b200.module_utils import linear_forward_rz, linear_forward_w4, pack_unsigned_codes
    M, N, K, group = 200, 301, 512, 64
    g = _gen('rz-int', bits, sym)
    codes = torch.randint(0, 1 << bits, (N, K), generator=g, device='cuda')
    s = torch.rand(K // group, N, generator=g, device='cuda') * 0.02 + 0.002
    z = None if sym else torch.randint(0, 1 << bits, (K // group, N), generator=g, device='cuda').float()
    gi = (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
    x = torch.randn(M, K, generator=g, device='cuda').to(torch.bfloat16)
    wq = pack_unsigned_codes(codes, bits, signed=False)
    y = linear_forward_rz(x, wq, s, z, bits, sym, 0, g_idx=gi)
    _same(y, linear_forward_w4(x, wq, s, z, group, bits=bits, qparams_t=True, g_idx=gi), 'rz vs gidx')


def _mask(kind, N, K, g):
    m = torch.zeros(N, K, dtype=torch.uint8, device='cuda')
    if kind == 'one':
        m[N // 3, K // 2 + 5] = 1
    elif kind in ('1%', '25%'):
        m = (torch.rand(N, K, generator=g, device='cuda') < (0.01 if kind == '1%' else 0.25)).to(torch.uint8)
    elif kind == 'row':
        m[N // 2] = 1
    elif kind == 'column':
        m[:, K // 3] = 1
    elif kind == 'edges':
        # both sides of a K step (k = 63 / 64) and of an N tile (n = 127 / 128), the last row / column
        for n in (0, 127, 128, N - 1):
            for k in (0, 63, 64, 127, 128, K - 1):
                m[n, k] = 1
    return m


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['none', 'one', '1%', '25%', 'row', 'column', 'edges'])
@pytest.mark.parametrize('axis', [0, 1], ids=['groups-k', 'groups-n'])
@pytest.mark.parametrize('bits', [3, 4])
def test_outliers_replace_their_elements(bits, axis, kind):
    M, N, K, group = 300, 320, 1024, 32
    g = _gen('rz-outliers', bits, axis, kind)
    y, ref = _case(bits, M, N, K, group, False, True, axis, torch.bfloat16, True, mask=_mask(kind, N, K, g),
                   key=kind)
    _same(y, ref, f'outliers {kind}')


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['1%', 'edges'])
def test_outliers_with_a_permuted_g_idx_and_the_persistent_loop(kind):
    """SpQR's shape: g16 act-order groups, outliers; more tiles than CTAs, so every CTA's cursors run
    across tiles and the two dequant groups' alternate steps."""
    M, N, K, group = 1100, 2096, 2048, 16
    g = _gen('rz-perm', kind)
    gi = (torch.argsort(torch.randperm(K, generator=g, device='cuda')) // group).to(torch.int32)
    y, ref = _case(4, M, N, K, group, False, True, 0, torch.float16, False, mask=_mask(kind, N, K, g), gi=gi,
                   key=kind)
    _same(y, ref, f'permuted g_idx, outliers {kind}')


# ---- HQQ and SpQR end to end (GPU) -----------------------------------------------------------------
def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


def _hqq(axis=0, bit=4):
    doc = _yaml('methods/HQQ/hqq_w_only.yml')
    doc['quant']['weight'] = dict(doc['quant']['weight'], bit=bit)
    doc['quant']['special'] = dict(doc['quant']['special'], axis=axis)
    return doc


def _spqr(actorder=True):
    doc = _yaml('methods/SpQR/spqr_w_only.yml')
    doc['quant']['special'] = dict(doc['quant']['special'], actorder=actorder)
    return doc


E2E = {
    'hqq_shipped_axis0': (lambda: _hqq(), 4.5),
    'hqq_axis1': (lambda: _hqq(axis=1), 4.5),
    'hqq_w2': (lambda: _hqq(bit=2), 2.5),
    'hqq_w3': (lambda: _hqq(bit=3), 3.5),
    'spqr_shipped': (lambda: _spqr(), None),
    'spqr_no_actorder': (lambda: _spqr(actorder=False), None),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(E2E))
def test_real_zero_recipes_deploy_packed_linears(name, tmp_path):
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
    assert wq.bit == doc['quant']['weight']['bit'] and not wq.round_zp
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
    bits = n_weights = nnz = 0
    for k, m in mods.items():
        assert isinstance(m, EffcientFakeQuantLinear) and m.packed and m.q_rz, k
        assert 'weight' not in m._buffers, k                       # no dense weight kept
        assert m.qweight.dtype == torch.int32 and m.q_bits == wq.bit, k
        _same(m.weight, w_qdq[k], f'{k} .weight vs w_qdq')
        R, K = m.out_features, m.in_features
        rows = (R + 1) // 2 * 2 if wq.bit == 3 else R
        assert m.qweight.numel() * 32 == rows * K * wq.bit, k
        tensors = [m.qweight, m.qscales] + ([m.qzeros] if m.qzeros is not None else [])
        if m.outlier_rows is not None:
            tensors += [m.outlier_rows, m.outlier_cols, m.outlier_vals]
            nnz += m.outlier_cols.numel()
        bits += 8 * sum(t.numel() * t.element_size() for t in tensors)
        n_weights += R * K
    bpw = bits / n_weights
    print(f'\n{name}: codes + qparams + outliers = {bpw:.4f} bits per weight (16-bit weight: 16); '
          f'{nnz} outliers of {n_weights} weights')
    if want_bpw is not None:
        assert bpw == want_bpw, bpw
    if name.startswith('spqr'):
        assert nnz > 0
    mods0, logits0, ppl0, saved0 = deploy('0')
    for k, m in mods0.items():
        assert not m.packed, k
        _same(m.weight, w_qdq[k], f'{k} materialised .weight vs w_qdq')
    _same(logits, logits0, 'logits')
    assert ppl == ppl0, (ppl, ppl0)
    assert sorted(saved) == sorted(saved0)
    for n in saved0:
        assert saved[n].dtype == saved0[n].dtype and torch.equal(saved[n], saved0[n]), n
