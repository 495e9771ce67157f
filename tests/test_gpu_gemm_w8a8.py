"""GPU: the W8A8 real-quant GEMM (csrc/gemm_8bit.cu) against the CPU oracle of tests/w8a8_oracle.py.

INT8 is bit for bit on any codes: the int32 sum is exact and the epilogue is the stated fp32 one.
FP8 is bit for bit on operands whose 128-deep partial sums are exact at any accumulator width, and
within wo.fp8_bound (the output's ulp plus 2^-8 of the scaled sum of |products|) of the float64 value
on random finite e4m3 inputs.  Shapes cover M, N and K at and off the 128 tile edges, the K tail of a
128-deep block, odd N (element-wise stores), one tile, many tiles, and the persistent loop at
16384 x 14336 x 4096 (there the oracle checks a sample of rows against every column)."""
import pytest
import torch

import w8a8_oracle as wo

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
DTYPES = [torch.bfloat16, torch.float16]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _run(kind, qx, s_x, qw, s_w, bias, dtype):
    from llmc_b200._lib import call, dtype_enum, ptr, stream_ptr
    M, K = qx.shape
    N = qw.shape[0]
    y = torch.empty((M, N), dtype=dtype, device='cuda')
    call(f'llmc_gemm_w8a8_{kind}', ptr(qx), ptr(s_x), int(s_x.numel() != 1), ptr(qw), ptr(s_w),
         int(s_w.numel() != 1), ptr(bias), ptr(y), M, N, K, dtype_enum(dtype), stream_ptr())
    return y


def _scales(n, per, g):
    """fp32 scales of several binades, or one per-tensor value."""
    s = torch.rand(n if per else 1, generator=g) * torch.exp2(torch.randint(-12, -6, (n if per else 1,),
                                                                           generator=g).float())
    return s.float().cuda()


def _rows(M, g, extra=48):
    """Every tile-edge row plus a random sample, for the oracle of very large M."""
    r = {0, M - 1}
    for e in range(128, M, 128):
        r.update((e - 1, e))
    r = sorted(r)
    if len(r) > 200:
        r = r[::len(r) // 200 + 1]
    return torch.tensor(sorted(set(r) | set(torch.randint(0, M, (extra,), generator=g).tolist())))


def _same(y, ref, what):
    y = y.cpu()
    if torch.equal(y.view(torch.int16), ref.view(torch.int16)):
        return
    bad = (y.view(torch.int16) != ref.view(torch.int16)).nonzero()
    i, j = bad[0].tolist()
    raise AssertionError(f'{what}: {bad.shape[0]} elements differ, first at ({i}, {j}): '
                         f'{y[i, j].item()} vs {ref[i, j].item()}')


SHAPES = [(1, 1, 16), (1, 4096, 4096), (7, 33, 32), (128, 128, 128), (129, 127, 144), (255, 257, 272),
          (300, 1000, 1040), (2048, 1024, 4096), (513, 384, 14336)]


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('per_token', [True, False])
@pytest.mark.parametrize('per_channel', [True, False])
@pytest.mark.parametrize('bias', [False, True])
@pytest.mark.parametrize('shape', SHAPES)
def test_int8_bit_for_bit(shape, bias, per_channel, per_token, dtype):
    M, N, K = shape
    g = _gen(hash((M, N, K)) % 1000)
    qx = torch.randint(-128, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    qw = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    s_x, s_w = _scales(M, per_token, g), _scales(N, per_channel, g)
    b = torch.randn(N, generator=g).to(dtype).cuda() if bias else None
    y = _run('i8', qx, s_x, qw, s_w, b, dtype)
    _same(y, wo.gemm_w8a8(qx, s_x, qw, s_w, b, dtype), f'int8 {shape}')


@pytest.mark.parametrize('dtype', DTYPES)
def test_int8_persistent_16384x14336x4096(dtype):
    M, N, K = 16384, 14336, 4096
    g = _gen(5)
    qx = torch.randint(-128, 128, (M, K), generator=g, dtype=torch.int8).cuda()
    qw = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8).cuda()
    s_x, s_w = _scales(M, True, g), _scales(N, True, g)
    b = torch.randn(N, generator=g).to(dtype).cuda()
    y = _run('i8', qx, s_x, qw, s_w, b, dtype)
    rows = _rows(M, g)
    ref = wo.gemm_w8a8(qx[rows.cuda()], s_x[rows.cuda()], qw, s_w, b, dtype)
    _same(y[rows.cuda()], ref, 'int8 16384 x 14336 x 4096')


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('per_token,per_channel,bias', [(True, True, False), (True, True, True),
                                                        (False, False, True), (True, False, False)])
@pytest.mark.parametrize('shape', SHAPES)
def test_fp8_bit_for_bit_on_exact_partial_sums(shape, per_token, per_channel, bias, dtype):
    M, N, K = shape
    g = _gen(hash((M, N, K, 8)) % 1000)
    qx, qw = wo.fp8_exact_operands(M, N, K, g, 'cuda')
    s_x, s_w = _scales(M, per_token, g), _scales(N, per_channel, g)
    b = torch.randn(N, generator=g).to(dtype).cuda() if bias else None
    y = _run('fp8', qx, s_x, qw, s_w, b, dtype)
    _same(y, wo.gemm_w8a8(qx, s_x, qw, s_w, b, dtype), f'fp8 {shape}')


@pytest.mark.parametrize('dtype', DTYPES)
def test_fp8_bit_for_bit_persistent_16384x14336x4096(dtype):
    M, N, K = 16384, 14336, 4096
    g = _gen(6)
    qx, qw = wo.fp8_exact_operands(M, N, K, g, 'cuda')
    s_x, s_w = _scales(M, True, g), _scales(N, True, g)
    y = _run('fp8', qx, s_x, qw, s_w, None, dtype)
    rows = _rows(M, g)
    _same(y[rows.cuda()], wo.gemm_w8a8(qx[rows.cuda()], s_x[rows.cuda()], qw, s_w, None, dtype),
          'fp8 16384 x 14336 x 4096')


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('shape', [(129, 257, 272), (300, 1000, 1040), (513, 384, 14336), (16384, 4096, 4096)])
def test_fp8_random_within_bound(shape, dtype):
    M, N, K = shape
    g = _gen(hash((M, N, K, 9)) % 1000)
    qx, qw = wo.fp8_finite_bytes((M, K), g, 'cuda'), wo.fp8_finite_bytes((N, K), g, 'cuda')
    s_x, s_w = _scales(M, True, g) * 1e-3, _scales(N, True, g) * 1e-3
    b = torch.randn(N, generator=g).to(dtype).cuda()
    y = _run('fp8', qx, s_x, qw, s_w, b, dtype)
    rows = _rows(M, g) if M > 1024 else torch.arange(M)
    y = y[rows.cuda()].cpu().double()
    y64, bound = wo.fp8_bound(qx[rows.cuda()], s_x[rows.cuda()], qw, s_w, b, dtype)
    err = (y - y64).abs()
    assert y.isfinite().all()
    assert bool((err <= bound).all()), f'{int((err > bound).sum())} elements beyond the bound'
    # the measured error in units of the scaled sum of |products|, beyond the output's ulp
    _, ulp_only = wo.fp8_bound(qx[rows.cuda()], s_x[rows.cuda()], qw, s_w, b, dtype, tol=0.0)
    mag = (bound - ulp_only) / 2.0 ** -8
    worst = float(((err - ulp_only).clamp(min=0) / mag).max())
    print(f'\nfp8 {shape} {dtype}: worst |err| - ulp = {worst:.3e} x s_x s_w sum|q_x q_w| '
          f'(bound 2^-8 = {2.0 ** -8:.3e}); mean |err| / |y| = {float((err / y64.abs().clamp(min=1e-30)).mean()):.3e}')


def test_ragged_k_tail_reads_zeros():
    """K = 144: the second 128-deep block is 16 columns of data and 112 of TMA zero fill; the bytes
    after column K of a row are the next row's codes and must not enter the sum."""
    g = _gen(10)
    M, N, K = 200, 136, 144
    big_x = torch.randint(-128, 128, (M, 256), generator=g, dtype=torch.int8).cuda()
    big_w = torch.randint(-128, 128, (N, 256), generator=g, dtype=torch.int8).cuda()
    qx, qw = big_x[:, :K].contiguous(), big_w[:, :K].contiguous()
    s_x, s_w = _scales(M, True, g), _scales(N, True, g)
    y = _run('i8', qx, s_x, qw, s_w, None, torch.bfloat16)
    _same(y, wo.gemm_w8a8(qx, s_x, qw, s_w, None, torch.bfloat16), 'K tail')


def test_linear_forward_w8a8_matches_the_oracle_on_its_own_codes():
    """linear_forward_w8a8 = the activation quantizer's codes and scales through the stated GEMM."""
    from llmc_b200.module_utils import act_quantizer, linear_forward_w8a8
    g = _gen(11)
    for dtype in DTYPES:
        x = (torch.randn(3, 70, 512, generator=g) * 4).to(dtype).cuda()
        for kind, act, wdt in [('i8', {'bit': 8, 'symmetric': True, 'granularity': 'per_token'}, torch.int8),
                               ('fp8', {'quant_type': 'float-quant', 'bit': 'e4m3', 'symmetric': True,
                                        'granularity': 'per_token', 'use_qtorch': True}, E4M3)]:
            if wdt == torch.int8:
                qw = torch.randint(-127, 128, (384, 512), generator=g, dtype=torch.int8).cuda()
            else:
                qw = wo.fp8_finite_bytes((384, 512), g, 'cuda')
            s_w = _scales(384, True, g).to(dtype).reshape(384, 1)
            b = torch.randn(384, generator=g).to(dtype).cuda()
            y = linear_forward_w8a8(x, qw, s_w, act, None, b)
            assert y.shape == (3, 70, 384) and y.dtype == dtype
            qx, s_x = act_quantizer(act).real_quant_act(x.reshape(-1, 512))
            ref = _run(kind, qx, s_x, qw, s_w.reshape(-1).float(), b, dtype)
            _same(y.reshape(-1, 384), ref.cpu(), f'{kind} linear_forward_w8a8')
            if kind == 'i8':
                _same(y.reshape(-1, 384), wo.gemm_w8a8(qx, s_x, qw, s_w.reshape(-1).float(), b, dtype),
                      'i8 linear_forward_w8a8 vs oracle')
        # no tokens: an empty output, no launch
        e = linear_forward_w8a8(x[:, :0], torch.zeros(8, 512, dtype=torch.int8, device='cuda'),
                                torch.ones(8, 1, device='cuda'), {'bit': 8, 'symmetric': True,
                                                                  'granularity': 'per_token'})
        assert e.shape == (3, 0, 8)
