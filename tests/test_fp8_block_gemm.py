"""CPU: the block-FP8 forward's oracle against the reference's own Triton kernels (run in Triton's
CPU interpreter by scripts/gen_fp8_gemm_golden.py), its fma and promotion order against exact
rational arithmetic, its NaN / inf rules, and the argument checks of llmc_fp8_act_quant /
llmc_gemm_fp8_block, which fail before any CUDA call."""
import ctypes
import math
import os
from fractions import Fraction

import pytest
import torch

import fp8_gemm_oracle as fgo
import w8a8_oracle as wo
from oracle.glue_oracle import fma32

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'fp8_gemm_kat.pt')


@pytest.fixture(scope='module')
def kat():
    return torch.load(GOLDEN)['cases']


def test_act_quant_scales_match_the_reference_exactly(kat):
    for c in kat:
        _, s = fgo.act_quant(c['x'], 128)
        assert s.dtype == c['a_s'].dtype == torch.float32
        assert s.shape == (c['M'], c['K'] // 128)
        assert torch.equal(s, c['a_s'])
        q, _ = fgo.act_quant(c['x'], 128)
        assert torch.equal(q.view(torch.uint8), c['a_q'])


def test_fp8_gemm_matches_the_reference_within_summation_order(kat):
    for c in kat:
        a = c['a_q'].view(torch.float8_e4m3fn)
        w = c['w_q'].view(torch.float8_e4m3fn)
        y = fgo.fp8_gemm(a, c['a_s'], w, c['w_s'])
        exact, mag = fgo.fp8_gemm_exact(a, c['a_s'], w, c['w_s'])
        # the oracle itself: one fp32 rounding per K block and per promotion step
        kb = c['K'] // 128
        assert ((y.double() - exact).abs() <= 2 * kb * 2.0 ** -24 * mag + 1e-30).all()
        for name in ('c_bm16_bn32', 'c_bm64_bn128'):
            ref = c[name]
            assert ref.dtype == torch.float32 and ref.shape == (c['M'], c['N'])
            # the interpreter's dot sums 128 fp32 products in its own order
            tol = (128 + 2 * kb) * 2.0 ** -24 * mag
            err = (ref.double() - y.double()).abs()
            assert (err <= tol).all(), (name, float((err - tol).max()))


def test_fp8_gemm_scale_indexing_is_pinned(kat):
    """Swapping the role of the scales (a_s per column, or b_s per row) breaks the match."""
    c = kat[0]
    a = c['a_q'].view(torch.float8_e4m3fn)
    w = c['w_q'].view(torch.float8_e4m3fn)
    ref = c['c_bm64_bn128'].double()
    y = fgo.fp8_gemm(a, c['a_s'], w, c['w_s']).double()
    bad = fgo.fp8_gemm(a, c['a_s'].flip(0), w, c['w_s']).double()
    scale = ref.abs().max()
    assert (y - ref).abs().max() / scale < 1e-5
    assert (bad - ref).abs().max() / scale > 1e-2


def test_all_zero_group_gives_a_zero_scale_and_nan_codes():
    x = torch.randn(2, 256)
    x[1, 128:] = 0
    q, s = fgo.act_quant(x)
    assert s[1, 1] == 0 and q[1, 128:].float().isnan().all()
    assert not q[0].float().isnan().any()


def test_act_quant_nan_and_inf_follow_max_f32():
    """The reference's compiled max (max.f32) skips a NaN element; +-inf makes s = inf."""
    x = torch.randn(6, 128)
    x[0, 5] = float('nan')                                        # one NaN: the others set s
    x[1] = float('nan')                                           # all NaN
    x[2, 7] = float('inf')
    x[3, 9] = float('-inf')
    x[3, 10] = float('nan')
    q, s = fgo.act_quant(x)
    qf = q.float()
    _, s_rest = fgo.act_quant(torch.cat([x[:1, :5], x[:1, 6:], torch.zeros(1, 1)], 1))
    assert s[0, 0] == s_rest[0, 0] and torch.isfinite(s[0, 0])
    assert qf[0, 5].isnan() and not qf[0, :5].isnan().any() and not qf[0, 6:].isnan().any()
    assert s[1, 0].isnan() and qf[1].isnan().all()
    for r, bad in ((2, [7]), (3, [9, 10])):
        assert s[r, 0] == float('inf')
        assert qf[r, bad].isnan().all()
        keep = torch.ones(128, dtype=torch.bool)
        keep[bad] = False
        # finite / inf = +-0, with the sign of x
        codes = q[r, keep].view(torch.uint8)
        assert torch.equal(codes, torch.where(x[r, keep] < 0, 0x80, 0x00).to(torch.uint8))


def _rn_f32(v):
    """A Fraction rounded to the nearest fp32 value, ties to even, overflow to +-inf (IEEE)."""
    if v == 0:
        return 0.0
    sign = -1.0 if v < 0 else 1.0
    v = abs(v)
    e = v.numerator.bit_length() - v.denominator.bit_length()
    if Fraction(2) ** e > v:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)                      # subnormals: 2^-149 apart
    n = v / ulp
    k = n.numerator // n.denominator
    rem = n - k
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and k % 2 == 1):
        k += 1
    r = k * ulp
    return sign * math.inf if r >= 2 ** 128 else sign * float(r)


def _fma_cases():
    """fp32 triples: random ones over the whole range and near one, and hand-made edges."""
    g = torch.Generator().manual_seed(3)
    bits = torch.randint(-2 ** 31, 2 ** 31, (3, 4000), generator=g, dtype=torch.int64)
    wide = bits.to(torch.int32).view(torch.float32)
    wide = wide[:, torch.isfinite(wide).all(0)]
    near = (1 + torch.rand(3, 4000, generator=g)) * \
        torch.exp2(torch.randint(-3, 4, (3, 4000), generator=g).float())
    near = near * torch.where(torch.rand(3, 4000, generator=g) < 0.5, -1.0, 1.0)
    # cancellation: c = -fp32(a * b) + a few ulp
    ulps = 1 + torch.randint(-4, 5, (1000,), generator=g) * 2.0 ** -23
    near[2, :1000] = -(near[0, :1000] * near[1, :1000]) * ulps
    # subnormal results: products below 2^-126 and subnormal addends
    sub = torch.stack([torch.rand(2000, generator=g) * 2.0 ** -60, torch.rand(2000, generator=g) * 2.0 ** -70,
                       torch.randint(-2 ** 20, 2 ** 20, (2000,), generator=g) * 2.0 ** -149])
    edges = []
    for i in (1, 3, 5, 1023, 4095):
        for j in (1, 7, 4095):
            a, b = (2.0 ** 12 + i) * 2.0 ** -12, (2.0 ** 12 + j) * 2.0 ** -12   # a * b: an fp32 midpoint
            if (2 ** 12 + i) * (2 ** 12 + j) >= 2 ** 25:
                continue
            for c in (0.0, 2.0 ** -149, -2.0 ** -149, 2.0 ** -100, -2.0 ** -60):
                edges.append((a, b, c))
                edges.append((-a, b, -c))
    a, b = 18631.0 * 2.0 ** 52, 1801.0 * 2.0 ** 51                   # a * b = fp32 max + half an ulp
    for c in (0.0, -2.0 ** 80, 2.0 ** 80, -2.0 ** 103, -2.0 ** 102, 2.0 ** -149):
        edges.append((a, b, c))
    edges.append((3.0e38, 2.0, -3.0e38))                          # overflow in a * b, back in range
    edges.append((2.0 ** 100, 2.0 ** 100, 1.0))                   # past the fp32 range: inf
    edges.append((2.0 ** -75, 2.0 ** -75, 0.0))                   # 2^-150: a tie to +0
    edges.append((3 * 2.0 ** -76, 2.0 ** -75, 0.0))               # 1.5 * 2^-150: up to 2^-149
    edges = torch.tensor(edges, dtype=torch.float32).T
    return torch.cat([wide, near, sub, edges], 1)


def test_fma32_is_one_correct_rounding():
    """The oracle's fp32 fma against exact rational arithmetic, bit for bit, at fp32 midpoints
    broken by an addend far below the sum's ulp, subnormal results and overflow."""
    a, b, c = _fma_cases()
    got = fma32(a.double(), b.double(), c)
    exp = torch.tensor([_rn_f32(Fraction(x) * Fraction(y) + Fraction(z))
                        for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], dtype=torch.float32)
    zero = exp == 0                                               # exact zeros: +0 under RN
    gb, eb = got.view(torch.int32), exp.view(torch.int32)
    bad = (gb != eb).nonzero().flatten()
    assert bad.numel() == 0, [(a[i].item(), b[i].item(), c[i].item(), got[i].item(), exp[i].item())
                              for i in bad[:5]]
    assert zero.any() and torch.isinf(exp).any() and (exp.abs() < 2.0 ** -126).logical_and(~zero).any()
    # the cases include ties that a float64 sum rounded straight to fp32 gets wrong
    naive = (a.double() * b.double() + c.double()).float()
    assert (naive.view(torch.int32) != eb).any()


def test_fp8_gemm_promotes_in_the_stated_order():
    """fp8_gemm against a scalar restatement in exact rationals, on operands with 24-bit scale
    mantissas where every fp32 step rounds; each other promotion order changes some bits."""
    g = torch.Generator().manual_seed(8)
    M, N, K = 9, 140, 512
    a, b = wo.fp8_exact_operands(M, N, K, g)
    a_s = _mantissa_scales((M, K // 128), g)
    b_s = _mantissa_scales((2, K // 128), g)
    y = fgo.fp8_gemm(a, a_s, b, b_s)
    A, B = a.float().tolist(), b.float().tolist()
    for m, n in ((0, 0), (3, 77), (8, 139), (5, 128)):
        acc = 0.0
        for k in range(K // 128):
            d = sum(Fraction(A[m][i]) * Fraction(B[n][i]) for i in range(128 * k, 128 * k + 128))
            t = _rn_f32(Fraction(_rn_f32(d)) * Fraction(a_s[m, k].item()))
            acc = _rn_f32(Fraction(t) * Fraction(b_s[n // 128, k].item()) + Fraction(acc))
        assert y[m, n].item() == acc, (m, n)
    for other in fgo.PROMOTIONS[1:]:
        assert not torch.equal(fgo.fp8_gemm(a, a_s, b, b_s, other), y), other


def test_fp8_gemm_nan_codes_poison_their_row_and_column():
    """A NaN code makes its whole K block's dot NaN, even against zeros (NaN * 0 = NaN)."""
    g = torch.Generator().manual_seed(9)
    a, b = wo.fp8_exact_operands(4, 6, 256, g)
    a, b = a.clone(), b.clone()
    a.view(torch.uint8)[1, 200] = 0x7f
    b.view(torch.uint8)[4, 3] = 0xff
    b.view(torch.float8_e4m3fn)[:, 200] = 0.0
    y = fgo.fp8_gemm(a, torch.ones(4, 2), b, torch.ones(1, 2))
    nan = torch.zeros(4, 6, dtype=torch.bool)
    nan[1, :] = True
    nan[:, 4] = True
    assert torch.equal(y.isnan(), nan)


def _mantissa_scales(shape, g):
    """Scales with random 24-bit mantissas over 2^-20 .. 2^20."""
    m = 1 + torch.randint(0, 1 << 23, shape, generator=g).double() * 2.0 ** -23
    return (m * torch.exp2(torch.randint(-20, 21, shape, generator=g).double())).float()


def test_bias_is_added_after_the_bf16_rounding():
    acc = torch.tensor([1.0 + 3 * 2.0 ** -10])                    # rounds down to 1.0 in bf16
    bias = torch.tensor([3 * 2.0 ** -10])
    assert fgo.bf16_plus_bias(acc, bias).float().item() == 1.0    # and 1 + bias rounds to 1.0 again
    assert (acc + bias).to(torch.bfloat16).float().item() == 1.0 + 2.0 ** -7


@pytest.fixture(scope='module')
def lib():
    from llmc_b200 import _lib, build
    build.build()
    return _lib.load()


def test_argument_validation_without_gpu(lib):
    null, p = ctypes.c_void_p(0), ctypes.c_void_p(256)

    def last():
        return lib.llmc_b200_last_error().decode()

    F32, F16, BF16 = 0, 1, 2
    # act_quant: K % 128, null pointers, dtype; rows == 0 is a no-op
    assert lib.llmc_fp8_act_quant(p, 4, 200, BF16, p, p, null) == -1 and 'multiple of 128' in last()
    assert lib.llmc_fp8_act_quant(p, 4, 256, 7, p, p, null) == -1 and 'bad dtype' in last()
    assert lib.llmc_fp8_act_quant(null, 4, 256, BF16, p, p, null) == -1 and 'null pointer' in last()
    assert lib.llmc_fp8_act_quant(p, 4, 256, BF16, p, null, null) == -1 and 'null pointer' in last()
    assert lib.llmc_fp8_act_quant(null, 0, 256, BF16, null, null, null) == 0
    # gemm: K % 128, out dtype, bias rules, null pointers; M == 0 is a no-op
    g = lib.llmc_gemm_fp8_block
    assert g(p, p, p, p, null, 0, p, F32, 16, 16, 200, null) == -1 and 'multiple of 128' in last()
    assert g(p, p, p, p, null, 0, p, F16, 16, 16, 256, null) == -1 and 'fp32 or bf16' in last()
    assert g(p, p, p, p, p, F32, p, F32, 16, 16, 256, null) == -1 and 'bf16 output' in last()
    assert g(p, p, p, p, p, 9, p, BF16, 16, 16, 256, null) == -1 and 'bias dtype' in last()
    assert g(p, p, p, p, null, 0, p, BF16, 16, 0, 256, null) == -1 and 'bad shape' in last()
    for i in (0, 1, 2, 3, 6):
        args = [p, p, p, p, null, 0, p, BF16, 16, 16, 256, null]
        args[i] = null
        assert g(*args) == -1 and 'null pointer' in last()
    assert g(null, null, null, null, null, 0, null, F32, 0, 16, 256, null) == 0


def test_python_interface_refuses_other_block_sizes():
    from llmc_b200.quant_float import act_quant
    with pytest.raises(NotImplementedError, match='kernel.py:143'):
        act_quant(torch.zeros(2, 256), 64)
