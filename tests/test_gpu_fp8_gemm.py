"""GPU: the block-FP8 linear forward on the FP8 tensor cores — act_quant (csrc/fp8.cu) and
llmc_gemm_fp8_block (csrc/gemm_8bit.cu) against the CPU oracle of tests/fp8_gemm_oracle.py.

The 128-deep dot runs in the Hopper FP8 accumulator, whose precision is below fp32, so bit-exact
comparisons use an integer grid: small integer codes and power-of-two scales keep every partial sum
exactly representable, and then everything else — operand layouts, swizzle, scale indexing,
promotion order, both epilogues — must match the oracle bit for bit."""
import numpy as np
import pytest
import torch

import fp8_gemm_oracle as fgo

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn


def _f32_bits(t):
    return t.contiguous().view(torch.int32).long()


# ---- act_quant ----------------------------------------------------------------------------------

@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('shape', [(2, 33, 512), (1, 7, 7168), (3, 1, 128)])
def test_act_quant_scales_and_codes(dtype, shape):
    from llmc_b200.quant_float import act_quant
    g = torch.Generator().manual_seed(sum(shape))
    K = shape[-1]
    x = torch.randn(*shape, generator=g) * torch.exp(torch.randn(K, generator=g) * 2)
    x.view(-1, K)[0, :128] *= 1e-4                                   # a tiny-scale group
    x = x.to(dtype)
    q, s = act_quant(x.cuda())
    assert q.dtype == E4M3 and q.shape == x.shape
    assert s.dtype == torch.float32 and s.shape == (*shape[:-1], K // 128)
    q, s = q.cpu(), s.cpu()
    _, s_o = fgo.act_quant(x)
    # div.full.f32 is within 2 ulp of the IEEE quotient (both scales positive)
    assert ((_f32_bits(s) - _f32_bits(s_o)).abs() <= 2).all()
    # every code is the RNE e4m3 code of x / s_kernel, except within 2^-21 of a rounding midpoint
    quo = x.double().reshape(*shape[:-1], K // 128, 128) / s.double()[..., None]
    quo = quo.reshape(shape).clamp(-448, 448)
    lo = (quo * (1 - 2.0 ** -21)).float().to(E4M3).view(torch.uint8)
    hi = (quo * (1 + 2.0 ** -21)).float().to(E4M3).view(torch.uint8)
    got = q.view(torch.uint8)
    ok = (got == lo) | (got == hi)
    bad = (~ok).nonzero()[:5].tolist()
    assert ok.all(), [(i, float(quo[tuple(i)]), int(got[tuple(i)]), int(lo[tuple(i)])) for i in bad]


def test_act_quant_all_zero_group_gives_zero_scale_and_nan_codes():
    from llmc_b200.quant_float import act_quant
    x = torch.randn(3, 384, dtype=torch.bfloat16)
    x[1, 128:256] = 0
    q, s = act_quant(x.cuda())
    q, s = q.cpu(), s.cpu()
    assert s[1, 1] == 0
    assert q[1, 128:256].float().isnan().all()
    assert not q[1, :128].float().isnan().any() and not q[1, 256:].float().isnan().any()
    assert (s[0] > 0).all() and (s[2] > 0).all()


# ---- GEMM on an integer grid: bit-exact -----------------------------------------------------------

def _grid_problem(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-3, 4, (M, K), generator=g).float().to(E4M3)
    b = torch.randint(-3, 4, (N, K), generator=g).float().to(E4M3)
    a_s = torch.pow(2.0, torch.randint(-3, 1, (M, K // 128), generator=g).float())
    b_s = torch.pow(2.0, torch.randint(-3, 1, (-(-N // 128), K // 128), generator=g).float())
    return a, a_s, b, b_s


_SHAPES = [(1, 1, 128), (77, 200, 256), (200, 77, 7168), (4160, 200, 256), (77, 4160, 128),
           (200, 4160, 7168), (4160, 77, 7168), (1, 4160, 256)]


@pytest.mark.parametrize('M,N,K', _SHAPES)
def test_gemm_integer_grid_bit_exact(M, N, K):
    from llmc_b200.quant_float import gemm_fp8_block
    a, a_s, b, b_s = _grid_problem(M, N, K, M * 7 + N * 3 + K)
    ref = fgo.fp8_gemm(a, a_s, b, b_s)
    args = (a.cuda(), a_s.cuda(), b.cuda(), b_s.cuda())
    y = gemm_fp8_block(*args, torch.float32)
    assert y.dtype == torch.float32 and torch.equal(y.cpu(), ref)
    g = torch.Generator().manual_seed(N)
    bias32 = torch.randn(N, generator=g) * 4
    for bias in (None, bias32, bias32.to(torch.bfloat16)):
        yb = gemm_fp8_block(*args, torch.bfloat16, bias=None if bias is None else bias.cuda())
        assert yb.dtype == torch.bfloat16
        assert torch.equal(yb.cpu(), fgo.bf16_plus_bias(ref, bias))


def test_fp8_gemm_public_interface_shape_and_dtype():
    from llmc_b200.quant_float import act_quant, fp8_gemm
    a, a_s, b, b_s = _grid_problem(2 * 9, 300, 384, 11)
    y = fp8_gemm(a.view(2, 9, 384).cuda(), a_s.view(2, 9, 3).cuda(), b.cuda(), b_s.cuda())
    assert y.dtype == torch.get_default_dtype() and y.shape == (2, 9, 300)
    assert torch.equal(y.cpu().view(18, 300), fgo.fp8_gemm(a, a_s, b, b_s))
    with pytest.raises(NotImplementedError, match='kernel.py:143'):
        act_quant(torch.zeros(2, 256, device='cuda'), 64)


# ---- GEMM on random data at real widths ------------------------------------------------------------

@pytest.mark.parametrize('M,N,K', [(64, 18432, 4096), (48, 7168, 7168), (130, 1536, 7168)])
def test_gemm_random_against_fp64(M, N, K):
    """|y - exact| <= 2^-10 * sum_k |a_s a_k b_s b_k| + fp32 promotion rounding, per element."""
    from llmc_b200.quant_float import act_quant, gemm_fp8_block, weight_cast_to_fp8
    g = torch.Generator().manual_seed(M + N + K)
    x = (torch.randn(M, K, generator=g) * torch.exp(torch.randn(K, generator=g))).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.02).bfloat16()
    a, a_s = act_quant(x.cuda())
    b, b_s = weight_cast_to_fp8(w.cuda(), 128)
    y = gemm_fp8_block(a, a_s, b, b_s, torch.float32).cpu().double()
    exact, mag = fgo.fp8_gemm_exact(a.cpu(), a_s.cpu(), b.cpu(), b_s.cpu())
    kb = K // 128
    err = (y - exact).abs()
    bound = 2.0 ** -10 * mag + 2 * kb * 2.0 ** -24 * mag
    ratio = float((err / mag.clamp_min(1e-30)).max())
    print(f'fp8 gemm M={M} N={N} K={K}: worst |err| / sum|a b| = {ratio:.3e} '
          f'(= 2^{np.log2(max(ratio, 1e-300)):.2f})')
    assert (err <= bound).all(), ratio


# ---- invariance ---------------------------------------------------------------------------------------

def test_gemm_results_do_not_depend_on_problem_size():
    from llmc_b200.quant_float import act_quant, gemm_fp8_block, weight_cast_to_fp8
    g = torch.Generator().manual_seed(5)
    M, N, K = 4200, 520, 1024
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) * 0.02).bfloat16().cuda()
    a, a_s = act_quant(x)
    b, b_s = weight_cast_to_fp8(w, 128)
    bias = torch.randn(N, device='cuda')
    for dt, bb in ((torch.float32, None), (torch.bfloat16, bias)):
        full = gemm_fp8_block(a, a_s, b, b_s, dt, bias=bb)
        # rows of a sub-problem (different tile count and tile assignment)
        rows = gemm_fp8_block(a[1000:1077], a_s[1000:1077], b, b_s, dt, bias=bb)
        assert torch.equal(rows, full[1000:1077])
        one = gemm_fp8_block(a[4199:], a_s[4199:], b, b_s, dt, bias=bb)
        assert torch.equal(one, full[4199:])
        # columns: a 128-aligned slice of the weight keeps its scale rows
        cb = None if bb is None else bb[128:333]
        cols = gemm_fp8_block(a, a_s, b[128:333], b_s[1:3], dt, bias=cb)
        assert torch.equal(cols, full[:, 128:333])
        nb = None if bb is None else bb[:77]
        both = gemm_fp8_block(a[7:200], a_s[7:200], b[:77], b_s[:1], dt, bias=nb)
        assert torch.equal(both, full[7:200, :77])


def test_gemm_empty_m_is_a_no_op():
    from llmc_b200.quant_float import gemm_fp8_block
    a = torch.zeros(0, 256, dtype=E4M3, device='cuda')
    a_s = torch.zeros(0, 2, device='cuda')
    b = torch.zeros(64, 256, dtype=E4M3, device='cuda')
    b_s = torch.ones(1, 2, device='cuda')
    assert gemm_fp8_block(a, a_s, b, b_s, torch.float32).shape == (0, 64)


# ---- modules ---------------------------------------------------------------------------------------------

def _fp8_module(out_f, in_f, bias, seed):
    from llmc_b200.module_utils import LlmcFp8Linear
    from llmc_b200.quant_float import weight_cast_to_fp8
    g = torch.Generator().manual_seed(seed)
    lin = torch.nn.Linear(in_f, out_f, bias=bias)
    m = LlmcFp8Linear.new(lin, 128).cuda()
    w = (torch.randn(out_f, in_f, generator=g) * 0.03).bfloat16().cuda()
    q, s = weight_cast_to_fp8(w, 128)
    m.weight.data, m.weight_scale_inv.data = q, s
    if bias:
        m.bias.data = (torch.randn(out_f, generator=g) * 0.1).cuda()
    x = torch.randn(2, 37, in_f, generator=g).bfloat16().cuda()
    return m, x, q, s, w


def test_origin_float_linear_runs_the_fp8_forward():
    from llmc_b200.module_utils import OriginFloatLinear, block_wise_fp8_forward_func
    m, x, q, s, _ = _fp8_module(300, 512, True, 1)
    o = OriginFloatLinear.new(m)
    assert o.fp8_forward and o.block_size == 128 and 'fp8_forward=True' in repr(o)
    y = o(x)
    assert y.dtype == torch.bfloat16 and y.shape == (2, 37, 300)
    assert torch.equal(y, block_wise_fp8_forward_func(x, q, s, 128, m.bias))
    # against the CPU oracle, up to the Hopper accumulator and 2-ulp scales
    yo = fgo.block_wise_fp8_forward(x.cpu(), q.cpu(), s.cpu(), m.bias.cpu())
    rel = (y.cpu().float() - yo.float()).norm() / yo.float().norm()
    assert rel < 1e-2, float(rel)


def test_llmc_fp8_linear_switch_keeps_the_weight_in_fp8(monkeypatch):
    from llmc_b200 import module_utils as mu
    from llmc_b200.module_utils import block_wise_fp8_forward_func, linear_forward
    from llmc_b200.quant_float import weight_cast_to_bf16
    m, x, q, s, w = _fp8_module(384, 1024, False, 2)
    assert 'use_fp8gemm_triton_kernel=False' in repr(m)
    monkeypatch.setattr(mu, 'USE_FP8GEMM_KERNEL', True)
    assert 'use_fp8gemm_triton_kernel=True' in repr(m)
    y = m(x)
    assert m.weight.dtype == E4M3
    assert torch.equal(y, block_wise_fp8_forward_func(x, q, s, 128, None))
    # sanity bar for the e4m3 activation rounding against the dequant-once bf16 path
    ref = linear_forward(x, weight_cast_to_bf16(q, s, 128))
    rel = (y.float() - ref.float()).norm() / ref.float().norm()
    assert rel < 6e-2, float(rel)
