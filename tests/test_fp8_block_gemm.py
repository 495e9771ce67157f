"""CPU: the block-FP8 forward's oracle against the reference's own Triton kernels (run in Triton's
CPU interpreter by scripts/gen_fp8_gemm_golden.py), and the argument checks of llmc_fp8_act_quant /
llmc_gemm_fp8_block, which fail before any CUDA call."""
import ctypes
import os

import pytest
import torch

import fp8_gemm_oracle as fgo

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
