"""CPU: the W8A8 real-quant GEMM's argument checks (returned before any launch), its oracle
(tests/w8a8_oracle.py) against exact integer arithmetic and the stated epilogue order, and the
reasons VllmRealQuantLinear gives for the layouts it does not run."""
import ctypes

import numpy as np
import pytest
import torch

import w8a8_oracle as wo

E4M3 = torch.float8_e4m3fn


# ---- argument checks ------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    from llmc_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize('name', ['llmc_gemm_w8a8_i8', 'llmc_gemm_w8a8_fp8'])
def test_arguments_are_checked_before_launch(lib, name):
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    f = getattr(lib, name)
    BF16, F16, F32 = 2, 1, 0

    def last():
        return lib.llmc_b200_last_error().decode()

    def run(x=p, sx=p, sxs=1, w=p, sw=p, sws=1, bias=null, y=p, M=64, N=64, K=128, dt=BF16):
        return f(x, sx, sxs, w, sw, sws, bias, y, M, N, K, dt, null)

    assert run(M=-1) == -1 and 'bad shape' in last()
    assert run(N=0) == -1 and 'bad shape' in last()
    assert run(K=0) == -1 and 'bad shape' in last()
    assert run(dt=F32) == -1 and 'bf16 or fp16' in last()
    assert run(sxs=2) == -1 and 's_x_stride' in last()
    assert run(sws=-1) == -1 and 's_w_stride' in last()
    assert run(K=136) == -1 and 'multiple of 16' in last()
    assert run(x=null) == -1 and 'null pointer' in last()
    assert run(sw=null) == -1 and 'null pointer' in last()
    assert run(y=null) == -1 and 'null pointer' in last()
    assert run(x=ctypes.c_void_p(264)) == -4 and 'aligned' in last()
    assert run(y=ctypes.c_void_p(258)) == -4 and 'aligned' in last()
    assert run(M=(1 << 24), N=(1 << 24)) == -1 and 'too many tiles' in last()
    if name.endswith('i8'):
        assert run(K=131072) == -1 and 'overflows' in last()
    # M == 0 is a no-op, even with null pointers
    assert run(x=null, sx=null, w=null, sw=null, y=null, M=0) == 0
    assert run(M=0, dt=F16) == 0


def test_python_wrapper_refuses_mismatched_operands():
    """linear_forward_w8a8's layout checks that need no device: CPU tensors are refused outright."""
    from llmc_b200._lib import LlmcB200Error
    from llmc_b200.module_utils import linear_forward_w8a8
    act = {'bit': 8, 'symmetric': True, 'granularity': 'per_token'}
    with pytest.raises(LlmcB200Error, match='CUDA tensors only'):
        linear_forward_w8a8(torch.zeros(2, 64, dtype=torch.bfloat16), torch.zeros(4, 64, dtype=torch.int8),
                            torch.ones(4, 1), act)


# ---- the oracle ------------------------------------------------------------------------------------
def test_exact_sum_is_the_integer_sum():
    g = torch.Generator().manual_seed(0)
    for M, N, K in [(1, 1, 16), (7, 5, 144), (33, 17, 1024)]:
        qx = torch.randint(-128, 128, (M, K), generator=g, dtype=torch.int8)
        qw = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8)
        ref = (qx.long().unsqueeze(1) * qw.long().unsqueeze(0)).sum(-1)
        assert torch.equal(wo.exact_sum(qx, qw).long(), ref)
    # the extreme: every code -128, the largest K the kernel takes: 131056 * 2^14 < 2^31
    K = 131056
    qx = torch.full((2, K), -128, dtype=torch.int8)
    acc = wo.exact_sum(qx, qx)
    assert acc[0, 0].item() == K * 16384 and K * 16384 < 2 ** 31


def test_exact_sum_on_e4m3_values():
    g = torch.Generator().manual_seed(1)
    qx = wo.fp8_finite_bytes((4, 512), g)
    qw = wo.fp8_finite_bytes((3, 512), g)
    # the same sum in exact rational arithmetic: every e4m3 value is an integer multiple of 2^-9
    ix = (qx.double() * 512).long()
    iw = (qw.double() * 512).long()
    assert torch.equal(ix.double() / 512, qx.double()) and torch.equal(iw.double() / 512, qw.double())
    ref = (ix.unsqueeze(1) * iw.unsqueeze(0)).sum(-1)
    assert torch.equal((wo.exact_sum(qx, qw) * 2 ** 18).long(), ref)


def test_fp8_exact_operands_keep_partial_sums_small():
    g = torch.Generator().manual_seed(2)
    qx, qw = wo.fp8_exact_operands(8, 16, 300, g)
    x, w = qx.double(), qw.double()
    assert set(x.unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0}
    assert set(w.unique().tolist()) <= {-1.0, 0.0, 1.0}
    for k0 in range(0, 300, 128):
        blk = w[:, k0:k0 + 128]
        assert int((blk != 0).sum(1).max()) <= 32
        # any partial sum of one block's products is an integer of magnitude <= 64
        prods = x[:, None, k0:k0 + 128] * blk[None]
        assert prods.abs().sum(-1).max() <= 64 and torch.equal(prods, prods.round())


def test_epilogue_order_is_the_stated_one():
    """fmul(fmul(fp32(acc), s_w), s_x), then the bias, then one rounding — a case where each other
    grouping gives a different result pins the order."""
    g = torch.Generator().manual_seed(3)
    acc = torch.randint(-(1 << 28), 1 << 28, (256, 256), generator=g).double()
    s_x = torch.rand(256, generator=g) * 1e-3
    s_w = torch.rand(256, generator=g) * 1e-3
    bias = torch.randn(256, generator=g).bfloat16()
    y = wo.epilogue(acc, s_x, s_w, None, torch.float32)
    a = acc.numpy().astype(np.float32)
    stated = (a * s_w.numpy()[None, :]) * s_x.numpy()[:, None]
    other = a * (s_w.numpy()[None, :] * s_x.numpy()[:, None])
    assert np.array_equal(y.numpy(), stated)
    assert not np.array_equal(stated, other)
    # fp32(acc) is one rounding of the exact sum: acc > 2^24 loses bits here
    assert (acc.abs() > 2 ** 24).any() and not torch.equal(acc.float().double(), acc)
    # the bias is added in fp32 before the single rounding to the output dtype
    yb = wo.epilogue(acc, s_x, s_w, bias, torch.bfloat16)
    before = torch.from_numpy(stated + bias.float().numpy()[None, :]).bfloat16()
    after = (torch.from_numpy(stated).bfloat16().float() + bias.float()[None, :]).bfloat16()
    assert torch.equal(yb, before) and not torch.equal(before, after)


def test_fp8_bound_covers_the_exact_formula():
    g = torch.Generator().manual_seed(4)
    qx, qw = wo.fp8_finite_bytes((16, 256), g), wo.fp8_finite_bytes((8, 256), g)
    s_x, s_w = torch.rand(16, generator=g) * 1e-2, torch.rand(8, generator=g) * 1e-2
    for dt in (torch.bfloat16, torch.float16):
        y = wo.gemm_w8a8(qx, s_x, qw, s_w, None, dt)
        y64, bound = wo.fp8_bound(qx, s_x, qw, s_w, None, dt, tol=0.0)
        ok = (y.double() - y64).abs() <= bound
        assert bool(ok[y.double().isfinite()].all())


# ---- what the real-quant module refuses ---------------------------------------------------------------
def _module(weight, scales_name='weight_scale', need_pack=False, act=None, input_scale=None):
    from llmc_b200.module_utils import VllmRealQuantLinear
    m = VllmRealQuantLinear(weight, None, torch.ones(weight.shape[0], 1), input_scale, need_pack, scales_name)
    m.act_cfg = act
    return m


INT_TOKEN = {'bit': 8, 'symmetric': True, 'granularity': 'per_token'}
FP8_TOKEN = {'quant_type': 'float-quant', 'bit': 'e4m3', 'symmetric': True, 'granularity': 'per_token',
             'use_qtorch': True}


@pytest.mark.parametrize('case,match', [
    ('packed', 'weight_packed'),
    ('per_block', 'per_block'),
    ('int8_weight_only', 'weight-only'),
    ('fp8_weight_only', 'weight-only'),
    ('int8_fp8_act', 'float-quant activations'),
    ('fp8_int_act', 'int-quant activations'),
    ('dynamic_per_tensor', 'dynamic per_tensor'),
    ('static_per_token', 'static per_token'),
    ('static_no_scale', 'input_scale'),
    ('e5m2', 'float8_e5m2'),
    ('bf16_int_act', 'bfloat16 weights'),
    ('bf16_off_grid', 'e4m3 grid'),
])
def test_unsupported_layouts_say_why(case, match):
    i8 = torch.zeros(4, 64, dtype=torch.int8)
    f8 = torch.zeros(4, 64, dtype=E4M3)
    m = {
        'packed': lambda: _module(torch.zeros(4, 16, dtype=torch.int32), need_pack=True, act=INT_TOKEN),
        'per_block': lambda: _module(f8, scales_name='weight_scale_inv', act=FP8_TOKEN),
        'int8_weight_only': lambda: _module(i8),
        'fp8_weight_only': lambda: _module(f8),
        'int8_fp8_act': lambda: _module(i8, act=FP8_TOKEN),
        'fp8_int_act': lambda: _module(f8, act=INT_TOKEN),
        'dynamic_per_tensor': lambda: _module(i8, act=dict(INT_TOKEN, granularity='per_tensor')),
        'static_per_token': lambda: _module(i8, act=dict(INT_TOKEN, static=True), input_scale=torch.ones(1)),
        'static_no_scale': lambda: _module(i8, act=dict(INT_TOKEN, granularity='per_tensor', static=True)),
        'e5m2': lambda: _module(torch.zeros(4, 64, dtype=torch.float8_e5m2), act=FP8_TOKEN),
        'bf16_int_act': lambda: _module(torch.zeros(4, 64, dtype=torch.bfloat16), act=INT_TOKEN),
        'bf16_off_grid': lambda: _module(torch.full((4, 64), 1.0625, dtype=torch.bfloat16), act=FP8_TOKEN),
    }[case]()
    with pytest.raises(NotImplementedError, match=match):
        m(torch.zeros(2, 64, dtype=torch.bfloat16))


def test_gptq_fp8_weight_in_the_model_dtype_gives_its_codes():
    """GPTQ's FP8 export holds e4m3 grid values in the model dtype: they are recovered exactly, once."""
    g = torch.Generator().manual_seed(5)
    codes = wo.fp8_finite_bytes((4, 64), g)
    m = _module(codes.to(torch.bfloat16), act=FP8_TOKEN)
    assert m.w8a8_unsupported() is None
    q = m.fp8_weight()
    assert q.dtype == E4M3 and torch.equal(q.view(torch.uint8), codes.view(torch.uint8))
    assert m.fp8_weight() is q
    assert 'weight' in m._buffers and '_w_e4m3' not in m.state_dict()


def test_supported_layouts_are_recognised():
    i8 = torch.zeros(4, 64, dtype=torch.int8)
    f8 = torch.zeros(4, 64, dtype=E4M3)
    assert _module(i8, act=INT_TOKEN).w8a8_unsupported() is None
    assert _module(f8, act=FP8_TOKEN).w8a8_unsupported() is None
    assert _module(i8, act=dict(INT_TOKEN, granularity='per_tensor', static=True),
                   input_scale=torch.ones(1)).w8a8_unsupported() is None
    assert _module(f8, act=dict(FP8_TOKEN, granularity='per_tensor', static=True),
                   input_scale=torch.tensor(0.5)).w8a8_unsupported() is None
