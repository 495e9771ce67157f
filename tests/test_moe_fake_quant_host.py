"""CPU: what the grouped FP8 MoE entry points refuse before any CUDA call, and which fake-quant expert
linears and activation fake-quants the grouped MoE path accepts (module_utils.fake_quant_forward_operands,
blockwise.a_qdq_routed) on CPU-built modules."""
import ctypes
import functools

import pytest
import torch
import torch.nn as nn

from llmc_b200 import _lib
from llmc_b200.blockwise import BaseBlockwiseQuantization
from llmc_b200.module_utils import (EffcientFakeQuantLinear, FakeQuantLinear, Fp8Operands, PackedOperands,
                                    dense_forward_weight, fake_quant_forward_operands, packed_forward_operands)
from llmc_b200.quant import IntegerQuantizer
from llmc_b200.quant_float import FloatQuantizer

CAP = _lib.MOE_MAX_EXPERTS


def _ptrs(n, addr=256):
    return (ctypes.c_void_p * n)(*([addr] * n))


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _last(lib):
    return lib.llmc_b200_last_error().decode()


def _swiglu(lib, xp=256, e5m2=0, wq1=None, wq3=None, s1=None, s3=None, g1=None, g3=None, qdt=_lib.BF16,
            group=128, ng=2, offsets=256, act=256, rows=256, inter=512, K=256, E=4, dtype=_lib.BF16):
    w = _ptrs(CAP + 1)
    return lib.llmc_moe_gemm_fp8a16_swiglu(
        ctypes.c_void_p(xp), e5m2, w if wq1 is None else wq1, w if wq3 is None else wq3, w if s1 is None else s1,
        w if s3 is None else s3, g1, g3, qdt, group, ng, ctypes.c_void_p(offsets), ctypes.c_void_p(act), rows,
        inter, K, E, dtype, None)


def _down(lib, act=256, e5m2=1, wq2=None, s2=None, g2=None, qdt=_lib.F32, group=-512, ng=1, offsets=256,
          w_route=256, y=256, rows=256, N=256, inter=512, E=4, dtype=_lib.F16):
    w = _ptrs(CAP + 1)
    return lib.llmc_moe_gemm_fp8a16_down(
        ctypes.c_void_p(act), e5m2, w if wq2 is None else wq2, w if s2 is None else s2, g2, qdt, group, ng,
        ctypes.c_void_p(offsets), ctypes.c_void_p(w_route), ctypes.c_void_p(y), rows, N, inter, E, dtype, None)


def test_e5m2_flag(lib):
    assert _swiglu(lib, e5m2=2) == -1 and 'e5m2 must be 0 (e4m3) or 1 (e5m2), got 2' in _last(lib)
    assert _down(lib, e5m2=-1) == -1 and 'got -1' in _last(lib)
    assert _swiglu(lib, e5m2=2, rows=0) == -1              # a scalar: refused before the rows == 0 return


def test_expert_count_and_shapes(lib):
    assert _swiglu(lib, E=CAP + 1) == -1 and 'experts outside 1..%d' % CAP in _last(lib)
    assert _down(lib, E=0) == -1 and 'experts outside' in _last(lib)
    assert _swiglu(lib, K=200) == -1 and 'K=200 must be a multiple of 64' in _last(lib)
    assert _swiglu(lib, inter=480) == -1 and 'inter=480 must be a multiple of 64' in _last(lib)
    assert _down(lib, N=100) == -1 and 'N=100 must be a multiple of 8' in _last(lib)
    assert _down(lib, inter=480) == -1 and 'K=480 must be a multiple of 64' in _last(lib)
    assert _swiglu(lib, group=96, ng=2) == -1 and 'group 96' in _last(lib)
    assert _swiglu(lib, group=-32) == -1 and 'group 32' in _last(lib)
    assert _swiglu(lib, ng=4) == -1 and 'ng=4' in _last(lib)


def test_dtypes(lib):
    assert _swiglu(lib, dtype=_lib.F32, qdt=_lib.F32) == -1 and 'dtype must be bf16 or fp16' in _last(lib)
    assert _swiglu(lib, qdt=_lib.F16) == -1 and 'qparam_dtype' in _last(lib)
    assert _down(lib, rows=0, qdt=_lib.BF16) == -1 and 'qparam_dtype' in _last(lib)


def test_null_arrays_and_entries_name_the_expert(lib):
    assert _swiglu(lib, offsets=0) == -1 and 'null pointer' in _last(lib)
    assert _down(lib, w_route=0) == -1 and 'null pointer' in _last(lib)
    w3 = _ptrs(4)
    w3[2] = None
    assert _swiglu(lib, wq3=w3) == -1 and 'null codes or scales of expert 2' in _last(lib)
    s2 = _ptrs(4)
    s2[3] = None
    assert _down(lib, s2=s2) == -1 and 'null codes or scales of expert 3' in _last(lib)


def test_gidx_for_some_experts_only(lib):
    g = _ptrs(4)
    g[1] = None
    assert _swiglu(lib, g1=g, g3=_ptrs(4), ng=4) == -1
    assert 'g_idx of expert 1 null while expert 0\'s is given' in _last(lib)
    assert _swiglu(lib, g1=_ptrs(4), g3=None, ng=4) == -1 and 'g_idx of expert 0 null' in _last(lib)


def test_misalignment_is_ealign(lib):
    assert _swiglu(lib, xp=258) == -4
    assert _down(lib, y=264) == -4
    wq = _ptrs(4)
    wq[1] = 264
    assert _swiglu(lib, wq1=wq) == -4 and 'expert 1 not 16-byte aligned' in _last(lib)
    g = _ptrs(4)
    g[2] = 260
    assert _down(lib, g2=g, ng=4) == -4 and 'expert 2 not 16-byte aligned' in _last(lib)


def test_no_rows_touches_no_pointer(lib):
    null = 0
    for f, kw in ((_swiglu, dict(xp=null, offsets=null, act=null)),
                  (_down, dict(act=null, offsets=null, w_route=null, y=null))):
        n = (ctypes.c_void_p * 4)()
        key = 'wq1' if f is _swiglu else 'wq2'
        assert f(lib, rows=0, **{key: n}, **kw) == 0


# ---- selection rules on CPU-built modules -------------------------------------------------------
def _algo(aq, static, cls=BaseBlockwiseQuantization):
    algo = object.__new__(cls)
    algo.wquantizer, algo.aquantizer, algo.act_static = IntegerQuantizer(8, True, 'per_channel'), aq, static
    return algo


def _a_qdq(aq, static=False, cls=BaseBlockwiseQuantization):
    return _algo(aq, static, cls).get_replacement_params('fake_quant')['a_qdq']


def _fp8_efq(a_qdq=None, N=128, K=256, grid=torch.float8_e4m3fn, sdt=torch.float32, gidx=False):
    ori = nn.Linear(K, N, bias=False)
    packed = dict(qweight=torch.zeros(N, K, dtype=grid), scales=torch.rand(N, 1).to(sdt), zeros=None, bits=8,
                  group=K, dtype=torch.bfloat16)
    if gidx:
        packed.update(scales=torch.rand(N, 2).to(sdt), group=128, g_idx=(torch.arange(K) // 128).to(torch.int32))
    m = EffcientFakeQuantLinear(None, None, ori, a_qdq, packed=packed)
    m.in_features, m.out_features = K, N
    return m


def _int_efq(a_qdq=None, N=128, K=256):
    ori = nn.Linear(K, N, bias=False)
    packed = dict(qweight=torch.zeros(N, K // 8, dtype=torch.int32), scales=torch.rand(N, 2).to(torch.bfloat16),
                  zeros=None, bits=4, group=128, dtype=torch.bfloat16)
    m = EffcientFakeQuantLinear(None, None, ori, a_qdq, packed=packed)
    m.in_features, m.out_features = K, N
    return m


@pytest.mark.parametrize('grid', [torch.float8_e4m3fn, torch.float8_e5m2])
@pytest.mark.parametrize('sdt', [torch.float32, torch.bfloat16])
def test_fp8_operands(grid, sdt):
    m = _fp8_efq(grid=grid, sdt=sdt)
    o, a = fake_quant_forward_operands(m, torch.bfloat16)
    assert isinstance(o, Fp8Operands) and a is None
    assert o.wq.dtype == torch.int32 and tuple(o.wq.shape) == (128, 64) and o.transposed and o.zeros is None
    assert o.e5m2 == int(grid == torch.float8_e5m2) and o.group == 256 and o.bits == 8
    assert o.scales.dtype == sdt and torch.equal(o.scales, m.qscales_t.to(sdt))   # as linear_forward_fp8w
    o16, _ = fake_quant_forward_operands(m, torch.float16)
    assert o16.scales.dtype == (torch.float32 if sdt == torch.bfloat16 else sdt)
    og, _ = fake_quant_forward_operands(_fp8_efq(gidx=True), torch.bfloat16)
    assert og.g_idx is not None and og.group == 128


def test_weight_forms_under_a_qdq():
    a = _a_qdq(IntegerQuantizer(8, True, 'per_token'))
    o, got = fake_quant_forward_operands(_int_efq(a), torch.bfloat16)
    assert isinstance(o, PackedOperands) and got is a
    assert packed_forward_operands(_int_efq(a), torch.bfloat16) is None        # its contract is unchanged
    lin = nn.Linear(256, 128, bias=False).bfloat16()
    fq = FakeQuantLinear.new(lin, lambda m: m.weight, a)
    w, got = fake_quant_forward_operands(fq, torch.bfloat16)
    assert torch.equal(w, lin.weight) and got is a
    assert dense_forward_weight(fq, torch.bfloat16) is None


@pytest.mark.parametrize('case', ['bias', 'hook', 'rz', 'w2', 'plain'])
def test_weight_forms_refused(case):
    if case == 'bias':
        ori = nn.Linear(256, 128, bias=True)
        m = FakeQuantLinear.new(ori, lambda m: m.weight, None)
    elif case == 'hook':
        m = _fp8_efq()
        m.register_forward_pre_hook(lambda *a: None)
    elif case in ('rz', 'w2'):
        m = _int_efq()
        if case == 'rz':
            m.q_rz = True
        else:
            m.q_bits = 2
    else:
        m = nn.Linear(256, 128, bias=False)
    assert fake_quant_forward_operands(m, torch.bfloat16) is None


class _Override(BaseBlockwiseQuantization):
    def a_qdq(self, act, module, aquantizer, input_index=0):
        return super().a_qdq(act, module, aquantizer, input_index)


def _static_linear(scale):
    m = _fp8_efq()
    m.register_buffer('buf_act_scales_0', scale)
    return m


def test_routed_twin_attached_by_the_defining_class():
    a = _a_qdq(IntegerQuantizer(8, True, 'per_token'))
    assert isinstance(a, functools.partial) and a.routed.func.__name__ == 'a_qdq_routed'
    assert not hasattr(_a_qdq(IntegerQuantizer(8, True, 'per_token'), cls=_Override), 'routed')
    assert _algo(None, False).get_replacement_params('fake_quant', w_only=True)['a_qdq'] is None


@pytest.mark.parametrize('aq', [IntegerQuantizer(8, True, 'per_token'), IntegerQuantizer(8, True, 'per_channel'),
                                IntegerQuantizer(4, False, 'per_group', group_size=128),
                                FloatQuantizer('e4m3', True, 'per_token', use_qtorch=True),
                                FloatQuantizer('e5m2', True, 'per_group', group_size=128, use_qtorch=True)])
def test_dynamic_row_local_forms_accepted(aq):
    a = _a_qdq(aq)
    assert a.routed([(_fp8_efq(),)]) is not None


@pytest.mark.parametrize('aq', [IntegerQuantizer(8, True, 'per_tensor'),
                                FloatQuantizer('e4m3', True, 'per_tensor', use_qtorch=True),
                                IntegerQuantizer(8, True, 'per_head', head_num=2),
                                IntegerQuantizer(8, True, 'per_token', calib_algo='mse')])
def test_dynamic_forms_refused(aq):
    assert _a_qdq(aq).routed([(_fp8_efq(),)]) is None


def test_static_forms():
    sym = IntegerQuantizer(8, True, 'per_tensor', calib_algo='static_minmax')
    s = torch.tensor(0.5)
    # CPU buffers: the gather runs on the device, so a CPU-built layer is refused; the rest of the
    # rules are checked through a stand-in whose scales report CUDA
    assert _a_qdq(sym, True).routed([(_static_linear(s),)]) is None

    class Cuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True

    def lin(v, shape=()):
        return _static_linear(torch.full(shape, v).as_subclass(Cuda))
    a = _a_qdq(sym, True)
    one = lin(0.5)
    assert a.routed([(one, one), (lin(0.25), lin(0.25))]) is not None
    assert a.routed([(lin(0.5), lin(0.25))]) is None                    # w1 and w3 scales differ
    assert a.routed([(lin(0.5, (1,)),)]) is None                        # not a 0-dim scale
    assert a.routed([(_fp8_efq(),)]) is None                            # no scale at all
    asym = IntegerQuantizer(8, False, 'per_tensor', calib_algo='static_minmax')
    assert _a_qdq(asym, True).routed([(lin(0.5),)]) is None
    fp8 = FloatQuantizer('e4m3', True, 'per_tensor', use_qtorch=True, calib_algo='static_minmax')
    assert _a_qdq(fp8, True).routed([(lin(0.5),)]) is not None
    per_token_static = IntegerQuantizer(8, True, 'per_token', calib_algo='static_minmax')
    assert _a_qdq(per_token_static, True).routed([(lin(0.5),)]) is None
