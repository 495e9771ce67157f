"""CPU: what the grouped packed MoE entry points refuse before any CUDA call, and which expert
linears module_utils.packed_forward_operands hands to them."""
import ctypes

import pytest
import torch
import torch.nn as nn

from llmc_b200 import _lib
from llmc_b200.module_utils import (EffcientFakeQuantLinear, PackedOperands, VllmRealQuantLinear,
                                    packed_forward_operands)

CAP = _lib.MOE_MAX_EXPERTS


def _ptrs(n, addr=256):
    return (ctypes.c_void_p * n)(*([addr] * n))


@pytest.fixture(scope='module')
def lib():
    return _lib.load()


def _last(lib):
    return lib.llmc_b200_last_error().decode()


def _swiglu(lib, xp=256, bits=4, wq1=None, wq3=None, s1=None, s3=None, z1=None, z3=None, g1=None, g3=None,
            qdt=_lib.BF16, group=128, ng=2, offsets=256, act=256, rows=256, inter=512, K=256, E=4,
            dtype=_lib.BF16):
    w = _ptrs(CAP + 1)
    return lib.llmc_moe_gemm_packed_swiglu(
        ctypes.c_void_p(xp), bits, w if wq1 is None else wq1, w if wq3 is None else wq3, w if s1 is None else s1,
        w if s3 is None else s3, z1, z3, g1, g3, qdt, group, ng, ctypes.c_void_p(offsets), ctypes.c_void_p(act),
        rows, inter, K, E, dtype, None)


def _down(lib, act=256, bits=8, wq2=None, s2=None, z2=None, g2=None, qdt=_lib.F32, group=-512, ng=1,
          offsets=256, w_route=256, y=256, rows=256, N=256, inter=512, E=4, dtype=_lib.F16):
    w = _ptrs(CAP + 1)
    return lib.llmc_moe_gemm_packed_down(
        ctypes.c_void_p(act), bits, w if wq2 is None else wq2, w if s2 is None else s2, z2, g2, qdt, group, ng,
        ctypes.c_void_p(offsets), ctypes.c_void_p(w_route), ctypes.c_void_p(y), rows, N, inter, E, dtype, None)


def test_bits_and_expert_count(lib):
    assert _swiglu(lib, bits=3) == -1 and 'bits=3 must be 4 or 8' in _last(lib)
    assert _down(lib, bits=2) == -1 and 'bits=2 must be 4 or 8' in _last(lib)
    assert _swiglu(lib, E=CAP + 1) == -1 and 'experts outside 1..%d' % CAP in _last(lib)
    assert _down(lib, E=0) == -1 and 'experts outside' in _last(lib)


def test_shapes_and_groups_not_multiples_of_64(lib):
    assert _swiglu(lib, K=200) == -1 and 'K=200 must be a multiple of 64' in _last(lib)
    assert _swiglu(lib, inter=480) == -1 and 'inter=480 must be a multiple of 64' in _last(lib)
    assert _down(lib, N=100) == -1 and 'N=100 must be a multiple of 8' in _last(lib)
    assert _down(lib, inter=480) == -1 and 'K=480 must be a multiple of 64' in _last(lib)
    assert _swiglu(lib, group=96, ng=2) == -1 and 'group 96' in _last(lib)
    assert _swiglu(lib, group=-32) == -1 and 'group 32' in _last(lib)
    assert _swiglu(lib, group=512) == -1 and 'group 512 must divide K=256' in _last(lib)
    assert _swiglu(lib, ng=4) == -1 and 'ng=4' in _last(lib)


def test_dtypes(lib):
    assert _swiglu(lib, dtype=_lib.F32, qdt=_lib.F32) == -1 and 'dtype must be bf16 or fp16' in _last(lib)
    assert _down(lib, dtype=_lib.F32) == -1 and 'dtype must be bf16 or fp16' in _last(lib)
    assert _swiglu(lib, qdt=_lib.F16) == -1 and 'qparam_dtype' in _last(lib)
    # scalar arguments are refused before the rows == 0 return
    assert _swiglu(lib, rows=0, dtype=_lib.F32, qdt=_lib.F32) == -1 and 'dtype must be bf16 or fp16' in _last(lib)
    assert _swiglu(lib, rows=0, qdt=_lib.F16) == -1 and 'qparam_dtype' in _last(lib)


def test_null_arrays_and_entries_name_the_expert(lib):
    assert _swiglu(lib, offsets=0) == -1 and 'null pointer' in _last(lib)
    assert _down(lib, w_route=0) == -1 and 'null pointer' in _last(lib)
    w3 = _ptrs(4)
    w3[2] = None
    assert _swiglu(lib, wq3=w3) == -1 and 'null codes or scales of expert 2' in _last(lib)
    s2 = _ptrs(4)
    s2[3] = None
    assert _down(lib, s2=s2) == -1 and 'null codes or scales of expert 3' in _last(lib)


def test_zeros_and_gidx_for_some_experts_only(lib):
    z = _ptrs(4)
    z[1] = None
    assert _swiglu(lib, z1=z, z3=_ptrs(4)) == -1
    assert 'zeros of expert 1 null while expert 0\'s are given' in _last(lib)
    # w1 with zeros, w3 without
    assert _swiglu(lib, z1=_ptrs(4), z3=None) == -1 and 'zeros of expert 0 null' in _last(lib)
    g = _ptrs(4)
    g[0] = None
    assert _down(lib, g2=g, group=512, ng=4) == -1
    assert 'g_idx of expert 1 given while expert 0\'s is null' in _last(lib)


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
        n = (ctypes.c_void_p * 4)()          # every entry null: never read with rows == 0
        key = 'wq1' if f is _swiglu else 'wq2'
        assert f(lib, rows=0, **{key: n}, **kw) == 0


# ---- packed_forward_operands on CPU-built modules ----------------------------------------------
def _packed(bits=4, N=128, K=256, group=128, zeros=True, qdt=torch.bfloat16, g_idx=False, rz=False):
    ng = K // group
    g = torch.Generator().manual_seed(bits * 7 + N)
    packed = dict(qweight=torch.randint(-2**31, 2**31 - 1, (N, K * bits // 32), generator=g, dtype=torch.int32),
                  scales=torch.rand(N, ng, generator=g).to(qdt),
                  zeros=torch.randint(0, 2**bits, (N, ng), generator=g).to(qdt) if zeros else None,
                  bits=bits, group=group, dtype=torch.bfloat16)
    if g_idx:
        packed['g_idx'] = (torch.randperm(K, generator=g) // group).to(torch.int32)
    if rz:
        packed.update(rz=True, group_axis=0, sym=False)
    return packed


def _efq(packed=None, bias=False, a_qdq=None, N=128, K=256):
    ori = nn.Linear(K, N, bias=bias)
    m = EffcientFakeQuantLinear(None if packed is not None else ori.weight.data,
                                ori.bias.data if bias else None, ori, a_qdq, packed=packed)
    m.in_features, m.out_features = K, N
    return m


def _vllm(bits=4, N=128, K=256, group=128, act_cfg=None, bias=False):
    words = torch.zeros(N, K * bits // 32, dtype=torch.int32)
    s = torch.rand(N, K // group).to(torch.float16)
    m = VllmRealQuantLinear(words, torch.zeros(N) if bias else None, s, None, True, 'weight_scale')
    m.in_features, m.out_features = K, N
    m.act_cfg = act_cfg
    return m


@pytest.mark.parametrize('bits', [4, 8])
@pytest.mark.parametrize('qdt', [torch.bfloat16, torch.float32])
def test_fake_quant_packed_int_forms_are_accepted(bits, qdt):
    m = _efq(_packed(bits=bits, qdt=qdt))
    for dtype in (torch.bfloat16, torch.float16):
        o = packed_forward_operands(m, dtype)
        assert isinstance(o, PackedOperands)
        native = qdt == dtype
        assert o.bits == bits and o.group == 128 and o.transposed and o.g_idx is None
        assert o.wq is m.qweight or torch.equal(o.wq, m.qweight)
        # what linear_forward_w4 hands to the kernel: [ng, N] in the activation dtype or fp32
        want = m.qscales_t.to(dtype if native else torch.float32)
        assert o.scales.dtype == want.dtype and torch.equal(o.scales, want) and o.scales.is_contiguous()
        assert torch.equal(o.zeros, m.qzeros_t.to(want.dtype))


def test_fake_quant_symmetric_and_gidx():
    m = _efq(_packed(zeros=False, g_idx=True, qdt=torch.float32))
    o = packed_forward_operands(m, torch.bfloat16)
    assert o.zeros is None and torch.equal(o.g_idx, m.g_idx) and o.g_idx.dtype == torch.int32


@pytest.mark.parametrize('case', ['w2', 'w3', 'rz', 'fp8', 'a_qdq', 'bias', 'hook', 'pre_hook', 'dense'])
def test_fake_quant_forms_refused(case):
    if case in ('w2', 'w3'):
        bits = int(case[1])
        p = _packed(bits=4)
        p['bits'] = bits
        m = _efq(p)
    elif case == 'rz':
        m = _efq(_packed(rz=True, qdt=torch.float32))
    elif case == 'fp8':
        p = _packed(bits=8, zeros=False)
        p['qweight'] = torch.zeros(128, 256, dtype=torch.float8_e4m3fn)
        m = _efq(p)
    elif case == 'a_qdq':
        m = _efq(_packed(), a_qdq=lambda x, layer: x)
    elif case == 'bias':
        m = _efq(_packed(), bias=True)
    elif case == 'dense':
        m = _efq(None)
    else:
        m = _efq(_packed())
        (m.register_forward_hook(lambda *a: None) if case == 'hook'
         else m.register_forward_pre_hook(lambda *a: None))
    assert packed_forward_operands(m, torch.bfloat16) is None


@pytest.mark.parametrize('bits', [4, 8])
def test_vllm_packed_export_is_accepted(bits):
    m = _vllm(bits=bits)
    o = packed_forward_operands(m, torch.bfloat16)
    assert o.bits == bits and o.group == 128 and not o.transposed and o.zeros is None and o.g_idx is None
    assert o.scales.dtype == torch.float32 and torch.equal(o.scales, m.weight_scale.float())
    o16 = packed_forward_operands(m, torch.float16)
    assert o16.scales.dtype == torch.float16 and torch.equal(o16.scales, m.weight_scale)


@pytest.mark.parametrize('case', ['w_act', 'bias', 'group32', 'hook', 'w8a8'])
def test_vllm_forms_refused(case):
    if case == 'w_act':
        m = _vllm(act_cfg={'bit': 8})
    elif case == 'bias':
        m = _vllm(bias=True)
    elif case == 'group32':
        m = _vllm(group=32)
    elif case == 'hook':
        m = _vllm()
        m.register_forward_hook(lambda *a: None)
    else:
        m = VllmRealQuantLinear(torch.zeros(128, 256, dtype=torch.int8), None, torch.ones(128, 1), None, False,
                                'weight_scale')
        m.in_features, m.out_features = 256, 128
    assert packed_forward_operands(m, torch.bfloat16) is None


def test_plain_linears_refused():
    assert packed_forward_operands(nn.Linear(256, 128, bias=False), torch.bfloat16) is None
