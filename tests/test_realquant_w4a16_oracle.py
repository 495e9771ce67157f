"""CPU: the weight-only real-quant forwards' oracle (tests/w4a16_export_oracle.py) pinned to the packed
words the reference's own packers wrote (tests/golden/pack_kat.pt), the argument checks of
llmc_gemm_w4a16_awq, and the reasons the real-quant modules give for the layouts they do not run."""
import ctypes
import os

import pytest
import torch

import w4a16_export_oracle as eo
from oracle import quant_oracle as qo


def _kat(golden_dir):
    return torch.load(os.path.join(golden_dir, 'pack_kat.pt'), weights_only=False)


def _reference_awq_codes(w, s, z, group):
    """The unclamped codes of the reference's gemm_pack (module_utils.py:1022-1029), [C, R]."""
    s16 = s.t().contiguous().to(torch.float16)
    z = z.t().contiguous()
    g = torch.arange(w.shape[1]) // group
    return torch.round((w + (z * s16)[g].t()) / s16[g].t()).to(torch.int32).t()


def test_awq_decoder_recovers_the_reference_codes(golden_dir):
    cases = _kat(golden_dir)['awq']
    checked = 0
    for c in cases:
        w, group = c['w'], c['group_size']
        _, s, z = qo.real_quant_dynamic(w, 4, False, 'per_group', group)
        codes = _reference_awq_codes(w, s, z, group)               # [K, N]
        got = eo.awq_nibbles(c['qweight'])
        # a word whose 8 codes all lie in 0..15 holds each of them in its own nibble
        in_range = ((codes >= 0) & (codes <= 15)).reshape(codes.shape[0], -1, 8).all(-1)
        mask = in_range.repeat_interleave(8, dim=1)
        assert torch.equal(got[mask], codes[mask])
        checked += int(mask.sum())
        # every word, carries included, is the OR of the shifted codes: what the forward decodes
        words = torch.zeros_like(c['qweight'])
        for i, col in enumerate(eo.AWQ_ORDER):
            words |= codes[:, col::8] << (4 * i)
        assert torch.equal(words, c['qweight'])
        assert torch.equal(eo.awq_nibbles(c['qzeros']), z.t().to(torch.int32))
        # the dequantised weight where every code of the word is in range is rT((code - z) * s)
        deq = eo.awq_dequant(c['qweight'], c['scales'], c['qzeros'], group, w.dtype).t()
        g = torch.arange(w.shape[1]) // group
        want = ((codes - z.t()[g]).float() * c['scales'].float()[g]).to(w.dtype)
        assert torch.equal(deq[mask], want[mask])
    assert checked >= 256 * 8


def test_vllm_decoder_recovers_the_reference_codes(golden_dir):
    for c in _kat(golden_dir)['vllm']:
        K = c['w'].shape[1]
        codes, s, _ = qo.real_quant_dynamic(c['w'], c['bit'], c['sym'], c['granularity'], c['group_size'])
        # stored as code + 2^(bits-1), also for an asymmetric grid, where a code can then overflow its
        # field and carry into the next: compare the words whose every stored code fits its field
        bit, pf = c['bit'], 32 // c['bit']
        stored = codes.to(torch.int32) + (1 << (bit - 1))
        pad = -K % pf
        fits = torch.nn.functional.pad((stored >= 0) & (stored < (1 << bit)), (0, pad), value=True)
        mask = fits.reshape(fits.shape[0], -1, pf).all(-1).repeat_interleave(pf, dim=1)[:, :K]
        got = eo.vllm_codes(c['packed'], bit, K)
        assert torch.equal(got[mask], stored[mask])
        assert c['sym'] <= bool(mask.all())                       # a symmetric grid always fits
        if c['sym'] and K % c['scales'].shape[1] == 0:
            deq = eo.vllm_dequant(c['packed'], c['scales'], c['bit'], K, c['w'].dtype)
            group = K // c['scales'].shape[1]
            g = torch.arange(K) // group
            assert torch.equal(deq, (codes.float() * c['scales'].float()[:, g]).to(c['w'].dtype))


def test_awq_entry_point_argument_errors_without_gpu():
    from llmc_b200 import _lib
    lib = _lib.load()
    null, p, odd = ctypes.c_void_p(0), ctypes.c_void_p(256), ctypes.c_void_p(260)

    def last():
        return lib.llmc_b200_last_error().decode()

    f = lib.llmc_gemm_w4a16_awq
    bf16 = _lib.dtype_enum(torch.bfloat16)
    assert f(p, p, p, p, null, p, 128, 256, 100, 100, bf16, null) == -1 and 'must divide K=100' in last()
    assert f(p, p, p, p, null, p, 128, 256, 256, 96, bf16, null) == -1 and 'group 96 must divide' in last()
    assert f(p, p, p, p, null, p, 128, 256, 192, 128, bf16, null) == -1 and 'group 128 must divide' in last()
    assert f(p, p, p, p, null, p, 128, 136, 128, 128, bf16, null) == -1 and 'N=136' in last()
    assert f(p, p, p, p, null, p, 128, 256, 128, 128, 7, null) == -1 and 'bf16 or fp16' in last()
    for i in range(5):
        args = [p, p, p, p, p]
        args[i] = null
        a = args[:4] + [null, args[4]]
        assert f(*a, 128, 256, 128, 128, bf16, null) == -1 and 'null pointer' in last()
    for i in range(5):
        args = [p, p, p, p, p]
        args[i] = odd
        a = args[:4] + [null, args[4]]
        assert f(*a, 128, 256, 128, 128, bf16, null) == -4 and '16-byte aligned' in last()
    assert f(null, null, null, null, null, null, 0, 256, 128, 128, bf16, null) == 0     # M = 0: no-op
    assert f(p, p, p, p, null, p, -1, 256, 128, 128, bf16, null) == -1 and 'bad shape' in last()


def _vllm(words, scales=None, act=None, in_features=64, scales_name='weight_scale'):
    from llmc_b200.module_utils import VllmRealQuantLinear
    s = torch.ones(words.shape[0], 1, dtype=torch.float16) if scales is None else scales
    m = VllmRealQuantLinear(words, None, s, None, True, scales_name)
    m.in_features, m.out_features = in_features, words.shape[0]
    m.act_cfg = act
    return m


def test_packed_modules_say_why_they_do_not_run():
    x = torch.zeros(2, 64, dtype=torch.bfloat16)
    cases = [
        (_vllm(torch.zeros(4, 8, dtype=torch.int32), act={'bit': 8, 'granularity': 'per_token'}),
         'weight_packed'),
        (_vllm(torch.zeros(4, 4, dtype=torch.int32)), '4- and 8-bit'),                 # 2-bit words
        (_vllm(torch.zeros(4, 12, dtype=torch.int32), in_features=96), 'multiples of 64'),
        (_vllm(torch.zeros(4, 8, dtype=torch.int32), torch.ones(4, 3, dtype=torch.float16)), 'groups'),
        (_vllm(torch.zeros(4, 16, dtype=torch.int32), torch.ones(4, 4, dtype=torch.float16), in_features=128),
         'group=32'),
        (_vllm(torch.zeros(4, 8, dtype=torch.int32), scales_name='weight_scale_inv'), 'weight_scale'),
    ]
    for m, match in cases:
        assert m.packed_unsupported() is not None
        with pytest.raises(NotImplementedError, match=match):
            m(x)
        assert m.w8a8_unsupported() is not None
    ok = _vllm(torch.zeros(4, 8, dtype=torch.int32))
    assert ok.packed_unsupported() is None
    w8 = _vllm(torch.zeros(4, 32, dtype=torch.int32), torch.ones(4, 1, dtype=torch.float16), in_features=128)
    assert w8.packed_unsupported() is None


def test_awq_module_and_forward_say_why():
    from llmc_b200.module_utils import AutoawqRealQuantLinear, linear_forward_w4a16_awq
    x = torch.zeros(2, 128, dtype=torch.bfloat16)
    qw = torch.zeros(128, 32, dtype=torch.int32)
    s = torch.ones(1, 256, dtype=torch.float16)
    qz = torch.zeros(1, 32, dtype=torch.int32)
    m = AutoawqRealQuantLinear(qw, None, s, None)
    m.in_features = 128
    with pytest.raises(NotImplementedError, match='without qzeros'):
        m(x)
    with pytest.raises(ValueError, match='fp16 scales'):
        linear_forward_w4a16_awq(x, qw, s.float(), qz, 128)
    with pytest.raises(ValueError, match='does not match K=128'):
        linear_forward_w4a16_awq(x, qw[:64], s, qz, 128)
    with pytest.raises(ValueError, match='do not match'):
        linear_forward_w4a16_awq(x, qw, s, qz, 64)
    with pytest.raises(ValueError, match='bf16 or fp16'):
        linear_forward_w4a16_awq(x.float(), qw, s, qz, 128)
    with pytest.raises(NotImplementedError, match='multiples of 64'):
        linear_forward_w4a16_awq(x, qw, torch.ones(4, 256, dtype=torch.float16), torch.zeros(4, 32, dtype=torch.int32), 32)
    with pytest.raises(NotImplementedError, match='N % 32'):
        linear_forward_w4a16_awq(x, qw[:, :3], torch.ones(1, 24, dtype=torch.float16),
                                 torch.zeros(1, 3, dtype=torch.int32), 128)
