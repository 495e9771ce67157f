"""GPU parity: the sm_90a quantize / pack kernels (through the C ABI, via the reference-shaped
Python classes) against the oracle and the reference-generated golden fixtures.
Bar: bit-exact for codes, packed words, zeros; scales bit-exact too (tolerance 0)."""
import os

import pytest
import torch

from oracle import quant_oracle as qo

pytestmark = pytest.mark.gpu


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name), weights_only=False)


def _q(bit, sym, gran, gs=None, **kw):
    from llmc_b200.quant import IntegerQuantizer
    if gs:
        kw['group_size'] = gs
    return IntegerQuantizer(bit, sym, gran, **kw)


def _same(a, b):
    a = a.cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    assert a.dtype == b.dtype, (a.dtype, b.dtype)
    if not torch.equal(a, b):
        bad = (a != b).sum().item()
        raise AssertionError(f'{bad}/{a.numel()} elements differ; first: '
                             f'{a[a != b][:4].tolist()} vs {b[a != b][:4].tolist()}')


def test_golden_dynamic(golden_dir):
    kat = _load(golden_dir, 'quant_kat.pt')
    for c in kat['dynamic']:
        q = _q(c['bit'], c['sym'], c['granularity'], c['group_size'])
        w = c['w'].cuda()
        _, s, z, qmax, qmin = q.get_tensor_qparams(w)
        _same(s, c['scales'])
        assert torch.equal(z.float().cpu().reshape(-1), c['zeros'].float().reshape(-1))
        codes, rs, rz = q.real_quant_weight_dynamic(w)
        _same(codes, c['codes'])
        _same(rs, c['real_scales'])
        if c['real_zeros'] is None:
            assert rz is None
        else:
            _same(rz, c['real_zeros'])
        _same(q.fake_quant_weight_dynamic(w), c['qdq'])


def test_golden_static_and_act(golden_dir):
    kat = _load(golden_dir, 'quant_kat.pt')
    for c in kat['static']:
        q = _q(c['bit'], c['sym'], 'per_group', c['group_size'])
        args = dict(scales=c['scales'].cuda(), zeros=c['zeros'].cuda(), qmax=c['qmax'],
                    qmin=c['qmin'])
        _same(q.fake_quant_weight_static(c['w'].cuda(), dict(args)), c['qdq'])
        codes, rs, rz = q.real_quant_weight_static(c['w'].cuda(), dict(args))
        _same(codes, c['codes'])
        _same(rz, c['real_zeros'])
    for c in kat['acts']:
        q = _q(c['bit'], c['sym'], 'per_token')
        _same(q.fake_quant_act_dynamic(c['x'].cuda()), c['qdq'])


def test_golden_pack(golden_dir):
    from llmc_b200.module_utils import AutoawqRealQuantLinear, VllmRealQuantLinear
    kat = _load(golden_dir, 'pack_kat.pt')
    for c in kat['vllm']:
        q = _q(c['bit'], c['sym'], c['granularity'], c['group_size'])
        lin = torch.nn.Linear(c['w'].shape[1], c['w'].shape[0], bias=False)
        lin.weight.data = c['w'].clone()
        lin = lin.cuda()
        cfg = {'weight': {'bit': c['bit'], 'need_pack': True, 'granularity': c['granularity']}}
        packed, scales = VllmRealQuantLinear.quant_pack(
            lin, lambda m: q.real_quant_weight_dynamic(m.weight.data), cfg)
        _same(packed, c['packed'])
        _same(scales, c['scales'])
    for c in kat['awq']:
        q = _q(4, False, 'per_group', c['group_size'])
        lin = torch.nn.Linear(c['w'].shape[1], c['w'].shape[0], bias=False)
        lin.weight.data = c['w'].clone()
        lin = lin.cuda()
        cfg = {'weight': {'bit': 4, 'group_size': c['group_size'], 'pack_version': 'gemm_pack'}}
        qweight, scales, qzeros = AutoawqRealQuantLinear.quant_pack(
            lin, lambda m: q.real_quant_weight_dynamic(m.weight.data), cfg)
        _same(qweight, c['qweight'])
        _same(scales, c['scales'])
        _same(qzeros, c['qzeros'])


SHAPES = [(4096, 4096), (1024, 4096), (3072, 768), (14336, 4096)]


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize('bit,sym,gran,gs', [
    (4, False, 'per_group', 128), (4, True, 'per_group', 128), (8, True, 'per_channel', None),
    (4, True, 'per_group', 64), (8, False, 'per_group', 256), (3, False, 'per_group', 128),
    (4, False, 'per_tensor', None), (8, True, 'per_group', 512),
    # asymmetric PACK on the fast kernels (the reference's overflowing +2^(bit-1) offset)
    (8, False, 'per_group', 128), (4, False, 'per_group', 64), (4, False, 'per_channel', None),
    (8, False, 'per_channel', None)])
def test_oracle_full_shapes(dtype, bit, sym, gran, gs):
    """Seeded random weights at model shapes; every output bit-exact vs the CPU oracle."""
    torch.manual_seed(1234 + bit)
    rows, cols = SHAPES[(bit + (gs or 0)) % len(SHAPES)]
    rows = min(rows, 1024)                           # keep the CPU oracle to seconds
    w = (torch.randn(rows, cols) * 0.02)
    w[:, ::97] *= 6
    w = w.to(dtype)
    q = _q(bit, sym, gran, gs)
    wc = w.cuda()
    codes, s, z = q.real_quant_weight_dynamic(wc)
    ocodes, os_, oz = qo.real_quant_dynamic(w, bit, sym, gran, gs)
    _same(codes, ocodes)
    _same(s, os_)
    if oz is None:
        assert z is None
    else:
        _same(z, oz)
    _same(q.fake_quant_weight_dynamic(wc), qo.fake_quant_dynamic(w, bit, sym, gran, gs))
    if gran != 'per_tensor' and bit in (4, 8):
        packed, ps, _ = q.real_quant_pack_vllm_dynamic(wc)
        opacked, _ = qo.pack_vllm(ocodes, os_, bit)
        _same(packed, opacked)


def test_ragged_and_empty():
    """cols not a multiple of 8 (generic kernels), per_group < group (falls back to rows),
    zero-row input, indivisible group -> ValueError like quant.py:627-630."""
    q = _q(4, True, 'per_channel')
    w = (torch.randn(7, 100) * 0.1).half()
    codes, s, z = q.real_quant_weight_dynamic(w.cuda())
    oc, os_, _ = qo.real_quant_dynamic(w, 4, True, 'per_channel')
    _same(codes, oc)
    _same(s, os_)
    _same(q.fake_quant_weight_dynamic(w.cuda()), qo.fake_quant_dynamic(w, 4, True, 'per_channel'))
    q = _q(4, False, 'per_group', 128)
    w = (torch.randn(5, 64) * 0.1).bfloat16()          # cols < group_size: per-row groups
    _same(q.fake_quant_weight_dynamic(w.cuda()), qo.fake_quant_dynamic(w, 4, False, 'per_group', 128))
    with pytest.raises(ValueError):
        q.fake_quant_weight_dynamic(torch.zeros(4, 200, dtype=torch.float16, device='cuda'))
    e = torch.zeros(0, 128, dtype=torch.float16, device='cuda')
    assert q.fake_quant_weight_dynamic(e).shape == (0, 128)


def test_cpu_tensor_fails_loudly():
    from llmc_b200._lib import LlmcB200Error
    q = _q(4, True, 'per_group', 128)
    with pytest.raises(LlmcB200Error):
        q.fake_quant_weight_dynamic(torch.zeros(4, 128, dtype=torch.float16))


def test_full_size_properties():
    """Llama-3-8B gate_proj shape: idempotence of fake-quant (qdq(qdq(w)) == qdq(w) holds for
    symmetric grids), codes within range, pack->unpack round trip."""
    torch.manual_seed(0)
    w = (torch.randn(14336, 4096, device='cuda') * 0.02).bfloat16()
    q = _q(4, True, 'per_group', 128)
    y = q.fake_quant_weight_dynamic(w)
    codes, s, _ = q.real_quant_weight_dynamic(w)
    assert int(codes.min()) >= -8 and int(codes.max()) <= 7
    packed, ps, _ = q.real_quant_pack_vllm_dynamic(w)
    shifts = torch.arange(8, device='cuda', dtype=torch.int32) * 4
    un = ((packed.unsqueeze(-1) >> shifts) & 0xF).reshape(14336, 4096) - 8
    assert torch.equal(un, codes)
    # dequantising the codes with the returned scales reproduces the fake-quant output
    deq = (codes.reshape(-1, 128).to(torch.bfloat16) * s.reshape(-1, 1)).reshape(14336, 4096)
    assert torch.equal(deq, y)
