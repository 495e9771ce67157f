"""GPU: FloatQuantizer (e4m3 / e5m2, use_qtorch semantics) vs the oracle restatement.
PARITY UNPINNED at the rounding boundary (qtorch absent, see oracle/fp8_oracle.py); what is
checked bit-exactly here is our kernel against IEEE RNE onto the fp8 grid + the reference's
dtype flow."""
import pytest
import torch

from oracle import fp8_oracle as fo

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('gran,gs', [('per_tensor', None), ('per_channel', None), ('per_group', 128)])
def test_fp8_weight_quant(dtype, bit, gran, gs):
    from llmc_b200.quant_float import FloatQuantizer
    torch.manual_seed(7)
    w = (torch.randn(96, 512) * 0.05)
    w[:, ::37] *= 7
    w = w.to(dtype)
    kw = {'group_size': gs} if gs else {}
    q = FloatQuantizer(bit, True, gran, use_qtorch=True, **kw)
    y = q.fake_quant_weight_dynamic(w.cuda())
    yo, so = fo.fake_quant_dynamic(w, bit, gran, gs)
    assert y.dtype == dtype and torch.equal(y.cpu(), yo)
    fw, s, z = q.real_quant_weight_dynamic(w.cuda())
    fo_w, fo_s = fo.real_quant_dynamic(w, bit, gran, gs)
    assert z is None and fw.dtype == fo.FP8[bit]
    assert torch.equal(fw.cpu().view(torch.uint8), fo_w.view(torch.uint8))
    assert torch.equal(s.cpu().float().reshape(-1), fo_s.float().reshape(-1))


def test_fp8_static_act_per_tensor():
    from llmc_b200.quant_float import FloatQuantizer
    torch.manual_seed(1)
    x = (torch.randn(4, 33, 256) * 3).bfloat16()
    q = FloatQuantizer('e4m3', True, 'per_tensor', use_qtorch=True, calib_algo='static_minmax')
    sc, zs, qmins, qmaxs = q.get_batch_tensors_qparams([x.cuda()])
    args = {'scales': sc[0], 'zeros': zs[0], 'qmax': qmaxs[0], 'qmin': qmins[0]}
    y = q.fake_quant_act_static(x.cuda(), args)
    # oracle: static min/max = mean of per-sample min/max (quant.py:253-263)
    mins = torch.stack([x[i].min().float() for i in range(4)]).mean()
    maxs = torch.stack([x[i].max().float() for i in range(4)]).mean()
    s = torch.max(maxs.abs(), mins.abs()).clamp(min=1e-5) / torch.tensor(448.0)
    assert torch.allclose(sc[0].cpu().float(), s, rtol=1e-6)
    yo = fo.fake_quant_static(x, sc[0].cpu().clone(), 'e4m3', 'per_tensor')
    assert torch.equal(y.cpu(), yo)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('M,N', [(256, 384), (200, 300), (128, 128), (1024, 4096)])
def test_block_fp8_cast_roundtrip_matches_oracle(dtype, M, N):
    """Q10: weight_cast_to_fp8 / weight_cast_to_bf16 (quant.py:18-43), 128x128 block scales, incl.
    ragged edges.  Exact vs the oracle restatement (rounding itself: parity unpinned, see header)."""
    from llmc_b200.quant_float import weight_cast_to_bf16, weight_cast_to_fp8
    from oracle import fp8_oracle as fo
    g = torch.Generator().manual_seed(M + N)
    w = (torch.randn(M, N, generator=g) * 0.05).to(dtype)
    w[:, ::37] *= 6
    q, s = weight_cast_to_fp8(w.cuda(), 128)
    q_o, s_o = fo.block_quant(w, 'e4m3', 128)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and s.shape == s_o.shape
    assert torch.equal(s.cpu(), s_o)
    qb, qo = q.cpu().view(torch.uint8), q_o.view(torch.uint8)
    bad = (qb != qo).nonzero()
    detail = [(int(i), int(j), float(w[i, j]), float(s_o[i // 128, j // 128]), int(qb[i, j]), int(qo[i, j]))
              for i, j in bad[:6].tolist()]
    assert len(bad) == 0, (len(bad), detail)
    back = weight_cast_to_bf16(q, s, 128)
    assert torch.equal(back.cpu(), fo.block_dequant(q_o, s_o, 128))


def test_llmc_fp8_linear_forward():
    from llmc_b200.module_utils import LlmcFp8Linear, linear_forward
    from llmc_b200.quant_float import weight_cast_to_bf16, weight_cast_to_fp8
    torch.manual_seed(0)
    lin = torch.nn.Linear(512, 384, bias=False)
    m = LlmcFp8Linear.new(lin, 128).cuda()
    w = (torch.randn(384, 512, device='cuda') * 0.05).bfloat16()
    q, s = weight_cast_to_fp8(w, 128)
    m.weight.data, m.weight_scale_inv.data = q, s
    x = torch.randn(4, 64, 512, device='cuda').bfloat16()
    y = m(x)
    assert m.weight.dtype == torch.bfloat16                      # dequantised once (module_utils.py:171-178)
    assert torch.equal(y, linear_forward(x, weight_cast_to_bf16(q, s, 128)))
