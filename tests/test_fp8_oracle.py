"""CPU: the FP8 oracle (oracle/fp8_oracle.py) on hand-computed cases, and the FloatQuantizer checks
that need no device.

The oracle restates the reference's FloatQuantizer (quant.py:1061-1081, 1161-1221) with IEEE
round-to-nearest-even standing in for qtorch (PARITY UNPINNED, see the oracle's header).  Every
value below is worked out by hand from the grids: e4m3fn has 3 mantissa bits, exponent bias 7,
smallest subnormal 2^-9 and maximum 448; e5m2 has 2 mantissa bits, bias 15, smallest subnormal
2^-16 and maximum 57344."""
import pytest
import torch

from oracle import fp8_oracle as fo

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2


def _codes(q):
    return q.view(torch.uint8).tolist()


@pytest.mark.parametrize('bit,x,expected', [
    # e4m3: spacing 1/8 in [1, 2); 1 + 1/16 lies half way between 1 (even) and 1.125 (odd)
    ('e4m3', 1.0625, 1.0), ('e4m3', 1.1875, 1.25), ('e4m3', -1.0625, -1.0),
    # e5m2: spacing 1/4 in [1, 2); 1.125 lies between 1 (even) and 1.25 (odd)
    ('e5m2', 1.125, 1.0), ('e5m2', 1.375, 1.5), ('e5m2', -1.375, -1.5),
    # just off the tie rounds to the nearer neighbour
    ('e4m3', 1.0625 + 2 ** -20, 1.125), ('e5m2', 1.125 - 2 ** -20, 1.0),
])
def test_rne_ties(bit, x, expected):
    assert fo.float_quantize(torch.tensor([x]), bit).item() == expected


@pytest.mark.parametrize('bit,tiny', [('e4m3', 2.0 ** -9), ('e5m2', 2.0 ** -16)])
def test_smallest_subnormal(bit, tiny):
    x = torch.tensor([tiny, tiny / 2, tiny * 0.75, tiny * 1.5, -tiny])
    q = fo.float_quantize(x, bit)
    # tiny / 2 is a tie between 0 (even) and tiny (code 1); 1.5 * tiny ties to 2 * tiny (code 2)
    assert q.tolist() == [tiny, 0.0, tiny, 2 * tiny, -tiny]
    assert _codes(q.to(fo.FP8[bit])) == [0x01, 0x00, 0x01, 0x02, 0x81]


@pytest.mark.parametrize('bit,fmax,code', [('e4m3', 448.0, 0x7E), ('e5m2', 57344.0, 0x7B)])
def test_saturation(bit, fmax, code):
    x = torch.tensor([fmax * 1.5, -fmax * 1.5, 1e30, float('inf'), -float('inf')])
    q = fo.float_quantize(x, bit)
    assert q.tolist() == [fmax, -fmax, fmax, fmax, -fmax]
    assert _codes(q.to(fo.FP8[bit])) == [code, code | 0x80, code, code, code | 0x80]


@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
def test_negative_zero_gives_code_zero(bit):
    """x / s + 0.0 (quant.py:1063): -0.0 + 0.0 is +0.0, so -0.0 quantises to code 0x00."""
    x = torch.tensor([[-0.0, 1.0]], dtype=torch.bfloat16)
    q = fo.quant(x, torch.tensor([[0.5]], dtype=torch.bfloat16), bit)
    assert _codes(q.to(fo.FP8[bit]))[0][0] == 0x00


def test_fp16_scale_underflow_exports_scale_one():
    """fp16, e5m2: absmax 1e-3 / 57344 = 1.7e-8 is below half the smallest fp16 subnormal (2^-25), so
    get_qparams gives 0; quant() sets it to 1 in place and the export returns that 1 with codes
    e5m2(x).  e4m3: an all-zero row gives 1e-5 / 448, which underflows too."""
    w = torch.tensor([[1e-3, -5e-4, 2.5e-4, 0.0], [0.5, -0.25, 0.125, 1.0]], dtype=torch.float16)
    s = fo.qparams(w, 'e5m2', 'per_channel')
    assert s.dtype == torch.float16 and s[0, 0].item() == 0.0 and s[1, 0].item() != 0.0
    q, sq = fo.real_quant_dynamic(w, 'e5m2', 'per_channel')
    assert sq[0, 0].item() == 1.0 and sq[1, 0].item() == s[1, 0].item()
    assert torch.equal(q[0].view(torch.uint8), w[0].float().to(E5M2).view(torch.uint8))
    assert q[0].float().tolist() == [1.0 / 1024, -1.0 / 2048, 1.0 / 4096, 0.0]    # all on the e5m2 grid
    y, _ = fo.fake_quant_dynamic(w, 'e5m2', 'per_channel')
    assert torch.equal(y, (q.float() * sq).to(torch.float16))

    z = torch.zeros(2, 8, dtype=torch.float16)
    assert fo.qparams(z, 'e4m3', 'per_channel').eq(0).all()
    qz, sz = fo.real_quant_dynamic(z, 'e4m3', 'per_channel')
    assert sz.eq(1).all() and qz.view(torch.uint8).eq(0).all()


def test_quant_sets_zero_scales_to_one_in_place():
    s = torch.tensor([[0.0], [0.5]])
    q = fo.quant(torch.tensor([[3.0, -2.0], [3.0, -2.0]]), s, 'e4m3')
    assert s.tolist() == [[1.0], [0.5]]
    assert q.tolist() == [[3.0, -2.0], [6.0, -4.0]]


def test_quant_dequant_is_fp32():
    x = torch.tensor([[1.0, 0.3]], dtype=torch.bfloat16)
    y = fo.quant_dequant(x, torch.tensor([[0.25]], dtype=torch.bfloat16), 'e4m3')
    assert y.dtype == torch.float32 and y.tolist() == [[1.0, 0.3125]]      # 0.3 / 0.25 = 1.203 -> 1.25


def test_static_scales_follow_torch_promotion():
    """1.0 / s with s = fp32(1 / 1.063): the fp32 quotient 1.063 lies above the e4m3 tie 1.0625 and
    rounds to 1.125; rounded to bf16 first it is exactly 1.0625, the tie, and goes to 1.0.  A 0-dim
    scale keeps the bf16 quotient, a [1, 1] fp32 scale promotes it to fp32, a [1, 1] bf16 one keeps bf16."""
    x = torch.tensor([[1.0]], dtype=torch.bfloat16)
    s = torch.tensor(1 / 1.063)
    assert (x / s).dtype == torch.bfloat16 and (x / s.view(1, 1)).dtype == torch.float32
    assert fo.quant(x, s.clone(), 'e4m3').item() == 1.0
    assert fo.quant(x, s.view(1, 1).clone(), 'e4m3').item() == 1.125
    sb = s.view(1, 1).bfloat16()
    assert fo.quant(x, sb, 'e4m3').item() == fo.float_quantize((x.float() / sb.float()).bfloat16(), 'e4m3').item()


def test_per_head_groups_rows_by_head():
    """quant.py:633-634: per_head reshapes to (head_num, -1), one scale over each head's rows."""
    w = torch.tensor([[1.0, 2.0], [4.0, 8.0], [0.5, 0.25], [0.125, 448.0]])
    t = fo.reshape(w, 'per_head', head_num=2)
    assert t.shape == (2, 4)
    assert torch.equal(fo.qparams(t, 'e4m3', 'per_head'), torch.tensor([[8.0], [448.0]]) / 448.0)


def test_block_quant_ragged_and_e5m2():
    """A 3 x 5 weight in 2 x 2 blocks: scales over the zero-padded blocks, codes cut to 3 x 5."""
    w = torch.tensor([[1.0, -2.0, 3.0, 0.0, 7.0], [0.5, 4.0, -6.0, 1.0, 0.0], [8.0, 0.0, 0.0, 0.0, -448.0]])
    q, s = fo.block_quant(w, 'e5m2', 2)
    assert s.shape == (2, 3) and q.shape == (3, 5)
    # block absmaxes 4, 6, 7 / 8, 0 (clamped to 1e-5), 448
    assert torch.equal(s, torch.tensor([[4.0, 6.0, 7.0], [8.0, 1e-5, 448.0]]) / 57344.0)
    full = s.repeat_interleave(2, 0)[:3].repeat_interleave(2, 1)[:, :5]
    assert torch.equal(q.float(), fo.float_quantize(w / full, 'e5m2'))
    y, _ = fo.block_fake_quant(w.bfloat16(), 'e5m2', 2)
    assert y.dtype == torch.bfloat16 and torch.equal(y, (q.float() * full).bfloat16())


def test_float_range_is_refused():
    """The kernels scale to finfo.max and saturate there, so a custom float_range would be honoured
    by the per-tensor path only; the quantizer refuses it instead."""
    from llmc_b200.quant_float import FloatQuantizer
    with pytest.raises(NotImplementedError, match='float_range'):
        FloatQuantizer('e4m3', True, 'per_channel', use_qtorch=True, float_range=(-240.0, 240.0))
    q = FloatQuantizer('e5m2', True, 'per_channel', use_qtorch=True)
    assert q.qmax.item() == 57344.0 and q.qmin.item() == -57344.0
