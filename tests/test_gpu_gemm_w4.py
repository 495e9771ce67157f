"""GPU: the fused dequant->GEMM (packed INT4 weights) must equal the wgmma GEMM on the
materialised fake-quant weight BIT FOR BIT (same tiles, same K order, identical operand bits),
for RTN-style (model dtype) and GPTQ-style (fp32) scales, sym and asym."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _pack_unsigned(codes_u):
    """[N, K] int (0..15) -> [N, K/8] int32, nibble i = element 8*w + i (vLLM order)."""
    N, K = codes_u.shape
    c = codes_u.to(torch.int64).reshape(N, K // 8, 8)
    sh = torch.arange(8, device=c.device, dtype=torch.int64) * 4
    w = (c << sh).sum(-1)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w)
    return w.to(torch.int32)


@pytest.mark.parametrize('native', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('sym', [True, False])
@pytest.mark.parametrize('M,N,K,g', [(128, 256, 128, 128), (300, 520, 512, 128), (2048, 4096, 4096, 128),
                                     (512, 1024, 1024, 64), (4096, 14336, 4096, 128),
                                     (300, 519, 512, 128)])
def test_fused_equals_materialised(dtype, sym, M, N, K, g, native):
    """native: qparams handed over in the activation dtype -> packed half2 / bf16x2 dequant;
    otherwise as fp32 -> fp32 dequant.  Both must reproduce the materialised weight bit for bit."""
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    from llmc_b200.quant import IntegerQuantizer
    torch.manual_seed(M + N + K + int(sym))
    w = (torch.randn(N, K, device='cuda') * 0.02).to(dtype)
    x = torch.randn(M, K, device='cuda').to(dtype)
    q = IntegerQuantizer(4, sym, 'per_group', group_size=g)
    codes, scales, zeros = q.real_quant_weight_dynamic(w)            # int32 codes, [N, ng] scales
    wqdq = q.fake_quant_weight_dynamic(w)                             # what FakeQuantLinear materialises
    qdt = dtype if native else torch.float32
    if sym:
        packed, z = _pack_unsigned(codes + 8), None                  # +8 offset, zero = 8
    else:
        packed, z = _pack_unsigned(codes), zeros.to(qdt)
    y_ref = linear_forward(x, wqdq)
    y = linear_forward_w4(x, packed, scales.to(qdt), z, g)
    assert torch.equal(y, y_ref)


def test_fused_with_fp32_gptq_scales_and_bias():
    """GPTQ dynamic groups carry fp32 scales: dequant = bf16(fp32((q - z) * s32))."""
    from llmc_b200.module_utils import linear_forward, linear_forward_w4
    torch.manual_seed(3)
    N, K, M, g = 768, 1024, 640, 128
    codes = torch.randint(0, 16, (N, K), device='cuda')
    s = (torch.rand(N, K // g, device='cuda') * 0.01 + 0.001)
    z = torch.randint(0, 16, (N, K // g), device='cuda').float()
    wdq = ((codes.reshape(N, -1, g).float() - z[..., None]) * s[..., None]).reshape(N, K).bfloat16()
    x = torch.randn(M, K, device='cuda').bfloat16()
    b = torch.randn(N, device='cuda').bfloat16()
    y = linear_forward_w4(x, _pack_unsigned(codes), s, z, g, bias=b)
    assert torch.equal(y, linear_forward(x, wdq, b))


@pytest.mark.parametrize('native', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('sym,gran,g', [(True, 'per_channel', None), (True, 'per_group', 128),
                                        (False, 'per_group', 128), (False, 'per_group', 64)])
@pytest.mark.parametrize('M,N,K', [(128, 256, 128), (300, 520, 512), (2048, 4096, 4096)])
def test_w8a16_fused_equals_materialised(dtype, sym, gran, g, M, N, K, native):
    """llmc_gemm_w8a16 (INT8 weights, W8A16 — rtn_w8a16.yml / per-channel W8): bit for bit the
    wgmma GEMM on the materialised fake-quant weight."""
    from llmc_b200.module_utils import linear_forward, linear_forward_w4, pack_unsigned_codes
    from llmc_b200.quant import IntegerQuantizer
    torch.manual_seed(M + N + K + int(sym))
    w = (torch.randn(N, K, device='cuda') * 0.02).to(dtype)
    x = torch.randn(M, K, device='cuda').to(dtype)
    kw = {'group_size': g} if g else {}
    q = IntegerQuantizer(8, sym, gran, **kw)
    codes, scales, zeros = q.real_quant_weight_dynamic(w)
    wqdq = q.fake_quant_weight_dynamic(w)
    qdt = dtype if native else torch.float32
    packed = pack_unsigned_codes(codes, 8, signed=sym)
    z = None if sym else zeros.to(qdt)
    y = linear_forward_w4(x, packed, scales.to(qdt), z, g or K, bits=8)
    assert torch.equal(y, linear_forward(x, wqdq))


@pytest.mark.parametrize('bit,sym,gran', [(4, True, 'per_group'), (4, False, 'per_group'),
                                          (8, True, 'per_channel')])
def test_efficient_fake_quant_linear_uses_the_packed_path(bit, sym, gran):
    """The product forward (deploy('fake_quant') -> EffcientFakeQuantLinear) keeps packed codes and
    runs the fused dequant-GEMM; output and `.weight` equal the materialised wrapper's bit for bit."""
    import os
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.module_utils import EffcientFakeQuantLinear
    from llmc_b200.rtn import RTN
    from llmc_b200.synth import SynthModel
    wcfg = {'bit': bit, 'symmetric': sym, 'granularity': gran}
    if gran == 'per_group':
        wcfg['group_size'] = 128
    outs = {}
    for fused in ('1', '0'):
        os.environ['LLMC_B200_FUSED_DEQUANT'] = fused
        try:
            model = SynthModel('tiny-llama', n_layers=1, device='cuda')
            cfg = AttrDict.wrap({'quant': {'method': 'RTN', 'weight': wcfg}})
            algo = RTN(model, cfg.quant, None, None, cfg)
            algo.run_block_loop()
            algo.deploy('fake_quant')
        finally:
            os.environ.pop('LLMC_B200_FUSED_DEQUANT', None)
        m = model.get_blocks()[0].mlp.down_proj
        assert isinstance(m, EffcientFakeQuantLinear) and m.packed == (fused == '1')
        x = torch.randn(3, 64, m.in_features, generator=torch.Generator().manual_seed(1)).bfloat16().cuda()
        outs[fused] = (m(x), m.weight.clone())
        if fused == '1':
            assert m.qweight.dtype == torch.int32 and m.qweight.shape == (m.out_features, m.in_features * bit // 32)
    assert torch.equal(outs['1'][0], outs['0'][0])
    assert torch.equal(outs['1'][1], outs['0'][1])


@pytest.mark.parametrize('bits', [4, 8])
def test_transposed_qparam_layout_is_identical(bits):
    """qparams handed over as [K/group, N] (coalesced loads) give the same bits as [N, K/group]."""
    from llmc_b200.module_utils import linear_forward_w4, pack_unsigned_codes
    from llmc_b200.quant import IntegerQuantizer
    torch.manual_seed(bits)
    N, K, M, g = 1024, 2048, 512, 128
    w = (torch.randn(N, K, device='cuda') * 0.02).bfloat16()
    x = torch.randn(M, K, device='cuda').bfloat16()
    q = IntegerQuantizer(bits, False, 'per_group', group_size=g)
    codes, s, z = q.real_quant_weight_dynamic(w)
    packed = pack_unsigned_codes(codes, bits, signed=False)
    for qdt in (torch.bfloat16, torch.float32):
        a = linear_forward_w4(x, packed, s.to(qdt), z.to(qdt), g, bits=bits)
        b = linear_forward_w4(x, packed, s.to(qdt).t().contiguous(), z.to(qdt).t().contiguous(), g, bits=bits,
                              qparams_t=True)
        assert torch.equal(a, b)
