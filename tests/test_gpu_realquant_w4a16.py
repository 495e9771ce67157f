"""GPU: the weight-only packed exports run.

  - llmc_gemm_w4a16_awq equals llmc_gemm_bf16 on the oracle-dequantised AutoAWQ weight bit for bit
    (tests/w4a16_export_oracle.py): random int32 words for qweight and qzeros, so every nibble
    pattern, including the carries of unclamped codes; bf16 and fp16, bias on and off, group 64 and
    128, M and N off the 128 tile, K = 64 * odd, and the Llama-3-8B linear shapes.
  - VllmRealQuantLinear's packed forward (llmc_gemm_w4a16 / w8a16 with the fp16 export scales) equals
    llmc_gemm_bf16 on the oracle-dequantised export bit for bit.
  - End to end, the shipped W4A16 / W8A16 backend recipes are calibrated on the tiny models and
    deployed once as fake-quant and once as the backend's real-quant modules: every linear runs on
    the packed GEMM; the logits equal, bit for bit, those of the model with each real-quant linear
    replaced by a dense B200Linear holding the oracle-dequantised export; they stay within a relative
    L2 of the fake-quant logits: 5e-2 for vLLM / SGLang, whose export differs from the fake-quant
    weight only by the scales' rounding to fp16 (measured: 0, the bf16 scales are fp16 values); 0.75
    for AutoAWQ / MLC-LLM, whose packer does not clamp: a group's extreme weight whose code
    round((w + z s) / s) comes out as 16 (or -1) stores as 0 and carries into the next column's nibble
    (or sets every higher nibble of the word), so the export moves such weights by up to the group's
    whole range (measured on an H100 80GB HBM3: 0.21 RTN, 0.25 AWQ, 0.48 GPTQ on tiny-llama, 0.07 RTN
    on tiny-opt); perplexity is finite; the saved safetensors are byte-identical before and after the
    forward."""
import json
import os

import pytest
import torch

import w4a16_export_oracle as eo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGIT_REL_L2 = {'vllm': 5e-2, 'awq': 0.75}


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _awq_case(M, N, K, group, dtype, bias, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = (torch.randn(M, K, device='cuda', generator=g) * 0.5).to(dtype)
    qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (K, N // 8), dtype=torch.int32, device='cuda', generator=g)
    qz = torch.randint(-2 ** 31, 2 ** 31 - 1, (K // group, N // 8), dtype=torch.int32, device='cuda', generator=g)
    # scales over 2^-14 .. 2^-2 with full fp16 mantissas
    s = (torch.rand(K // group, N, device='cuda', generator=g) * 2 ** -2 + 2 ** -14).half()
    b = (torch.randn(N, device='cuda', generator=g)).to(dtype) if bias else None
    return x, qw, s, qz, b


def _check_awq(M, N, K, group, dtype, bias, seed=0):
    from llmc_b200.module_utils import linear_forward, linear_forward_w4a16_awq
    x, qw, s, qz, b = _awq_case(M, N, K, group, dtype, bias, seed)
    y = linear_forward_w4a16_awq(x, qw, s, qz, group, b)
    w = eo.awq_dequant(qw, s, qz, group, dtype)
    ref = linear_forward(x, w, b)
    torch.cuda.synchronize()
    assert _bits_equal(y, ref), (M, N, K, group, int((y != ref).sum()))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('bias', [False, True])
@pytest.mark.parametrize('group', [64, 128])
@pytest.mark.parametrize('M,N,Kmul', [(1, 160, 3), (127, 160, 5), (129, 256, 1), (300, 416, 7), (64, 128, 9)])
def test_awq_gemm_bit_exact(dtype, bias, group, M, N, Kmul):
    _check_awq(M, N, group * Kmul, group, dtype, bias, seed=M + N + Kmul)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('N,K', [(4096, 4096), (1024, 4096), (14336, 4096), (4096, 14336)])
def test_awq_gemm_llama3_8b_shapes(dtype, N, K):
    _check_awq(2048, N, K, 128, dtype, False, seed=N + K)


@pytest.mark.parametrize('act', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('bits,group', [(4, 128), (8, 128), (8, None)])
@pytest.mark.parametrize('bias', [False, True])
def test_vllm_packed_forward_bit_exact(act, bits, group, bias):
    from llmc_b200.module_utils import VllmRealQuantLinear, linear_forward
    M, N, K = 200, 416, 640
    group = group or K
    g = torch.Generator(device='cuda').manual_seed(bits * 1000 + group)
    words = torch.randint(-2 ** 31, 2 ** 31 - 1, (N, K * bits // 32), dtype=torch.int32, device='cuda', generator=g)
    s = (torch.rand(N, K // group, device='cuda', generator=g) * 2 ** -2 + 2 ** -14).half()
    b = torch.randn(N, device='cuda', generator=g).to(act) if bias else None
    m = VllmRealQuantLinear(words, b, s, None, True, 'weight_scale')
    m.in_features, m.out_features = K, N
    assert m.packed_unsupported() is None
    x = torch.randn(3, M // 3 + 1, K, device='cuda', generator=g).to(act)
    y = m(x)
    ref = linear_forward(x, eo.vllm_dequant(words, s, bits, K, act), b)
    torch.cuda.synchronize()
    assert _bits_equal(y, ref), int((y != ref).sum())


def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


FORMATS = {'vllm': 'vllm_quant', 'sglang': 'sgl_quant', 'autoawq': 'autoawq_quant', 'mlcllm': 'mlcllm_quant'}
RECIPES = {f'{be}/{algo}_w4a16': (f'backend/{be}/{algo}_w4a16.yml', 'tiny-llama', fmt)
           for be, fmt in FORMATS.items() for algo in ('rtn', 'awq', 'gptq')}
RECIPES.update({f'{be}/rtn_w8a16': (f'backend/{be}/rtn_w8a16.yml', 'tiny-llama', FORMATS[be])
                for be in ('vllm', 'sglang')})
RECIPES.update({f'opt/{be}/rtn_w{b}a16': (f'backend/{be}/rtn_w{b}a16.yml', 'tiny-opt', FORMATS[be])
                for be, b in (('vllm', 4), ('vllm', 8), ('autoawq', 4))})


def _export_weight(m, dtype):
    from llmc_b200.module_utils import AutoawqRealQuantLinear
    if isinstance(m, AutoawqRealQuantLinear):
        return eo.awq_dequant(m.qweight, m.scales, m.qzeros, m.in_features // m.scales.shape[0], dtype)
    bits = 32 * m.weight_packed.shape[1] // m.in_features
    return eo.vllm_dequant(m.weight_packed, m.weight_scale, bits, m.in_features, dtype)


@pytest.mark.parametrize('name', list(RECIPES))
def test_realquant_w4a16_forward(name, tmp_path):
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.export import save_model
    from llmc_b200.module_utils import AutoawqRealQuantLinear, VllmRealQuantLinear
    from llmc_b200.prof import TIMER
    from llmc_b200.synth import B200Linear, SynthModel, perplexity
    rel, shape, fmt = RECIPES[name]
    doc = _yaml(rel)
    doc.pop('save', None)
    cfg = adapt_reference_config(doc, shape, n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['eval']['eval_pos'] = []
    algo, model, _ = main(cfg, quiet=True)
    blocks = model.get_blocks()
    calibrated = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    ids = torch.randint(0, model.shape['vocab'], (2, 128), generator=torch.Generator().manual_seed(4))
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(5))

    algo.deploy('fake_quant')
    logits_f = model.logits(ids).float()

    for (i, n), m in calibrated.items():
        SynthModel._set(blocks[i], n, m)
    algo.deploy(fmt)
    real = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    awq = fmt in ('autoawq_quant', 'mlcllm_quant')
    assert all(isinstance(m, AutoawqRealQuantLinear if awq else VllmRealQuantLinear) for m in real.values())
    if not awq:
        assert all(m.packed_unsupported() is None for m in real.values()), \
            {k: m.packed_unsupported() for k, m in real.items()}
    before = os.path.join(str(tmp_path), 'before')
    save_model(model, before)
    n_buffers = {k: len(list(m.buffers())) for k, m in real.items()}

    TIMER.reset()
    TIMER.enabled = True
    try:
        logits_r = model.logits(ids).float()
        torch.cuda.synchronize()
        spans = TIMER.summary()
    finally:
        TIMER.enabled = False
        TIMER.reset()
    want = {'gemm_w4a16_awq'} if awq else {f'gemm_w{b}a16' for b in (4, 8) if f'w{b}a16' in rel}
    assert want <= set(spans), spans
    assert sum(spans[s]['calls'] for s in want) == len(real) * 1, (spans, len(real))
    assert not {s for s in spans if s.startswith('gemm_w')} - want, spans

    # the same model with each real-quant linear replaced by its dequantised export
    dtype = model.shape['dtype']
    for (i, n), m in real.items():
        d = B200Linear(m.in_features, m.out_features, bias=m.bias is not None).to('cuda', dtype)
        d.weight.data = _export_weight(m, dtype)
        if m.bias is not None:
            d.bias.data = m.bias.to(dtype)
        SynthModel._set(blocks[i], n, d)
    logits_d = model.logits(ids).float()
    for (i, n), m in real.items():
        SynthModel._set(blocks[i], n, m)
    assert torch.equal(logits_r, logits_d), float((logits_r - logits_d).abs().max())

    rel_l2 = ((logits_r - logits_f).norm() / logits_f.norm()).item()
    print(f'\n{name}: logits relative L2 (real-quant vs fake-quant) = {rel_l2:.3e}')
    assert logits_r.isfinite().all() and rel_l2 <= LOGIT_REL_L2['awq' if awq else 'vllm'], rel_l2
    ppl = perplexity(model, tokens, 128, ce_dtype=torch.float32)
    assert ppl == ppl and ppl < float('inf'), ppl

    after = os.path.join(str(tmp_path), 'after')
    save_model(model, after)
    with open(os.path.join(before, 'model.safetensors'), 'rb') as fa, \
            open(os.path.join(after, 'model.safetensors'), 'rb') as fb:
        assert fa.read() == fb.read()
    assert {k: len(list(m.buffers())) for k, m in real.items()} == n_buffers
