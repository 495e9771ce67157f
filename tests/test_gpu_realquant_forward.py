"""GPU: the exported W8A8 linears run.  Shipped INT8 and FP8 recipes are calibrated on the tiny models,
deployed once as fake-quant and once as the backend's real-quant modules (VllmRealQuantLinear /
SglRealQuantLinear), and compared:
  - every real-quant linear runs on llmc_gemm_w8a8_* (no NotImplementedError);
  - on the input each real-quant linear sees, its activation codes and scales give exactly the fake-quant
    module's QDQ activation, rT(code * scale), and its scales are the quantizer's own;
  - the logits stay within a relative L2 distance of the fake-quant logits: 5e-2 for INT8, 8e-2 for FP8
    (the forwards differ by the fake-quant weight's and activation's rounding to the model dtype and
    the GEMM's arithmetic; a code that then lands on the other side of a rounding boundary moves by a
    step of the grid, 1/127 of the row's range for INT8, up to 1/8 of the value for e4m3);
  - perplexity is finite;
  - the saved safetensors are byte-identical before and after the forward runs, and hold only the
    export's tensors (the recorded activation config is not a buffer; a tensor shared by several
    linears, like the input_scale of q/k/v, is saved once, under the first)."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGIT_REL_L2 = {'int': 5e-2, 'fp8': 8e-2}


def _yaml(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]


def _mixtral_static():
    import yaml
    with open(os.path.join(ROOT, 'configs', 'rtn_fp8_static_mixtral.yml')) as fh:
        return yaml.safe_load(fh)


def _int8_static():
    doc = _yaml('backend/vllm/rtn_w8a8.yml')
    doc['quant']['act'] = dict(doc['quant']['act'], granularity='per_tensor', static=True,
                               calib_algo='static_minmax')
    doc['calib'] = {'name': 'synthetic', 'n_samples': 8, 'bs': 1, 'seq_len': 128, 'seed': 0}
    return doc


RECIPES = {
    'vllm/rtn_w8a8': (lambda: _yaml('backend/vllm/rtn_w8a8.yml'), 'tiny-llama', 'vllm_quant'),
    'sglang/rtn_w8a8': (lambda: _yaml('backend/sglang/rtn_w8a8.yml'), 'tiny-llama', 'sgl_quant'),
    'vllm/smoothquant_w8a8': (lambda: _yaml('backend/vllm/smoothquant_w8a8.yml'), 'tiny-llama', 'vllm_quant'),
    'sglang/smoothquant_w8a8': (lambda: _yaml('backend/sglang/smoothquant_w8a8.yml'), 'tiny-llama', 'sgl_quant'),
    'vllm/rtn_fp8': (lambda: _yaml('backend/vllm/fp8/rtn_fp8.yml'), 'tiny-llama', 'vllm_quant'),
    'sglang/rtn_fp8': (lambda: _yaml('backend/sglang/fp8/rtn_fp8.yml'), 'tiny-llama', 'sgl_quant'),
    'vllm/smoothquant_fp8': (lambda: _yaml('backend/vllm/fp8/smoothquant_fp8.yml'), 'tiny-llama', 'vllm_quant'),
    'vllm/gptq_fp8': (lambda: _yaml('backend/vllm/fp8/gptq_fp8.yml'), 'tiny-llama', 'vllm_quant'),
    'sglang/gptq_fp8': (lambda: _yaml('backend/sglang/fp8/gptq_fp8.yml'), 'tiny-llama', 'sgl_quant'),
    'rtn_fp8_static_mixtral': (_mixtral_static, 'tiny-mixtral', 'vllm_quant'),
    'rtn_w8a8_static': (_int8_static, 'tiny-llama', 'vllm_quant'),
}


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize('name', list(RECIPES))
def test_realquant_forward(name, tmp_path):
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.export import save_model
    from llmc_b200.module_utils import VllmRealQuantLinear
    from llmc_b200.quant import IntegerQuantizer
    from llmc_b200.synth import SynthModel, perplexity
    make, shape, fmt = RECIPES[name]
    doc = make()
    doc.pop('save', None)
    cfg = adapt_reference_config(doc, shape, n_samples=8, seq_len=128, eval_seq_len=128)
    cfg['eval']['eval_pos'] = []
    algo, model, _ = main(cfg, quiet=True)
    blocks = model.get_blocks()
    calibrated = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    ids = torch.randint(0, model.shape['vocab'], (2, 128), generator=torch.Generator().manual_seed(4))
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(5))

    algo.deploy('fake_quant')
    fake = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    logits_f = model.logits(ids).float()

    for (i, n), m in calibrated.items():
        SynthModel._set(blocks[i], n, m)
    algo.deploy(fmt)
    real = {(i, n): m for i, b in enumerate(blocks) for n, m in model.get_block_linears(b).items()}
    assert all(isinstance(m, VllmRealQuantLinear) for m in real.values())
    assert all(m.w8a8_unsupported() is None for m in real.values()), \
        {k: m.w8a8_unsupported() for k, m in real.items()}
    before = os.path.join(str(tmp_path), 'before')
    save_model(model, before)

    seen = {}
    hooks = [m.register_forward_pre_hook(lambda mod, a, k=k: seen.__setitem__(k, a[0].detach().clone()))
             for k, m in real.items()]
    logits_r = model.logits(ids).float()
    for h in hooks:
        h.remove()
    ran = set(seen)
    experts = {k for k in real if '.experts.' in k[1]}
    assert set(real) - experts <= ran, set(real) - experts - ran
    assert not experts or experts & ran

    # activation codes and scales: the fake-quant module's QDQ activation, on the same input
    for k in sorted(ran):
        x, r, f = seen[k], real[k], fake[k]
        if x.numel() == 0:
            continue
        static = bool(r.act_cfg.get('static', False))
        aq = r.activation_quantizer()
        x2 = x.reshape(-1, x.shape[-1])
        qx, sx = aq.real_quant_act(x2, r.input_scale if static else None)
        # GPTQ's FP8 export holds its e4m3 codes in the model dtype
        assert qx.dtype == (torch.int8 if r.weight.dtype == torch.int8 else torch.float8_e4m3fn), k
        deq = (qx.float() * sx.reshape(-1, 1)).to(x.dtype)
        fq = f.a_qdq(x, f).reshape(-1, x.shape[-1])
        assert _bits_equal(deq, fq), (k, int((deq != fq).sum()))
        if static:
            assert torch.equal(sx, r.input_scale.reshape(1).float()), k
        elif isinstance(aq, IntegerQuantizer):
            from llmc_b200._lib import OUT_NONE
            s, _ = aq._dynamic(x2, OUT_NONE)
            assert torch.equal(sx, s.reshape(-1).float()), k
        else:
            _, s = aq._dynamic(x2, 0)
            s = s.reshape(-1).float()
            assert torch.equal(sx, s.masked_fill(s == 0, 1.0)), k

    rel = ((logits_r - logits_f).norm() / logits_f.norm()).item()
    print(f'\n{name}: logits relative L2 (real-quant vs fake-quant) = {rel:.3e}')
    kind = 'int' if next(iter(real.values())).weight.dtype == torch.int8 else 'fp8'
    assert logits_r.isfinite().all() and rel <= LOGIT_REL_L2[kind], rel
    ppl = perplexity(model, tokens, 128, ce_dtype=torch.float32)
    assert ppl == ppl and ppl < float('inf'), ppl

    after = os.path.join(str(tmp_path), 'after')
    save_model(model, after)
    with open(os.path.join(before, 'model.safetensors'), 'rb') as fa, \
            open(os.path.join(after, 'model.safetensors'), 'rb') as fb:
        assert fa.read() == fb.read()
    from safetensors.torch import load_file
    saved = load_file(os.path.join(after, 'model.safetensors'))
    for (i, n), m in real.items():
        prefix = f'layers.{i}.{n}.'
        leaves = {key[len(prefix):] for key in saved if key.startswith(prefix)}
        want = {'weight', 'weight_scale'} | ({'input_scale'} if m.input_scale is not None else set()) \
            | ({'bias'} if m.bias is not None else set())
        assert {'weight', 'weight_scale'} <= leaves <= want, (n, leaves)
