"""Generate tests/golden/gptq_fp8_kat.pt by RUNNING THE REFERENCE'S OWN GPTQ on FP8 weight grids, on CPU.

Build container only (needs /root/reference):

    python oracle/gen_gptq_fp8_golden.py

The reference's FloatQuantizer with `use_qtorch: True` rounds with `qtorch.quant.float_quantize`,
which is absent here (SURVEY.md §8c).  A stub module `qtorch.quant` is installed whose
`float_quantize(x, exp, man, rounding='nearest')` is fp8_oracle.float_quantize (clamp to
+-finfo.max, then IEEE round-to-nearest-even): that one step is the project's restatement, and
everything around it — scale search, the in-place zero-scale fix, the column loop, Losses, the
trailing updates, update_model_qparams, w_qdq — is the reference's own code (oracle/ref_harness.py
runs a CPU copy of it).  Every sweep runs on one thread, so the trailing GEMMs have one summation
order (tests/test_gptq_fp8_golden.py runs the oracle the same way).
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import fp8_oracle as fo  # noqa: E402
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(HERE, '..', 'tests', 'golden', 'gptq_fp8_kat.pt')
_BITS = {(4, 3): 'e4m3', (5, 2): 'e5m2'}


def install_qtorch_stub():
    def float_quantize(x, exp, man, rounding='nearest'):
        assert rounding == 'nearest' and x.dtype == torch.float32
        return fo.float_quantize(x, _BITS[(exp, man)])
    pkg = types.ModuleType('qtorch')
    quant = types.ModuleType('qtorch.quant')
    quant.float_quantize = float_quantize
    pkg.quant = quant
    sys.modules['qtorch'] = pkg
    sys.modules['qtorch.quant'] = quant


# name, R, C, tokens per batch, batches, dtype, weight kwargs, special, saturating.  Kept small (the
# [C, C] factor dominates the file): three two-block layers (128 + 64 columns), four one-block layers
SPECS = [
    ('e4m3_channel_actorder_fp16', 16, 128, 64, 2, torch.float16,
     dict(bit='e4m3', granularity='per_channel'), dict(actorder=True, static_groups=False), False),
    ('e4m3_channel_actorder_bf16_saturating', 16, 192, 64, 2, torch.bfloat16,
     dict(bit='e4m3', granularity='per_channel'), dict(actorder=True, static_groups=False), True),
    ('e5m2_channel_noorder_bf16_saturating', 16, 128, 64, 2, torch.bfloat16,
     dict(bit='e5m2', granularity='per_channel'), dict(actorder=False, static_groups=False), True),
    ('e4m3_g64_actorder_dynamic_bf16', 16, 192, 96, 2, torch.bfloat16,
     dict(bit='e4m3', granularity='per_group', group_size=64), dict(actorder=True, static_groups=False), False),
    ('e5m2_g128_actorder_dynamic_fp16', 16, 128, 96, 2, torch.float16,
     dict(bit='e5m2', granularity='per_group', group_size=128), dict(actorder=True, static_groups=False), False),
    ('e4m3_g64_actorder_static_fp16', 16, 192, 80, 2, torch.float16,
     dict(bit='e4m3', granularity='per_group', group_size=64), dict(actorder=True, static_groups=True), False),
    ('e4m3_tensor_noorder_fp16', 16, 128, 80, 2, torch.float16,
     dict(bit='e4m3', granularity='per_tensor'), dict(actorder=False, static_groups=False), False),
]


def pack_upper(U):
    """The upper factor's upper triangle, row by row (its lower triangle is exactly zero;
    gptq_fp8_oracle.unpack_upper restores it)."""
    C = U.shape[0]
    assert torch.equal(U, torch.triu(U))
    i, j = torch.triu_indices(C, C)
    return U[i, j].clone()


def make_layer(R, C, T, nb, dtype, seed, saturating):
    gen = torch.Generator().manual_seed(seed)
    if saturating:
        # every weight of a row near the row's absmax, inputs that share one strong direction: the
        # compensation of one column lands on the next ones with the same sign and pushes them past
        # absmax, i.e. past finfo.max * scale
        W = torch.sign(torch.randn(R, C, generator=gen)) * (0.9 + 0.1 * torch.rand(R, C, generator=gen)) * 0.02
        common = torch.randn(1, T, 1, generator=gen)
        batches = [((common + 0.05 * torch.randn(1, T, C, generator=gen)) * torch.sign(W[0])).to(dtype)
                   for _ in range(nb)]
    else:
        W = torch.randn(R, C, generator=gen) * 0.02
        chan = torch.exp(torch.randn(C, generator=gen))
        batches = [(torch.randn(1, T, C, generator=gen) * chan).to(dtype) for _ in range(nb)]
    W[1] = 0                       # an all-zero row: its 16-bit per-channel scale underflows to 0
    return W.to(dtype), batches


def run(rg, rq, name, R, C, T, nb, dtype, wkw, sp, saturating, seed):
    W0, batches = make_layer(R, C, T, nb, dtype, seed, saturating)
    layer = torch.nn.Linear(C, R, bias=False)
    layer.weight.data = W0.clone()
    g = rg.GPTQ.__new__(rg.GPTQ)
    g.dev = torch.device('cpu')
    g.model_dtype = dtype
    g.wquantizer = rq.FloatQuantizer(symmetric=True, use_qtorch=True, **wkw)
    g.actorder, g.static_groups = sp['actorder'], sp['static_groups']
    g.owq, g.percdamp, g.blocksize, g.chunk_num = False, 0.01, 128, 1
    g.need_perm = (wkw['granularity'] == 'per_group' and not g.static_groups and g.actorder)
    # collect_block_qparams (base_blockwise_quantization.py:337-365)
    _, s, z, qmax, qmin = g.wquantizer.get_tensor_qparams(layer.weight.data)
    layer.register_buffer('buf_scales', s.detach())
    layer.register_buffer('buf_zeros', z.detach())
    layer.register_buffer('buf_qmax', qmax.clone())
    layer.register_buffer('buf_qmin', qmin.clone())
    rtn_scales = s.clone()
    g.layers_cache = {'l': {}}
    g.named_layers = {'l': layer}
    g.layer_init(layer, 'l')
    for b in batches:
        g.add_batch(layer, 'l', b, None)
    g.initialize_qparams_and_prepare_weights(layer, 'l')
    Wp, Hinv = g.process_hessian_and_weights(layer, 'l')
    Wp_in = Wp.clone()
    Losses, tmp = torch.zeros_like(Wp), torch.zeros_like(Wp)
    g.n_nonout = g.columns
    g.weight_transform(Wp, Hinv, Losses, tmp)
    tmp_perm = tmp.clone()
    perm = g.perm if g.actorder else None
    if g.actorder:
        tmp = tmp[:, g.invperm]
    layer.weight.data = tmp.reshape(layer.weight.shape)
    if wkw['granularity'] == 'per_group' and not g.static_groups:
        g.update_model_qparams(layer)
    qdq = g.w_qdq(layer, g.wquantizer)
    # saturation: compensated weights beyond finfo.max * scale of their row (per-channel cases)
    sat = 0
    if wkw['granularity'] == 'per_channel':
        fmax = torch.finfo(fo.FP8[wkw['bit']]).max
        s_rows = layer.buf_scales.float().reshape(-1, 1)
        sat = int((tmp_perm.abs() > fmax * s_rows).sum())
    assert sat > 0 or not saturating, name
    print(f' {name}: loss {Losses.sum().item():.6g}, saturated {sat}')
    return dict(name=name, weight_kwargs=wkw, special=sp, dtype=dtype, perm=perm, Wp=Wp_in,
                Hinv_upper=pack_upper(Hinv), rtn_scales=rtn_scales, tmp_perm=tmp_perm, Losses=Losses,
                losses_sum=Losses.sum().item(), buf_scales=layer.buf_scales.clone(), qdq=qdq, saturated=sat)


def main():
    install_qtorch_stub()
    ref_harness.setup()
    torch.set_num_threads(1)
    from llmc.compression.quantization import gptq as rg
    from llmc.compression.quantization import quant as rq
    assert rq.float_quantize is not None
    out = [run(rg, rq, *spec, seed=3000 + k) for k, spec in enumerate(SPECS)]
    torch.save(out, OUT)
    print('wrote', os.path.normpath(OUT), len(out), 'layers')


if __name__ == '__main__':
    main()
