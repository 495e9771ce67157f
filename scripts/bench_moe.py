"""The Mixtral-8x7B sparse-MoE layer on the grouped expert GEMMs (module_utils.moe_forward) next to the
per-expert loop (MixtralSparseMoe.expert_loop) it replaces.

    python scripts/bench_moe.py [--reps 10] [--tokens 2048 65536] [--awq-samples 128] [--awq-rounds 3]
                                [--packed] [--ppl-rounds 3] [--w8a8] [--fake-quant] [--out DIR]

1. One MoE layer (hidden 4096, inter 14336, 8 experts, top-2, bf16) at 2048 tokens (one GPTQ
   calibration forward at batch size 1) and 65536 tokens (the AWQ inspect batch, 128 x 512): the
   module forward, router included, both ways.  Both paths are checked to give the same bits first;
   after warm-up the two alternate for `reps` rounds between CUDA events, and the medians are
   reported with the achieved TFLOP/s of the expert GEMMs (2 * tokens * top_k * 3 * hidden * inter).
2. One AWQ run_block_loop (w4 g128, scale search + auto-clip) on a one-block Mixtral-8x7B-shaped
   model with awq_samples x 512 calibration tokens, end to end on a host clock that ends in a device
   synchronise: awq_rounds rounds of grouped path then loop, each run on a fresh model (the first
   runs include the caching allocator's first allocations at this shape); every round's two runs
   must leave the same weights.  All times are reported, the speed-up is of the medians.
With --packed, instead of 1. and 2.: the same layer with PACKED experts on the grouped dequant GEMMs
(module_utils.PackedOperands, csrc/gemm_w4.cu) against the loop over their packed forwards, for W4
g128 with bf16 qparams, W4 g128 act-order (fp32 qparams, a g_idx per linear) and W8 per-channel
(random codes and qparams: the kernels' work does not depend on the values), at each of `tokens`,
timed as in 1.; then the fake-quant perplexity of a one-block Mixtral-8x7B-shaped model after an RTN
W4 g128 deploy (8 x 2048 tokens), grouped then loop for ppl_rounds alternated rounds on a host
clock that ends in a device synchronise, with equal perplexities checked.
With --w8a8, instead: the same layer with W8A8 experts (exported VllmRealQuantLinear int8 / e4m3
linears) on the grouped W8A8 GEMMs (module_utils.W8A8Operands, csrc/gemm_8bit.cu) against the loop
over their real-quant forwards, for e4m3 per-tensor weights with static per-tensor activations
(configs/rtn_fp8_static_mixtral.yml), e4m3 per-channel with per-token dynamic activations and int8
per-channel with per-token dynamic activations (random codes and scales), at each of `tokens`, timed
as in 1.
With --fake-quant, instead: the same layer with fake-quant experts under activation fake-quant
(module_utils.fake_quant_forward_operands, the routed twin of blockwise's a_qdq) against the loop over
their fake-quant forwards, for e4m3 per-tensor weights with static e4m3 activations
(configs/rtn_fp8_static_mixtral.yml), e4m3 per-channel weights with per-token e4m3 activations and
int8 per-channel weights with per-token int8 activations, weights quantised from random ones, static
scales random per expert; at each of `tokens`, timed as in 1.  Then the fake-quant perplexity of a
one-block Mixtral-8x7B-shaped model under configs/rtn_fp8_static_mixtral.yml (RTN with static
calibration on 16 x 512 tokens, then 8 x 2048 eval tokens), grouped then loop for ppl_rounds
alternated rounds as with --packed, with equal perplexities checked.
Prints, and writes to DIR/bench_moe.json, one JSON object with the card name and power limit.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from llmc_b200 import synth  # noqa: E402
from llmc_b200.synth import MixtralSparseMoe  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def loop_forward(moe, hs):
    """MixtralSparseMoe.forward with the expert loop forced."""
    B, S, H = hs.shape
    x = hs.reshape(-1, H)
    sel, w = moe.route(x)
    return moe.expert_loop(x, sel, w).reshape(B, S, H)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def compare_and_time(res, key, moe, hs, flops, reps):
    """The module forward (grouped) and loop_forward on hs: the same bits first, then after warm-up
    `reps` alternated rounds between CUDA events; records the medians, the TFLOP/s of `flops` and the
    speed-up under `key`."""
    grouped, loop = moe(hs), loop_forward(moe, hs)
    assert torch.equal(grouped.view(torch.int16), loop.view(torch.int16)), key
    del grouped, loop
    runs = {'grouped': lambda: moe(hs), 'loop': lambda: loop_forward(moe, hs)}
    for fn in runs.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n in runs}
    for _ in range(reps):
        for n, fn in runs.items():
            times[n].append(timed(fn))
    med = {n: round(statistics.median(v), 3) for n, v in times.items()}
    res['layer_ms'][key] = med
    res['layer_tflops'][key] = {n: round(flops / (v * 1e-3) / 1e12, 1) for n, v in med.items()}
    res['layer_speedup'][key] = round(med['loop'] / med['grouped'], 3)
    print(key, med, res['layer_tflops'][key], flush=True)


def bench_layer(res, tokens, reps):
    s = synth.SHAPES['mixtral-8x7b']
    H, I, E, k = s['hidden'], s['inter'], s['experts'], s['top_k']
    g = torch.Generator(device='cuda').manual_seed(0)
    with torch.device('meta'):
        moe = MixtralSparseMoe(H, I, E, k)
    moe = moe.to(torch.bfloat16).to_empty(device='cuda')
    for p in moe.parameters():
        p.data.normal_(0, 0.02, generator=g)
    for T in tokens:
        hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
        assert moe.grouped_weights(hs.view(T, H)) is not None
        compare_and_time(res, f'moe_layer[T={T}]', moe, hs, 2.0 * T * k * 3 * H * I, reps)
        del hs
        torch.cuda.empty_cache()
    del moe
    torch.cuda.empty_cache()


def packed_moe(form, g):
    """The Mixtral-8x7B MoE layer (bf16) with every expert linear packed in `form`, random values."""
    from llmc_b200.module_utils import EffcientFakeQuantLinear, pack_unsigned_codes
    s = synth.SHAPES['mixtral-8x7b']
    with torch.device('meta'):
        moe = MixtralSparseMoe(s['hidden'], s['inter'], s['experts'], s['top_k'])
    moe.gate = moe.gate.to_empty(device='cuda').to(torch.bfloat16)
    moe.gate.weight.data.normal_(0, 0.02, generator=g)
    for ex in moe.experts:
        for n in ('w1', 'w3', 'w2'):
            lin = getattr(ex, n)
            N, K = lin.out_features, lin.in_features
            bits, group = (8, K) if form == 'w8_channel' else (4, 128)
            qdt = torch.float32 if form == 'w4_g128_gidx_f32' else torch.bfloat16
            codes = torch.randint(0, 2**bits, (N, K), generator=g, device='cuda', dtype=torch.int32)
            packed = dict(qweight=pack_unsigned_codes(codes, bits, signed=False),
                          scales=(torch.rand(N, K // group, generator=g, device='cuda') * 0.01).to(qdt),
                          zeros=torch.randint(0, 2**bits, (N, K // group), generator=g, device='cuda').to(qdt),
                          bits=bits, group=group, dtype=torch.bfloat16)
            if form == 'w4_g128_gidx_f32':
                packed['g_idx'] = (torch.randperm(K, generator=g, device='cuda') // group).to(torch.int32)
            del codes
            m = EffcientFakeQuantLinear(None, None, lin, None, packed=packed)
            m.in_features, m.out_features = K, N
            setattr(ex, n, m)
    return moe


def bench_packed_layer(res, tokens, reps):
    s = synth.SHAPES['mixtral-8x7b']
    H, I, k = s['hidden'], s['inter'], s['top_k']
    g = torch.Generator(device='cuda').manual_seed(0)
    for form in ('w4_g128_native', 'w4_g128_gidx_f32', 'w8_channel'):
        moe = packed_moe(form, g)
        for T in tokens:
            hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
            assert moe.grouped_packed_operands(hs.view(T, H)) is not None
            compare_and_time(res, f'moe_layer[{form}, T={T}]', moe, hs, 2.0 * T * k * 3 * H * I, reps)
            del hs
            torch.cuda.empty_cache()
        del moe
        torch.cuda.empty_cache()


# form: (codes, static input scales, per-channel weight scales)
W8A8_FORMS = {'e4m3_tensor_static': ('e4m3', True, False), 'e4m3_channel_dynamic': ('e4m3', False, True),
              'int8_channel_dynamic': ('int8', False, True)}


def w8a8_moe(form, g):
    """The Mixtral-8x7B MoE layer (bf16) with every expert linear a W8A8 export (VllmRealQuantLinear) of
    `form`, random codes and scales; static input scales differ per expert, w1's and w3's alike."""
    from llmc_b200.module_utils import VllmRealQuantLinear
    kind, static, per_channel = W8A8_FORMS[form]
    act = ({'bit': 8, 'symmetric': True} if kind == 'int8' else
           {'quant_type': 'float-quant', 'bit': 'e4m3', 'symmetric': True, 'use_qtorch': True})
    act.update({'granularity': 'per_tensor', 'static': True, 'calib_algo': 'static_minmax'} if static
               else {'granularity': 'per_token'})
    s = synth.SHAPES['mixtral-8x7b']
    with torch.device('meta'):
        moe = MixtralSparseMoe(s['hidden'], s['inter'], s['experts'], s['top_k'])
    moe.gate = moe.gate.to_empty(device='cuda').to(torch.bfloat16)
    moe.gate.weight.data.normal_(0, 0.02, generator=g)
    for ex in moe.experts:
        in_scale = torch.rand(1, generator=g, device='cuda') * 0.01 + 0.005
        for n in ('w1', 'w3', 'w2'):
            lin = getattr(ex, n)
            N, K = lin.out_features, lin.in_features
            if kind == 'int8':
                w = torch.randint(-127, 128, (N, K), generator=g, device='cuda', dtype=torch.int8)
                sw = torch.rand(N if per_channel else 1, 1, generator=g, device='cuda') * 2e-4 + 5e-5
            else:
                w = torch.randn(N, K, generator=g, device='cuda').to(torch.float8_e4m3fn)
                sw = torch.rand(N if per_channel else 1, 1, generator=g, device='cuda') * 0.01 + 0.002
            if n == 'w2':
                in_scale = torch.rand(1, generator=g, device='cuda') * 0.01 + 0.005
            m = VllmRealQuantLinear(w, None, sw, in_scale.clone() if static else None, False, 'weight_scale')
            m.in_features, m.out_features, m.act_cfg = K, N, dict(act)
            setattr(ex, n, m)
    return moe


def bench_w8a8_layer(res, tokens, reps):
    s = synth.SHAPES['mixtral-8x7b']
    H, I, k = s['hidden'], s['inter'], s['top_k']
    g = torch.Generator(device='cuda').manual_seed(0)
    for form in W8A8_FORMS:
        moe = w8a8_moe(form, g)
        for T in tokens:
            hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
            assert moe.grouped_w8a8_operands(hs.view(T, H)) is not None
            compare_and_time(res, f'moe_layer[{form}, T={T}]', moe, hs, 2.0 * T * k * 3 * H * I, reps)
            del hs
            torch.cuda.empty_cache()
        del moe
        torch.cuda.empty_cache()


# form: (weight quantizer, activation quantizer, static activations)
FAKE_QUANT_FORMS = {
    'e4m3_tensor_w_e4m3_static_a': ({'quant_type': 'float-quant', 'bit': 'e4m3', 'granularity': 'per_tensor'},
                                    {'quant_type': 'float-quant', 'bit': 'e4m3', 'granularity': 'per_tensor',
                                     'calib_algo': 'static_minmax'}, True),
    'e4m3_channel_w_e4m3_token_a': ({'quant_type': 'float-quant', 'bit': 'e4m3', 'granularity': 'per_channel'},
                                    {'quant_type': 'float-quant', 'bit': 'e4m3', 'granularity': 'per_token'}, False),
    'int8_channel_w_int8_token_a': ({'bit': 8, 'granularity': 'per_channel'},
                                    {'bit': 8, 'granularity': 'per_token'}, False),
}


def fake_quant_moe(form, g):
    """The Mixtral-8x7B MoE layer (bf16) with every expert linear replaced as a fake-quant deploy
    replaces it (EffcientFakeQuantLinear.new with blockwise's w_qdq / a_qdq), weights quantised from
    random ones; static activation scales random per expert, w1's and w3's one tensor."""
    from llmc_b200.blockwise import BaseBlockwiseQuantization
    from llmc_b200.module_utils import EffcientFakeQuantLinear, act_quantizer
    wcfg, acfg, static = FAKE_QUANT_FORMS[form]
    fp8 = {'symmetric': True, 'use_qtorch': True}
    wq = act_quantizer({**fp8, **wcfg} if 'quant_type' in wcfg else {'symmetric': True, **wcfg})
    aq = act_quantizer({**fp8, **acfg} if 'quant_type' in acfg else {'symmetric': True, **acfg})
    algo = object.__new__(BaseBlockwiseQuantization)
    algo.wquantizer, algo.aquantizer, algo.act_static = wq, aq, static
    params = algo.get_replacement_params('fake_quant')
    s = synth.SHAPES['mixtral-8x7b']
    with torch.device('meta'):
        moe = MixtralSparseMoe(s['hidden'], s['inter'], s['experts'], s['top_k'])
    moe = moe.to(torch.bfloat16).to_empty(device='cuda')
    for p in moe.parameters():
        p.data.normal_(0, 0.02, generator=g)
    for ex in moe.experts:
        s_in = torch.rand((), generator=g, device='cuda') * 0.02 + 0.01
        for n in ('w1', 'w3', 'w2'):
            m = EffcientFakeQuantLinear.new(getattr(ex, n), params['w_qdq'], params['a_qdq'])
            if static:
                sc = s_in if n != 'w2' else torch.rand((), generator=g, device='cuda') * 0.004 + 1e-3
                m.register_buffer('buf_act_scales_0', sc)
                m.register_buffer('buf_act_zeros_0', torch.tensor(0.0, device='cuda'))
                m.register_buffer('buf_act_qmin_0', aq.qmin.to('cuda'))
                m.register_buffer('buf_act_qmax_0', aq.qmax.to('cuda'))
            setattr(ex, n, m)
    return moe


def bench_fake_quant_layer(res, tokens, reps):
    s = synth.SHAPES['mixtral-8x7b']
    H, I, k = s['hidden'], s['inter'], s['top_k']
    g = torch.Generator(device='cuda').manual_seed(0)
    for form in FAKE_QUANT_FORMS:
        moe = fake_quant_moe(form, g)
        for T in tokens:
            hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
            assert moe.grouped_fake_quant_operands(hs.view(T, H)) is not None
            compare_and_time(res, f'moe_layer[{form}, T={T}]', moe, hs, 2.0 * T * k * 3 * H * I, reps)
            del hs
            torch.cuda.empty_cache()
        del moe
        torch.cuda.empty_cache()


def time_ppl(res, key, model, tokens, seq_len, rounds):
    """Perplexity of `model` on `tokens`, grouped then loop for `rounds` alternated rounds after one
    warm-up each, on a host clock that ends in a device synchronise; equal perplexities checked."""
    saved = MixtralSparseMoe.forward

    def run(loop):
        if loop:
            MixtralSparseMoe.forward = loop_forward
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ppl = synth.perplexity(model, tokens, seq_len, 1)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, ppl
        finally:
            MixtralSparseMoe.forward = saved
    run(False), run(True)                          # warm-up
    times, ppls = {'grouped': [], 'loop': []}, {'grouped': set(), 'loop': set()}
    for _ in range(rounds):
        for path in times:
            dt, ppl = run(path == 'loop')
            times[path].append(round(dt, 3))
            ppls[path].add(ppl)
    assert ppls['grouped'] == ppls['loop'] and len(ppls['loop']) == 1, ppls
    med = {n: statistics.median(v) for n, v in times.items()}
    res['ppl_s'][key] = times
    res['ppl_speedup'][key] = round(med['loop'] / med['grouped'], 3)
    print(key, times, flush=True)


def bench_fake_quant_ppl(res, rounds):
    import yaml
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.rtn import RTN
    with open(os.path.join(ROOT, 'configs', 'rtn_fp8_static_mixtral.yml')) as fh:
        cfg = AttrDict.wrap(yaml.safe_load(fh))
    model = synth.SynthModel('mixtral-8x7b', n_layers=1, seed=0, device='cuda', init='device')
    c = cfg.calib
    inp = model.first_block_input(c.n_samples, c.seq_len, bs=c.bs, seed=1, device='cuda')
    algo = RTN(model, cfg.quant, inp, None, cfg)
    algo.run_block_loop()
    algo.deploy('fake_quant')
    del inp
    x = torch.zeros(1, model.shape['hidden'], dtype=model.shape['dtype'], device='cuda')
    assert all(blk.block_sparse_moe.grouped_fake_quant_operands(x) is not None for blk in model.get_blocks())
    tokens = torch.randint(0, model.shape['vocab'], (1, 2048 * 8), generator=torch.Generator().manual_seed(4))
    time_ppl(res, 'fake_quant_ppl[mixtral-8x7b 1 block, rtn_fp8_static_mixtral.yml, 8x2048 tokens]', model,
             tokens, 2048, rounds)


def bench_packed_ppl(res, rounds):
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.rtn import RTN
    cfg = AttrDict.wrap({'base': {'seed': 0},
                         'quant': {'method': 'RTN', 'weight': {'bit': 4, 'symmetric': False,
                                                               'granularity': 'per_group', 'group_size': 128}}})
    model = synth.SynthModel('mixtral-8x7b', n_layers=1, seed=0, device='cuda', init='device')
    algo = RTN(model, cfg.quant, None, None, cfg)
    algo.run_block_loop()
    algo.deploy('fake_quant')
    tokens = torch.randint(0, model.shape['vocab'], (1, 2048 * 8), generator=torch.Generator().manual_seed(4))
    saved = MixtralSparseMoe.forward

    def run(loop):
        if loop:
            MixtralSparseMoe.forward = loop_forward
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ppl = synth.perplexity(model, tokens, 2048, 1)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, ppl
        finally:
            MixtralSparseMoe.forward = saved
    run(False), run(True)                          # warm-up
    times, ppls = {'grouped': [], 'loop': []}, {'grouped': set(), 'loop': set()}
    for _ in range(rounds):
        for path in times:
            dt, ppl = run(path == 'loop')
            times[path].append(round(dt, 3))
            ppls[path].add(ppl)
    assert ppls['grouped'] == ppls['loop'] and len(ppls['loop']) == 1, ppls
    key = 'fake_quant_ppl[mixtral-8x7b 1 block, RTN w4 g128, 8x2048 tokens]'
    med = {n: statistics.median(v) for n, v in times.items()}
    res['ppl_s'][key] = times
    res['ppl_speedup'][key] = round(med['loop'] / med['grouped'], 3)
    print(key, times, flush=True)


def run_awq(name, n_samples, seq_len, loop):
    from llmc_b200.awq import Awq
    from llmc_b200.blockwise import AttrDict
    cfg = {'calib': {'seq_len': seq_len},
           'quant': {'method': 'Awq',
                     'weight': {'bit': 4, 'symmetric': True, 'granularity': 'per_group', 'group_size': 128},
                     'special': {'trans': True, 'trans_version': 'v2', 'weight_clip': True,
                                 'clip_sym': True}}}
    saved = MixtralSparseMoe.forward
    if loop:
        MixtralSparseMoe.forward = loop_forward
    try:
        model = synth.SynthModel(name, n_layers=1, seed=0, device='cuda', with_head=False, init='device')
        inp = model.first_block_input(n_samples, seq_len, bs=-1, seed=1, device='cuda')
        c = AttrDict.wrap(copy.deepcopy(cfg))
        algo = Awq(model, c.quant, inp, None, c)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        algo.run_block_loop()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        MixtralSparseMoe.forward = saved
    state = [p.detach().clone() for p in model.get_model().layers.parameters()]
    del algo, inp, model
    torch.cuda.empty_cache()
    return dt, state


def bench_awq(res, n_samples, rounds):
    for loop in (False, True):                     # warm-up: every kernel both paths launch
        run_awq('tiny-mixtral', 8, 64, loop)
    times, states = {'grouped': [], 'loop': []}, {}
    for _ in range(rounds):                        # alternated: grouped, loop, grouped, loop, ...
        for path in times:
            dt, states[path] = run_awq('mixtral-8x7b', n_samples, 512, path == 'loop')
            times[path].append(round(dt, 3))
        assert all(torch.equal(a, b) for a, b in zip(states['grouped'], states['loop']))
    key = f'awq_run_block_loop[mixtral-8x7b 1 block, {n_samples}x512 tokens]'
    med = {n: statistics.median(v) for n, v in times.items()}
    res['awq_s'][key] = times
    res['awq_speedup'][key] = round(med['loop'] / med['grouped'], 3)
    print(key, times, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--tokens', type=int, nargs='+', default=[2048, 65536])
    ap.add_argument('--awq-samples', type=int, default=128)
    ap.add_argument('--awq-rounds', type=int, default=3)
    ap.add_argument('--packed', action='store_true')
    ap.add_argument('--w8a8', action='store_true')
    ap.add_argument('--fake-quant', action='store_true')
    ap.add_argument('--ppl-rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    res = {'card': card(), 'reps': args.reps, 'layer_ms': {}, 'layer_tflops': {}, 'layer_speedup': {}}
    if args.fake_quant:
        res.update(ppl_s={}, ppl_speedup={})
        with torch.no_grad():
            bench_fake_quant_layer(res, args.tokens, args.reps)
        if args.ppl_rounds > 0:
            bench_fake_quant_ppl(res, args.ppl_rounds)
    elif args.w8a8:
        with torch.no_grad():
            bench_w8a8_layer(res, args.tokens, args.reps)
    elif args.packed:
        res.update(ppl_s={}, ppl_speedup={})
        with torch.no_grad():
            bench_packed_layer(res, args.tokens, args.reps)
        if args.ppl_rounds > 0:
            bench_packed_ppl(res, args.ppl_rounds)
    else:
        res.update(awq_s={}, awq_speedup={})
        with torch.no_grad():
            bench_layer(res, args.tokens, args.reps)
        if args.awq_samples > 0:
            bench_awq(res, args.awq_samples, args.awq_rounds)
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_moe.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
