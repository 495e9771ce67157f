"""One DeepSeek-V2-Lite layer's two new paths next to what they replace: the sparse-MoE layer (64
routed experts, top-6, fp32 routing weights, 2 ungated shared experts) on the grouped expert GEMMs
and llmc_moe_combine_weighted against its per-expert loop, and the MLA attention with its fused
projection pair (llmc_gemm_mla_qkv / llmc_gemm_mla_kv_b) against the unfused module path.

    python scripts/bench_deepseek_v2.py [--reps 10] [--tokens 2048 65536] [--seq 2048] [--out DIR]

Token counts: 2048 is one calibration forward at batch size 1, 65536 an inspect batch (32 x 2048).
Every pair first gives the same bits; after three warm-up calls each, the two alternate for `reps`
rounds between CUDA events and the medians are reported (the attention includes SDPA and o_proj,
which both paths share).  Prints, and writes to DIR/bench_deepseek_v2.json, one JSON object with the
card name and power limit.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench_moe  # noqa: E402
from llmc_b200 import synth  # noqa: E402
from llmc_b200.synth import DeepseekV2Attention, DeepseekV2SparseMoe  # noqa: E402


def alternate(res, key, runs, reps, flops):
    """runs: {'name': fn} of two paths that give the same bits (checked here); their medians."""
    outs = [fn() for fn in runs.values()]
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), key
    del outs
    for fn in runs.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n in runs}
    for _ in range(reps):
        for n, fn in runs.items():
            times[n].append(bench_moe.timed(fn))
    med = {n: round(statistics.median(v), 3) for n, v in times.items()}
    res['ms'][key] = med
    res['tflops'][key] = {n: round(flops / (v * 1e-3) / 1e12, 1) for n, v in med.items()}
    names = list(runs)
    res['speedup'][key] = round(med[names[1]] / med[names[0]], 3)
    print(key, med, res['tflops'][key], flush=True)


def _init(mod, g):
    for p in mod.parameters():
        p.data.normal_(0, 0.02, generator=g)


def bench_moe_layer(res, s, tokens, reps):
    H, I, E, k, ns = s['hidden'], s['moe_inter'], s['experts'], s['top_k'], s['shared_experts']
    g = torch.Generator(device='cuda').manual_seed(0)
    with torch.device('meta'):
        moe = DeepseekV2SparseMoe(H, I, E, k, ns, s['routed_scale'])
    moe = moe.to(torch.bfloat16).to_empty(device='cuda')
    _init(moe, g)

    def loop(hs):
        x = hs.reshape(-1, H)
        sel, w = moe.route(x)
        return moe.shared_loop(x, sel, w).reshape(hs.shape)

    for T in tokens:
        hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
        assert moe.grouped_weights(hs.view(T, H)) is not None
        flops = 2.0 * T * (k + ns) * 3 * H * I
        alternate(res, f'moe_layer[T={T}]', {'grouped': lambda: moe(hs), 'loop': lambda: loop(hs)}, reps, flops)
        del hs
        torch.cuda.empty_cache()
    del moe
    torch.cuda.empty_cache()


def bench_mla(res, s, tokens, seq, reps):
    H, nh, r = s['hidden'], s['heads'], s['kv_lora']
    g = torch.Generator(device='cuda').manual_seed(1)
    with torch.device('meta'):
        a = DeepseekV2Attention(H, nh, r, eps=s['rms_eps'])
    a = a.to(torch.bfloat16).to_empty(device='cuda')
    _init(a, g)
    a.kv_a_layernorm.weight.data.fill_(1.0)
    assert a.fused_weights(torch.bfloat16) is not None
    real = DeepseekV2Attention.fused_weights

    def unfused(x, pos):
        DeepseekV2Attention.fused_weights = lambda self, dtype: None
        try:
            return a(x, position_embeddings=pos)
        finally:
            DeepseekV2Attention.fused_weights = real

    pos = synth.mla_rope_cos_sin(seq, 64, 'cuda', s['rope_theta'])
    for T in tokens:
        S = min(seq, T)
        x = torch.randn(T // S, S, H, device='cuda', generator=g).to(torch.bfloat16)
        proj = 2.0 * T * H * (nh * 192 + r + 64) + 2.0 * T * r * nh * 256 + 2.0 * T * nh * 128 * H
        alternate(res, f'mla_attention[T={T}, S={S}]',
                  {'fused': lambda: a(x, position_embeddings=pos), 'unfused': lambda: unfused(x, pos)}, reps, proj)
        del x
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--tokens', type=int, nargs='+', default=[2048, 65536])
    ap.add_argument('--seq', type=int, default=2048)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    s = synth.SHAPES['deepseek-v2-lite']
    # tflops: of the expert GEMMs (routed and shared) / of the attention's projections (not SDPA)
    res = {'card': bench_moe.card(), 'reps': args.reps, 'ms': {}, 'tflops': {}, 'speedup': {}}
    bench_moe_layer(res, s, args.tokens, args.reps)
    bench_mla(res, s, args.tokens, args.seq, args.reps)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_deepseek_v2.json'), 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
