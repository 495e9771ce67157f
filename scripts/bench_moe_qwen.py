"""The Qwen1.5-MoE-A2.7B sparse-MoE layer (60 routed experts, top-4, a gated shared expert) on the
grouped expert GEMMs and llmc_moe_combine_shared, next to the per-expert loop it replaces; and the
Mixtral-8x7B layer of scripts/bench_moe.py on this library against another build of it.

    python scripts/bench_moe_qwen.py [--reps 10] [--tokens 2048 65536] [--ab-lib PATH] [--ab-rounds 3]
                                     [--out DIR]

1. One Qwen1.5-MoE layer (hidden 2048, moe_inter 1408, shared_inter 5632, 60 experts, top-4, bf16)
   at 2048 tokens (one calibration forward at batch size 1) and 65536 tokens (an AWQ inspect batch,
   128 x 512): the module forward, router and shared expert included, grouped and with the expert
   loop forced (Qwen2MoeSparseMoe.shared_loop).  Both give the same bits first; after warm-up the two
   alternate for `reps` rounds between CUDA events (bench_moe.compare_and_time), and the medians are
   reported with the achieved TFLOP/s of the routed and shared expert GEMMs.
2. With --ab-lib PATH (a libllmc_b200.so built from another revision): bench_moe.py's Mixtral-8x7B
   layer timing (bench_moe.bench_layer, grouped and loop at each of `tokens`) in a fresh process per
   run, alternating this tree's library and PATH (and which of them goes first) for ab_rounds
   rounds, so that run-to-run spread and
   the difference between the builds are measured the same way.  The grouped launches' parameter block
   grew from about 2.5 KB to about 16 KB when the expert cap went from 8 to 64; this is how that cost
   is measured.
Prints, and writes to DIR/bench_moe_qwen.json, one JSON object with the card name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench_moe  # noqa: E402
from llmc_b200 import _lib, synth  # noqa: E402
from llmc_b200.synth import Qwen2MoeSparseMoe  # noqa: E402


class _Loop(torch.nn.Module):
    """The layer with its expert loop forced, as bench_moe.loop_forward forces Mixtral's."""

    def __init__(self, moe):
        super().__init__()
        self.moe = moe

    def forward(self, hs):
        B, S, H = hs.shape
        x = hs.reshape(-1, H)
        sel, w = self.moe.route(x)
        return self.moe.shared_loop(x, sel, w).reshape(B, S, H)


def bench_qwen_layer(res, tokens, reps):
    s = synth.SHAPES['qwen1.5-moe-a2.7b']
    H, I, Is, E, k = s['hidden'], s['moe_inter'], s['shared_inter'], s['experts'], s['top_k']
    g = torch.Generator(device='cuda').manual_seed(0)
    with torch.device('meta'):
        moe = Qwen2MoeSparseMoe(H, I, Is, E, k)
    moe = moe.to(torch.bfloat16).to_empty(device='cuda')
    for p in moe.parameters():
        p.data.normal_(0, 0.02, generator=g)
    loop = _Loop(moe)
    real_loop = bench_moe.loop_forward
    bench_moe.loop_forward = lambda m, hs: loop(hs)
    try:
        for T in tokens:
            hs = torch.randn(1, T, H, device='cuda', generator=g).to(torch.bfloat16)
            assert moe.grouped_weights(hs.view(T, H)) is not None
            flops = 2.0 * T * (k * 3 * H * I + 3 * H * Is)
            bench_moe.compare_and_time(res, f'qwen_moe_layer[T={T}]', moe, hs, flops, reps)
            del hs
            torch.cuda.empty_cache()
    finally:
        bench_moe.loop_forward = real_loop
    del moe, loop
    torch.cuda.empty_cache()


def mixtral_once(lib, tokens, reps):
    """bench_moe.bench_layer on the library at `lib`, in this process; returns its medians."""
    _lib.LIB_PATH = lib
    res = {'layer_ms': {}, 'layer_tflops': {}, 'layer_speedup': {}}
    bench_moe.bench_layer(res, tokens, reps)
    return res['layer_ms']


def bench_ab(res, other, tokens, reps, rounds):
    libs = {'this': _lib.LIB_PATH, 'other': os.path.abspath(other)}
    runs = {n: [] for n in libs}
    for r in range(rounds):
        # which build runs first alternates too: a card near its power limit is faster when it starts cool
        for name, lib in (list(libs.items()) if r % 2 == 0 else list(libs.items())[::-1]):
            cmd = [sys.executable, os.path.abspath(__file__), '--mixtral-once', lib, '--reps', str(reps),
                   '--tokens', *map(str, tokens)]
            out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
            runs[name].append(json.loads(out.strip().splitlines()[-1]))
            print(name, runs[name][-1], flush=True)
    summary = {}
    for key in runs['this'][0]:
        for path in ('grouped', 'loop'):
            vals = {n: [r[key][path] for r in runs[n]] for n in runs}
            summary[f'{key}.{path}'] = {
                'this_ms': vals['this'], 'other_ms': vals['other'],
                'median_ratio_this_over_other': round(statistics.median(vals['this'])
                                                      / statistics.median(vals['other']), 4)}
    res['mixtral_ab'] = summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--tokens', type=int, nargs='+', default=[2048, 65536])
    ap.add_argument('--ab-lib', default=None)
    ap.add_argument('--ab-rounds', type=int, default=3)
    ap.add_argument('--mixtral-once', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if args.mixtral_once:
        print(json.dumps(mixtral_once(args.mixtral_once, args.tokens, args.reps)))
        return
    res = {'card': bench_moe.card(), 'layer_ms': {}, 'layer_tflops': {}, 'layer_speedup': {}}
    bench_qwen_layer(res, args.tokens, args.reps)
    if args.ab_lib:
        bench_ab(res, args.ab_lib, args.tokens, args.reps, args.ab_rounds)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_moe_qwen.json'), 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
