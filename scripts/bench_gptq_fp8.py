"""Per-linear span of the GPTQ column sweep on an FP8 grid next to the INT4 sweep, at the Llama-3-8B
linear shapes (q/k/v and gate/up stacked, as GPTQ sweeps them).

    python scripts/bench_gptq_fp8.py [--reps 3] [--out DIR]

Each shape gets one Hessian (bf16 activations through the SYRK), one Cholesky factor and one
permuted weight; then the sweeps alternate — INT4 asym g128 (the flagship configuration),
e4m3 per-channel with model-dtype scales (the shipped vLLM / SGLang FP8 recipe) and e4m3 g128
dynamic groups — after one warm-up each.  Times are the `gptq_colblock[...]` /
`gptq_colblock_fp8[...]` TIMER spans (CUDA events around the C-ABI call), the median over reps.
Prints, and writes to DIR/bench_gptq_fp8.json, one JSON object with the card name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llmc_b200 import gptq_ops as ops  # noqa: E402
from llmc_b200.prof import TIMER  # noqa: E402

SHAPES = {'qkv': (6144, 4096), 'o': (4096, 4096), 'gate_up': (28672, 4096), 'down': (4096, 14336)}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'shapes': {}}
    for name, (R, C) in SHAPES.items():
        W = (torch.randn(R, C, device='cuda') * 0.02).bfloat16()
        chan = torch.exp(torch.randn(C, device='cuda') * 0.7)
        H = torch.zeros(C, C, device='cuda')
        n = 0
        for _ in range(2):
            n = ops.hessian_add_batch(H, n, (torch.randn(1, 2048, C, device='cuda') * chan).bfloat16())
        perm = torch.argsort(torch.diag(H), descending=True)
        Wp, Hp = ops.prepare(W, H, perm, 0.01)
        Hinv = ops.chol_inv_upper(Hp)
        del Hp, H
        s_ch = (W.float().abs().amax(1, keepdim=True).clamp(min=1e-5) / 448).bfloat16()
        runs = {
            'int4_g128': lambda: ops.weight_transform(Wp.clone(), Hinv, 4, False, 128, out_perm=perm),
            'e4m3_channel': lambda: ops.weight_transform(Wp.clone(), Hinv, 'e4m3', True, C,
                                                         static_qparams=(s_ch.reshape(-1), None), out_perm=perm),
            'e4m3_g128': lambda: ops.weight_transform(Wp.clone(), Hinv, 'e4m3', True, 128, out_perm=perm),
        }
        times = {k: [] for k in runs}
        TIMER.enabled = True
        for rep in range(args.reps + 1):
            for k, fn in runs.items():
                TIMER.reset()
                fn()
                torch.cuda.synchronize()
                (span,) = [v for s, v in TIMER.summary().items() if s.startswith('gptq_colblock')]
                if rep:
                    times[k].append(span['ms'])
        TIMER.enabled = False
        res['shapes'][f'{name}[{R}x{C}]'] = {k: round(statistics.median(v), 3) for k, v in times.items()}
        del Wp, Hinv
        torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gptq_fp8.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
