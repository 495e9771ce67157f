"""The fake-quant forward on 2- and 3-bit weights (llmc_gemm_w2a16 / w3a16[_gidx]) next to the W4A16
packed GEMM and the bf16 GEMM on a materialised weight, at the Llama-3-8B linear shapes.

    python scripts/bench_gemm_lowbit.py [--reps 10] [--out DIR]

For each (M, N, K), M in {2048, 16384}, five forwards of the same bf16 activations:
  bf16         llmc_gemm_bf16 on the materialised W4 g128 weight
  w4_g128      llmc_gemm_w4a16, asymmetric g128, bf16 scale + zero (the shipped AWQ / RTN W4 recipes)
  w3_g128      llmc_gemm_w3a16, asymmetric g128, bf16 scale + zero (awq_comb_omni w3a16g128)
  w2_g64       llmc_gemm_w2a16, asymmetric g64, bf16 scale + zero (awq_comb_omni w2a16g64)
  w3_actorder  llmc_gemm_w3a16_gidx, fp32 g128 scale + zero, g_idx from a random permutation (GPTQ
               act-order)
Before timing, every packed forward is checked bit for bit against llmc_gemm_bf16 on its own
materialised weight.  Each form is warmed up, then the five alternate for `reps` rounds, one call
per round between CUDA events; the median is reported.  Prints, and writes to
DIR/bench_gemm_lowbit.json, one JSON object with the card name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llmc_b200.module_utils import linear_forward, linear_forward_w4, pack_unsigned_codes  # noqa: E402

SHAPES = {'q_o': (4096, 4096), 'k_v': (1024, 4096), 'gate_up': (14336, 4096), 'down': (4096, 14336)}
MS = (2048, 16384)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def packed_form(N, K, bits, group, qdt, g_idx=None):
    """Random unsigned codes with qparams [ng, N] (transposed, as EffcientFakeQuantLinear holds them)
    and the weight they materialise, rT((code - zero) * scale)."""
    ng = K // group
    codes = torch.randint(0, 1 << bits, (N, K), device='cuda')
    s = (torch.rand(N, ng, device='cuda') * 0.01 + 0.001).to(qdt)
    z = torch.randint(0, 1 << bits, (N, ng), device='cuda').to(qdt)
    gi = (g_idx if g_idx is not None else torch.arange(K, device='cuda') // group).long()
    w = ((codes.float() - z.float()[:, gi]) * s.float()[:, gi]).bfloat16()
    return pack_unsigned_codes(codes, bits, signed=False), s.t().contiguous(), z.t().contiguous(), w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'reps': args.reps, 'ms': {}}
    bf = torch.bfloat16
    for name, (N, K) in SHAPES.items():
        g_idx = (torch.argsort(torch.randperm(K, device='cuda')) // 128).to(torch.int32)
        w4, s4, z4, m4 = packed_form(N, K, 4, 128, bf)
        w3, s3, z3, m3 = packed_form(N, K, 3, 128, bf)
        w2, s2, z2, m2 = packed_form(N, K, 2, 64, bf)
        w3a, s3a, z3a, m3a = packed_form(N, K, 3, 128, torch.float32, g_idx)
        for M in MS:
            x = torch.randn(M, K, device='cuda').bfloat16()
            runs = {
                'bf16': lambda: linear_forward(x, m4),
                'w4_g128': lambda: linear_forward_w4(x, w4, s4, z4, 128, bits=4, qparams_t=True),
                'w3_g128': lambda: linear_forward_w4(x, w3, s3, z3, 128, bits=3, qparams_t=True),
                'w2_g64': lambda: linear_forward_w4(x, w2, s2, z2, 64, bits=2, qparams_t=True),
                'w3_actorder': lambda: linear_forward_w4(x, w3a, s3a, z3a, 128, bits=3, qparams_t=True,
                                                         g_idx=g_idx),
            }
            for k, mat in (('w4_g128', m4), ('w3_g128', m3), ('w2_g64', m2), ('w3_actorder', m3a)):
                ref = runs['bf16']() if k == 'w4_g128' else linear_forward(x, mat)
                assert torch.equal(runs[k]().view(torch.int16), ref.view(torch.int16)), (name, M, k)
            for fn in runs.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in runs}
            for _ in range(args.reps):
                for k, fn in runs.items():
                    times[k].append(timed(fn))
            res['ms'][f'{name}[M={M},N={N},K={K}]'] = {k: round(statistics.median(v), 4) for k, v in times.items()}
            del x
        del w4, w3, w2, w3a, m4, m3, m2, m3a
        torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gemm_lowbit.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
