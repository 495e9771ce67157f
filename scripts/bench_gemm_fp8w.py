"""The fake-quant forward on FP8 weights (llmc_gemm_fp8a16[_gidx]) next to the W8A16 packed GEMM and
the bf16 GEMM on the materialised weight, at the Llama-3-8B linear shapes.

    python scripts/bench_gemm_fp8w.py [--reps 10] [--out DIR]

For each (M, N, K), M in {2048, 16384}, four forwards of the same bf16 activations:
  fp8_channel   e4m3 bytes + bf16 per-channel scales (the shipped RTN / SmoothQuant / GPTQ recipes)
  fp8_actorder  e4m3 bytes + fp32 g128 scales with a random group index (GPTQ act-order)
  w8a16         llmc_gemm_w8a16, INT8 codes + bf16 per-channel scales
  bf16          llmc_gemm_bf16 on the materialised e4m3 weight
Each is warmed up, then the four alternate for `reps` rounds, one call per round between CUDA
events; the median is reported.  Before timing, fp8_channel's output is checked bit for bit
against bf16's (the same weight).  Prints, and writes to DIR/bench_gemm_fp8w.json, one JSON object
with the card name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llmc_b200.module_utils import linear_forward, linear_forward_fp8w, linear_forward_w4  # noqa: E402
from llmc_b200.quant_float import FloatQuantizer  # noqa: E402

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'reps': args.reps, 'ms': {}}
    q_ch = FloatQuantizer(bit='e4m3', symmetric=True, granularity='per_channel', use_qtorch=True)
    q_g = FloatQuantizer(bit='e4m3', symmetric=True, granularity='per_group', group_size=128, use_qtorch=True)
    for name, (N, K) in SHAPES.items():
        W = (torch.randn(N, K, device='cuda') * 0.02).bfloat16()
        wq, s_ch = q_ch._dynamic(W, 2)                         # e4m3 bytes, bf16 [N, 1]
        s_ch = s_ch.reshape(N, 1)
        w_mat = (wq.float() * s_ch.float()).bfloat16()
        perm = torch.randperm(K, device='cuda')
        invperm = torch.argsort(perm)
        wq_p, s_g = q_g._dynamic(W[:, perm].float().contiguous(), 2)
        wq_g = wq_p.view(torch.uint8)[:, invperm].view(torch.float8_e4m3fn).contiguous()
        s_g = s_g.reshape(N, -1).t().contiguous()               # fp32 [ng, N]
        g_idx = (invperm // 128).to(torch.int32)
        codes = torch.randint(0, 256, (N, K // 4), device='cuda', dtype=torch.int32)   # any bytes: same work
        s8 = s_ch.reshape(1, N).contiguous()
        for M in MS:
            x = torch.randn(M, K, device='cuda').bfloat16()
            runs = {
                'fp8_channel': lambda: linear_forward_fp8w(x, wq, s8, K, qparams_t=True),
                'fp8_actorder': lambda: linear_forward_fp8w(x, wq_g, s_g, 128, qparams_t=True, g_idx=g_idx),
                'w8a16': lambda: linear_forward_w4(x, codes, s8, None, K, bits=8, qparams_t=True),
                'bf16': lambda: linear_forward(x, w_mat),
            }
            assert torch.equal(runs['fp8_channel']().view(torch.int16), runs['bf16']().view(torch.int16)), name
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
        del W, wq, w_mat, wq_p, wq_g, codes
        torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gemm_fp8w.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
