"""The W8A8 real-quant GEMM (llmc_gemm_w8a8_i8 / llmc_gemm_w8a8_fp8) next to the bf16 GEMM on the
dequantised weight, at the Llama-3-8B linear shapes and M = 2048 and 16384.

    python scripts/bench_gemm_w8a8.py [--reps 20] [--out DIR]

For each (M, N, K), five calls:
  bf16        llmc_gemm_bf16: bf16 activations times the dequantised int8 weight (what the fake-quant
              forward's GEMM does)
  i8          llmc_gemm_w8a8_i8 on int8 codes, per-token and per-channel fp32 scales
  fp8         llmc_gemm_w8a8_fp8 on e4m3 codes, the same scales
  i8_fwd      linear_forward_w8a8 with an int8 weight: the per-token activation quantizer pass
              (llmc_quant_dynamic, codes out) plus the i8 GEMM — the real-quant module's forward
  fp8_fwd     the same with an e4m3 weight (llmc_fp8_quant, bytes out, plus the fp8 GEMM)
Before timing, the i8 GEMM is checked bit for bit against the CPU oracle on a sample of rows.  Each
call is warmed up, then the five alternate for `reps` rounds, one call per round between CUDA events;
the median is reported with the achieved TFLOP/s (2 M N K over the median).  Prints, and writes to
DIR/bench_gemm_w8a8.json, one JSON object with the card name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import w8a8_oracle as wo  # noqa: E402
from llmc_b200._lib import call, dtype_enum, ptr, stream_ptr  # noqa: E402
from llmc_b200.module_utils import linear_forward, linear_forward_w8a8  # noqa: E402

SHAPES = {'qkv': (6144, 4096), 'o': (4096, 4096), 'gate_up': (28672, 4096), 'down': (4096, 14336)}
MS = (2048, 16384)
ACT_I8 = {'bit': 8, 'symmetric': True, 'granularity': 'per_token'}
ACT_FP8 = {'quant_type': 'float-quant', 'bit': 'e4m3', 'symmetric': True, 'granularity': 'per_token',
           'use_qtorch': True}


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


def gemm(kind, qx, s_x, qw, s_w, y):
    M, K = qx.shape
    call(f'llmc_gemm_w8a8_{kind}', ptr(qx), ptr(s_x), 1, ptr(qw), ptr(s_w), 1, None, ptr(y), M, qw.shape[0], K,
         dtype_enum(y.dtype), stream_ptr())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'reps': args.reps, 'ms': {}, 'tflops': {}}
    bf = torch.bfloat16
    for M in MS:
        for name, (N, K) in SHAPES.items():
            qw = torch.randint(-127, 128, (N, K), device='cuda', dtype=torch.int8)
            s_w = torch.rand(N, device='cuda') * 1e-3 + 1e-4
            w_bf = (qw.float() * s_w[:, None]).to(bf)
            fw = wo.fp8_finite_bytes((N, K), torch.Generator().manual_seed(1), 'cuda')
            x = torch.randn(M, K, device='cuda').to(bf)
            qx = torch.randint(-127, 128, (M, K), device='cuda', dtype=torch.int8)
            fx = wo.fp8_finite_bytes((M, K), torch.Generator().manual_seed(2), 'cuda')
            s_x = torch.rand(M, device='cuda') * 1e-2 + 1e-3
            y = torch.empty(M, N, device='cuda', dtype=bf)
            s_w16 = s_w.to(bf).reshape(N, 1)
            runs = {
                'bf16': lambda: linear_forward(x, w_bf),
                'i8': lambda: gemm('i8', qx, s_x, qw, s_w, y),
                'fp8': lambda: gemm('fp8', fx, s_x, fw, s_w, y),
                'i8_fwd': lambda: linear_forward_w8a8(x, qw, s_w16, ACT_I8),
                'fp8_fwd': lambda: linear_forward_w8a8(x, fw, s_w16, ACT_FP8),
            }
            runs['i8']()
            rows = torch.tensor([0, 1, 127, 128, M // 2, M - 1])
            ref = wo.gemm_w8a8(qx[rows.cuda()], s_x[rows.cuda()], qw, s_w, None, bf)
            assert torch.equal(y[rows.cuda()].cpu().view(torch.int16), ref.view(torch.int16)), (M, name)
            for fn in runs.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in runs}
            for _ in range(args.reps):
                for k, fn in runs.items():
                    times[k].append(timed(fn))
            key = f'{name}[M={M},N={N},K={K}]'
            med = {k: round(statistics.median(v), 4) for k, v in times.items()}
            res['ms'][key] = med
            res['tflops'][key] = {k: round(2.0 * M * N * K / (v * 1e-3) / 1e12, 1) for k, v in med.items()}
            print(key, med, flush=True)
            del qw, w_bf, fw, x, qx, fx, y
            torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gemm_w8a8.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
