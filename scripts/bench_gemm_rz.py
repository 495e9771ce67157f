"""The fake-quant forward with real-valued zero-points (llmc_gemm_w4a16_rz: HQQ, SpQR) next to the
contiguous W4A16 packed GEMM and the bf16 GEMM on a materialised weight, at the Llama-3-8B linear
shapes.

    python scripts/bench_gemm_rz.py [--reps 20] [--out DIR]

For each (N, K) at M = 2048, five forwards of the same bf16 activations:
  bf16        llmc_gemm_bf16 on the materialised weight of hqq_axis0
  w4_g128     llmc_gemm_w4a16, asymmetric g128, bf16 scale + integer zero (the shipped AWQ / RTN W4)
  hqq_axis0   llmc_gemm_w4a16_rz, group_axis 1: fp32 [K, N/128] scales + fractional zeros, groups
              of 128 rows (the shipped HQQ recipe, axis 0)
  hqq_axis1   llmc_gemm_w4a16_rz, group_axis 0: fp32 [K/128, N] qparams, g_idx = k // 128 (HQQ axis 1)
  spqr_g16    llmc_gemm_w4a16_rz, group_axis 0: fp32 g16 qparams, g_idx from a random permutation
              (act-order), 1 % random outliers as a CSR
Before timing, every packed forward is checked bit for bit against llmc_gemm_bf16 on its own
materialised weight.  Each form is warmed up, then the five alternate for `reps` rounds, one call
per round between CUDA events; the median is reported.  Prints, and writes to DIR/bench_gemm_rz.json,
one JSON object with the card name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llmc_b200.module_utils import (linear_forward, linear_forward_rz, linear_forward_w4,  # noqa: E402
                                    outliers_to_csr, pack_unsigned_codes)

SHAPES = {'qkv': (6144, 4096), 'o': (4096, 4096), 'gate_up': (28672, 4096), 'down': (4096, 14336)}
M = 2048


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


def qparams(rows, cols):
    s = torch.rand(rows, cols, device='cuda') * 0.01 + 0.001
    z = torch.rand(rows, cols, device='cuda') * 16 - 0.5
    return s, z


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'reps': args.reps, 'M': M, 'ms': {}, 'outliers': {}}
    bf = torch.bfloat16
    for name, (N, K) in SHAPES.items():
        codes = torch.randint(0, 16, (N, K), device='cuda')
        wq = pack_unsigned_codes(codes, 4, signed=False)
        c = codes.float()
        # W4 g128, integer zero-points in bf16 (the contiguous form)
        s4 = (torch.rand(N, K // 128, device='cuda') * 0.01 + 0.001).to(bf)
        z4 = torch.randint(0, 16, (N, K // 128), device='cuda').to(bf)
        m4 = ((c - z4.float().repeat_interleave(128, 1)) * s4.float().repeat_interleave(128, 1)).to(bf)
        # groups along N: [K, N/128]
        sn, zn = qparams(K, N // 128)
        mn = ((c - zn.repeat_interleave(128, 1).t()) * sn.repeat_interleave(128, 1).t()).to(bf)
        # groups along K: [K/128, N], g_idx = k // 128
        gk = (torch.arange(K, device='cuda') // 128).to(torch.int32)
        sk, zk = qparams(K // 128, N)
        mk = ((c - zk[gk.long()].t()) * sk[gk.long()].t()).to(bf)
        # SpQR-like: g16 act-order, 1 % outliers
        gp = (torch.argsort(torch.randperm(K, device='cuda')) // 16).to(torch.int32)
        sp, zp = qparams(K // 16, N)
        mask = torch.rand(N, K, device='cuda') < 0.01
        wo = (torch.randn(N, K, device='cuda') * 0.05).to(bf)
        mp = torch.where(mask, wo, ((c - zp[gp.long()].t()) * sp[gp.long()].t()).to(bf))
        csr = outliers_to_csr(mask, wo)
        res['outliers'][name] = int(csr[1].numel())
        del c, codes
        x = torch.randn(M, K, device='cuda').to(bf)
        runs = {
            'bf16': lambda: linear_forward(x, mn),
            'w4_g128': lambda: linear_forward_w4(x, wq, s4, z4, 128, bits=4),
            'hqq_axis0': lambda: linear_forward_rz(x, wq, sn, zn, 4, False, 1, group=128),
            'hqq_axis1': lambda: linear_forward_rz(x, wq, sk, zk, 4, False, 0, g_idx=gk),
            'spqr_g16': lambda: linear_forward_rz(x, wq, sp, zp, 4, False, 0, g_idx=gp, outliers=csr),
        }
        for k, mat in (('w4_g128', m4), ('hqq_axis0', mn), ('hqq_axis1', mk), ('spqr_g16', mp)):
            assert torch.equal(runs[k]().view(torch.int16), linear_forward(x, mat).view(torch.int16)), (name, k)
        for fn in runs.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(args.reps):
            for k, fn in runs.items():
                times[k].append(timed(fn))
        res['ms'][f'{name}[M={M},N={N},K={K}]'] = {k: round(statistics.median(v), 4) for k, v in times.items()}
        del x, wq, m4, mn, mk, mp, wo, mask, csr
        torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gemm_rz.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
