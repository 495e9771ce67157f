"""The real-quant forward of the AutoAWQ export (llmc_gemm_w4a16_awq, qweight packed along N) next to the
vLLM export on the packed W4 GEMM (llmc_gemm_w4a16, codes packed along K) and the bf16 GEMM on the
materialised weight, at the Llama-3-8B linear shapes.

    python scripts/bench_gemm_awq.py [--reps 10] [--out DIR]

For each (M, N, K), M in {2048, 16384}, three forwards of the same bf16 activations on one W4 g128
weight, rT((code - 8) * s) with fp16 scales:
  bf16   llmc_gemm_bf16 on the materialised weight
  vllm   llmc_gemm_w4a16 on the vLLM export (weight_packed [N, K/8], fp16 weight_scale [N, K/128],
         widened to fp32 as a bf16 model's export runs it)
  awq    llmc_gemm_w4a16_awq on the AutoAWQ export (qweight [K, N/8], qzeros, fp16 scales), as stored
Before timing, both packed forwards are checked bit for bit against llmc_gemm_bf16.  Each form is
warmed up, then the three alternate for `reps` rounds, one call per round between CUDA events; the
median is reported.  Prints, and writes to DIR/bench_gemm_awq.json, one JSON object with the card
name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llmc_b200.module_utils import linear_forward, linear_forward_w4, linear_forward_w4a16_awq  # noqa: E402

SHAPES = {'q_o': (4096, 4096), 'k_v': (1024, 4096), 'gate_up': (14336, 4096), 'down': (4096, 14336)}
MS = (2048, 16384)
GROUP = 128
AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)


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


def pack8(codes):
    """int [R, C] codes 0..15 -> int32 [R, C/8], code 8w + i in nibble i of word w."""
    c = codes.to(torch.int64).reshape(codes.shape[0], -1, 8)
    w = sum(c[:, :, i] << (4 * i) for i in range(8))
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def forms(N, K):
    """One symmetric W4 g128 weight as the vLLM and the AutoAWQ export, and its materialised bf16 form."""
    ng = K // GROUP
    codes = torch.randint(0, 16, (N, K), device='cuda')
    s = (torch.rand(N, ng, device='cuda') * 0.01 + 0.001).half()
    gi = torch.arange(K, device='cuda') // GROUP
    w = ((codes - 8).float() * s.float()[:, gi]).bfloat16()
    vllm = pack8(codes)
    ct = codes.t().contiguous()                                        # [K, N]
    qweight = pack8(torch.stack([ct[:, o::8] for o in AWQ_ORDER], dim=-1).reshape(K, N))
    qzeros = pack8(torch.full((ng, N), 8, device='cuda'))
    return vllm, s, qweight, s.t().contiguous(), qzeros, w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a CUDA device'
    torch.manual_seed(0)
    res = {'card': card(), 'reps': args.reps, 'ms': {}}
    for name, (N, K) in SHAPES.items():
        vllm, s_v, qweight, s_a, qzeros, w = forms(N, K)
        for M in MS:
            x = torch.randn(M, K, device='cuda').bfloat16()
            runs = {
                'bf16': lambda: linear_forward(x, w),
                'vllm': lambda: linear_forward_w4(x, vllm, s_v, None, GROUP, bits=4),
                'awq': lambda: linear_forward_w4a16_awq(x, qweight, s_a, qzeros, GROUP),
            }
            ref = runs['bf16']()
            for k in ('vllm', 'awq'):
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
            del x, ref
        del vllm, qweight, qzeros, w
        torch.cuda.empty_cache()
    doc = json.dumps(res)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gemm_awq.json'), 'w') as fh:
            fh.write(doc + '\n')


if __name__ == '__main__':
    main()
