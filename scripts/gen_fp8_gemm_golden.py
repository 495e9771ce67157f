"""Generate tests/golden/fp8_gemm_kat.pt from the reference's own Triton block-FP8 kernels
(llmc/compression/quantization/kernel.py), run in Triton's CPU interpreter.

    python scripts/gen_fp8_gemm_golden.py --llmc-root /path/to/llmc-checkout

The autotuned `fp8_gemm_kernel` needs a GPU driver to time its configs, so its inner jitted function
is launched directly with fixed configs (TRITON_INTERPRET=1).  The golden pins fp8_gemm's fp32
output, its scale indexing (a_s per row, b_s per 128 columns) and the per-K-block promotion, and
act_quant's scale under IEEE division (the interpreter divides with numpy).  The e4m3 codes are made
by torch, never taken from the interpreter: its fp32 -> e4m3 encode is wrong at binade edges.
"""
import argparse
import importlib.util
import os

os.environ['TRITON_INTERPRET'] = '1'

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'fp8_gemm_kat.pt')


def load_kernels(llmc_root):
    path = os.path.join(llmc_root, 'llmc', 'compression', 'quantization', 'kernel.py')
    spec = importlib.util.spec_from_file_location('llmc_fp8_kernel', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def case(kern, M, N, K, seed):
    import triton
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * torch.exp(torch.randn(K, generator=g))).to(torch.bfloat16)
    x[M // 2, :128] = x[M // 2, :128] * 1e-3                             # a small-scale group
    w = torch.randn(N, K, generator=g) * 0.05
    kb, nb = K // 128, -(-N // 128)
    w_s = (torch.rand(nb, kb, generator=g) * 2e-4 + 5e-5).float()
    w_q = (w / w_s.repeat_interleave(128, 0)[:N].repeat_interleave(128, 1)).clamp(-448, 448)
    w_q = w_q.to(torch.float8_e4m3fn)
    # act_quant in the interpreter: keep its scales, make the codes with torch from those scales
    _, a_s = kern.act_quant(x, 128)
    xs = x.float().view(M, kb, 128)
    a_q = (xs / a_s[..., None]).clamp(-448, 448).to(torch.float8_e4m3fn).view(M, K)
    outs = {}
    for bm, bn in [(16, 32), (64, 128)]:
        c = torch.empty(M, N, dtype=torch.get_default_dtype())
        grid = (triton.cdiv(M, bm), triton.cdiv(N, bn))
        kern.fp8_gemm_kernel.fn[grid](a_q, w_q, c, a_s, w_s, M, N, K, BLOCK_SIZE_M=bm, BLOCK_SIZE_N=bn,
                                      BLOCK_SIZE_K=128)
        outs[f'c_bm{bm}_bn{bn}'] = c
    return dict(M=M, N=N, K=K, x=x, a_s=a_s, a_q=a_q.view(torch.uint8), w_q=w_q.view(torch.uint8),
                w_s=w_s, **outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--llmc-root', required=True, help='checkout of ModelTC/llmc')
    args = ap.parse_args()
    kern = load_kernels(args.llmc_root)
    cases = [case(kern, M, N, K, seed) for seed, (M, N, K) in
             enumerate([(37, 200, 384), (5, 130, 256), (70, 64, 128)])]
    torch.save({'cases': cases}, OUT)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
