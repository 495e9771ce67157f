"""Times the 3xTF32 update (llmc_gemm_f32x3, tf32.cu) alone, at the shapes the GPTQ workload of
bench.py calls it with (Llama-3-8B: Cholesky inverse of the 14336-column Hessian, column sweeps
of 4096 x 14336 and 28672 x 4096 weights).

    python scripts/bench_tf32x3.py [--lib A.so [--lib B.so ...]] [--out FILE.json]

Per shape: ms per call (CUDA events over many back-to-back launches after a warm-up), fp32-equivalent
TFLOP/s (2 M N K, or 2 * 128 * 128 * K per computed tile for the lower-triangle calls) and the
bytes of C read and written (8 per computed element).  Operands are compact (ld = K or M / N);
the workload reads them out of larger matrices, which TMA loads in the same 128-byte rows.

With several --lib, each shape is timed with every library in turn (alternating, same inputs),
and the outputs of one seeded call per mode are compared bit for bit across the libraries.  The card name
and power limit are printed with the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from llmc_b200 import _lib  # noqa: E402

BM = BN = 128

# (name, M, N, K, lower_only); see chol.cu (look-ahead schedule) and gptq.cu (sweep)
SHAPES = [
    ('chol14336 factor bulk (lower)', 13824, 13824, 512, 1),   # L[sp1:, sp0:sp1] twice, sp1 = 512
    ('chol14336 factor bulk (lower)', 7168, 7168, 512, 1),     # sp1 = 7168
    ('chol14336 factor chain K=128', 7168, 128, 128, 0),       # G[k0:, k0:k0+128], k0 = 7168
    ('chol14336 factor chain K=256', 7168, 128, 256, 0),
    ('chol14336 factor chain K=384', 7168, 128, 384, 0),
    ('chol14336 inverse bulk', 7168, 7168, 512, 0),            # Z[0:sp1, sp0:sp1] x L[sp1:, ..]
    ('chol14336 inverse chain', 7168, 128, 128, 0),            # Z[0:k0, k-block] x Y_kk
    ('sweep 4096x14336 bulk', 4096, 13312, 512, 0),             # Err1 x Hinv^T[n0:, k-block]
    ('sweep 4096x14336 bulk', 4096, 6656, 512, 0),
    ('sweep 4096x14336 chain', 4096, 512, 512, 0),
    ('sweep 4096x14336 in-panel', 4096, 384, 128, 0),
    ('sweep 28672x4096 bulk', 28672, 3072, 512, 0),
    ('sweep 28672x4096 chain', 28672, 512, 512, 0),
    ('sweep 28672x4096 in-panel', 28672, 384, 128, 0),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return name, q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return name, 'power limit not readable'


def load(path):
    lib = ctypes.CDLL(path)
    res, args = _lib.SIGNATURES['llmc_gemm_f32x3']
    lib.llmc_gemm_f32x3.restype, lib.llmc_gemm_f32x3.argtypes = res, args
    lib.llmc_b200_last_error.restype = ctypes.c_char_p
    return lib


def lower_tiles(M, N):
    return sum(min((mi * BM + BM - 1) // BN + 1, (N + BN - 1) // BN) for mi in range((M + BM - 1) // BM))


class Case:
    """Seeded operands (tf32 split) and C for one shape; the split itself is done in torch,
    which matches tf32_split only approximately: timing and cross-library equality need inputs,
    not a particular split."""

    def __init__(self, M, N, K, lower, seed=0):
        g = torch.Generator(device='cuda').manual_seed(seed)
        def split(shape):
            x = torch.randn(*shape, device='cuda', generator=g)
            hi = (x.view(torch.int32) & ~0x1fff).view(torch.float32)
            return hi.contiguous(), (x - hi).contiguous()
        self.a = split((M, K))
        self.b = split((N, K))
        self.c0 = torch.randn(M, N, device='cuda', generator=g)
        self.c = self.c0.clone()
        self.M, self.N, self.K, self.lower = M, N, K, lower

    def call(self, lib, c=None, mode=0):
        c = self.c if c is None else c
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = _lib.ptr
        rc = lib.llmc_gemm_f32x3(p(self.a[0]), p(self.a[1]), self.K, p(self.b[0]), p(self.b[1]), self.K,
                                 p(c), self.N, self.M, self.N, self.K, mode, self.lower, st)
        if rc != 0:
            raise RuntimeError('llmc_gemm_f32x3: %s' % lib.llmc_b200_last_error().decode())


def time_call(case, lib, reps):
    for _ in range(3):
        case.call(lib)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        case.call(lib)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', default=None,
                    help='library to time (repeatable); default: this tree\'s build')
    ap.add_argument('--rounds', type=int, default=3, help='alternating timing rounds per library')
    ap.add_argument('--out', default=None, help='also write the results as JSON here')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_tf32x3 needs a CUDA device'
    paths = args.lib or [_lib.LIB_PATH]
    libs = [load(p) for p in paths]
    name, power = card()
    print(f'# {name}, power limit / max SM clock: {power}')
    for i, p in enumerate(paths):
        print(f'# lib{i}: {p}')
    rows = []
    for sname, M, N, K, lower in SHAPES:
        case = Case(M, N, K, lower)
        tiles = lower_tiles(M, N) if lower else None
        elems = tiles * BM * BN if lower else M * N
        flop = 2.0 * elems * K
        # one seeded call per library and mode (0: C -= AB from the same C, 1: C = AB), compared
        # bit for bit
        same = True
        for mode in (0, 1):
            outs = []
            for lib in libs:
                c = case.c0.clone()
                case.call(lib, c, mode)
                outs.append(c)
            same = same and all(torch.equal(outs[0], o) for o in outs[1:])
            del outs
        t1 = time_call(case, libs[0], 1)
        reps = max(5, min(200, int(0.15 / max(t1 * 1e-3, 1e-6))))
        ms = [[] for _ in libs]
        for _ in range(args.rounds):
            for i, lib in enumerate(libs):
                ms[i].append(time_call(case, lib, reps))
        row = {'shape': sname, 'M': M, 'N': N, 'K': K, 'lower': lower,
               'c_rmw_bytes': 8 * elems, 'reps': reps, 'bitwise_equal': same,
               'ms': [min(m) for m in ms], 'ms_max': [max(m) for m in ms],
               'tflops_fp32eq': [flop / min(m) / 1e9 for m in ms]}
        rows.append(row)
        cols = '  '.join(f'lib{i} {row["ms"][i]:8.3f} ms ({row["ms_max"][i]:7.3f}) {row["tflops_fp32eq"][i]:6.1f} TF/s'
                         for i in range(len(libs)))
        extra = f'  x{row["ms"][0] / row["ms"][1]:.2f}' if len(libs) > 1 else ''
        print(f'{sname:32s} M={M:6d} N={N:6d} K={K:4d} C rmw {8 * elems / 1e6:8.1f} MB  {cols}{extra}'
              f'  {"same bits" if same else "BITS DIFFER"}', flush=True)
        del case
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump({'card': name, 'power_limit_max_sm_clock': power, 'libs': paths, 'shapes': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
