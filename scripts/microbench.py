"""Kernel-level timings on one GPU (CUDA events, warm-up, inputs larger than L2 or L2 flushed).
Writes gpurun_out/microbench.json.  Not the headline bench (bench.py); used to steer tuning."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from llmc_b200 import gptq_ops as ops  # noqa: E402
from llmc_b200.module_utils import linear_forward  # noqa: E402
from llmc_b200.quant import IntegerQuantizer  # noqa: E402

PEAKS = {}
try:
    PEAKS = json.load(open(os.path.join(os.path.dirname(__file__), '..', 'MEASURED_PEAKS.json')))
except Exception:
    pass
# H100 SXM data sheet (dense, 700 W card): 3.35 TB/s HBM3, 989 TFLOP/s bf16, 1,979 TFLOP/s fp8
HBM = PEAKS.get('hbm_gbs', 3350.0)
TF = PEAKS.get('bf16_tflops', 989.0)
TF_FP8 = PEAKS.get('fp8_tflops', 1979.0)

flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')


def timeit(fn, iters=5, warm=2, do_flush=True):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if do_flush:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def _device():
    """The card every number of this run was measured on, and its power limit."""
    import subprocess
    d = {'name': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm',
                              '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        d['power_limit'], d['max_sm_clock'] = [v.strip() for v in out.split(',')]
    except Exception as e:                                   # noqa: BLE001
        d['power_limit'] = f'unknown ({type(e).__name__})'
    return d


res = {'_device': _device()}
print('device', res['_device'], flush=True)


def rec(name, ms, **kw):
    res[name] = dict(ms=round(ms, 4), **kw)
    print(name, res[name], flush=True)


only = sys.argv[1:] or ['quant', 'gemm', 'syrk', 'gptq']

if 'quant' in only:
    for dt in (torch.bfloat16, torch.float16):
        w = (torch.randn(28672, 4096, device='cuda') * 0.02).to(dt)
        n = w.numel()
        q = IntegerQuantizer(4, False, 'per_group', group_size=128)
        ms = timeit(lambda: q.real_quant_pack_vllm_dynamic(w))
        by = n * (2 + 0.5 + 4 / 128)
        rec(f'quant_pack_w4g128_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        ms = timeit(lambda: q.fake_quant_weight_dynamic(w))
        by = n * (4 + 4 / 128)
        rec(f'fake_quant_w4g128_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        qs = IntegerQuantizer(4, True, 'per_group', group_size=128)
        ms = timeit(lambda: qs.real_quant_pack_vllm_dynamic(w))
        by = n * (2 + 0.5 + 2 / 128)
        rec(f'quant_pack_w4g128_sym_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        ms = timeit(lambda: qs.fake_quant_weight_dynamic(w))
        by = n * (4 + 2 / 128)
        rec(f'fake_quant_w4g128_sym_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        q8g = IntegerQuantizer(8, True, 'per_group', group_size=128)
        ms = timeit(lambda: q8g.real_quant_pack_vllm_dynamic(w))
        by = n * (2 + 1 + 2 / 128)
        rec(f'quant_pack_w8g128_sym_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        q8 = IntegerQuantizer(8, True, 'per_channel')
        ms = timeit(lambda: q8.real_quant_weight_dynamic(w))
        by = n * 3
        rec(f'quant_w8_perchannel_{dt}', ms, gbs=by / ms / 1e6, frac=by / ms / 1e6 / HBM)
        del w

if 'gemm' in only:
    for (M, N, K) in ((8192, 4096, 4096), (32768, 4096, 4096), (16384, 14336, 4096),
                      (16384, 4096, 14336), (2048, 14336, 4096)):
        x = torch.randn(M, K, device='cuda').bfloat16()
        w = (torch.randn(N, K, device='cuda') * 0.02).bfloat16()
        fl = 2.0 * M * N * K
        ms = timeit(lambda: linear_forward(x, w), do_flush=False)
        rec(f'gemm_{M}x{N}x{K}', ms, tflops=fl / ms / 1e9, frac=fl / ms / 1e9 / TF)
        ms = timeit(lambda: torch.nn.functional.linear(x, w), do_flush=False)
        rec(f'cublas_{M}x{N}x{K}', ms, tflops=fl / ms / 1e9, frac=fl / ms / 1e9 / TF)
        del x, w

if 'syrk' in only:
    for (T, C) in ((32768, 4096), (131072, 4096), (16384, 14336)):
        x = torch.randn(T, C, device='cuda').bfloat16()
        H = torch.zeros(C, C, device='cuda')
        fl = 2.0 * T * C * C
        ms = timeit(lambda: ops.hessian_add_batch(H, 1, x.unsqueeze(0)), do_flush=False)
        rec(f'syrk_T{T}_C{C}', ms, tflops_full=fl / ms / 1e9, frac_full=fl / ms / 1e9 / TF,
            tflops_half=fl / 2 / ms / 1e9)
        xt = x.float()
        ms = timeit(lambda: xt.t() @ xt, iters=2, warm=1, do_flush=False)
        rec(f'torch_fp32_xtx_T{T}_C{C}', ms, tflops=fl / ms / 1e9)
        del x, H, xt

if 'gptq' in only:
    for (R, C) in ((4096, 4096), (14336, 4096), (4096, 14336)):
        W = (torch.randn(R, C, device='cuda') * 0.02).bfloat16()
        x = torch.randn(1, 8192, C, device='cuda').bfloat16()
        H = torch.zeros(C, C, device='cuda')
        ops.hessian_add_batch(H, 0, x)
        perm = torch.argsort(torch.diag(H), descending=True)
        t_prep = timeit(lambda: ops.prepare(W, H, perm, 0.01), iters=3, warm=1, do_flush=False)
        Wp, Hp = ops.prepare(W, H, perm, 0.01)
        t_chol = timeit(lambda: ops.chol_inv_upper(Hp), iters=3, warm=1, do_flush=False)
        Hinv = ops.chol_inv_upper(Hp)
        t_col = timeit(lambda: ops.weight_transform(Wp.clone(), Hinv, 4, False, 128, out_perm=perm),
                       iters=3, warm=1, do_flush=False)
        rec(f'gptq_layer_{R}x{C}', t_prep + t_chol + t_col, prepare_ms=t_prep, chol_ms=t_chol,
            colblock_ms=t_col, trailing_tflops=(R * C * C) / t_col / 1e9)
        del W, x, H, Wp, Hp, Hinv

if 'spqr' in only:
    # SpQR's sweep (spqr_w_only.yml: W4 asym g16, bilevel 3-bit qparams, threshold 0.2) next to the
    # GPTQ sweep of the same layer (W4 asym g128)
    for (R, C) in ((4096, 4096),):
        W = (torch.randn(R, C, device='cuda') * 0.02).bfloat16()
        x = torch.randn(1, 8192, C, device='cuda').bfloat16()
        H = torch.zeros(C, C, device='cuda')
        ops.hessian_add_batch(H, 0, x)
        perm = torch.argsort(torch.diag(H), descending=True)
        Wp, Hp = ops.prepare(W, H, perm, 1.0)
        Hinv = ops.chol_inv_upper(Hp)
        thr = ops.spqr_threshold(Wp, Hinv, 0.2)
        cfg = ((4, False, False, 16), (3, False, False), (3, False, False))
        t_sp = timeit(lambda: ops.spqr_transform(Wp.clone(), Hinv, *cfg, thr, False, out_perm=perm),
                      iters=3, warm=1, do_flush=False)
        t_g = timeit(lambda: ops.weight_transform(Wp.clone(), Hinv, 4, False, 128, out_perm=perm),
                     iters=3, warm=1, do_flush=False)
        mask = ops.spqr_transform(Wp.clone(), Hinv, *cfg, thr, False, out_perm=perm)[1]
        rec(f'spqr_colblock_{R}x{C}_g16', t_sp, gptq_colblock_g128_ms=t_g,
            us_per_128_columns=t_sp * 1e3 / (C / 128), outlier_frac=float(mask.float().mean()))
        del W, x, H, Wp, Hp, Hinv

if 'w4' in only:
    # SURVEY 8(d) config 3: the dequant-GEMM at M = 65536 (AWQ, bs -1) and M = 2048 (PPL eval)
    from llmc_b200.module_utils import linear_forward_w4
    for (M, N, K) in ((65536, 4096, 4096), (65536, 11008, 4096), (65536, 4096, 11008), (2048, 4096, 4096),
                      (2048, 11008, 4096)):
        x = torch.randn(M, K, device='cuda').half()
        w = (torch.randn(N, K, device='cuda') * 0.02).half()
        q = IntegerQuantizer(4, False, 'per_group', group_size=128)
        packed, s, z = q.real_quant_pack_vllm_dynamic(w)
        fl = 2.0 * M * N * K
        ms = timeit(lambda: linear_forward_w4(x, packed, s.float(), None if z is None else z.float(), 128),
                    do_flush=False)
        rec(f'gemm_w4a16_f32qparams_{M}x{N}x{K}', ms, tflops=fl / ms / 1e9, frac=fl / ms / 1e9 / TF)
        zt = None if z is None else z.to(x.dtype)
        ms = timeit(lambda: linear_forward_w4(x, packed, s.to(x.dtype), zt, 128), do_flush=False)
        rec(f'gemm_w4a16_native_{M}x{N}x{K}', ms, tflops=fl / ms / 1e9, frac=fl / ms / 1e9 / TF)
        wd = q.fake_quant_weight_dynamic(w)
        ms = timeit(lambda: linear_forward(x, wd), do_flush=False)
        rec(f'gemm_f16_materialised_{M}x{N}x{K}', ms, tflops=fl / ms / 1e9, frac=fl / ms / 1e9 / TF)
        del x, w, packed, wd

if 'awq' in only:
    # SURVEY 8(d) config 3: AWQ W4A16 g128 scale search + auto-clip, ONE Llama-2-7B-shape block,
    # calibration [128, 512] token ids in one batch (bs -1), configs/awq_w_only.yml
    import copy
    import yaml
    from llmc_b200.awq import Awq
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.synth import SynthModel
    cfg = yaml.safe_load(open(os.path.join(os.path.dirname(__file__), '..', 'configs', 'awq_w_only.yml')))
    for rep in range(2):
        model = SynthModel('llama-2-7b', n_layers=1, seed=0, device='cuda', with_head=False, init='device')
        inp = model.first_block_input(128, 512, bs=-1, seed=1, device='cuda')
        c = AttrDict.wrap(copy.deepcopy(cfg))
        algo = Awq(model, c.quant, inp, None, c)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        algo.run_block_loop()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rec(f'awq_block_llama2_7b_rep{rep}', dt * 1e3, layers_per_s=7 / dt)
        del algo, model, inp

if 'fp8' in only:
    # The block-FP8 linear forward (act_quant + gemm_fp8_block, csrc/fp8.cu + csrc/gemm_fp8.cu) next
    # to the dequant-once path (llmc_fp8_block_dequant + llmc_gemm_bf16) and, where this
    # torch / cuBLAS build takes it, torch._scaled_mm with 1 x 128 / 128 x 128 block scales.
    from llmc_b200.quant_float import act_quant, gemm_fp8_block, weight_cast_to_bf16, weight_cast_to_fp8
    shapes = [(1536, 7168), (18432, 7168), (7168, 18432), (2048, 7168), (7168, 2048),   # DeepSeek-V3
              (14336, 4096), (4096, 14336)]                                          # Llama-3-8B
    scaled_mm = None
    for M in (16384, 4096):
        for (N, K) in shapes:
            tag = f'{M}x{N}x{K}'
            x = torch.randn(M, K, device='cuda').bfloat16()
            w = (torch.randn(N, K, device='cuda') * 0.02).bfloat16()
            wq, ws = weight_cast_to_fp8(w, 128)
            xq, xs = act_quant(x)
            fl = 2.0 * M * N * K
            ms = timeit(lambda: act_quant(x))
            by = M * K * (2 + 1 + 4 / 128)
            rec(f'fp8_act_quant_{M}x{K}', ms, gbs=by / ms / 1e6, frac_hbm=by / ms / 1e6 / HBM)
            ms_g = timeit(lambda: gemm_fp8_block(xq, xs, wq, ws, torch.bfloat16), do_flush=False)
            rec(f'gemm_fp8_block_{tag}', ms_g, tflops=fl / ms_g / 1e9, frac_fp8=fl / ms_g / 1e9 / TF_FP8)
            ms_f = timeit(lambda: gemm_fp8_block(*act_quant(x), wq, ws, torch.bfloat16), do_flush=False)
            rec(f'fp8_forward_{tag}', ms_f, tflops=fl / ms_f / 1e9)
            wd = weight_cast_to_bf16(wq, ws, 128)
            ms_b = timeit(lambda: linear_forward(x, wd), do_flush=False)
            ms_d = timeit(lambda: weight_cast_to_bf16(wq, ws, 128))
            rec(f'dequant_once_bf16_gemm_{tag}', ms_b, tflops=fl / ms_b / 1e9, frac_bf16=fl / ms_b / 1e9 / TF,
                dequant_ms=round(ms_d, 4), fp8_forward_speedup=ms_b / ms_f)
            if scaled_mm is None or scaled_mm is True:
                try:
                    # 1 x 128 activation scales and 128 x 128 weight scales, both outer-dim-major
                    sa = xs.t().contiguous().t()
                    sb = ws.t().contiguous().t()
                    f = lambda: torch._scaled_mm(xq, wq.t(), scale_a=sa, scale_b=sb.t(),  # noqa: E731
                                                 out_dtype=torch.bfloat16)
                    f()
                    ms_s = timeit(f, do_flush=False)
                    rec(f'torch_scaled_mm_block_{tag}', ms_s, tflops=fl / ms_s / 1e9)
                    scaled_mm = True
                except Exception as e:                       # noqa: BLE001
                    scaled_mm = False
                    rec('torch_scaled_mm_block', 0.0, status='unsupported',
                        error=f'{type(e).__name__}: {str(e).splitlines()[0][:200]}')
            del x, w, wq, ws, xq, xs, wd

os.makedirs('gpurun_out', exist_ok=True)
json.dump(res, open('gpurun_out/microbench.json', 'w'), indent=1)

# ---- short, fixed-shape launches for `ncu --set full -k regex:<kernel>` captures -------------------
if 'prof' in only:
    x = torch.randn(32768, 4096, device='cuda').bfloat16()
    w = (torch.randn(4096, 4096, device='cuda') * 0.02).bfloat16()
    for _ in range(3):
        linear_forward(x, w)                                   # wgmma_gemm_kernel<false,true>
    H = torch.zeros(4096, 4096, device='cuda')
    for _ in range(3):
        ops.hessian_add_batch(H, 1, x.unsqueeze(0))            # wgmma_gemm_kernel<true,true> + finalize
    wq = (torch.randn(14336, 4096, device='cuda') * 0.02).bfloat16()
    q = IntegerQuantizer(4, False, 'per_group', group_size=128)
    for _ in range(3):
        q.real_quant_pack_vllm_dynamic(wq)                     # quant_dynamic_warp_kernel
        q.fake_quant_weight_dynamic(wq)
    Hs = torch.zeros(4096, 4096, device='cuda')
    ops.hessian_add_batch(Hs, 0, torch.randn(1, 8192, 4096, device='cuda').bfloat16())
    Hs += 0.01 * torch.diag(Hs).mean() * torch.eye(4096, device='cuda')
    for _ in range(2):
        ops.chol_inv_upper(Hs)                                 # tf32x3_wgmma_kernel, diag_kernel
    Wp, Hp = ops.prepare(w, Hs, None, 0.0)
    Hinv = ops.chol_inv_upper(Hp)
    ops.weight_transform(Wp, Hinv, 4, False, 128)              # gptq_inblock_kernel, tf32x3_wgmma_kernel
    torch.cuda.synchronize()

if 'cholq' in only:
    # Does the latency-bound Cholesky loop run slower behind a deep queue of tensor-core work
    # (the situation inside bench.py) than on an idle GPU (the situation in `gptq` above)?
    for C in (4096, 14336):
        Hs = torch.zeros(C, C, device='cuda')
        ops.hessian_add_batch(Hs, 0, torch.randn(1, 4096, C, device='cuda').bfloat16())
        Hs += 0.01 * torch.diag(Hs).mean() * torch.eye(C, device='cuda')
        x = torch.randn(32768, 4096, device='cuda').bfloat16()
        w = (torch.randn(4096, 4096, device='cuda') * 0.02).bfloat16()
        ops.chol_inv_upper(Hs)
        torch.cuda.synchronize()
        for label, pre in (('idle', 0), ('behind_60_gemms', 60)):
            ts = []
            for _ in range(3):
                for _ in range(pre):
                    linear_forward(x, w)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                ops.chol_inv_upper(Hs)
                e.record()
                torch.cuda.synchronize()
                ts.append(round(s.elapsed_time(e), 3))
            print(f'cholq C={C} {label}: {ts}', flush=True)

if 'prof2' in only:
    # one Cholesky-inverse + one column sweep at C = 4096, for a per-launch ncu list of the two
    # latency-bound host loops (csrc/chol.cu, csrc/gptq.cu)
    w = (torch.randn(4096, 4096, device='cuda') * 0.02).bfloat16()
    Hs = torch.zeros(4096, 4096, device='cuda')
    ops.hessian_add_batch(Hs, 0, torch.randn(1, 8192, 4096, device='cuda').bfloat16())
    Hs += 0.01 * torch.diag(Hs).mean() * torch.eye(4096, device='cuda')
    Wp, Hp = ops.prepare(w, Hs, None, 0.0)
    Hinv = ops.chol_inv_upper(Hp)
    ops.weight_transform(Wp, Hinv, 4, False, 128)
    torch.cuda.synchronize()
