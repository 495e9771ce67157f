"""GPU: parity at the BENCHMARK's own widths (VERDICT r1 item 1b).

bench.py's timed configuration runs C = K = 14336 (Llama-3-8B down_proj / intermediate size);
round 1 only tested SYRK / Cholesky / sweep up to C = 4096.  tests/golden/gptq_fullwidth_kat.pt
holds what the REFERENCE's GPTQ layer path produced on CPU for one 4096 x 14336 linear with
8 x 2048 calibration tokens (oracle/gen_fullwidth_golden.py); inputs are regenerated from the
same seeds here.  Bars: Hessian / Hinv <= 1e-3 relative (north_star), Losses.sum() <= 1e-3.
"""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
_cache = {}


def _setup(golden_dir):
    if 'k' in _cache:
        return _cache
    from oracle.gen_fullwidth_golden import make_inputs
    k = torch.load(os.path.join(golden_dir, 'gptq_fullwidth_kat.pt'), weights_only=False)
    W, batches = make_inputs(k['R'], k['C'], k['NB'], k['S'], k['seed'])
    _cache.update(k=k, W=W.cuda(), X=torch.cat(batches, 0).cuda())
    return _cache


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _note(key, val):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
    try:
        os.makedirs(out, exist_ok=True)
        p = os.path.join(out, 'fullwidth_parity_report.json')
        d = json.load(open(p)) if os.path.exists(p) else {}
        d[key] = val
        json.dump(d, open(p, 'w'), indent=1)
    except (OSError, ValueError):
        pass


def test_fullwidth_hessian_cholesky_sweep(golden_dir):
    from llmc_b200 import gptq_ops as ops
    from oracle.gen_fullwidth_golden import COLS, ROWS
    c = _setup(golden_dir)
    k, W, X = c['k'], c['W'], c['X']
    C = k['C']
    # G2: 8 add_batch calls of [1, 2048, 14336] (gptq.py:253-290) on the wgmma SYRK
    H = torch.zeros(C, C, device='cuda')
    n = 0
    for b in range(k['NB']):
        n = ops.hessian_add_batch(H, n, X[b:b + 1])
    r_diag = _rel(torch.diag(H), k['H_diag'])
    r_samp = float((H[ROWS, COLS].double().cpu() - k['H_sample'].double()).abs().max() / k['H_absmax'])
    assert r_diag <= 1e-3 and r_samp <= 1e-3, (r_diag, r_samp)
    assert torch.equal(H, H.t())
    # G3: act-order; equal up to near-ties of diag(H) (fp32 summation order)
    perm = torch.argsort(torch.diag(H), descending=True)
    same_perm = float((perm.cpu() == k['perm']).float().mean())
    d_ref = k['H_diag'][k['perm']]
    assert _rel(torch.diag(H)[perm], d_ref) <= 1e-3
    # chain the later stages from the REFERENCE's permutation so they are comparable element-wise
    perm = k['perm'].cuda()
    Wp, Hp = ops.prepare(W, H, perm, k['percdamp'])
    # G4: the Cholesky triple at C = 14336 (cuSOLVER/LAPACK potrf + potri + potrf in the reference)
    Hinv, info = ops.chol_inv_upper(Hp, return_info=True)
    assert int(info.item()) == 0
    r_hd = _rel(torch.diag(Hinv), k['Hinv']['diag'])
    r_hs = float((Hinv[ROWS, COLS].double().cpu() - k['Hinv']['sample'].double()).abs().max() / k['Hinv']['absmax'])
    r_h4 = float((Hinv[:4].double().cpu() - k['Hinv']['first_rows'].double()).abs().max() / k['Hinv']['absmax'])
    fro = float(Hinv.double().pow(2).sum().sqrt())
    assert max(r_hd, r_hs, r_h4) <= 1e-3, (r_hd, r_hs, r_h4)
    assert abs(fro - k['Hinv']['fro']) <= 1e-3 * k['Hinv']['fro']
    assert torch.equal(Hinv, torch.triu(Hinv))
    # G5: the column sweep over 112 blocks
    tmp, losses, scales, zeros = ops.weight_transform(Wp, Hinv, 4, False, 128)
    ls = float(losses.double().sum())
    r_loss = abs(ls - k['losses_sum']) / k['losses_sum']
    r_rows = _rel(losses, k['losses_rows'])
    tf = tmp[ROWS, :128].cpu()
    first_bad = float(((tf - k['tmp_first_block']).abs() > 1e-4 * k['tmp_absmax']).float().mean())
    ts = tmp[ROWS, COLS].cpu()
    samp_bad = float(((ts - k['tmp_sample']).abs() > 1e-2 * k['tmp_absmax']).float().mean())
    sc = scales[ROWS].cpu()
    r_sc = float(((sc - k['group_scales_rows']).abs() / k['group_scales_rows'].abs().clamp(min=1e-12)).median())
    z_same = float((zeros[ROWS].cpu() == k['group_zeros_rows']).float().mean())
    _note('gptq_4096x14336', dict(H_diag_rel=r_diag, H_sample_rel=r_samp, perm_same_frac=same_perm,
                                   Hinv_diag_rel=r_hd, Hinv_sample_rel=r_hs, Hinv_rows_rel=r_h4,
                                   losses_sum=ls, losses_sum_ref=k['losses_sum'], losses_sum_rel=r_loss,
                                   losses_rows_rel=r_rows, tmp_first_block_bad_frac=first_bad,
                                   tmp_sample_bad_frac=samp_bad, scales_median_rel=r_sc,
                                   zeros_same_frac=z_same))
    assert r_loss <= 1e-3, (ls, k['losses_sum'])
    assert r_rows <= 2e-2, r_rows
    assert first_bad <= 1e-3, first_bad            # first block: no cross-block reduction involved
    assert samp_bad <= 2e-2, samp_bad              # chaotic w.r.t. rounding flips: bounded fraction
    assert r_sc <= 1e-3 and z_same >= 0.97, (r_sc, z_same)


def test_fullwidth_gemm_k14336(golden_dir):
    """K6 / M1 at the widest contraction of the bench (down_proj: K = 14336), vs fp32 torch."""
    from llmc_b200.module_utils import linear_forward
    c = _setup(golden_dir)
    x = (c['X'][:2048].float() / c['X'][:2048].float().abs().amax(dim=0, keepdim=True).clamp(min=1e-3)).bfloat16()
    w = c['W']
    y = linear_forward(x, w).float()
    ref = x.float() @ w.float().t()
    err = float((y - ref).abs().max() / ref.abs().max())
    _note('gemm_2048x4096x14336', dict(max_rel_err=err))
    assert err <= 2 ** -8, err                     # one bf16 rounding of an fp32-accumulated sum


def test_fullwidth_syrk_k_matches_fp64_sample(golden_dir):
    """SYRK at C = 14336 against the definition (fp64 on a strided sample of entries)."""
    from llmc_b200 import gptq_ops as ops
    c = _setup(golden_dir)
    X = c['X'][:2].reshape(-1, c['X'].shape[-1])          # 4096 tokens
    C = X.shape[1]
    H = torch.zeros(C, C, device='cuda')
    ops.hessian_add_batch(H, 0, X.unsqueeze(0))
    idx = torch.arange(0, C, 89, device='cuda')
    Xs = X[:, idx].double()
    ref = 2.0 * (Xs.t() @ Xs)
    got = H[idx][:, idx].double()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err <= 1e-5, err
