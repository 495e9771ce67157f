"""GPTQ layer math on the CUDA kernels — the tensor-level pieces of
llmc/compression/quantization/gptq.py (add_batch :253-295, process_hessian_and_weights
:128-176, weight_transform :198-244) behind small functions; llmc_b200/gptq.py wires them into
the reference's class / hook structure.
"""
import math

import torch

from ._lib import F32, call, dtype_enum, load, ptr, require_cuda, stream_ptr
from .prof import TIMER

_ws_cache = {}
_FP8_GRIDS = {'e4m3': 0, 'e5m2': 1}      # FloatQuantizer.bit -> the e5m2 flag of llmc_gptq_colblock_fp8


def _workspace(nbytes, device, tag):
    """Grow-only scratch buffers (split-K slabs, Err1) keyed by (device, tag)."""
    key = (device, tag)
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def free_workspaces():
    _ws_cache.clear()


@torch.no_grad()
def hessian_add_batch(H, nsamples, inp):
    """gptq.py:253-290 for nn.Linear inputs.  H [C,C] fp32 updated in place:
    H <- H*n/(n+b) + 2/(n+b) * X^T X with X = inp.reshape(-1, C); returns the new nsamples.
    One wgmma SYRK launch (csrc/gemm.cu) instead of an fp32 SGEMM on X.float()."""
    require_cuda(H, inp)
    if inp.dim() == 2:
        inp = inp.unsqueeze(0)
    b = inp.shape[0]
    x = inp.reshape(-1, inp.shape[-1])
    if not x.is_contiguous():
        x = x.contiguous()
    T, C = x.shape
    assert H.shape == (C, C) and H.dtype == torch.float32 and H.is_contiguous()
    nbytes = load().llmc_syrk_workspace_bytes(T, C)
    ws = _workspace(nbytes, x.device, 'syrk')
    # algorithmic flops: C(C+1)/2 unique entries x 2T (DESIGN.md); bytes: X once + H in/out
    with TIMER.span('syrk', flops=float(T) * C * (C + 1), nbytes=2.0 * T * C + 8.0 * C * C):
        call('llmc_syrk_accum', ptr(x), T, C, dtype_enum(x.dtype), ptr(H), float(nsamples),
             float(b), ptr(ws), ws.numel(), stream_ptr(x.device))
    return nsamples + b


@torch.no_grad()
def prepare(W, H, perm, percdamp, want_h=True, wp_out=None):
    """gptq.py:128-171 minus the Cholesky: returns (Wp fp32 [R,C], Hp fp32 [C,C]).
    W None: only Hp.  want_h False: only Wp (Hp returned as None).  wp_out: a contiguous fp32
    [R, C] destination (a row slice of a shared buffer, see GPTQ._transform_fused)."""
    require_cuda(W, H)
    C = H.shape[0]
    dev = H.device
    Wp, R, wdt = None, 0, F32
    if W is not None:
        W = W.contiguous()
        R = W.shape[0]
        wdt = dtype_enum(W.dtype)
        Wp = wp_out if wp_out is not None else torch.empty((R, C), dtype=torch.float32, device=dev)
        assert Wp.shape == (R, C) and Wp.dtype == torch.float32 and Wp.is_contiguous()
    Hp = torch.empty((C, C), dtype=torch.float32, device=dev) if want_h else None
    scratch = torch.empty(4, dtype=torch.float32, device=dev)
    p = perm.to(torch.int64).contiguous() if perm is not None else None
    nb = (8.0 * C * C if want_h else 0.0) + ((W.element_size() + 4.0) * R * C if W is not None else 0.0)
    with TIMER.span('gptq_prepare', nbytes=nb):
        call('llmc_gptq_prepare', ptr(H), C, ptr(p), float(percdamp), ptr(Hp), ptr(W), R,
             wdt, ptr(Wp), ptr(scratch), stream_ptr(dev))
    return Wp, Hp


@torch.no_grad()
def chol_inv_upper(Hp, backend='b200', inplace=False, return_info=False):
    """gptq.py:172-174: U = cholesky(cholesky_inverse(cholesky(Hp)), upper=True).

    backend 'b200' (default): csrc/chol.cu — one reverse-ordered blocked factorisation + one
    blocked triangular inverse, all O(C^3) work as 3xTF32 rank-128 updates on tensor cores.
    backend 'cusolver': the reference's three library calls, kept only so tests can compare the
    two (never used by the algorithms).
    return_info: also return the device int32[1] status flag (0 = positive-definite, k = the
    leading minor of order k is not); the caller owns checking it (GPTQ.check_factorizations)."""
    C = Hp.shape[0]
    if backend == 'cusolver':
        with TIMER.span('cholesky_triple(cusolver)', flops=4.0 / 3.0 * C ** 3):
            L = torch.linalg.cholesky(Hp)
            Hinv = torch.cholesky_inverse(L)
            U = torch.linalg.cholesky(Hinv, upper=True).contiguous()
            return (U, torch.zeros(1, dtype=torch.int32, device=Hp.device)) if return_info else U
    require_cuda(Hp)
    assert Hp.dtype == torch.float32 and Hp.shape == (C, C)
    A = Hp if (inplace and Hp.is_contiguous()) else Hp.contiguous().clone()
    nbytes = load().llmc_chol_workspace_bytes(C)
    ws = _workspace(nbytes, A.device, 'chol')
    info = torch.empty(1, dtype=torch.int32, device=A.device)
    with TIMER.span(f'chol_inv_upper[{C}]', flops=2.0 / 3.0 * C ** 3, nbytes=16.0 * C ** 3 / (6 * 128)):
        call('llmc_chol_inv_upper', ptr(A), C, ptr(ws), ws.numel(), ptr(info), stream_ptr(A.device))
    return (A, info) if return_info else A


@torch.no_grad()
def weight_transform(Wp, Hinv, bit, sym, group, static_qparams=None, gmap=None, out_perm=None):
    """gptq.py:198-244 (+ :186-193 when out_perm is given).

    Wp [R,C] fp32 permuted weights (consumed as scratch), Hinv [C,C] upper factor.
    bit: an integer width (IntegerQuantizer, llmc_gptq_colblock), or 'e4m3' / 'e5m2'
      (FloatQuantizer with use_qtorch, llmc_gptq_colblock_fp8: symmetric, no zeros).
    group: group size, or C for per_channel.
    static_qparams: None -> dynamic groups (qparams searched while sweeping, returned fp32
      [R, ng] in permuted column order); else (scales [R*ng], zeros|None) inputs.
    gmap: int32 [C], static groups with act-order: group of permuted column idx (perm[idx]//g).
    out_perm: int64 [C]; tmp is scattered back to the original column order
      (tmp_out[:, out_perm[i]] = tmp[:, i]  ==  tmp[:, invperm]).
    Returns (tmp [R,C] fp32, losses [R] fp32, scales, zeros).
    """
    require_cuda(Wp, Hinv)
    Wp = Wp if Wp.is_contiguous() else Wp.contiguous()
    Hinv = Hinv if Hinv.is_contiguous() else Hinv.contiguous()   # cholesky(upper=True) is a .mH view
    assert Wp.dtype == torch.float32 and Hinv.dtype == torch.float32
    R, C = Wp.shape
    ng = C // group
    dev = Wp.device
    fp8 = bit in _FP8_GRIDS
    if fp8:
        sym = True                      # FloatQuantizer is symmetric (quant.py:966)
    tmp = torch.empty_like(Wp)
    losses = torch.empty(R, dtype=torch.float32, device=dev)
    if static_qparams is None:
        scales = torch.empty((R, ng), dtype=torch.float32, device=dev)
        zeros = None if sym else torch.empty((R, ng), dtype=torch.float32, device=dev)
        qdt, static = F32, 0
    else:
        scales, zeros = static_qparams
        scales = scales.contiguous()
        zeros = None if (sym or zeros is None) else zeros.to(scales.dtype).contiguous()
        qdt, static = dtype_enum(scales.dtype), 1
    nbytes = load().llmc_gptq_workspace_bytes(R, C)
    ws = _workspace(nbytes, dev, 'gptq_err')
    op = out_perm.to(torch.int64).contiguous() if out_perm is not None else None
    flops, nbytes = float(R) * C * C + float(R) * C * 128, 8.0 * R * C + 2.0 * C * C
    if fp8:
        with TIMER.span(f'gptq_colblock_fp8[{R}x{C}]', flops=flops, nbytes=nbytes):
            call('llmc_gptq_colblock_fp8', ptr(Wp), ptr(Hinv), R, C, int(group), _FP8_GRIDS[bit],
                 static, ptr(gmap), ptr(scales), qdt, ptr(tmp), ptr(op), ptr(losses), ptr(ws),
                 ws.numel(), stream_ptr(dev))
        return tmp, losses, scales, None
    with TIMER.span(f'gptq_colblock[{R}x{C}]', flops=flops, nbytes=nbytes):
        call('llmc_gptq_colblock', ptr(Wp), ptr(Hinv), R, C, int(group), int(bit),
             int(bool(sym)), static, ptr(gmap), ptr(scales), ptr(zeros), qdt, ptr(tmp), ptr(op),
             ptr(losses), ptr(ws), ws.numel(), stream_ptr(dev))
    return tmp, losses, scales, zeros


@torch.no_grad()
def spqr_threshold(Wp, Hinv, relative_threshold):
    """spqr.py:194-195 as a DEVICE fp32 scalar (no host read): relative_threshold *
    mean(var(W, dim=0) / diag(Hinv)^2), the product taken in double like the reference's Python
    float arithmetic and rounded to fp32 where the reference's comparisons round it."""
    rel = math.inf if relative_threshold == 'inf' else float(relative_threshold)
    if math.isinf(rel):
        return torch.full((1,), math.inf, dtype=torch.float32, device=Wp.device)
    outlier_scale = (Wp.var(dim=0) / torch.diag(Hinv).square()).mean()
    return (outlier_scale.double() * rel).float().reshape(1)


@torch.no_grad()
def spqr_transform(Wp, Hinv, wcfg, scale_cfg, zero_cfg, threshold, simplified_outliers, out_perm=None):
    """spqr.py:172-268 (+ :163-165 when out_perm is given) on the permuted fp32 weight.

    wcfg / scale_cfg / zero_cfg: (bit, symmetric, round_zp) of the weight quantizer and of
    special.scale / special.zero; wcfg carries the group size as a fourth element.
    threshold: device fp32 scalar from spqr_threshold.
    Returns (tmp [R,C] fp32, mask [R,C] uint8, losses [R], scales [R,ng], zeros [R,ng])."""
    require_cuda(Wp, Hinv, threshold)
    Wp = Wp if Wp.is_contiguous() else Wp.contiguous()
    Hinv = Hinv if Hinv.is_contiguous() else Hinv.contiguous()
    assert Wp.dtype == torch.float32 and Hinv.dtype == torch.float32 and threshold.dtype == torch.float32
    R, C = Wp.shape
    bit, sym, rzp, group = wcfg
    ng = C // group
    dev = Wp.device
    tmp = torch.empty_like(Wp)
    mask = torch.empty((R, C), dtype=torch.uint8, device=dev)
    losses = torch.empty(R, dtype=torch.float32, device=dev)
    scales = torch.empty((R, ng), dtype=torch.float32, device=dev)
    zeros = torch.empty((R, ng), dtype=torch.float32, device=dev)
    nbytes = load().llmc_gptq_workspace_bytes(R, C)
    ws = _workspace(nbytes, dev, 'gptq_err')
    op = out_perm.to(torch.int64).contiguous() if out_perm is not None else None
    with TIMER.span(f'spqr_colblock[{R}x{C}]', flops=float(R) * C * C + float(R) * C * 128,
                    nbytes=9.0 * R * C + 2.0 * C * C):
        call('llmc_spqr_colblock', ptr(Wp), ptr(Hinv), R, C, int(group), int(bit), int(bool(sym)),
             int(bool(rzp)), int(scale_cfg[0]), int(bool(scale_cfg[1])), int(bool(scale_cfg[2])),
             int(zero_cfg[0]), int(bool(zero_cfg[1])), int(bool(zero_cfg[2])), ptr(threshold),
             int(bool(simplified_outliers)), ptr(scales), ptr(zeros), ptr(tmp), ptr(mask), ptr(op),
             ptr(losses), ptr(ws), ws.numel(), stream_ptr(dev))
    return tmp, mask, losses, scales, zeros
