"""ORACLE (test infrastructure only) — CPU restatement of llmc's integer quantizer and packers.

This file is the checker, never the product: only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import it.  llmc_b200/ must not.

Why torch-on-CPU rather than numpy/C: the reference's arithmetic IS torch eager arithmetic on
fp16/bf16/fp32 tensors — every elementwise op is evaluated in fp32 and rounded once to the
tensor dtype (SURVEY.md Appendix A.1).  numpy has no bfloat16, so the only faithful CPU
restatement of those rounding points is the same torch ops on CPU tensors; integer packing
is restated in numpy.

Pinned by tests/golden/*.pt, which oracle/gen_golden.py produced by running the reference's
own code (/root/reference, imported read-only) on CPU; tests/test_oracle_golden.py checks
every function here against them.

Each function cites the reference lines (relative to /root/reference/llmc/compression/
quantization/) it restates.
"""
import math

import numpy as np
import torch


def int_range(bit, sym, qrange=None):
    """quant.py:665-677 -> (qmin, qmax) as 0-dim tensors with the reference's dtypes.  `qrange`
    is the quantizer's `int_range: [qmin, qmax]` option (quant.py:665-666)."""
    if qrange is not None:
        return torch.tensor(qrange[0]), torch.tensor(qrange[1])
    if sym:
        return torch.tensor(-(2 ** (bit - 1))), torch.tensor(2 ** (bit - 1) - 1)
    return torch.tensor(0.0), torch.tensor(2 ** bit - 1)


def group_view(w, granularity, group_size=None):
    """quant.py:612-642 (reshape_tensor) for per_group / per_channel / per_tensor."""
    if granularity == 'per_group' and w.shape[-1] >= group_size:
        if w.shape[-1] % group_size:
            raise ValueError(f'Dimension {w.shape[-1]} not divisible by group size {group_size}')
        return w.reshape(-1, group_size)
    return w


def minmax(t, granularity):
    """quant.py:132-143."""
    if granularity == 'per_tensor':
        return torch.min(t), torch.max(t)
    return t.amin(dim=-1, keepdim=True), t.amax(dim=-1, keepdim=True)


def qparams(min_val, max_val, bit, sym, round_zp=True, qrange=None):
    """quant.py:545-559 (qmin / qmax moved to the device of the range, :547-548)."""
    qmin, qmax = (t.to(min_val.device) for t in int_range(bit, sym, qrange))
    if sym:
        abs_max = torch.max(max_val.abs(), min_val.abs()).clamp(min=1e-5)
        return abs_max / qmax, torch.tensor(0.0), qmax, qmin
    scales = (max_val - min_val).clamp(min=1e-5) / (qmax - qmin)
    zeros = (qmin - torch.round(min_val / scales)).clamp(qmin, qmax)
    if not round_zp:
        zeros = qmin - (min_val / scales)
    return scales, zeros, qmax, qmin


def quant(t, scales, zeros, qmax, qmin, round_zp=True):
    """quant.py:699-708; round_zp=False adds the real-valued zero-point before the rounding."""
    if not round_zp:
        return torch.clamp(torch.round(t / scales.clamp_min(1e-9) + zeros), qmin, qmax)
    return torch.clamp(torch.round(t / scales) + zeros, qmin, qmax)


def dequant(q, scales, zeros):
    """quant.py:710-712."""
    return (q - zeros) * scales


def tensor_qparams(w, bit, sym, granularity, group_size=None, qrange=None):
    """quant.py:690-697 -> (grouped view, scales, zeros, qmax, qmin)."""
    t = group_view(w, granularity, group_size)
    mn, mx = minmax(t, granularity)
    s, z, qmax, qmin = qparams(mn, mx, bit, sym, qrange=qrange)
    return t, s, z, qmax, qmin


def fake_quant_dynamic(w, bit, sym, granularity, group_size=None, qrange=None):
    """quant.py:833-869 (no int_indices / dim / current_bit)."""
    t, s, z, qmax, qmin = tensor_qparams(w, bit, sym, granularity, group_size, qrange)
    y = dequant(quant(t, s, z, qmax, qmin), s, z)
    return y.reshape(w.shape).to(w.dtype)


def fake_quant_static(w, scales, zeros, qmax, qmin, granularity, group_size=None):
    """quant.py:785-831."""
    t = group_view(w, granularity, group_size)
    y = dequant(quant(t, scales, zeros, qmax, qmin), scales, zeros)
    return y.reshape(w.shape).to(w.dtype)


def quant_static_gmap(w, scales, zeros, gmap, qmax, qmin, round_zp=True):
    """Static qparams [R, ng] applied through a column -> group map (gptq.py:424-452: act-order
    quantises W[:, perm] group by group, so column c of W uses group invperm[c] // group_size).
    -> (codes, dequantised values), both in the promoted dtype of w and the qparams."""
    s = scales[:, gmap]
    z = zeros[:, gmap] if torch.is_tensor(zeros) and zeros.dim() else zeros
    q = quant(w, s, z, qmax, qmin, round_zp)
    return q, dequant(q, s, z)


def code_dtype(bit, sym):
    """quant.py:890-896."""
    if bit == 8:
        return torch.int8 if sym else torch.uint8
    return torch.int32


def real_quant_dynamic(w, bit, sym, granularity, group_size=None, qrange=None):
    """quant.py:916-953 -> (codes, scales [R, ng] | [1], zeros | None)."""
    t, s, z, qmax, qmin = tensor_qparams(w, bit, sym, granularity, group_size, qrange)
    codes = quant(t, s, z, qmax, qmin).reshape(w.shape).to(code_dtype(bit, sym))
    shape = 1 if granularity == 'per_tensor' else (w.shape[0], -1)
    zeros = None if sym else z.to(code_dtype(bit, sym)).view(shape)
    return codes, s.view(shape), zeros


def real_quant_static(w, scales, zeros, qmax, qmin, bit, sym, granularity, group_size=None):
    """quant.py:871-914."""
    t = group_view(w, granularity, group_size)
    codes = quant(t, scales, zeros, qmax, qmin).reshape(w.shape).to(code_dtype(bit, sym))
    shape = 1 if granularity == 'per_tensor' else (w.shape[0], -1)
    z = None if sym else zeros.to(code_dtype(bit, sym)).view(shape)
    return codes, scales.view(shape), z


def pack_vllm(codes, scales, bit):
    """module_utils.py:836-862 (VllmRealQuantLinear.pack): codes + 2^(bit-1) -> uint8 ->
    32/bit codes per int32 along the input dim, little-end first, zero padded."""
    offset = pow(2, bit) // 2
    u = (codes + offset).to(torch.uint8).numpy().astype(np.uint32)
    pf = 32 // bit
    ncols = math.ceil(u.shape[1] / pf)
    u = np.pad(u, [(0, 0), (0, ncols * pf - u.shape[1])], constant_values=0)
    packed = np.zeros((u.shape[0], ncols), dtype=np.uint32)
    for i in range(pf):
        packed |= u[:, i::pf] << np.uint32(bit * i)
    return torch.from_numpy(packed.view(np.int32).copy()), scales.to(torch.float16)


AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)


def pack_awq(weight, scales, zeros, group_size, bit=4):
    """module_utils.py:1004-1065 (AutoawqRealQuantLinear.gemm_pack), vectorised over columns.

    weight [R, C] model dtype; scales [R, ng]; zeros [R, ng] int32.
    -> qweight [C, R/8] int32, scales [ng, R] fp16, qzeros [ng, R/8] int32.
    """
    assert bit == 4 and scales is not None and zeros is not None
    s = scales.t().contiguous().to(torch.float16)          # [ng, R]
    z = zeros.t().contiguous()                             # [ng, R] int32
    sz = z * s                                             # fp16
    R, C = weight.shape
    g = torch.arange(C) // group_size
    # (W[:, c] + sz[g(c)]) / s[g(c)], promoted exactly like the per-column loop (:1022-1029)
    iw = torch.round((weight + sz[g].t()) / s[g].t()).to(torch.int)   # [R, C]
    iw = iw.t().contiguous().numpy().astype(np.int32)                 # [C, R]
    qweight = np.zeros((C, R // 32 * bit), dtype=np.int32)
    zz = z.numpy().astype(np.int32)
    qzeros = np.zeros((zz.shape[0], R // 32 * bit), dtype=np.int32)
    for i, o in enumerate(AWQ_ORDER):
        qweight |= iw[:, o::8] << (i * bit)
        qzeros |= zz[:, o::8] << (i * bit)
    return torch.from_numpy(qweight), s, torch.from_numpy(qzeros)


# ---- granularities beyond per_group / per_channel / per_tensor (quant.py:612-658) -----------------
def reshape_tensor(w, granularity, group_size=None, head_num=None, block_size=None):
    if granularity == 'per_head':
        return w.reshape(head_num, -1)
    if granularity == 'per_block':
        m, n = w.shape
        bs = block_size
        pm, pn = -(-m // bs) * bs, -(-n // bs) * bs
        padded = torch.zeros((pm, pn), dtype=w.dtype)
        padded[:m, :n] = w
        return padded.view(-1, bs, pn // bs, bs)
    return group_view(w, granularity, group_size)


def restore_tensor(t, shape, granularity):
    if t.shape == shape:
        return t
    if granularity == 'per_block':
        return t.reshape(-1, t.shape[2] * t.shape[3])[:shape[0], :shape[1]]
    return t.reshape(shape)


def fake_quant_dynamic_any(w, bit, sym, granularity, **kw):
    """quant.py:833-869 for per_head (reshape(head_num, -1), row-wise range) and per_block
    (128x128 tiles, abs range over dims (1, 3) computed in fp32, :137-139)."""
    t = reshape_tensor(w, granularity, **kw)
    if granularity == 'per_block':
        mn = t.abs().float().amin(dim=(1, 3), keepdim=True)
        mx = t.abs().float().amax(dim=(1, 3), keepdim=True)
    else:
        mn, mx = t.amin(dim=-1, keepdim=True), t.amax(dim=-1, keepdim=True)
    s, z, qmax, qmin = qparams(mn, mx, bit, sym)
    y = dequant(quant(t, s, z, qmax, qmin), s, z)
    return restore_tensor(y, w.shape, granularity).to(w.dtype), s, z


# ---- calib_algo: mse (quant.py:145-203) -------------------------------------------------------------
def mse_range(t, bit, sym, mse_grid=100, maxshrink=0.8, norm=2.4):
    """t: reshaped [groups, g] tensor.  The reference writes `best_min_val, best_max_val = _min_val,
    _max_val` (:165): the best range ALIASES the running range, so `best_min_val[tmp] = xmin[tmp]`
    also changes the base that later shrink levels multiply — kept as is."""
    t = t.float()
    mn, mx = t.amin(dim=-1, keepdim=True), t.amax(dim=-1, keepdim=True)
    best = torch.full([t.shape[0]], float('inf'))
    for i in range(int(maxshrink * mse_grid)):
        p = 1 - i / mse_grid
        xmin, xmax = p * mn, p * mx
        s, z, qmax, qmin = qparams(xmin, xmax, bit, sym)
        q = dequant(quant(t, s, z, qmax, qmin), s, z)
        q -= t
        q.abs_()
        q.pow_(norm)
        err = torch.sum(q, 1)
        better = err < best
        if torch.any(better):
            best[better] = err[better]
            mn[better] = xmin[better]          # in place: the aliasing
            mx[better] = xmax[better]
    return mn, mx


def fake_quant_mse(w, bit, sym, granularity, group_size=None):
    """fake_quant_weight_dynamic with calib_algo 'mse': fp32 qparams on a model-dtype tensor
    (type promotion makes the quantise-dequantise fp32), cast back at the end (:852-867)."""
    t = group_view(w, granularity, group_size)
    mn, mx = mse_range(t, bit, sym)
    s, z, qmax, qmin = qparams(mn, mx, bit, sym)
    y = dequant(quant(t, s, z, qmax, qmin), s, z)
    return y.reshape(w.shape).to(w.dtype), s, z, mn, mx


# ---- static histogram observer (quant.py:265-522) -----------------------------------------------------
def _hist_error(hist, min_val, max_val, first, last, bins, dst_nbins):
    """get_quantization_error (:279-330) + get_norm (:265-277)."""
    bin_width = (max_val.item() - min_val.item()) / bins
    dst_w = bin_width * (last - first + 1) / dst_nbins
    if dst_w == 0.0:
        return 0.0
    src = torch.arange(bins)
    b0 = (src - first) * bin_width
    b1 = b0 + bin_width
    d0 = torch.clamp(torch.div(b0, dst_w, rounding_mode='floor'), 0, dst_nbins - 1)
    d0c = (d0 + 0.5) * dst_w
    d1 = torch.clamp(torch.div(b1, dst_w, rounding_mode='floor'), 0, dst_nbins - 1)
    density = hist / bin_width

    def gn(a, b):
        return density * ((b * b * b - a * a * a) / 3)
    norm = torch.zeros(bins)
    norm += gn(b0 - d0c, torch.ones(bins) * (dst_w / 2))
    norm += (d1 - d0 - 1) * gn(torch.tensor(-dst_w / 2), torch.tensor(dst_w / 2))
    d1c = d1 * dst_w + dst_w / 2
    norm += gn(torch.tensor(-dst_w / 2), b1 - d1c)
    return norm.sum().item()


def hist_threshold(hist, min_val, max_val, bins, dst_nbins):
    """get_hist_threshold (:403-460)."""
    bin_width = (max_val - min_val) / bins
    total = torch.sum(hist).item()
    csum = torch.cumsum(hist, dim=0)
    step, alpha, beta = 1e-8, 0.0, 1.0
    first, last, best = 0, bins - 1, float('inf')
    while alpha < beta:
        na, nb = alpha + step, beta - step
        lo, hi = first, last
        while lo < last and csum[lo] < na * total:
            lo += 1
        while hi > first and csum[hi] > nb * total:
            hi -= 1
        nf, nl = first, last
        if (lo - first) > (last - hi):
            nf, alpha = lo, na
        else:
            nl, beta = hi, nb
        if nf == first and nl == last:
            continue
        e = _hist_error(hist, min_val, max_val, nf, nl, bins, dst_nbins)
        if e > best:
            break
        best, first, last = e, nf, nl
    return min_val + bin_width * first, min_val + bin_width * (last + 1)


def static_hist_range(tensors, bins=2048, dst_nbins=256, upsample=16):
    """get_static_hist_range (:462-522) for ONE hooked input given as a list of per-sample tensors."""
    lo = hi = None
    hist = torch.zeros(bins)
    for x in tensors:
        x = x.float()
        x_min, x_max = torch.min(x), torch.max(x)
        if lo is None:
            hist = torch.histc(x, bins, min=x_min.item(), max=x_max.item())
            lo, hi = x_min, x_max
            continue
        n_min, n_max = torch.min(lo, x_min), torch.max(hi, x_max)
        upd = torch.histc(x, bins, min=n_min.item(), max=n_max.item())
        if n_min == lo and n_max == hi:
            hist = hist + upd
        elif lo == hi:
            hist = torch.histc(lo, bins=bins, min=n_min, max=n_max) * torch.sum(upd) + upd
        else:                                                    # _upscale_histogram (:332-366)
            fine = hist.repeat_interleave(upsample) / upsample
            size = (hi - lo) / (bins * upsample)
            mids = torch.linspace(lo, hi, bins * upsample + 1)[:-1] + 0.5 * size
            edges = torch.linspace(n_min, n_max, bins + 1)
            idx = torch.bucketize(mids, edges, right=True) - 1
            idx[idx >= bins] = bins - 1
            idx[idx < 0] = 0
            hist = upd + torch.bincount(idx, weights=fine, minlength=bins)
        lo, hi = n_min, n_max
    return hist_threshold(hist, lo, hi, bins, dst_nbins)
