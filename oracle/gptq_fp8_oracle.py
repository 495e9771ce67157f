"""ORACLE (test infrastructure only) — GPTQ's column sweep on an FP8 weight grid: gptq.py:198-244
with FloatQuantizer and `use_qtorch: True` (quant.py:1043-1081), the CPU counterpart of
llmc_gptq_colblock_fp8.

Same loop as gptq_oracle.weight_transform; what differs is the grid: symmetric, zero-point
tensor(0.0), scale = max(|max|, |min|).clamp(1e-5) / finfo.max, and the rounding of
fp8_oracle.float_quantize (PARITY UNPINNED w.r.t. qtorch, see fp8_oracle.py).  Pinned by
tests/golden/gptq_fp8_kat.pt (oracle/gen_gptq_fp8_golden.py runs the reference's own GPTQ).
"""
import torch

from . import fp8_oracle as fo
from .gptq_oracle import tf32_split


def unpack_upper(v, C):
    """[C, C] upper-triangular matrix from its upper triangle stored row by row (the fixture's
    layout of the Cholesky factor)."""
    i, j = torch.triu_indices(C, C)
    U = torch.zeros(C, C, dtype=v.dtype)
    U[i, j] = v
    return U


def qdq(w, s, bit):
    """quant.py:1061-1081 on a column: quant() sets zero scales to 1 IN PLACE (:1062), so dequant
    sees 1 as well; everything in fp32 (fp32 w / model-dtype s)."""
    s = s.clone()
    s[s == 0] = 1
    return ((fo.quant(w.unsqueeze(1), s, bit) - torch.tensor(0.0)) * s).squeeze(1)


def weight_transform(W, Hinv, bit, granularity, group_size=None, blocksize=128, static_qparams=None,
                     perm=None, trailing_split=False):
    """gptq.py:198-244 on the `bit` ('e4m3' / 'e5m2') grid.  W [R, C] fp32 (permuted), Hinv upper factor.

    dynamic groups (static_qparams None, per_group): scales searched on the compensated columns
      [idx, idx+g) when idx % g == 0 (:215-223), fp32;
    static groups / per_channel / per_tensor: static_qparams = scales, a list over groups of [R, 1]
      tensors (per_group, indexed perm[idx] // g, :225-227) or one tensor ([R, 1] or 0-dim).
    trailing_split: as gptq_oracle.weight_transform (the 3xTF32 kernel's split of Err1).
    Returns (tmp [R,C], Losses [R,C], list of the dynamic group scales [R, 1])."""
    W = W.clone()
    R, C = W.shape
    tmp = torch.zeros_like(W)
    Losses = torch.zeros_like(W)
    groups = {}
    per_group = granularity == 'per_group'
    s = None if per_group else static_qparams
    for i1 in range(0, C, blocksize):
        i2 = min(i1 + blocksize, C)
        W1 = W[:, i1:i2].clone()
        Hinv1 = Hinv[i1:i2, i1:i2]
        Err1 = torch.zeros_like(W1)
        for i in range(i2 - i1):
            w, d = W1[:, i], Hinv1[i, i]
            idx = i1 + i
            if per_group:
                if static_qparams is None:
                    if idx % group_size == 0:
                        s = fo.qparams(W[:, idx:min(idx + group_size, C)], bit, 'per_group')
                        groups[idx // group_size] = s
                else:
                    s = static_qparams[int((perm[idx] if perm is not None else idx) // group_size)]
            q = qdq(w, s, bit)
            tmp[:, idx] = w
            Losses[:, idx] = ((w - q) ** 2) / (2 * d ** 2)
            err1 = (w - q) / d
            W1[:, i:] -= err1.unsqueeze(1).matmul(Hinv1[i, i:].unsqueeze(0))
            Err1[:, i] = err1
        if trailing_split:
            hi, lo = tf32_split(Err1)
            Err1 = hi + lo
        W[:, i2:] -= Err1.matmul(Hinv[i1:i2, i2:])
    return tmp, Losses, [groups[k] for k in sorted(groups)]


def w_qdq(weight, buf_scales, bit, granularity, group_size, perm, invperm, model_dtype):
    """gptq.py:424-452: W[:, perm] -> FloatQuantizer.fake_quant_weight_static (quant.py:1111-1140)
    -> model dtype -> [:, invperm]."""
    w = weight[:, perm] if perm is not None else weight
    t = w.reshape(-1, group_size) if granularity == 'per_group' else w
    s = buf_scales.clone()
    s[s == 0] = 1
    t = (fo.quant(t, s, bit) - torch.tensor(0.0)) * s
    w = t.reshape(w.shape).to(w.dtype).to(model_dtype)
    return w[:, invperm] if perm is not None else w
