"""ORACLE (test infrastructure only) — CPU restatement of llmc's GPTQ layer math.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this.  Pinned by tests/golden/gptq_*.pt (oracle/gen_golden.py runs the reference's
GPTQ methods on CPU).  Citations: /root/reference/llmc/compression/quantization/gptq.py.
"""
import math

import torch

from . import quant_oracle as qo


def hessian_add_batch(H, nsamples, inp, chunk_num=1):
    """gptq.py:253-295 (one add_batch call, world_size 1).

    inp [bs, S, C] (or [S, C]) in the model dtype.  Returns (H, nsamples).
    """
    if inp.dim() == 2:
        inp = inp.unsqueeze(0)
    b = inp.shape[0]
    x = inp.reshape(-1, inp.shape[-1]).t()                 # [C, T]
    H = H * (nsamples / (nsamples + b))
    nsamples += b
    for chunk in torch.chunk(x, chunk_num, dim=1):
        chunk = math.sqrt(2 / nsamples) * chunk.float()
        H = H + chunk.matmul(chunk.t())
    return H, nsamples


def hessian(batches, C, chunk_num=1):
    H, n = torch.zeros(C, C), 0
    for inp in batches:
        H, n = hessian_add_batch(H, n, inp, chunk_num)
    return H, n


def prepare(W, H, actorder, percdamp):
    """gptq.py:58-64, 128-176: dead columns, act-order permutation, damping, Cholesky triple.

    Returns (Wp fp32 [R, C] permuted, Hinv_U, perm or None).  H is not modified.
    """
    W = W.clone().float()
    H = H.clone()
    C = H.shape[0]
    perm = torch.argsort(torch.diag(H), descending=True) if actorder else None
    dead = torch.diag(H) == 0
    H[dead, dead] = 1
    W[:, dead] = 0
    if perm is not None:
        W = W[:, perm]
        H = H[perm][:, perm]
    damp = percdamp * torch.mean(torch.diag(H))
    idx = torch.arange(C)
    H[idx, idx] += damp
    H = torch.linalg.cholesky(H)
    H = torch.cholesky_inverse(H)
    H = torch.linalg.cholesky(H, upper=True)
    return W, H, perm


def tf32_split(x):
    """hi = tf32(x), lo = tf32(x - hi) of an fp32 tensor, each rounded like cvt.rna.tf32.f32
    (nearest, ties away from zero, to 10 mantissa bits): on the int32 view, add 0x1000 to the
    magnitude and clear the low 13 bits.  This is the split the library's 3xTF32 updates
    multiply (llmc_b200/csrc/tf32.cu)."""
    def rna(v):
        return ((v.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)
    hi = rna(x)
    return hi, rna(x - hi)


def weight_transform(W, Hinv, bit, sym, granularity, group_size=None, blocksize=128,
                     static_qparams=None, perm=None, trailing_split=False):
    """gptq.py:198-244.  W [R, C] fp32 (permuted), Hinv upper factor.

    dynamic groups (static_qparams None, per_group): qparams searched on the compensated
      columns [idx, idx+g) when idx % g == 0 (:215-223, search_column_qparams :358-366);
    static groups / per_channel: static_qparams = (scales, zeros) each a list over groups of
      [R,1] tensors (per_group, indexed perm[idx] // g, :225-227) or a single [R,1] pair.
    trailing_split: the trailing update multiplies hi + lo of tf32_split(Err1) instead of Err1,
      as the 3xTF32 kernel does.  The default is the reference's arithmetic.
    Returns (tmp [R,C], Losses [R,C], groups list of (scale, zero)).
    """
    W = W.clone()
    R, C = W.shape
    qmin, qmax = qo.int_range(bit, sym)
    tmp = torch.zeros_like(W)
    Losses = torch.zeros_like(W)
    groups = {}
    per_group = granularity == 'per_group'
    cur = None
    if not per_group:
        cur = static_qparams
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
                        cols = W[:, idx:min(idx + group_size, C)]
                        _, s, z, _, _ = qo.tensor_qparams(cols, bit, sym, 'per_group', group_size)
                        cur = (s, z)
                        groups[idx // group_size] = cur
                else:
                    gi = (perm[idx] if perm is not None else idx) // group_size
                    cur = (static_qparams[0][int(gi)], static_qparams[1][int(gi)])
            s, z = cur
            q = qo.dequant(qo.quant(w.unsqueeze(1), s, z, qmax, qmin), s, z).squeeze(1)
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


def merged_group_qparams(groups):
    """gptq.py:343-356, 397-409: buf_scales / buf_zeros [R*ng, 1] in PERMUTED column order."""
    scales = torch.stack([g[0] for g in groups], dim=1).reshape(-1, 1)
    zeros = torch.stack([g[1] for g in groups], dim=1).reshape(-1, 1)
    return scales, zeros


def w_qdq(weight, buf_scales, buf_zeros, bit, sym, group_size, perm, invperm, model_dtype):
    """gptq.py:424-452 with need_perm: W[:, perm] -> static qdq -> model dtype -> [:, invperm]."""
    qmin, qmax = qo.int_range(bit, sym)
    w = weight[:, perm] if perm is not None else weight
    w = qo.fake_quant_static(w, buf_scales, buf_zeros, qmax, qmin, 'per_group', group_size)
    w = w.to(model_dtype)
    return w[:, invperm] if perm is not None else w
