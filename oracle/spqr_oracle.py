"""ORACLE (test infrastructure only) — SpQR (llmc/compression/quantization/spqr.py:116-351).

A CPU restatement of the reference's layer_transform / weight_transform / get_group_qparams /
w_qdq in fp32 torch, vectorised over the weight rows (which are independent given Hinv and the
layer's outlier threshold) and with every sum over a group taken in ASCENDING INDEX ORDER — the
order llmc_b200/csrc/spqr_row.cuh uses, so that the CUDA kernel (and its host build) can be
compared with this file bit for bit.  torch's own `sum(-1)` over 15 / 16 contiguous floats
(spqr.py:186-190, 236-238) may associate differently; against the reference-generated goldens
(tests/golden/spqr_kat.pt, oracle/gen_spqr_golden.py) that shows up as rare flips of
`E > threshold` next to the threshold, which tests/test_oracle_golden.py bounds.

Pinned: tests/test_oracle_golden.py::test_spqr_oracle_matches_reference.
"""
import math

import torch

from .gptq_oracle import tf32_split


def qcfg(bit, sym, round_zp=True):
    """quant.py:661-678."""
    if sym:
        return dict(qmin=float(-(2 ** (bit - 1))), qmax=float(2 ** (bit - 1) - 1), sym=True, round_zp=round_zp)
    return dict(qmin=0.0, qmax=float(2 ** bit - 1), sym=False, round_zp=round_zp)


def qparams(mn, mx, c):
    """quant.py:545-559."""
    qmin, qmax = torch.tensor(c['qmin']), torch.tensor(c['qmax'])
    if c['sym']:
        am = torch.maximum(mx.abs(), mn.abs()).clamp(min=1e-5)
        return am / qmax, torch.zeros_like(am)
    s = (mx - mn).clamp(min=1e-5) / (qmax - qmin)
    if c['round_zp']:
        z = (qmin - torch.round(mn / s)).clamp(c['qmin'], c['qmax'])
    else:
        z = qmin - (mn / s)
    return s, z


def qdq(x, s, z, c):
    """quant.py:699-717."""
    if c['round_zp']:
        q = torch.clamp(torch.round(x / s) + z, c['qmin'], c['qmax'])
    else:
        q = torch.clamp(torch.round(x / s.clamp_min(1e-9) + z), c['qmin'], c['qmax'])
    return (q - z) * s


def second_level(v, c):
    """spqr.py:337-351: the [R, 1] scale / zero tensor through a per_group quantizer whose
    reshape_tensor leaves it [R, 1] (quant.py:612-632) — statistics of one value per row."""
    s, z = qparams(v, v, c)
    return qdq(v, s, z, c)


def _seq_sum(t):
    """Sum over the last dim in ascending index order (see the module docstring)."""
    acc = torch.zeros(t.shape[:-1], dtype=t.dtype)
    for k in range(t.shape[-1]):
        acc = acc + t[..., k]
    return acc


def group_qparams(G, hd, cfg):
    """spqr.py:174-192, 228-243, 326-351.  G [R, gs] current weights of the group, hd [gs] the
    matching diag(Hinv).  Returns the second-level quantised (scale, zero), each [R]."""
    R, gs = G.shape
    if not cfg['outliers']:
        newG = G
    else:
        loo = cfg['loo']
        s, z = qparams(G.amin(1), G.amax(1), loo)
        base = _seq_sum(((qdq(G, s[:, None], z[:, None], loo) - G) / hd) ** 2)
        M = torch.zeros_like(G)
        for j in range(gs):
            keep = [k for k in range(gs) if k != j]
            Gj = G[:, keep]
            s, z = qparams(Gj.amin(1), Gj.amax(1), loo)
            e = _seq_sum(((qdq(Gj, s[:, None], z[:, None], loo) - Gj) / hd[keep]) ** 2)
            M[:, j] = ((base - e) > cfg['thr']).float()
        mean = _seq_sum(G * (1 - M)) / _seq_sum(1 - M).clamp_min(1)
        newG = G * (1 - M) + mean[:, None] * M
    s, z = qparams(newG.amin(1), newG.amax(1), cfg['w'])
    return second_level(s, cfg['sc']), second_level(z, cfg['zc'])


def row_block(Wb, Hb, cfg):
    """One <= 128-column block, all rows (spqr.py:215-268 without the trailing update).
    Returns tmp [R, cnt], Err1 [R, cnt], mask [R, cnt] (uint8), scales / zeros [R, cnt / gs],
    losses [R]."""
    Wb = Wb.clone()
    R, cnt = Wb.shape
    gs = cfg['gs']
    err = torch.zeros_like(Wb)
    mask = torch.zeros((R, cnt), dtype=torch.uint8)
    S = torch.zeros((R, (cnt + gs - 1) // gs))
    Z = torch.zeros_like(S)
    loss = torch.zeros(R)
    hd = torch.diag(Hb)
    thr = torch.tensor(cfg['thr'], dtype=torch.float32)
    s = z = None
    for c in range(cnt):
        if c % gs == 0:
            s, z = group_qparams(Wb[:, c:c + gs], hd[c:c + gs], cfg)
            S[:, c // gs], Z[:, c // gs] = s, z
        w = Wb[:, c].clone()
        d = Hb[c, c]
        q = qdq(w, s, z, cfg['w'])
        e = (w - q) / d
        if cfg['has_thr']:
            m = (e * e) > thr
            mf = m.float()
            newq = q * (1 - mf) + w * mf
            e = (w - newq) / d
            mask[:, c] = m.to(torch.uint8)
        err[:, c] = e
        loss = loss + e * e
        if c + 1 < cnt:
            Wb[:, c + 1:] = Wb[:, c + 1:] - e[:, None] * Hb[c, c + 1:][None, :]
    return Wb, err, mask, S, Z, loss


def make_cfg(wkw, special, level2_scale, level2_zero, thr):
    w = qcfg(wkw['bit'], wkw['symmetric'], wkw.get('round_zp', True))
    has_thr = not math.isinf(thr)
    return dict(w=w, loo=qcfg(wkw['bit'], wkw['symmetric'], False),
                sc=qcfg(level2_scale['bit'], level2_scale['symmetric'], level2_scale.get('round_zp', True)),
                zc=qcfg(level2_zero['bit'], level2_zero['symmetric'], level2_zero.get('round_zp', True)),
                gs=wkw['group_size'], thr=float(thr), has_thr=has_thr,
                outliers=bool(has_thr and not special['simplified_outliers']))


def threshold_of(Wp, Hinv, relative_threshold):
    """spqr.py:194-195 (a Python float: the fp32 mean widened, times the relative threshold)."""
    rel = math.inf if relative_threshold == 'inf' else float(relative_threshold)
    outlier_scale = (Wp.var(dim=0) / torch.diag(Hinv).square()).mean().item()
    thr = rel * outlier_scale
    return float(torch.tensor(thr, dtype=torch.float32)) if not math.isinf(thr) else math.inf


def weight_transform(Wp, Hinv, cfg, blocksize=128, trailing_split=False):
    """spqr.py:172-268 on the permuted weight.  Returns tmp, mask (uint8), scales, zeros [R, ng],
    per-row losses.  trailing_split: the trailing update multiplies hi + lo of the tf32 split of
    the block's errors, as the 3xTF32 kernel does (gptq_oracle.tf32_split)."""
    W = Wp.clone()
    R, C = W.shape
    gs = cfg['gs']
    tmp = torch.zeros_like(W)
    mask = torch.zeros((R, C), dtype=torch.uint8)
    S = torch.zeros((R, C // gs))
    Z = torch.zeros_like(S)
    losses = torch.zeros(R)
    for i1 in range(0, C, blocksize):
        i2 = min(i1 + blocksize, C)
        t, e, m, s, z, l = row_block(W[:, i1:i2], Hinv[i1:i2, i1:i2], cfg)
        tmp[:, i1:i2], mask[:, i1:i2] = t, m
        S[:, i1 // gs:i1 // gs + s.shape[1]], Z[:, i1 // gs:i1 // gs + s.shape[1]] = s, z
        losses = losses + l
        if trailing_split:
            hi, lo = tf32_split(e)
            e = hi + lo
        W[:, i2:] -= e.matmul(Hinv[i1:i2, i2:])
    return tmp, mask, S, Z, losses


def layer_transform(W, H, wkw, special, level2_scale, level2_zero):
    """spqr.py:116-170: act-order, dead columns, damping, Cholesky triple, sweep, un-permute."""
    W = W.float().clone()
    H = H.clone()
    C = W.shape[1]
    perm = None
    if special['actorder']:
        perm = torch.argsort(torch.diag(H), descending=True)
        W = W[:, perm]
        H = H[perm][:, perm]
    dead = torch.diag(H) == 0
    if special['percdamp'] > 0:
        damp = special['percdamp'] * abs(torch.diag(H)).mean()
        idx = torch.arange(C)
        H[idx, idx] += damp
    H[dead, dead] = 1
    W[:, dead] = 0
    H = torch.linalg.cholesky(H)
    H = torch.cholesky_inverse(H)
    Hinv = torch.linalg.cholesky(H, upper=True)
    thr = threshold_of(W, Hinv, special['relative_threshold'])
    cfg = make_cfg(wkw, special, level2_scale, level2_zero, thr)
    tmp, mask, S, Z, losses = weight_transform(W, Hinv, cfg)
    out = dict(perm=perm, Wp=W, Hinv=Hinv, thr=thr, tmp_perm=tmp, mask_perm=mask, losses_rows=losses,
               buf_scales=S.reshape(-1, 1), buf_zeros=Z.reshape(-1, 1))
    if perm is not None:
        inv = torch.argsort(perm)
        tmp, mask = tmp[:, inv], mask[:, inv]
    out.update(new_weight=tmp, buf_mask=mask.float())
    return out


def w_qdq(new_weight, buf_scales, buf_zeros, buf_mask, perm, wkw, dtype):
    """spqr.py:363-386."""
    c = qcfg(wkw['bit'], wkw['symmetric'], wkw.get('round_zp', True))
    gs = wkw['group_size']
    out = (buf_mask * new_weight).to(dtype)
    w = new_weight[:, perm] if perm is not None else new_weight
    shape = w.shape
    y = qdq(w.reshape(-1, gs), buf_scales, buf_zeros, c).reshape(shape).to(new_weight.dtype).to(dtype)
    if perm is not None:
        y = y[:, torch.argsort(perm)]
    return (y * (1 - buf_mask) + out).to(dtype)
