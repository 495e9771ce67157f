"""ORACLE (test infrastructure only) — CPU restatement of llmc's AWQ scale search and weight
auto-clip.  Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import it.

Pinned by tests/golden/awq_kat.pt (oracle/gen_golden.py runs the reference's Awq /
AutoClipper methods on CPU).  Citations: /root/reference/llmc/compression/quantization/awq.py,
auto_clip.py, base_blockwise_quantization.py.
"""
import torch

from . import quant_oracle as qo


def weight_scale(weights, granularity, group_size):
    """awq.py:48-72 (get_weight_scale): mean over rows of |W| / group-max, averaged over layers."""
    total = None
    for w in weights:
        w = w.clone()
        shape = w.shape
        r = qo.group_view(w, granularity, group_size)
        a = r.abs()
        mx = a.amax(dim=1, keepdim=True)
        ls = a.div_(mx).view(shape)
        total = ls.mean(0) if total is None else total.add_(ls.mean(0))
    return total.div_(len(weights))


def act_scale(x):
    """awq.py:74-85 with _bs == x.shape[0]."""
    return x.abs().view(-1, x.shape[-1]).mean(0)


def get_scales(x, w_max, ratio, version='v2'):
    """awq.py:87-108 (no GQA branch)."""
    xs = act_scale(x)
    if version == 'v1':
        s = (xs.pow(ratio) / w_max.pow(1 - ratio)).clamp(min=1e-4).view(-1)
    else:
        s = xs.pow(ratio).clamp(min=1e-4).view(-1)
    return s / (s.max() * s.min()).sqrt()


def fake_quantize_weight(w, scales, bit, sym, granularity, group_size):
    """awq.py:147-164: W.mul_(s.view(1,-1)) then dynamic fake quant (returns a new tensor)."""
    return qo.fake_quant_dynamic(w * scales.view(1, -1), bit, sym, granularity, group_size)


def loss(org_out, out):
    """awq.py:134-145 with a single batch."""
    return (org_out - out).float().pow(2).mean().item()


def search_scale(weights, x, forward, bit, sym, granularity, group_size, version='v2', n_grid=20):
    """awq.py:178-253 for one input batch, world size 1.

    weights: list of [R_i, C] tensors of the subset; forward(list_of_weights, x) -> module output.
    Returns (best_scales, losses[n_grid])."""
    w_max = weight_scale(weights, granularity, group_size)
    org_out = forward(weights, x)
    best_err, best_scales, losses = float('inf'), None, []
    for n in range(n_grid):
        ratio = n * 1 / n_grid
        s = get_scales(x, w_max, ratio, version)
        qws = [fake_quantize_weight(w, s, bit, sym, granularity, group_size) for w in weights]
        out = forward(qws, x / s.view(1, -1))
        l = loss(org_out, out)
        losses.append(l)
        if l < best_err:
            best_err, best_scales = l, s
    return best_scales, losses


def auto_clip_layer(w, x, bit, sym, granularity, group_size, clip_sym=True, n_grid=20,
                    max_shrink=0.5, n_sample_token=512):
    """auto_clip.py:83-191, clip_version v1, w_only, one input tensor.
    w [R, C]; x [..., C].  Returns (best_max [R, ng, 1], best_min [R, ng, 1])."""
    gs = group_size if granularity == 'per_group' else w.shape[1]
    w = w.reshape(w.shape[0], 1, -1, gs)
    ocb = 256 if w.shape[0] % 256 == 0 else 64     # blocking sizes memory only; the last block may be short
    x = x.view(-1, x.shape[-1])
    x = x.reshape(1, x.shape[0], -1, gs)
    step = max(1, x.shape[1] // n_sample_token)
    x = x[:, 0::step]
    best_max_all, best_min_all = [], []
    for ib in range(-(-w.shape[0] // ocb)):
        wb = w[ib * ocb:(ib + 1) * ocb]
        org_max = wb.abs().amax(dim=-1, keepdim=True) if clip_sym else wb.amax(dim=-1, keepdim=True)
        org_min = wb.amin(dim=-1, keepdim=True)
        best_max, best_min = org_max.clone(), org_min.clone()
        min_errs = torch.ones_like(org_max) * 1e9
        org_out = (x * wb).sum(dim=-1)
        for i_s in range(int(max_shrink * n_grid)):
            max_val = org_max * (1 - i_s / n_grid)
            min_val = -max_val if clip_sym else org_min * (1 - i_s / n_grid)
            cur_w = torch.clamp(wb, min_val, max_val)
            q_w = qo.fake_quant_dynamic(cur_w, bit, sym, granularity, group_size)
            cur_out = (x * q_w).sum(dim=-1)
            err = (cur_out - org_out).pow(2).mean(dim=1).view(min_errs.shape)
            better = err < min_errs
            min_errs[better] = err[better]
            best_max[better] = max_val[better]
            best_min[better] = min_val[better]
        best_max_all.append(best_max)
        best_min_all.append(best_min)
    return torch.cat(best_max_all, 0).squeeze(1), torch.cat(best_min_all, 0).squeeze(1)


def apply_clip(w, max_val, clip_sym=True, min_val=None):
    """auto_clip.py:193-211, v1."""
    shape = w.shape
    w = w.reshape(*max_val.shape[:2], -1)
    mn = -max_val if clip_sym else min_val
    return torch.clamp(w, mn, max_val).reshape(shape)
