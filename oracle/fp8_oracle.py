"""ORACLE (test infrastructure only) — FloatQuantizer with use_qtorch (quant.py:963-1229).

*** PARITY UNPINNED ***  The rounding step of the reference is `qtorch.quant.float_quantize`
(third-party, unpinned in requirements/runtime.txt:29, not vendored, not installed here, no
network), and the reference holds no test or golden vector at that boundary.  It is restated as
`x.float().to(torch.float8_e4m3fn / float8_e5m2).float()` — IEEE round-to-nearest-even with
subnormals, identical to any correct nearest rounding for |x| <= finfo.max (which holds for
weights because scale = absmax / finfo.max).  torch's cast gives NaN above 448 (e4m3) and inf above
61440 (e5m2) where the kernels saturate, so the value is clamped to +-finfo.max first.  Everything
else follows the cited lines, including the object flow: quant() sets zero scales to 1 in the
caller's tensor, and dequant and the real-quant export use those scales.
"""
import torch

FP8 = {'e4m3': torch.float8_e4m3fn, 'e5m2': torch.float8_e5m2}


def float_quantize(x, bit):
    fi = torch.finfo(FP8[bit])
    return x.float().clamp(fi.min, fi.max).to(FP8[bit]).float()


def qparams(t, bit, granularity):
    """quant.py:132-143 + 545-553 (symmetric, qmax = finfo.max as a 0-dim fp32 tensor)."""
    qmax = torch.tensor(torch.finfo(FP8[bit]).max)
    if granularity == 'per_tensor':
        mn, mx = torch.min(t), torch.max(t)
    else:
        mn, mx = t.amin(dim=-1, keepdim=True), t.amax(dim=-1, keepdim=True)
    abs_max = torch.max(mx.abs(), mn.abs()).clamp(min=1e-5)
    return abs_max / qmax


def quant(t, scales, bit, zeros=None):
    """quant.py:1061-1072: `scales[scales == 0] = 1` IN PLACE on the caller's tensor (:1062), then
    float_quantize(tensor / scales + zeros) -> fp32 grid values.  The division follows torch's
    promotion: a 0-dim scale keeps the tensor's dtype T, scales with dimensions of another dtype
    promote the quotient to fp32."""
    scales[scales == 0] = 1
    zeros = torch.tensor(0.0) if zeros is None else zeros
    return float_quantize((t / scales + zeros).float(), bit)


def dequant(q, scales, zeros=None):
    """quant.py:1074-1076: (q - zeros) * scales, fp32 for fp32 grid values."""
    return (q - (torch.tensor(0.0) if zeros is None else zeros)) * scales


def quant_dequant(t, scales, bit):
    """quant.py:1078-1081 -> fp32 (dequant sees the scales quant() changed)."""
    return dequant(quant(t, scales, bit), scales)


def reshape(w, granularity, group_size=None, head_num=None):
    """quant.py:612-642 for the row-wise granularities."""
    if granularity == 'per_group' and w.shape[-1] >= group_size:
        return w.reshape(-1, group_size)
    if granularity == 'per_head':
        return w.reshape(head_num, -1)
    return w


def fake_quant_dynamic(w, bit, granularity, group_size=None, head_num=None):
    """quant.py:1142-1159 -> (w's dtype and shape, the scales get_qparams returned, after quant())."""
    t = reshape(w, granularity, group_size, head_num)
    s = qparams(t, bit, granularity)
    y = quant_dequant(t, s, bit)
    return y.reshape(w.shape).to(w.dtype), s


def real_quant_dynamic(w, bit, granularity, group_size=None, head_num=None):
    """quant.py:1195-1221 -> (fp8 weight, scales): the scales are the ones quant() changed."""
    t = reshape(w, granularity, group_size, head_num)
    s = qparams(t, bit, granularity)
    q = quant(t, s, bit).reshape(w.shape).to(FP8[bit])
    return q, (s.view(1) if granularity == 'per_tensor' else s.view(w.shape[0], -1))


def fake_quant_static(w, scales, bit, granularity, group_size=None, head_num=None):
    """quant.py:1083-1098 / 1111-1140 (scales: the caller's args['scales'], changed in place)."""
    t = reshape(w, granularity, group_size, head_num)
    return quant_dequant(t, scales, bit).reshape(w.shape).to(w.dtype)


def real_quant_static(w, scales, bit, granularity, group_size=None, head_num=None):
    """quant.py:1161-1193 -> (fp8 weight, scales viewed as the reference exports them)."""
    t = reshape(w, granularity, group_size, head_num)
    q = quant(t, scales, bit).reshape(w.shape).to(FP8[bit])
    return q, (scales.view(1) if granularity == 'per_tensor' else scales.view(w.shape[0], -1))


def _block_view(w, bs):
    M, N = w.shape
    pm, pn = -(-M // bs) * bs, -(-N // bs) * bs
    padded = torch.zeros((pm, pn), dtype=w.dtype)
    padded[:M, :N] = w
    return padded.view(-1, bs, pn // bs, bs)


def block_qparams(t, bit):
    """quant.py:137-139 + 545-553 on the [Mb, bs, Nb, bs] view: fp32 scales [Mb, 1, Nb, 1]."""
    qmax = torch.tensor(torch.finfo(FP8[bit]).max)
    mx = t.abs().float().amax(dim=(1, 3), keepdim=True)
    mn = t.abs().float().amin(dim=(1, 3), keepdim=True)
    return torch.max(mx.abs(), mn.abs()).clamp(min=1e-5) / qmax


def block_quant(w, bit='e4m3', block_size=128):
    """weight_cast_to_fp8 (quant.py:32-43) = FloatQuantizer(per_block).real_quant_weight_dynamic:
    zero-padded [Mb, bs, Nb, bs] view (:633-642), abs().float() amax over dims (1, 3) (:137-139),
    scale = amax.clamp(min=1e-5) / finfo.max in fp32, q = float_quantize(x / scale)."""
    M, N = w.shape
    t = _block_view(w, block_size)
    s = block_qparams(t, bit)
    q = quant(t, s, bit)
    q2 = q.reshape(t.shape[0] * block_size, -1)[:M, :N]
    return q2.to(FP8[bit]), s.view(s.shape[0], s.shape[2])


def block_fake_quant(w, bit, block_size):
    """FloatQuantizer(per_block).fake_quant_weight_dynamic: the fp32 quotient and product of the
    block path, cast back to w's dtype; the padding is cut off (the reference's restore_tensor
    reshapes the padded view, which keeps the layout only when N is a multiple of the block)."""
    M, N = w.shape
    t = _block_view(w, block_size)
    s = block_qparams(t, bit)
    y = quant_dequant(t, s, bit)
    return y.reshape(t.shape[0] * block_size, -1)[:M, :N].to(w.dtype), s.view(s.shape[0], s.shape[2])


def block_dequant(w_fp8, scale, block_size=128):
    """weight_cast_to_bf16 (quant.py:18-29)."""
    M, N = w_fp8.shape
    bs = block_size
    sc = scale.repeat_interleave(bs, 0)[:M].repeat_interleave(bs, 1)[:, :N]
    return ((w_fp8.float() - 0) * sc).to(torch.bfloat16)
