"""Exact oracle of the weight-only real-quant forwards: the stored codes of the exported packed layouts
and the weight they dequantise to.

  AutoAWQ (AutoawqRealQuantLinear / MlcllmRealQuantLinear, gemm_pack): qweight [K, N/8] and qzeros
  [K/group, N/8] int32 packed along N, nibble i of word j = column 8j + AWQ_ORDER[i]; scales
  [K/group, N] fp16.  W[n, k] = rT(fp32(q - z) * fp32(s)), q and z the nibbles as stored.
  vLLM / SGLang (VllmRealQuantLinear, need_pack): weight_packed [N, ceil(K*bits/32)] int32, 32/bits
  unsigned codes per word along K, little end first, stored as code + 2^(bits-1); weight_scale
  [N, K/group] fp16.  W[n, k] = rT(fp32(stored - 2^(bits-1)) * fp32(s)).

The product of a small integer and an fp16 scale is exact in fp32, so the one rounding is to the
model dtype.  Plain torch integer ops, on whichever device the tensors are."""
import torch

AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)


def awq_nibbles(words):
    """int32 [R, C/8] AutoAWQ words -> int32 [R, C] codes as stored: column 8j + AWQ_ORDER[i] is
    nibble i of word j."""
    R, W = words.shape
    out = torch.empty((R, W, 8), dtype=torch.int32, device=words.device)
    for i, col in enumerate(AWQ_ORDER):
        out[:, :, col] = (words >> (4 * i)) & 0xF
    return out.reshape(R, W * 8)


def awq_dequant(qweight, scales, qzeros, group, dtype):
    """The [N, K] weight of an AutoAWQ export."""
    q = awq_nibbles(qweight)                                   # [K, N]
    g = torch.arange(q.shape[0], device=q.device) // group
    z = awq_nibbles(qzeros)[g]                                 # [K, N]
    s = scales.float()[g]
    return ((q - z).float() * s).to(dtype).t().contiguous()


def vllm_codes(packed, bits, K):
    """int32 [N, ceil(K*bits/32)] -> int32 [N, K] stored (unsigned) codes: element pf*w + e is field e
    of word w, pf = 32 / bits."""
    pf = 32 // bits
    mask = (1 << bits) - 1
    N, W = packed.shape
    out = torch.empty((N, W, pf), dtype=torch.int32, device=packed.device)
    for e in range(pf):
        out[:, :, e] = (packed >> (bits * e)) & mask
    return out.reshape(N, W * pf)[:, :K]


def vllm_dequant(packed, scales, bits, K, dtype):
    """The [N, K] weight of a vLLM / SGLang packed export (symmetric: zero = 2^(bits-1))."""
    codes = vllm_codes(packed, bits, K) - (1 << (bits - 1))
    group = K // scales.shape[1]
    g = torch.arange(K, device=packed.device) // group
    return (codes.float() * scales.float()[:, g]).to(dtype)
