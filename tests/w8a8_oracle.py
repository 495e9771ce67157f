"""CPU oracle of the W8A8 real-quant GEMM (llmc_gemm_w8a8_i8 / llmc_gemm_w8a8_fp8, include/llmc_b200.h
K7), written from the stated numerics:

    acc = sum_k qx[m, k] * qw[n, k]                                     exact
    y   = rT(fadd(fmul(fmul(fp32(acc), s_w[n]), s_x[m]), bias[n]))      fp32 ops, one rounding

The exact sum is taken as a float64 matmul.  That is exact whatever order or fusion the matmul uses,
because every product and partial sum is representable in float64:
  int8 codes   products are integers of magnitude <= 2^14, sums below 2^31 for K <= 131056;
  e4m3 values  products are multiples of 2^-18 of magnitude < 2^17.6, so sums of K <= 2^17 of them
               are multiples of 2^-18 below 2^35, within float64's 53 bits.
fp32(acc) is then one round-to-nearest-even conversion, and the fp32 multiplies and the add are
torch's elementwise CPU ops (IEEE, one rounding each, no contraction).
"""
import torch

E4M3 = torch.float8_e4m3fn


def exact_sum(qx, qw):
    """[M, K] x [N, K] codes (int8 or e4m3, any device) -> the exact sums [M, N] as float64 (CPU)."""
    return qx.cpu().double() @ qw.cpu().double().t()


def epilogue(acc, s_x, s_w, bias, dtype):
    """acc [M, N] (float64, exact), s_x [M] or [1], s_w [N] or [1] fp32, bias [N] or None -> [M, N]
    of `dtype`, in the stated order: fmul(fmul(fp32(acc), s_w), s_x), fadd bias, one rounding."""
    f = acc.to(torch.float32)
    v = f * s_w.cpu().float().reshape(1, -1)
    v = v * s_x.cpu().float().reshape(-1, 1)
    if bias is not None:
        v = v + bias.cpu().float().reshape(1, -1)
    return v.to(dtype)


def gemm_w8a8(qx, s_x, qw, s_w, bias, dtype):
    """The oracle of llmc_gemm_w8a8_i8 (exact for any inputs) and of llmc_gemm_w8a8_fp8 on inputs whose
    128-deep partial sums are exact at the tensor core's accumulator width."""
    return epilogue(exact_sum(qx, qw), s_x, s_w, bias, dtype)


def fp8_exact_operands(M, N, K, gen, device='cpu'):
    """e4m3 operands on which every partial sum of llmc_gemm_w8a8_fp8 is exact at any accumulator width
    of 7 significant bits or more: x in {0, +-1, +-2}, w in {0, +-1} with at most 32 nonzeros in each
    128-deep K block of a row.  Every product is an integer of magnitude <= 2, so every partial sum
    inside a block is an integer of magnitude <= 64, and the fp32 sum over blocks is an integer below
    2^24 for K < 2^18."""
    x = torch.randint(-2, 3, (M, K), generator=gen).float()
    w = torch.randint(0, 2, (N, K), generator=gen).float() * 2 - 1
    keep = torch.zeros(N, K, dtype=torch.bool)
    for k0 in range(0, K, 128):
        width = min(128, K - k0)
        idx = torch.rand(N, width, generator=gen).argsort(dim=1)[:, :min(32, width)]
        keep[:, k0:k0 + width].scatter_(1, idx, True)
    w = w * keep
    return x.to(E4M3).to(device), w.to(E4M3).to(device)


def fp8_finite_bytes(shape, gen, device='cpu'):
    """Uniformly random finite e4m3 values (every byte but the two NaNs)."""
    b = torch.randint(0, 254, shape, generator=gen)
    b = b + (b >= 0x7f).long()                        # skip 0x7f; 0xff is never drawn
    return b.to(torch.uint8).view(E4M3).to(device)


def fp8_bound(qx, s_x, qw, s_w, bias, dtype, tol=2.0 ** -8):
    """(y64, bound) for llmc_gemm_w8a8_fp8 on arbitrary inputs: y64 the float64 value of the stated
    formula on the exact sum, bound = ulp_dtype(|y64|) + tol * s_x s_w sum_k |qx qw|.  The first term
    covers the output rounding and the fp32 epilogue, the second the tensor core's reduced-precision
    adds inside each 128-deep block."""
    acc = exact_sum(qx, qw)
    mag = qx.cpu().double().abs() @ qw.cpu().double().abs().t()
    s = s_x.cpu().double().reshape(-1, 1) * s_w.cpu().double().reshape(1, -1)
    y64 = acc * s
    if bias is not None:
        y64 = y64 + bias.cpu().double().reshape(1, -1)
    mant = {torch.bfloat16: 8, torch.float16: 11}[dtype]
    ulp = torch.exp2(torch.floor(torch.log2(y64.abs().clamp(min=2.0 ** -24))) - (mant - 1))
    if dtype == torch.float16:
        ulp = ulp.clamp(min=2.0 ** -24)                # fp16 subnormal spacing
    return y64, ulp + tol * mag * s
