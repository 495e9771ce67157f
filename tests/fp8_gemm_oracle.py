"""ORACLE (test infrastructure only) — the reference's block-FP8 linear forward, restated on the CPU:
act_quant and fp8_gemm (llmc/compression/quantization/kernel.py:7-53, 153-242) and
block_wise_fp8_forward_func (module_utils.py:40-45).

  * act_quant: s = max|x| / 448 and y = e4m3(x / s) per contiguous group of 128, with IEEE
    division.  The reference's compiled kernel (and csrc/fp8.cu) divides with the approximate
    div.full.f32 (<= 2 ulp), so a GPU scale may differ from this one by up to 2 ulp.  The max is
    the reference's compiled `max.f32`, which returns the other operand when one is NaN: a NaN
    element does not reach the scale unless its whole group is NaN.  +-inf gives s = inf, so the
    group's finite elements quantise to +-0 and its infinite ones to NaN; an all-zero group gives
    s = 0 and NaN codes.
  * fp8_gemm: per 128-deep K block, ascending, d = the dot of exact products rounded once to fp32
    (NaN wherever the block's row of a or column of b holds a NaN code, as on the tensor core),
    then acc = fma(fp32(d * a_s[m]), b_s[n / 128], acc), one correctly rounded fp32 fma.  The
    Hopper tensor core's reduced-precision dot is not modelled: on operands whose 128-deep dots
    are exact (w8a8_oracle.fp8_exact_operands) the kernel must match this bit for bit.
  * fp8_gemm_exact: the same sum in float64 without intermediate rounding, plus the per-element
    magnitude sum_k |a_s a_k b_s b_k| that error bounds scale with.
"""
import torch

from oracle.glue_oracle import fma32

FMAX = 448.0

# the order fp8_gemm promotes in, and three others that must give different bits when the
# promotion rounds (the sanity check of a test that claims to pin the order)
PROMOTIONS = ('a_s-then-b_s', 'b_s-then-a_s', 'a_s*b_s-fused', 'k-descending')


def act_quant(x, block_size=128):
    """-> (e4m3 codes of x's shape, fp32 scales [*x.shape[:-1], K / block_size])."""
    K = x.shape[-1]
    assert K % block_size == 0
    xs = x.float().reshape(*x.shape[:-1], K // block_size, block_size)
    ax = xs.abs()
    mx = ax.masked_fill(ax.isnan(), -1.0).amax(-1)                     # max.f32 skips NaN ...
    mx = torch.where(mx < 0, torch.nan, mx)                             # ... unless all are NaN
    s = mx / torch.tensor(FMAX)
    q = (xs / s[..., None]).clamp(-FMAX, FMAX).to(torch.float8_e4m3fn)   # satfinite; NaN stays NaN
    return q.reshape(x.shape), s


def _blocks(a, a_s, b, b_s):
    K = a.shape[-1]
    kb = K // 128
    A = a.float().double().reshape(-1, kb, 128)
    B = b.float().double().reshape(b.shape[0], kb, 128)
    sa = a_s.float().reshape(-1, kb)
    sb = b_s.float().repeat_interleave(128, 0)[:b.shape[0]]             # [N, kb]
    return A, B, sa, sb, kb


def _dot(Ak, Bk):
    """[M, 128] x [N, 128] e4m3 values (float64) -> fp32 [M, N]: exact in float64 (products are
    multiples of 2^-18 below 2^18), rounded once; NaN where either operand row holds a NaN."""
    d = (Ak.nan_to_num(0.0) @ Bk.nan_to_num(0.0).T).float()
    nan = Ak.isnan().any(-1)[:, None] | Bk.isnan().any(-1)[None, :]
    return d.masked_fill(nan, torch.nan)


def fp8_gemm(a, a_s, b, b_s, promotion='a_s-then-b_s'):
    """a [..., K], b [N, K] e4m3; a_s [..., K/128], b_s [ceil(N/128), K/128] -> fp32 [..., N].
    `promotion` other than the first of PROMOTIONS computes a wrong order on purpose."""
    assert promotion in PROMOTIONS, promotion
    A, B, sa, sb, kb = _blocks(a, a_s, b, b_s)
    acc = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float32, device=A.device)
    order = range(kb - 1, -1, -1) if promotion == 'k-descending' else range(kb)
    for k in order:
        d = _dot(A[:, k], B[:, k])
        s_m, s_n = sa[:, k:k + 1], sb[:, k][None, :]
        if promotion == 'b_s-then-a_s':
            acc = fma32((d * s_n).double(), s_m.double(), acc)
        elif promotion == 'a_s*b_s-fused':
            acc = fma32(d.double(), (s_m * s_n).double(), acc)
        else:
            acc = fma32((d * s_m).double(), s_n.double(), acc)             # mul.rn, then fma.rn
    return acc.reshape(*a.shape[:-1], b.shape[0])


def fp8_gemm_exact(a, a_s, b, b_s):
    """-> (float64 sum_kb dot_kb * a_s * b_s, float64 sum_k |a_s a_k b_s b_k|), both [..., N]."""
    A, B, sa, sb, kb = _blocks(a, a_s, b, b_s)
    out = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float64)
    mag = torch.zeros_like(out)
    for k in range(kb):
        w = sa[:, k:k + 1].double() * sb[:, k].double()
        out += (A[:, k] @ B[:, k].T) * w
        mag += (A[:, k].abs() @ B[:, k].abs().T) * w.abs()
    shape = (*a.shape[:-1], b.shape[0])
    return out.reshape(shape), mag.reshape(shape)


def bf16_plus_bias(acc, bias):
    """module_utils.py:42-44: y = acc.to(bf16); y += bias (fp32 sum, one rounding)."""
    y = acc.to(torch.bfloat16)
    if bias is not None:
        y = (y.float() + bias.float()).to(torch.bfloat16)
    return y


def block_wise_fp8_forward(x, w, w_scale, bias=None, block_size=128):
    xq, s = act_quant(x, block_size)
    return bf16_plus_bias(fp8_gemm(xq, s, w, w_scale), bias)


def block_wise_fp8_forward_exact(x, w, w_scale, bias=None, block_size=128):
    """The fp64 value of the same forward after the activation quantisation (no fp32 or bf16
    rounding), and its magnitude sum."""
    xq, s = act_quant(x, block_size)
    y, mag = fp8_gemm_exact(xq, s, w, w_scale)
    if bias is not None:
        y = y + bias.double()
    return y, mag
