"""ORACLE (test infrastructure only) — the block-forward glue (llmc_b200/csrc/block_ops.cu) and
GPTQ's prepare gathers (llmc_gptq_prepare, csrc/gptq.cu) restated in the kernels' own order.

Each function spells out the kernel's fp32 operations and its roundings to the tensor dtype T
(`_rT`).  Everything here is elementwise IEEE arithmetic (plus float64 where it is exact), so it
gives the same bits on any device torch runs it on: the GPU tests evaluate the largest cases on
the GPU, the CPU tests pin the functions against the torch expressions the kernels replace.

Not restated: `rsqrtf` (RMSNorm's reciprocal square root, within 2 ulp on the device; `rmsnorm`
takes the fp32 `inv` as an argument) and `expf` (SiLU; the CPU's and the GPU's differ, so SiLU is
checked against torch's own CUDA `F.silu`).  The AutoAWQ packer's oracle is
`quant_oracle.pack_awq`, pinned to the reference's golden.
"""
import torch

THREADS = 256          # every kernel here runs 256-thread CTAs
WARPS = THREADS // 32


def _rT(x32, dtype):
    """Round an fp32 tensor to `dtype` and widen it back (exact)."""
    return x32.to(dtype).float() if dtype != torch.float32 else x32


def fma32(a64, b64, c32):
    """fp32 fmaf(a, b, c) for fp32-representable a, b: a*b is exact in float64 (≤ 48-bit
    significands, no float64 underflow), the sum is rounded to odd in float64 and then to fp32,
    which is a single correct rounding because float64 carries more than 24 + 1 bits.  The TwoSum
    error's sign says which way an inexact sum was rounded; it can lie far below the sum's ulp
    (an fp32 subnormal c beside a product near 1), so it picks the direction, not its size."""
    p = a64 * b64
    c = c32.double()
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                     # TwoSum: p + c = s + err exactly
    odd = (s.view(torch.int64) & 1) == 1
    fix = (err != 0) & ~odd & torch.isfinite(s)
    s = torch.where(fix, torch.nextafter(s, torch.full_like(s, torch.inf).copysign(err)), s)
    return s.float()


def _butterfly(v):
    """warp_sum (common.cuh): xor shuffles 16, 8, 4, 2, 1 over the last dim of 32 lanes; lane 0's
    result.  Adds are commutative, so lane l and lane l^o hold the same bits after each step."""
    for o in (16, 8, 4, 2, 1):
        v = v[..., :o] + v[..., o:2 * o]
    return v[..., 0]


def rmsnorm_sumsq(x):
    """rmsnorm_kernel's sum of squares of each row of x [rows, cols] (cols % 8 == 0) as fp32:
    thread t folds its 8-wide chunks t, t+256, ... in element order with fmaf(v, v, acc), each warp
    reduces with warp_sum, warp 0 reduces the 8 warp sums (padded to 32 lanes with zeros)."""
    rows, cols = x.shape
    chunks = cols // 8
    it = -(-chunks // THREADS)
    xp = torch.zeros(rows, it * THREADS * 8, dtype=torch.float64, device=x.device)
    xp[:, :cols] = x.double()
    xp = xp.view(rows, it, THREADS, 8)
    acc = torch.zeros(rows, THREADS, dtype=torch.float32, device=x.device)
    for i in range(it):
        for k in range(8):
            v = xp[:, i, :, k]
            acc = fma32(v, v, acc)
    warp = _butterfly(acc.view(rows, WARPS, 32))
    lanes = torch.zeros(rows, 32, dtype=torch.float32, device=x.device)
    lanes[:, :WARPS] = warp
    return _butterfly(lanes)


def _div32(a, n):
    """fp32 a / n correctly rounded (the kernels' IEEE division).  torch divides a CUDA tensor by a
    Python scalar through the scalar's reciprocal, so the quotient is taken in float64, between
    tensors, and rounded once more: exact, as float64 carries more than 2 * 24 + 1 bits."""
    a64 = a.double()
    return (a64 / torch.full_like(a64, float(n))).float()


def rmsnorm_mean_eps(sumsq, cols, eps):
    """The argument of rsqrtf: sumsq / cols (IEEE division) + eps, in fp32."""
    eps32 = torch.tensor(eps, dtype=torch.float32, device=sumsq.device)
    return _div32(sumsq, cols) + eps32


def rmsnorm_inv_candidates(sumsq, cols, eps, ulps=2):
    """[rows, 2*ulps+1] fp32 values around the correctly rounded 1/sqrt(mean + eps) (computed in
    float64 from the fp32 argument), offsets -ulps..ulps; column `ulps` is the correctly rounded
    value.  An infinite argument gives 0 (rsqrt(inf)), as torch's fallback does."""
    m = rmsnorm_mean_eps(sumsq, cols, eps).double()
    c = (1.0 / torch.sqrt(m)).float()
    cols_ = [c]
    lo = hi = c
    inf = torch.tensor(float('inf'), device=c.device)
    for _ in range(ulps):
        lo = torch.nextafter(lo, -inf)
        hi = torch.nextafter(hi, inf)
        cols_ = [lo] + cols_ + [hi]
    return torch.stack(cols_, dim=-1)


def rmsnorm(x, w, inv):
    """The kernel's output for x [rows, cols] and a per-row fp32 inv [rows]: T(w * T(x * inv)),
    each product one fp32 multiply.  With w in another dtype (the module fallback) the product
    is promoted as torch promotes it."""
    T = x.dtype
    y = _rT(x.float() * inv.float()[:, None], T)
    out = torch.result_type(w, x.to(T))
    return _rT(w.float()[None, :] * y, out).to(out)


def rope(x, cos, sin, heads, head_dim):
    """rope_kernel on x [B, S, heads*head_dim] with cos / sin [S, head_dim]: for the pair
    (a, b) = (x_i, x_{i+D/2}),  T(T(a*c1) + T((-b)*s1))  and  T(T(b*c2) + T(a*s2)).  cos / sin
    may be wider than x (torch promotes), which the module fallback does."""
    B, S, _ = x.shape
    T = torch.result_type(x, cos)
    h = head_dim // 2
    q = x.float().view(B, S, heads, head_dim)
    c = cos.float()[None, :, None, :]
    s = sin.float()[None, :, None, :]
    a, b = q[..., :h], q[..., h:]
    oa = _rT(_rT(a * c[..., :h], T) + _rT((-b) * s[..., :h], T), T)
    ob = _rT(_rT(b * c[..., h:], T) + _rT(a * s[..., h:], T), T)
    return torch.cat((oa, ob), dim=-1).reshape(B, S, heads * head_dim).to(T)


def add(a, b):
    """add_kernel: T(a + b) in fp32."""
    return (a.float() + b.float()).to(a.dtype)


def diag_mean(H, percdamp):
    """diag_mean_kernel: percdamp * (sum / C) over diag(H) with zeros replaced by 1, summed as
    one CTA does it — thread t adds d[t], d[t+256], ... in order, warp_sum, then warp 0's
    warp_sum of the 8 warp sums."""
    C = H.shape[0]
    d = torch.diagonal(H).float()
    d = torch.where(d == 0, torch.ones_like(d), d)
    it = -(-C // THREADS)
    dp = torch.zeros(it * THREADS, dtype=torch.float32, device=H.device)
    dp[:C] = d
    dp = dp.view(it, THREADS)
    acc = torch.zeros(THREADS, dtype=torch.float32, device=H.device)
    for i in range(it):
        acc = acc + dp[i]
    lanes = torch.zeros(32, dtype=torch.float32, device=H.device)
    lanes[:WARPS] = _butterfly(acc.view(WARPS, 32))
    v = _butterfly(lanes)
    p = torch.tensor(percdamp, dtype=torch.float32, device=H.device)
    return p * _div32(v, C)


def prepare(W, H, perm, percdamp):
    """llmc_gptq_prepare -> (Wp fp32 [R, C] or None, Hp fp32 [C, C]).

    Wp[:, j] = W[:, perm[j]] in fp32, or 0 where H's ORIGINAL diagonal at perm[j] is 0 (a dead
    column); Hp = H[perm][:, perm] with its diagonal's zeros replaced by 1 and the damping added
    (gptq.py:58-64, 128-171)."""
    C = H.shape[0]
    p = torch.arange(C, device=H.device) if perm is None else perm.to(H.device).long()
    dead = torch.diagonal(H) == 0
    Wp = None
    if W is not None:
        Wp = W.float()[:, p].clone()
        Wp[:, dead[p]] = 0
    Hp = H[p][:, p].clone()
    dg = torch.diagonal(Hp)
    dg.copy_(torch.where(dg == 0, torch.ones_like(dg), dg) + diag_mean(H, percdamp))
    return Wp, Hp
