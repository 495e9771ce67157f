"""GPU: the block-forward glue (csrc/block_ops.cu), the AutoAWQ packer (csrc/pack_awq.cu) and GPTQ's
prepare gathers (llmc_gptq_prepare) bit for bit against the oracles (oracle/glue_oracle.py,
oracle/quant_oracle.pack_awq), on every grid-stride loop, tile edge, dtype and value edge.

RMSNorm's reciprocal square root is rsqrtf (2 ulp): each row must equal the oracle at one fp32
`inv` within 2 ulp of the correctly rounded value, everything else (the sum of squares in the
kernel's order, the products and roundings) is exact.  SiLU is compared with torch's own CUDA
`F.silu(g) * u` (expf cannot be restated on the CPU).  The oracles are elementwise IEEE
arithmetic, so the large cases evaluate them on the GPU."""
import collections
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import glue_oracle as glo
from oracle import quant_oracle as qo

pytestmark = pytest.mark.gpu

NUM_SMS = 132                              # kNumSMs, common.cuh
RMSNORM_BLOCKS = NUM_SMS * 16              # block_ops.cu:128  — rows per rmsnorm grid pass
ELTWISE_UNITS = NUM_SMS * 32 * 256         # block_ops.cu:143-144, 158-159, 172-173 (threads)
PACK_QPARAM_UNITS = NUM_SMS * 16 * 256     # pack_awq.cu:112-113
EINVAL = -1
DT16 = [torch.bfloat16, torch.float16]
DTYPES = DT16 + [torch.float32]
_INT = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}
INV_OFFSETS = collections.Counter()        # rsqrtf: ulp offsets from the correctly rounded inv


def _lib():
    from llmc_b200 import _lib
    return _lib.load()


def _launches():
    return int(_lib().llmc_b200_launch_count())


def _bits_equal(a, b):
    """Per element: the same bits, or both NaN (NaN payloads differ between torch and the kernels)."""
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    it = _INT[a.dtype]
    return (a.view(it) == b.view(it)) | (torch.isnan(a) & torch.isnan(b))


def _assert_bits(a, b, what=''):
    ok = _bits_equal(a, b)
    if not bool(ok.all()):
        i = int((~ok).nonzero()[0][0]) if ok.dim() == 1 else tuple((~ok).nonzero()[0].tolist())
        raise AssertionError(f'{what}: {int((~ok).sum())}/{ok.numel()} differ, first at {i}: '
                             f'{a[i].item()} vs {b[i].item()}')


def _specials(dtype):
    fi = torch.finfo(dtype)
    return torch.tensor([0.0, -0.0, fi.tiny, -fi.tiny, fi.tiny / 4, -fi.tiny / 8, fi.max, -fi.max,
                         float('inf'), float('-inf'), float('nan'), 1.0, -1.0], dtype=dtype)


# ---- RMSNorm ----------------------------------------------------------------------------------------
def _check_rmsnorm(x, w, eps, y=None):
    """y = block_ops.rmsnorm(x, w, eps) equals glue_oracle.rmsnorm at one inv within 2 ulp of the
    correctly rounded one, row by row.  Returns y."""
    from llmc_b200 import block_ops
    rows, cols = x.shape
    if y is None:
        y = block_ops.rmsnorm(x, w, eps)
    cand = glo.rmsnorm_inv_candidates(glo.rmsnorm_sumsq(x), cols, eps)
    ok = torch.stack([_bits_equal(glo.rmsnorm(x, w, cand[:, k]), y).all(-1) for k in range(5)], -1)
    bad = ~ok.any(-1)
    assert not bool(bad.any()), (f'{int(bad.sum())}/{rows} rows match no inv within 2 ulp; first row '
                                 f'{int(bad.nonzero()[0])}')
    # the matching offset nearest to the correctly rounded inv, per row
    dist = torch.tensor([2, 1, 0, 1, 2], device=x.device)
    signed = torch.tensor([-2, -1, 0, 1, 2], device=x.device)
    best = torch.where(ok, dist, 99).argmin(-1)
    INV_OFFSETS.update(signed[best].tolist())
    return y


@pytest.mark.parametrize('cols', [8, 2048, 4096, 5120, 8192])
@pytest.mark.parametrize('dtype', DTYPES)
def test_rmsnorm_rows_and_grid_stride(dtype, cols):
    """Rows 1 .. 3 grid passes + 5; copies of a row in different grid-stride passes give the same
    bits; a weight that is not all ones."""
    torch.manual_seed(cols)
    w = (1 + 0.25 * torch.randn(cols, device='cuda')).to(dtype)
    for i, rows in enumerate([1, RMSNORM_BLOCKS - 1, RMSNORM_BLOCKS, RMSNORM_BLOCKS + 1,
                              3 * RMSNORM_BLOCKS + 5]):
        eps = (1e-5, 1e-6)[i % 2]
        x = (torch.randn(rows, cols, device='cuda') * torch.exp(torch.randn(rows, 1, device='cuda'))).to(dtype)
        if rows > 3 * RMSNORM_BLOCKS:
            assert rows > 3 * RMSNORM_BLOCKS           # four passes of the row loop, the last ragged
            x[RMSNORM_BLOCKS:2 * RMSNORM_BLOCKS] = x[:RMSNORM_BLOCKS]
            x[3 * RMSNORM_BLOCKS:3 * RMSNORM_BLOCKS + 5] = x[:5]
        y = _check_rmsnorm(x, w, eps)
        if rows > 3 * RMSNORM_BLOCKS:
            _assert_bits(y[RMSNORM_BLOCKS:2 * RMSNORM_BLOCKS], y[:RMSNORM_BLOCKS], 'pass 2 vs pass 1')
            _assert_bits(y[3 * RMSNORM_BLOCKS:], y[:5], 'pass 4 vs pass 1')


def test_rmsnorm_production_shape_and_torch_parity():
    """8192 tokens x 4096 bf16 (a Llama-3-8B chunk): the oracle, and the fraction of elements that
    differ from torch's CUDA RMSNorm expression (LlamaRMSNorm; another summation order and rsqrt)."""
    torch.manual_seed(0)
    x = (torch.randn(8192, 4096, device='cuda') * 2).bfloat16()
    w = (1 + 0.1 * torch.randn(4096, device='cuda')).bfloat16()
    assert 8192 > 3 * RMSNORM_BLOCKS
    y = _check_rmsnorm(x, w, 1e-5)
    xf = x.float()
    ref = w * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5)).bfloat16()
    frac = float((y != ref).float().mean())
    print(f'\nrmsnorm vs torch CUDA RMSNorm, 8192x4096 bf16: {frac:.3e} of elements differ')
    assert frac < 0.02


@pytest.mark.parametrize('dtype', DTYPES)
def test_rmsnorm_edge_rows(dtype):
    fi = torch.finfo(dtype)
    cols = 4096
    torch.manual_seed(1)
    rows = torch.randn(8, cols, device='cuda').to(dtype)
    rows[0] = 0                                               # inv = rsqrt(eps), output +-0
    rows[1] = -0.0
    rows[2] = fi.max if dtype != torch.bfloat16 else 2.0 ** 70      # sum of squares overflows
    rows[2, ::3] *= -1
    rows[3] = fi.tiny / 4 * torch.randint(-3, 4, (cols,), device='cuda').to(dtype)   # subnormals
    rows[4, :] = fi.tiny
    rows[5, ::7] = fi.max                                     # a few maxima among random values
    w = (torch.randn(cols, device='cuda') * 3).to(dtype)
    w[::5] = -0.0
    for eps in (1e-5, 1e-6):
        y = _check_rmsnorm(rows, w, eps)
        assert bool((y[0] == 0).all() & (y[1] == 0).all())
    if dtype == torch.bfloat16:
        assert float(glo.rmsnorm_sumsq(rows[2:3])) == float('inf')
        assert bool((y[2] == 0).all())                         # inv = rsqrt(inf) = 0, as torch gives


# ---- RoPE -------------------------------------------------------------------------------------------
def _rope_check(B, S, heads, D, dtype, x=None):
    from llmc_b200 import block_ops
    from llmc_b200.synth import _rot_half, rope_cos_sin
    if x is None:
        x = (torch.randn(B, S, heads * D, device='cuda') * 4).to(dtype)
    cos, sin = rope_cos_sin(S + 13, D, 'cuda', dtype)         # longer tables, sliced as attend does
    cos, sin = cos[:S], sin[:S]
    out = block_ops.rope_(x.clone(), cos, sin, heads, D)
    _assert_bits(out, glo.rope(x, cos, sin, heads, D), f'rope B{B} S{S} H{heads} D{D} {dtype}')
    q = x.view(B, S, heads, D).transpose(1, 2)
    ref = (q * cos[None, None] + _rot_half(q) * sin[None, None]).transpose(1, 2).reshape(x.shape)
    _assert_bits(out, ref, 'rope vs torch')
    return out


@pytest.mark.parametrize('heads', [1, 8, 32])
@pytest.mark.parametrize('D', [16, 64, 128, 256])
def test_rope_shapes(D, heads):
    torch.manual_seed(D + heads)
    for dtype in DTYPES:
        for S in (1, 7, 2048):
            _rope_check(2 if S < 2048 else 1, S, heads, D, dtype)


def test_rope_grid_stride():
    B, S, H, D = 16, 2048, 8, 128
    assert B * S * H * (D // 16) > ELTWISE_UNITS > B * S * H * (D // 16) - ELTWISE_UNITS
    torch.manual_seed(2)
    _rope_check(B, S, H, D, torch.bfloat16)


@pytest.mark.parametrize('dtype', DTYPES)
def test_rope_special_values(dtype):
    B, S, H, D = 2, 7, 4, 64
    torch.manual_seed(3)
    x = (torch.randn(B, S, H * D, device='cuda')).to(dtype)
    sp = _specials(dtype).cuda()
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), device='cuda')[: 20 * sp.numel()]
    flat[idx] = sp.repeat(20)
    _rope_check(B, S, H, D, dtype, x=x)


# ---- SiLU * up --------------------------------------------------------------------------------------
def _ups(dtype):
    fi = torch.finfo(dtype)
    return torch.tensor([0.0, -0.0, 1.0, -1.0, fi.max, -fi.max, float('inf'), float('-inf'),
                         float('nan'), fi.tiny / 4, -fi.tiny, 0.37, -2.5, 3.0e-3, 17.0, -0.8125],
                        dtype=dtype, device='cuda')


@pytest.mark.parametrize('dtype', DT16)
def test_silu_mul_every_16bit_gate(dtype):
    """All 65,536 gate bit patterns against 16 up values."""
    from llmc_b200 import block_ops
    g = torch.arange(-32768, 32768, dtype=torch.int32, device='cuda').to(torch.int16).view(dtype)
    u = _ups(dtype)
    G = g.repeat(u.numel())
    U = u.repeat_interleave(g.numel())
    _assert_bits(block_ops.silu_mul(G, U), F.silu(G) * U, f'silu_mul {dtype}')


def test_silu_mul_fp32_and_sizes():
    from llmc_b200 import block_ops
    torch.manual_seed(4)
    g = torch.randn(1 << 20, device='cuda') * 8
    u = torch.randn(1 << 20, device='cuda')
    sp = _specials(torch.float32).cuda()
    g[: sp.numel() ** 2] = sp.repeat(sp.numel())
    u[: sp.numel() ** 2] = sp.repeat_interleave(sp.numel())
    _assert_bits(block_ops.silu_mul(g, u), F.silu(g) * u, 'fp32')
    for dtype in DTYPES:
        for n in (8, (1 << 24) + 8):
            if n > 8:
                assert n // 8 > ELTWISE_UNITS                 # a full pass plus a ragged tail
            g = (torch.randn(n, device='cuda') * 6).to(dtype)
            u = torch.randn(n, device='cuda').to(dtype)
            _assert_bits(block_ops.silu_mul(g, u), F.silu(g) * u, f'n={n} {dtype}')
            del g, u


def test_silu_mul_refuses_ragged_n_and_mlp_falls_back(monkeypatch):
    from llmc_b200 import _lib, block_ops
    from llmc_b200.synth import LlamaMLP
    g = torch.randn(13, device='cuda').bfloat16()
    y = torch.empty_like(g)
    n0 = _launches()
    rc = _lib.load().llmc_silu_mul(_lib.ptr(g), _lib.ptr(g), _lib.ptr(y), 12, _lib.BF16,
                                   _lib.stream_ptr(g.device))
    assert rc == EINVAL and _launches() == n0
    calls = []
    real = block_ops.silu_mul
    monkeypatch.setattr(block_ops, 'silu_mul', lambda *a, **k: calls.append(1) or real(*a, **k))
    m = LlamaMLP(8, 16)
    for shape in [(3, 5), (2, 8)]:
        g = torch.randn(*shape, device='cuda').bfloat16()
        u = torch.randn(*shape, device='cuda').bfloat16()
        calls.clear()
        _assert_bits(m.act(g, u), F.silu(g) * u, str(shape))
        assert len(calls) == (1 if g.numel() % 8 == 0 else 0)
    g = torch.randn(4, 16, device='cuda').bfloat16()
    u = torch.randn(4, 16, device='cuda').bfloat16()
    calls.clear()
    _assert_bits(m.act(g.t(), u.t()), F.silu(g.t()) * u.t(), 'strided')      # not contiguous
    assert calls == []
    calls.clear()
    out = m.act(g, u.float())                                                # up in another dtype
    assert calls == [] and out.dtype == torch.float32
    _assert_bits(out, F.silu(g) * u.float(), 'mixed')
    out = torch.empty(4, 16, device='cuda').bfloat16()
    assert m.act(g, u, out=out) is out and calls == [1]
    _assert_bits(out, F.silu(g) * u, 'out=')


def test_silu_mul_and_add_refuse_a_bad_out():
    from llmc_b200 import block_ops
    g = torch.randn(64, 16, device='cuda').bfloat16()
    bad = [torch.empty(16, 64, device='cuda').bfloat16().t(),        # strided
           torch.empty(64, 16, device='cuda').half(),                  # dtype
           torch.empty(32, 16, device='cuda').bfloat16()]               # shape
    for out in bad:
        with pytest.raises(AssertionError):
            block_ops.silu_mul(g, g, out=out)
        with pytest.raises(AssertionError):
            block_ops.add(g, g, out=out)
    with pytest.raises(AssertionError):
        block_ops.silu_mul(g, g.half())
    with pytest.raises(AssertionError):
        block_ops.add(g, g.half())


# ---- add --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', DTYPES)
def test_add_bit_patterns_and_grid_stride(dtype):
    from llmc_b200 import block_ops
    it = _INT[dtype]
    if dtype == torch.float32:
        a = torch.randn(1 << 20) * torch.exp(torch.randn(1 << 20) * 20)
        b = torch.randn(1 << 20) * torch.exp(torch.randn(1 << 20) * 20)
    else:
        a = torch.randint(-32768, 32768, (1 << 20,), dtype=torch.int32).to(it).view(dtype)
        b = torch.randint(-32768, 32768, (1 << 20,), dtype=torch.int32).to(it).view(dtype)
    sp = _specials(dtype)
    a[: sp.numel() ** 2] = sp.repeat(sp.numel())
    b[: sp.numel() ** 2] = sp.repeat_interleave(sp.numel())
    ref = glo.add(a, b)                                       # on the CPU
    _assert_bits(block_ops.add(a.cuda(), b.cuda()).cpu(), ref, 'add')
    n = (1 << 24) + 8
    assert n // 8 > ELTWISE_UNITS
    a = (torch.randn(n, device='cuda') * 100).to(dtype)
    b = (torch.randn(n, device='cuda') * 100).to(dtype)
    ref = glo.add(a, b)
    _assert_bits(block_ops.add(a, b), ref, 'add n=2^24+8')
    y = block_ops.add(a, b, out=a)                            # in place, as gptq.py's residual add
    assert y.data_ptr() == a.data_ptr()
    _assert_bits(a, ref, 'add in place')


# ---- dispatch guards ------------------------------------------------------------------------------
def _counting(monkeypatch, name):
    from llmc_b200 import block_ops
    calls = []
    real = getattr(block_ops, name)
    monkeypatch.setattr(block_ops, name, lambda *a, **k: calls.append(1) or real(*a, **k))
    return calls


def test_rmsnorm_guards(monkeypatch):
    from llmc_b200.gptq import norm_into
    from llmc_b200.synth import RMSNorm
    calls = _counting(monkeypatch, 'rmsnorm')
    torch.manual_seed(5)
    for cols, wdt, fused in [(64, torch.bfloat16, True), (60, torch.bfloat16, False),
                             (64, torch.float32, False)]:
        ln = RMSNorm(cols, eps=1e-6).cuda().to(wdt)
        ln.weight.data = (1 + 0.1 * torch.randn(cols, device='cuda')).to(wdt)
        # integer rows: every summation order gives the same mean, so the fallback's torch rsqrt is
        # the correctly rounded-ish inv the window contains
        x = torch.randint(-9, 10, (3, 5, cols), device='cuda').bfloat16()
        calls.clear()
        y = ln(x)
        assert len(calls) == int(fused), (cols, wdt)
        x2 = x.reshape(-1, cols)
        cand = glo.rmsnorm_inv_candidates(glo.rmsnorm_sumsq(x2), cols, 1e-6)
        y2 = y.reshape(-1, cols)
        ok = torch.stack([_bits_equal(glo.rmsnorm(x2, ln.weight.data, cand[:, k]), y2).all(-1)
                          for k in range(5)], -1)
        assert bool(ok.any(-1).all()), (cols, wdt)
        dst = torch.empty_like(y)
        calls.clear()
        norm_into(ln, x, dst)
        assert len(calls) == int(fused)
        _assert_bits(dst, y, 'norm_into')
    # a strided activation still runs the kernel (block_ops.rmsnorm makes it contiguous)
    ln = RMSNorm(64).cuda().bfloat16()
    x = torch.randn(64, 6, device='cuda').bfloat16().t()
    calls.clear()
    _check_rmsnorm(x.contiguous(), ln.weight.data, 1e-5, y=ln(x))
    assert calls == [1]


@pytest.mark.parametrize('head_dim,contig,cos_dt,fused', [
    (64, True, torch.bfloat16, True), (48, True, torch.bfloat16, True),
    (8, True, torch.bfloat16, False), (24, True, torch.bfloat16, False),
    (64, False, torch.bfloat16, False), (64, True, torch.float32, False)])
def test_rope_guard(monkeypatch, head_dim, contig, cos_dt, fused):
    """LlamaAttention.attend: the kernel exactly when head_dim % 16 == 0, q / k are contiguous and the
    tables are in q's dtype; either way q and k reach attention rotated as the oracle rotates
    them (GQA: 8 query heads, 2 kv heads sharing the table)."""
    from llmc_b200 import synth
    calls = _counting(monkeypatch, 'rope_')
    seen = {}

    def sdpa(q, k, v, **kw):
        seen['q'], seen['k'] = q, k
        return torch.zeros_like(q)
    monkeypatch.setattr(synth.F, 'scaled_dot_product_attention', sdpa)
    heads, kv, B, S = 8, 2, 2, 9
    a = synth.LlamaAttention(heads * head_dim, heads, kv)
    torch.manual_seed(6)
    q0 = torch.randn(B, S, heads * head_dim, device='cuda').bfloat16()
    k0 = torch.randn(B, S, kv * head_dim, device='cuda').bfloat16()
    v0 = torch.randn(B, S, kv * head_dim, device='cuda').bfloat16()
    cos, sin = synth.rope_cos_sin(S + 3, head_dim, 'cuda', cos_dt)
    if contig:
        q, k = q0.clone(), k0.clone()
    else:
        q = torch.cat([q0, q0], -1)[..., : heads * head_dim]
        k = torch.cat([k0, k0], -1)[..., : kv * head_dim]
    a.attend(q, k, v0, (cos, sin))
    assert len(calls) == (2 if fused else 0)
    for name, x, h in (('q', q0, heads), ('k', k0, kv)):
        got = seen[name].transpose(1, 2).reshape(B, S, h * head_dim)
        _assert_bits(got, glo.rope(x, cos[:S], sin[:S], h, head_dim), name)


# ---- AutoAWQ pack -----------------------------------------------------------------------------------
def _awq_pack(w, scales, zeros, group):
    from llmc_b200 import _lib
    R, C = w.shape
    ng = C // group
    qweight = torch.empty((C, R // 8), dtype=torch.int32, device='cuda')
    qzeros = torch.empty((ng, R // 8), dtype=torch.int32, device='cuda')
    sout = torch.empty((ng, R), dtype=torch.float16, device='cuda')
    rc = _lib.load().llmc_pack_awq(_lib.ptr(w), R, C, _lib.dtype_enum(w.dtype), _lib.ptr(scales),
                                   _lib.dtype_enum(scales.dtype), _lib.ptr(zeros), group,
                                   _lib.ptr(qweight), _lib.ptr(qzeros), _lib.ptr(sout),
                                   _lib.stream_ptr(w.device))
    assert rc == 0
    return qweight, sout, qzeros


def _check_awq(w, s, z, group, got):
    ref = qo.pack_awq(w.cpu(), s.cpu(), z.cpu().to(torch.int32), group)
    for name, a, b in zip(('qweight', 'scales', 'qzeros'), got, ref):
        a = a.cpu()
        assert a.shape == b.shape and a.dtype == b.dtype, name
        if not torch.equal(a, b):
            bad = (a != b).nonzero()[0].tolist()
            raise AssertionError(f'{name}: {int((a != b).sum())} words differ, first at {bad}')


AWQ_SHAPES = [(32, 32, 32), (224, 96, 32), (288, 96, 96), (4128, 32, 32), (288, 4096, 64),
              (4128, 4096, 128), (224, 4096, 4096)]


@pytest.mark.parametrize('s_fp32', [False, True])
@pytest.mark.parametrize('dtype', DTYPES)
def test_awq_pack_through_quant_pack(dtype, s_fp32):
    """AutoawqRealQuantLinear.quant_pack with the 4-bit asymmetric integer quantiser: R with
    partial 256-row tiles (224, 288, 4128), C with partial 64-column tiles (32, 96), groups 32 / 64 /
    128 / C, scales in the weight dtype and in fp32."""
    from llmc_b200.module_utils import AutoawqRealQuantLinear
    from llmc_b200.quant import IntegerQuantizer
    torch.manual_seed(7)
    for R, C, group in AWQ_SHAPES:
        q = IntegerQuantizer(4, False, 'per_group', group_size=group, round_zp=True)
        lin = torch.nn.Linear(C, R, bias=False).cuda()
        lin.weight.data = (torch.randn(R, C, device='cuda') * 0.05).to(dtype)
        out = {}

        def w_q(m):
            codes, s, z = q.real_quant_weight_dynamic(m.weight.data)
            out['s'], out['z'] = (s.float() if s_fp32 else s), z
            return codes, out['s'], z
        cfg = {'weight': {'bit': 4, 'group_size': group, 'pack_version': 'gemm_pack'}}
        got = AutoawqRealQuantLinear.quant_pack(lin, w_q, cfg)
        assert out['s'].dtype == (torch.float32 if s_fp32 else dtype)
        _check_awq(lin.weight.data, out['s'], out['z'], group, got)


def test_awq_pack_qparams_grid_stride():
    R, C, group = 4096, 8192, 32
    assert (C // group) * R > PACK_QPARAM_UNITS
    torch.manual_seed(8)
    w = (torch.randn(R, C, device='cuda') * 0.05).half()
    s = (torch.rand(R, C // group, device='cuda') * 0.01 + 1e-3).half()
    z = torch.randint(0, 16, (R, C // group), dtype=torch.int32, device='cuda')
    _check_awq(w, s, z, group, _awq_pack(w, s, z, group))


@pytest.mark.parametrize('dtype', DTYPES)
def test_awq_pack_codes_outside_the_nibble(dtype):
    """Codes -1 and 16 (the reference does not clamp, module_utils.py:1022-1029, and spills them
    into the neighbouring nibble), and codes beyond int8 that every bit of reaches the word."""
    R, C, group = 288, 96, 32
    torch.manual_seed(9)
    codes = torch.randint(0, 16, (R, C), device='cuda')
    big = [-1, 16, 17, -2, 127, 128, 255, -128, -129, -200, 1000, -4097, 30000, -30000]
    if dtype == torch.float32:
        big += [1 << 20, -(1 << 20) - 5, (1 << 23) + 1]
    elif dtype == torch.float16:
        big += [65504 - 15]
    else:
        big = [c for c in big if abs(c) <= 240]          # bf16 holds integers exactly up to 256
    flat = codes.view(-1)
    idx = torch.randperm(flat.numel(), device='cuda')[: 40 * len(big)]
    flat[idx] = torch.tensor(big, device='cuda').repeat(40)
    z = torch.randint(0, 16, (R, C // group), dtype=torch.int32, device='cuda')
    z[0, 0], z[1, 1] = 16, -1                             # zeros outside the nibble too
    s = torch.ones(R, C // group, dtype=dtype, device='cuda')
    zr = z.repeat_interleave(group, 1)
    w = (codes - zr).to(dtype)                           # (w + z*s) / s: the codes, up to w's rounding
    q = w.float() + zr
    assert float(q.max()) >= 128 and float(q.min()) <= -129
    _check_awq(w, s, z, group, _awq_pack(w, s, z, group))


# ---- GPTQ prepare -----------------------------------------------------------------------------------
def _hessian(C, dead, gen_seed):
    g = torch.Generator(device='cuda').manual_seed(gen_seed)
    H = torch.rand(C, C, device='cuda', generator=g)
    H.mul_(torch.exp(torch.randn(C, 1, device='cuda', generator=g)))
    H.diagonal().mul_(8)
    H.diagonal()[dead] = 0
    return H


def _check_prepare(W, H, perm, percdamp, Wp, Hp):
    C = H.shape[0]
    if Wp is not None:                                    # glue_oracle.prepare's weight gather
        p = torch.arange(C, device='cuda') if perm is None else perm
        rWp = W.float()[:, p].clone()
        rWp[:, (torch.diagonal(H) == 0)[p]] = 0
        _assert_bits(Wp, rWp, 'Wp')
    if Hp is not None:
        p = torch.arange(C, device='cuda') if perm is None else perm
        damp = glo.diag_mean(H, percdamp)
        for i0 in range(0, C, 2048):                      # row blocks: no second C x C buffer
            i1 = min(C, i0 + 2048)
            ref = H[p[i0:i1]][:, p]
            d = ref[torch.arange(i1 - i0), torch.arange(i0, i1)]
            ref[torch.arange(i1 - i0), torch.arange(i0, i1)] = torch.where(d == 0, torch.ones_like(d), d) + damp
            _assert_bits(Hp[i0:i1], ref, f'Hp rows {i0}:{i1}')


@pytest.mark.parametrize('C,R', [(1, 1), (7, 333), (128, 4096), (4096, 333), (4096, 4096),
                                 (8192, 333), (14336, 333)])
def test_prepare(C, R):
    from llmc_b200 import gptq_ops as ops
    torch.manual_seed(C)
    dead = torch.randperm(C)[: max(1, C // 50)].cuda() if C > 1 else torch.tensor([], dtype=torch.long)
    H = _hessian(C, dead.cuda(), C)
    for j, dtype in enumerate(DTYPES):
        W = (torch.randn(R, C, device='cuda') * 0.05).to(dtype)
        for permuted in (False, True):
            perm = torch.argsort(torch.diagonal(H), descending=True) if permuted else None
            if permuted and C > 1:                       # dead columns move to the end
                assert bool((perm[-len(dead):].sort().values == dead.sort().values).all())
            percdamp = (0.01, 1.0)[(j + permuted) % 2]
            if C > 8192 and dtype != torch.bfloat16:
                Wp, _ = ops.prepare(W, H, perm, percdamp, want_h=False)
                _check_prepare(W, H, perm, percdamp, Wp, None)
                continue
            Wp, Hp = ops.prepare(W, H, perm, percdamp)
            _check_prepare(W, H, perm, percdamp, Wp, Hp)
            if C <= 4096:
                rWp, rHp = glo.prepare(W, H, perm, percdamp)
                _assert_bits(Wp, rWp, 'Wp vs glue_oracle.prepare')
                _assert_bits(Hp, rHp, 'Hp vs glue_oracle.prepare')
                del rWp, rHp
            del Hp
        del W, Wp
    Wp, Hp = ops.prepare(None, H, None, 0.01)             # Hessian only
    assert Wp is None
    _check_prepare(None, H, None, 0.01, None, Hp)


def test_prepare_refuses_more_columns_than_the_row_buffer():
    """C * 4 bytes must fit the 200 KiB shared-memory row buffer: C = 51201 is refused before any
    launch (nothing of that size is allocated: the kernels never run)."""
    from llmc_b200 import _lib
    H = torch.zeros(8, device='cuda')
    W = torch.zeros(8, device='cuda')
    out = torch.zeros(8, device='cuda')
    n0 = _launches()
    rc = _lib.load().llmc_gptq_prepare(_lib.ptr(H), 51201, None, ctypes.c_float(0.01), _lib.ptr(out),
                                       _lib.ptr(W), 1, _lib.F32, _lib.ptr(out), _lib.ptr(out),
                                       _lib.stream_ptr(H.device))
    assert rc == EINVAL and _launches() == n0
    assert b'51201' in _lib.load().llmc_b200_last_error()


def test_report_rsqrtf_offsets():
    """Runs after the RMSNorm tests in this module: prints which ulp offsets of the correctly
    rounded inv the kernel's rows matched (the nearest matching offset per row)."""
    if INV_OFFSETS:
        print('\nrmsnorm rows by nearest matching inv offset (ulp):', dict(sorted(INV_OFFSETS.items())))
