"""GPU: the bf16/fp16 GEMM (`llmc_gemm_bf16`), the packed W4/W8 GEMM (`llmc_gemm_w4a16`,
`llmc_gemm_w8a16`) and the Hessian SYRK (`llmc_syrk_accum`) bit for bit against an exact oracle, at
every tile edge.

The oracle is an integer grid.  With integer operands (and, for W4/W8, small integer codes and
zero-points with power-of-two scales, so that every dequantised weight is exact in bf16 / fp16)
every partial sum the kernels form is a multiple of a fixed power of two and below 2^24 of it.  It
is then exact in fp32 in any summation order, tensor-core accumulation included, and the kernel's
output must be one RNE rounding, to the output dtype, of the exact value, computed here as an fp64
matmul (exact below 2^53).  Operand ranges keep most outputs above 256 (bf16) or 2048 (fp16), so
the final rounding is not trivial: a bias added after the rounding, a column pair stored from the
wrong lane, a tile the raster order skips, a slab entry the SYRK finalize reads but the kernel did
not write all change bits.

Each path-table entry is named by the case its shape reaches and asserts that it reaches it, from
a restatement of the host-side plans: `l2_group_width` and the tile counts for the GEMMs, the split
count read back from `llmc_syrk_workspace_bytes` for SYRK.  Around the tables: random data against
a worst-case bound for fp32 accumulation at real widths, outputs that do not depend on the problem
size, special values against torch's own F.linear on the same GPU, and M = 0."""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from llmc_b200._lib import call, dtype_enum, load, ptr, stream_ptr
from llmc_b200.gptq_ops import hessian_add_batch
from llmc_b200.module_utils import linear_forward, linear_forward_w4

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
NUM_SMS = 132                   # persistent kernels run min(units, 132) CTAs
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
EXACT_LIMIT = 1 << 24           # |partial sum| below this many units of its spacing: exact in fp32


# ---- helpers -------------------------------------------------------------------------------------
def _gen(*key):
    g = torch.Generator(device='cuda')
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def _randint(lo, hi, shape, g):
    """Integers in [lo, hi] as fp64 on the GPU."""
    return torch.randint(lo, hi + 1, shape, generator=g, device='cuda').double()


def _same(got, exp, what):
    """Bit-exact equality; NaN matches NaN whatever its payload."""
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert got.dtype == exp.dtype, (what, got.dtype, exp.dtype)
    gn, en = torch.isnan(got), torch.isnan(exp)
    iv = INT_VIEW[got.dtype]
    bad = (gn != en) | (~gn & (got.view(iv) != exp.view(iv)))
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        first = [(i, got[tuple(i)].item(), exp[tuple(i)].item()) for i in idx]
        raise AssertionError(f'{what}: {int(bad.sum())}/{got.numel()} elements differ; first '
                             f'(index, got, expected): {first}')


def _nontrivial(ref, dtype, what):
    """Most outputs lie where the dtype cannot hold every integer, so the rounding matters."""
    if ref.numel() < 64:
        return
    big = 256 if dtype == torch.bfloat16 else 2048
    frac = (ref.abs() > big).double().mean().item()
    assert frac > 0.25, (what, frac)


# ---- host-side plans, restated -------------------------------------------------------------------
def l2_group_width(divisor, n_tiles):
    """tc.cuh l2_group_width: as many n-tiles as 32 MB of L2 holds, at least 1, at most n_tiles."""
    return min(max((32 << 20) // divisor, 1), n_tiles)


def _cdiv(a, b):
    return -(-a // b)


def _raster_cases(m_tiles, n_tiles, gn):
    cases = set()
    if m_tiles * n_tiles > NUM_SMS:
        cases.add('persistent')
    if n_tiles % gn:
        cases.add('partial-group')
    elif n_tiles // gn >= 2:
        cases.add('full-groups')
    else:
        cases.add('one-group')
    return cases


def gemm_cases(M, N, K):
    """The cases llmc_gemm_bf16 (tile 128 x 256 x 64, two 64-row consumer warpgroups) reaches."""
    m_tiles, n_tiles = _cdiv(M, 128), _cdiv(N, 256)
    cases = _raster_cases(m_tiles, n_tiles, l2_group_width(256 * K * 2, n_tiles))
    cases.add('wg1-empty' if M - (m_tiles - 1) * 128 <= 64 else 'both-wg')
    if M % 128:
        cases.add('partial-m')
    if N % 2:
        cases.add('odd-n')            # element-wise store_pair16
    if N % 256:
        cases.add('partial-n')
    if K % 64:
        cases.add('k-tail')
    if K <= 64:
        cases.add('one-kb')
    return cases


def w_cases(M, N, K, bits, group):
    """The cases llmc_gemm_w{4,8}a16 (tile 128 x 128 x 64) reaches."""
    m_tiles, n_tiles = _cdiv(M, 128), _cdiv(N, 128)
    cases = _raster_cases(m_tiles, n_tiles, l2_group_width(128 * K * bits // 8 + 1, n_tiles))
    if M % 128:
        cases.add('partial-m')
    if N % 2:
        cases.add('odd-n')
    if N % 128:
        cases.add('partial-n')
    cases.add('per-channel' if group == K else f'g{group}')
    return cases


def syrk_plan(T, C):
    """(splits, k-blocks, k-blocks per split, upper tiles, m-blocks) of llmc_syrk_accum; the split
    count is the library's own, read back from its workspace size."""
    splits = load().llmc_syrk_workspace_bytes(T, C) // (4 * C * C)
    kb = _cdiv(T, 64)
    kbps = _cdiv(kb, splits)
    assert _cdiv(kb, kbps) == splits, (T, C, splits)
    m_tiles, n_tiles = _cdiv(C, 128), _cdiv(C, 256)
    tiles = sum(n_tiles - (m >> 1) for m in range(m_tiles))
    return splits, kb, kbps, tiles, m_tiles


def syrk_cases(T, C):
    splits, kb, kbps, tiles, m_tiles = syrk_plan(T, C)
    cases = {f'split{splits}'}
    if splits > 2:
        cases.add('splits>2')
    if kb % kbps:
        cases.add('uneven-split')
    if T % 64:
        cases.add('ragged-t')
    if C % 32:
        cases.add('ragged-c')         # the finalize's 32 x 32 diagonal tiles overhang C
    if m_tiles > 12:
        cases.add('super-rows')       # decode_unit's 12-m-block super-rows
    if tiles * splits > NUM_SMS:
        cases.add('persistent')
    return cases


# ---- the exact integer-grid oracle ---------------------------------------------------------------
def _int_range(K, dtype):
    """Operand magnitude for a K-deep integer product: every partial sum (and a bias below 256)
    stays below 2^23, and for fp16 a typical |y| ~ sqrt(K) r^2 / 3 of about 8000, above 2048 but
    mostly finite."""
    r = min(64, math.isqrt((1 << 23) // K))
    if dtype == torch.float16:
        r = min(r, math.isqrt(int(24000 / math.sqrt(K))))
    return r


def gemm_grid(M, N, K, dtype, bias, key=()):
    """Integer x [M, K], w [N, K], bias [N] (or None) in dtype and the exact y in fp64."""
    g = _gen('gemm', M, N, K, str(dtype), bias, key)
    r = _int_range(K, dtype)
    assert K * r * r + 256 < EXACT_LIMIT
    x = _randint(-r, r, (M, K), g)
    w = _randint(-r, r, (N, K), g)
    ref = x @ w.t()
    b = None
    if bias:
        b = _randint(-255, 255, (N,), g)
        ref += b
        b = b.to(dtype)
    return x.to(dtype), w.to(dtype), b, ref


def pack_codes(codes, bits):
    """[N, K] unsigned codes -> [N, K * bits / 32] int32, element per * w + i in bit field i (the
    LLMC_OUT_PACK_VLLM layout), written out here so that the library's packer is not part of the
    oracle."""
    N, K = codes.shape
    per = 32 // bits
    c = codes.to(torch.int64).reshape(N, K // per, per)
    w = (c << (torch.arange(per, device=c.device, dtype=torch.int64) * bits)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


class WGrid:
    """Packed W4/W8 weights on the integer grid: codes and zero-points in [0, 2^bits), scales
    2^-3 .. 2^1, so (q - z) s is exact in bf16 / fp16, and integer activations small enough that
    every partial sum is below 2^24 units of 2^-3.  zeros None: the kernel's default 2^(bits-1)."""

    def __init__(self, M, N, K, bits, group, sym, dtype, bias, key=()):
        g = _gen('w', M, N, K, bits, group, sym, str(dtype), bias, key)
        qmax = (1 << bits) - 1
        ng = K // group
        self.bits, self.group, self.dtype = bits, group, dtype
        self.codes = _randint(0, qmax, (N, K), g)
        self.scales = torch.pow(2.0, _randint(-3, 1, (N, ng), g))
        self.zeros = None if sym else _randint(0, qmax, (N, ng), g)
        z = torch.full((N, ng), float(1 << (bits - 1)), dtype=torch.float64, device='cuda') \
            if sym else self.zeros
        wdq = (self.codes.view(N, ng, group) - z[..., None]) * self.scales[..., None]
        self.wdq = wdq.reshape(N, K)
        wmax = qmax * 2
        r = min(64, (EXACT_LIMIT // 8 - 256) // (K * wmax))
        assert r >= 1 and K * r * wmax + 256 < EXACT_LIMIT // 8
        x = _randint(-r, r, (M, K), g)
        self.ref = x @ self.wdq.t()
        self.bias = None
        if bias:
            b = _randint(-255, 255, (N,), g)
            self.ref += b
            self.bias = b.to(dtype)
        self.x = x.to(dtype)
        self.packed = pack_codes(self.codes, bits)

    def run(self, native, transposed, x=None, rows=None):
        """linear_forward_w4 with qparams in fp32 or (native) the activation dtype, stored [N, ng]
        or (transposed) [ng, N]; rows: a slice of output features."""
        qdt = self.dtype if native else torch.float32
        rows = rows or slice(None)
        s = self.scales[rows].to(qdt)
        z = self.zeros[rows].to(qdt) if self.zeros is not None else None
        if transposed:
            s = s.t().contiguous()
            z = z.t().contiguous() if z is not None else None
        b = self.bias[rows] if self.bias is not None else None
        return linear_forward_w4(self.x if x is None else x, self.packed[rows].contiguous(), s, z,
                                 self.group, bias=b, bits=self.bits, qparams_t=transposed)


# ---- GEMM: path table ----------------------------------------------------------------------------
GEMM_PATHS = [
    # name, M, N, K, x shape (None: [M, K]), cases the shape must reach
    ('m1-wg1-empty-k-tail', 1, 257, 72, None, {'wg1-empty', 'odd-n', 'k-tail'}),
    ('m63-odd-n', 63, 263, 200, None, {'wg1-empty', 'odd-n', 'k-tail'}),
    ('m64-n2-k8', 64, 2, 8, None, {'wg1-empty', 'one-kb', 'k-tail'}),
    ('m65-both-wg-n7-k56', 65, 7, 56, None, {'both-wg', 'odd-n', 'one-kb', 'k-tail'}),
    ('m127-n255-one-kb', 127, 255, 64, None, {'both-wg', 'odd-n', 'one-kb', 'partial-m'}),
    ('m129-n520-k4104', 129, 520, 4104, None, {'wg1-empty', 'partial-n', 'k-tail'}),
    ('m300-n1', 300, 1, 200, None, {'wg1-empty', 'odd-n', 'partial-m'}),
    ('persistent', 1100, 4100, 200, None, {'persistent', 'one-group', 'k-tail'}),
    ('partial-group', 300, 14336, 4096, None, {'partial-group', 'persistent', 'partial-m'}),
    ('partial-group-odd-n', 257, 14335, 4096, None, {'partial-group', 'persistent', 'odd-n'}),
    ('full-groups-k14336', 256, 4096, 14336, None, {'full-groups'}),
    ('3d-input', 300, 264, 200, (2, 150, 200), {'partial-n', 'k-tail'}),
]


@pytest.mark.parametrize('bias', [False, True], ids=['nobias', 'bias'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,M,N,K,xshape,want', GEMM_PATHS, ids=[p[0] for p in GEMM_PATHS])
def test_gemm_path_table(name, M, N, K, xshape, want, dtype, bias):
    got_cases = gemm_cases(M, N, K)
    assert want <= got_cases, (name, want - got_cases)
    x, w, b, ref = gemm_grid(M, N, K, dtype, bias)
    _nontrivial(ref, dtype, name)
    y = linear_forward(x.reshape(xshape) if xshape else x, w, b)
    assert y.shape == (xshape[:-1] if xshape else (M,)) + (N,)
    _same(y.reshape(M, N), ref.to(dtype), name)


GEMM_MS = (1, 63, 64, 65, 127, 129, 300)
GEMM_NS = (1, 2, 7, 255, 257, 263, 520)
GEMM_KS = (8, 56, 64, 72, 200, 4104)


@pytest.mark.parametrize('bias', [False, True], ids=['nobias', 'bias'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_gemm_grid_sweep(dtype, bias):
    """Every combination of the edge M, N and K above."""
    for K in GEMM_KS:
        for N in GEMM_NS:
            for M in GEMM_MS:
                x, w, b, ref = gemm_grid(M, N, K, dtype, bias)
                _same(linear_forward(x, w, b), ref.to(dtype), f'M={M} N={N} K={K}')


# ---- W4 / W8: path table -------------------------------------------------------------------------
W_PATHS = [
    # name, bits, M, N, K, group, sym, native qparams, transposed qparams, bias, cases
    ('w4-g64-n1', 4, 65, 1, 512, 64, False, False, False, True, {'g64', 'odd-n', 'partial-m'}),
    ('w4-g128-n127-native', 4, 129, 127, 512, 128, True, True, False, False, {'g128', 'odd-n'}),
    ('w4-g256-n129-t', 4, 300, 129, 512, 256, False, True, True, True, {'g256', 'odd-n'}),
    ('w4-per-channel-n519', 4, 1, 519, 1024, 1024, True, False, True, True,
     {'per-channel', 'odd-n'}),
    ('w4-n14336-one-group', 4, 300, 14336, 4096, 128, False, True, True, True,
     {'one-group', 'persistent'}),
    ('w8-g64-n519-native', 8, 77, 519, 512, 64, False, True, False, True, {'g64', 'odd-n'}),
    ('w8-per-channel-n127', 8, 300, 127, 512, 512, True, False, False, False,
     {'per-channel', 'odd-n'}),
    ('w8-partial-group', 8, 300, 14336, 4096, 128, False, False, False, True,
     {'partial-group', 'persistent', 'partial-m'}),
    ('w8-partial-group-sym-native-t', 8, 256, 14336, 4096, 4096, True, True, True, False,
     {'partial-group', 'persistent', 'per-channel'}),
]


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,bits,M,N,K,group,sym,native,transposed,bias,want', W_PATHS,
                         ids=[p[0] for p in W_PATHS])
def test_w_path_table(name, bits, M, N, K, group, sym, native, transposed, bias, want, dtype):
    got_cases = w_cases(M, N, K, bits, group)
    assert want <= got_cases, (name, want - got_cases)
    wg = WGrid(M, N, K, bits, group, sym, dtype, bias)
    _nontrivial(wg.ref, dtype, name)
    _same(wg.run(native, transposed), wg.ref.to(dtype), name)


@pytest.mark.parametrize('transposed', [False, True], ids=['nk', 'kn'])
@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('bits', [4, 8])
def test_w_grid_sweep(bits, dtype, native, transposed):
    """group 64 / 128 / 256 / per channel x sym / asym x N 1 / 127 / 129 / 519 x bias, at ragged M."""
    K = 512
    ms = (1, 77, 129, 300)
    i = 0
    for group in (64, 128, 256, K):
        for sym in (True, False):
            for N in (1, 127, 129, 519):
                for bias in (False, True):
                    M = ms[i % len(ms)]
                    i += 1
                    wg = WGrid(M, N, K, bits, group, sym, dtype, bias)
                    _same(wg.run(native, transposed), wg.ref.to(dtype),
                          f'M={M} N={N} group={group} sym={sym} bias={bias}')


# ---- SYRK ----------------------------------------------------------------------------------------
def _syrk_x(T, C, dtype, limit, key=()):
    """Integer X [T, C] whose column products summed over T stay below `limit`."""
    g = _gen('syrk', T, C, str(dtype), key)
    r = min(64, math.isqrt((limit - 1) // T))
    assert r >= 1
    return _randint(-r, r, (T, C), g)


def syrk_call(x, H, n, b, ws):
    T, C = x.shape
    call('llmc_syrk_accum', ptr(x), T, C, dtype_enum(x.dtype), ptr(H), float(n), float(b), ptr(ws),
         ws.numel() * ws.element_size(), stream_ptr())


SYRK_PATHS = [
    # name, C, T, cases
    ('c8-t1', 8, 1, {'split1', 'ragged-t', 'ragged-c'}),
    ('c8-t4096-even-split4', 8, 4096, {'split4', 'splits>2'}),
    ('c136-t16421-split16-uneven', 136, 16421, {'split16', 'uneven-split', 'ragged-t', 'ragged-c'}),
    ('c264-t2100-uneven-split2', 264, 2100, {'split2', 'uneven-split', 'ragged-t', 'ragged-c'}),
    ('c392-t65', 392, 65, {'split1', 'ragged-t', 'ragged-c'}),
    ('c1544-super-rows-split12', 1544, 16421, {'super-rows', 'split12', 'uneven-split'}),
    ('c1544-super-rows-split7', 1544, 8192, {'super-rows', 'split7', 'uneven-split'}),
    ('c3080-persistent', 3080, 2100, {'super-rows', 'persistent', 'uneven-split', 'ragged-c'}),
    ('c3080-t16421-split8', 3080, 16421, {'super-rows', 'persistent', 'split8', 'uneven-split'}),
]


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,C,T,want', SYRK_PATHS, ids=[p[0] for p in SYRK_PATHS])
def test_syrk_path_table(name, C, T, want, dtype):
    """Through the C ABI with the workspace pre-filled with NaN and H's strict lower triangle NaN:
    the finalize must read only slab entries the kernel wrote and only H's upper triangle.
    n = 3, b = 1 makes n / (n + b) = 3/4 and 2 / (n + b) = 1/2, so the exact H is an fp32 value."""
    got_cases = syrk_cases(T, C)
    assert want <= got_cases, (name, want - got_cases)
    x = _syrk_x(T, C, dtype, 1 << 21)
    g = _gen('syrk-h', C)
    h0 = torch.triu(_randint(-(1 << 20), 1 << 20, (C, C), g))
    h0 = h0 + torch.triu(h0, 1).t()
    ref = 0.75 * h0 + 0.5 * (x.t() @ x)
    H = h0.float()
    H[torch.ones(C, C, dtype=torch.bool, device='cuda').tril(-1)] = float('nan')
    ws = torch.full((load().llmc_syrk_workspace_bytes(T, C) // 4,), float('nan'), device='cuda')
    syrk_call(x.to(dtype), H, 3, 1, ws)
    _same(H, ref.float(), name)


SYRK_CS = (8, 136, 264, 392, 1544, 3080)
SYRK_TS = (1, 63, 65, 2100, 16421)


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_syrk_grid_sweep(dtype):
    """Every C x T above through hessian_add_batch (H = 2 X^T X from zero), and H exactly
    symmetric.  The cached workspace holds the previous shape's slabs when the next one starts."""
    for C in SYRK_CS:
        for T in SYRK_TS:
            x = _syrk_x(T, C, dtype, EXACT_LIMIT)
            H = torch.zeros(C, C, device='cuda')
            assert hessian_add_batch(H, 0, x.to(dtype)) == 1
            ref = torch.zeros(C, C, dtype=torch.float64, device='cuda') + 2 * (x.t() @ x)
            _same(H, ref.float(), f'C={C} T={T}')     # 0 + (-0) = +0, as the update's formula
            assert torch.equal(H, H.t())


@pytest.mark.parametrize('C', [136, 1544])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_syrk_running_mean_chain(dtype, C):
    """Batches of b = 1, 1, 2, 4: every n / (n + b) and 2 / (n + b) is dyadic, so the running
    mean stays exact in fp32 and must equal the fp64 recurrence bit for bit."""
    tokens = 300
    H = torch.zeros(C, C, device='cuda')
    ref = torch.zeros(C, C, dtype=torch.float64, device='cuda')
    n = 0
    for i, b in enumerate((1, 1, 2, 4)):
        x = _syrk_x(8 * tokens, C, dtype, 1 << 21, key=i)[:b * tokens]
        ref = ref * (n / (n + b)) + (2 / (n + b)) * (x.t() @ x)
        n = hessian_add_batch(H, n, x.to(dtype).reshape(b, tokens, C))
        _same(H, ref.float(), f'after batch {i} (n={n})')
        assert torch.equal(H, H.t())
    assert n == 8


# ---- random data: a worst-case bound for fp32 accumulation ----------------------------------------
def _ulp(v, dtype):
    """ulp of dtype at |v| (the subnormal spacing below the normal range)."""
    p, emin = (8, -126) if dtype == torch.bfloat16 else (11, -14)
    _, e = torch.frexp(v)
    e = torch.clamp(torch.where(v == 0, emin, e - 1), min=emin)
    return torch.ldexp(torch.ones_like(v), e - (p - 1))


def _check_bound(y, ref, absum, K, dtype, what):
    """|y - ref| <= ulp(ref) + 2 K 2^-24 sum_k |x_k w_k| for every element; returns the largest
    ratio of the error to that bound."""
    bound = _ulp(ref, dtype) + 2 * K * 2.0 ** -24 * absum
    ratio = ((y.double() - ref).abs() / bound).max().item()
    print(f'{what}: largest error / bound = {ratio:.4f}')
    assert ratio <= 1.0, (what, ratio)
    return ratio


REAL_WIDTHS = [(256, 768, 768), (256, 4096, 4096), (256, 14336, 4096), (256, 4096, 14336)]


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('M,N,K', REAL_WIDTHS)
def test_gemm_random_within_bound(M, N, K, dtype):
    g = _gen('gemm-rand', M, N, K, str(dtype))
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    w = (torch.randn(N, K, generator=g, device='cuda') * 0.02).to(dtype)
    b = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype)
    xd, wd, bd = x.double(), w.double(), b.double()
    ref = xd @ wd.t() + bd
    absum = xd.abs() @ wd.abs().t() + bd.abs()
    _check_bound(linear_forward(x, w, b), ref, absum, K, dtype, f'gemm {M}x{N}x{K} {dtype}')


@pytest.mark.parametrize('native', [False, True], ids=['q-fp32', 'q-native'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('M,N,K', REAL_WIDTHS)
def test_w4_random_within_bound(M, N, K, dtype, native):
    """Random codes, zero-points and scales; the weight is the materialised rT((q - z) s)."""
    g = _gen('w4-rand', M, N, K, str(dtype), native)
    group = 128
    ng = K // group
    codes = torch.randint(0, 16, (N, K), generator=g, device='cuda')
    qdt = dtype if native else torch.float32
    s = (torch.rand(N, ng, generator=g, device='cuda') * 0.004 + 0.001).to(qdt)
    z = torch.randint(0, 16, (N, ng), generator=g, device='cuda').to(qdt)
    wdq = ((codes.view(N, ng, group).float() - z.float()[..., None]) * s.float()[..., None])
    wdq = wdq.reshape(N, K).to(dtype)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    b = (torch.randn(N, generator=g, device='cuda') * 0.1).to(dtype)
    xd, wd, bd = x.double(), wdq.double(), b.double()
    y = linear_forward_w4(x, pack_codes(codes, 4), s, z, group, bias=b)
    _check_bound(y, xd @ wd.t() + bd, xd.abs() @ wd.abs().t() + bd.abs(), K, dtype,
                 f'w4 {M}x{N}x{K} {dtype} native={native}')


# ---- results do not depend on the problem size ---------------------------------------------------
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_gemm_outputs_independent_of_problem_size(dtype):
    """On random data, any rows or columns of the product computed as a smaller (or wider) problem
    are the same rows / columns of the full product bit for bit: unaligned row ranges, the last row
    alone, unaligned and tile-aligned column ranges, and N widened from one raster group (16 n-tiles
    at K = 4096) to 56 n-tiles in four groups."""
    M, N, K = 1300, 4096, 4096
    g = _gen('gemm-inv', str(dtype))
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    w = (torch.randn(14336, K, generator=g, device='cuda') * 0.02).to(dtype)
    b = torch.randn(14336, generator=g, device='cuda').to(dtype)
    y = linear_forward(x, w[:N], b[:N])
    _same(linear_forward(x[1000:1077], w[:N], b[:N]), y[1000:1077], 'rows 1000:1077')
    _same(linear_forward(x[-1:], w[:N], b[:N]), y[-1:], 'last row')
    _same(linear_forward(x[3:4], w[:N], b[:N]), y[3:4], 'row 3')
    _same(linear_forward(x, w[256:1280], b[256:1280]), y[:, 256:1280], 'columns 256:1280')
    _same(linear_forward(x, w[37:1037], b[37:1037]), y[:, 37:1037], 'columns 37:1037')
    _same(linear_forward(x, w[4095:4096], b[4095:4096]), y[:, 4095:4096], 'last column')
    assert 'one-group' in gemm_cases(M, N, K) and 'partial-group' in gemm_cases(M, 14336, K)
    _same(linear_forward(x, w, b)[:, :N], y, 'N widened to 14336')


@pytest.mark.parametrize('bits', [4, 8])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_w_outputs_independent_of_problem_size(dtype, bits):
    """As for the GEMM, on random codes, zero-points and scales; N widened from one raster group
    to 112 n-tiles (W8 at K = 4096: groups of 63)."""
    M, N, K, group = 1300, 4096, 4096, 128
    Nw = 14336
    g = _gen('w-inv', str(dtype), bits)
    ng = K // group
    codes = torch.randint(0, 1 << bits, (Nw, K), generator=g, device='cuda')
    s = torch.rand(Nw, ng, generator=g, device='cuda') * 0.004 + 0.001
    z = torch.randint(0, 1 << bits, (Nw, ng), generator=g, device='cuda').float()
    b = torch.randn(Nw, generator=g, device='cuda').to(dtype)
    x = torch.randn(M, K, generator=g, device='cuda').to(dtype)
    packed = pack_codes(codes, bits)

    def run(xx, rows):
        return linear_forward_w4(xx, packed[rows].contiguous(), s[rows], z[rows], group,
                                 bias=b[rows], bits=bits)

    y = run(x, slice(0, N))
    _same(run(x[1000:1077], slice(0, N)), y[1000:1077], 'rows 1000:1077')
    _same(run(x[-1:], slice(0, N)), y[-1:], 'last row')
    _same(run(x, slice(128, 1152)), y[:, 128:1152], 'columns 128:1152')
    _same(run(x, slice(37, 1037)), y[:, 37:1037], 'columns 37:1037')
    want = 'partial-group' if bits == 8 else 'one-group'
    assert want in w_cases(M, Nw, K, bits, group)
    _same(run(x, slice(0, Nw))[:, :N], y, 'N widened to 14336')


# ---- special values: torch's F.linear on the same GPU is the oracle ------------------------------
@pytest.fixture
def fp32_reductions():
    """cuBLAS keeps its split-K reductions in fp32, so that F.linear is exact on integer grids."""
    m = torch.backends.cuda.matmul
    old = (m.allow_fp16_reduced_precision_reduction, m.allow_bf16_reduced_precision_reduction)
    m.allow_fp16_reduced_precision_reduction = False
    m.allow_bf16_reduced_precision_reduction = False
    yield
    m.allow_fp16_reduced_precision_reduction, m.allow_bf16_reduced_precision_reduction = old


@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_special_values_match_f_linear(dtype, fp32_reductions):
    """A NaN in a row of x; +inf and -inf in x where the matching column of W holds zeros in some
    rows (inf * 0 = NaN there, +-inf elsewhere).  The rest of the grid is exact in both.  N is even:
    with a bias and an odd N, torch's bf16 F.linear rounds the product before adding the bias
    (DESIGN.md §4), which the kernel does not."""
    M, N, K = 300, 264, 200
    x, w, b, _ = gemm_grid(M, N, K, dtype, True, key='special')
    x[5, 17] = float('nan')
    x[130, 10] = float('inf')
    x[131, 20] = float('-inf')
    for col, zero_rows in ((10, slice(0, None, 3)), (20, slice(1, None, 4))):
        w[:, col] = torch.where(w[:, col] == 0, 1, w[:, col])
        w[zero_rows, col] = 0
    y = linear_forward(x, w, b)
    assert bool(torch.isnan(y[5]).all())
    assert bool(torch.isnan(y[130, ::3]).all()) and bool(torch.isinf(y[130, 1::3]).all())
    _same(y, F.linear(x, w, b), 'special values')
    wg = WGrid(M, N, 256, 4, 128, False, dtype, True, key='special')
    wg.x[5, 17] = float('nan')
    yw = wg.run(False, False)
    assert bool(torch.isnan(yw[5]).all())
    ref = wg.ref.to(dtype)
    ref[5] = float('nan')
    _same(yw, ref, 'w4 NaN row')


def test_fp16_overflow_and_subnormals_match_f_linear(fp32_reductions):
    """fp16 outputs beyond 65504 become +-inf; subnormal fp16 activations and weights
    (k * 2^-24, |k| < 1024) multiply and round like F.linear's."""
    dt = torch.float16
    M, N, K = 300, 263, 200
    x, w, b, ref = gemm_grid(M, N, K, dt, True, key='overflow')
    x[:2] = 200
    w[:4] = 200
    w[2:4] = -200
    y = linear_forward(x, w, b)
    assert bool(torch.isinf(y[:2, :4]).all())
    _same(y, F.linear(x, w, b), 'fp16 overflow')
    g = _gen('subnormal')
    tiny = 2.0 ** -24
    xs = (_randint(-1000, 1000, (M, K), g) * tiny).to(dt)
    ws = _randint(-8, 8, (N, K), g).to(dt)
    assert bool(((xs != 0) & (xs.abs() < 2.0 ** -14)).any())
    _same(linear_forward(xs, ws), F.linear(xs, ws), 'subnormal activations')
    wsub = (_randint(-1000, 1000, (N, K), g) * tiny).to(dt)
    xi = _randint(-8, 8, (M, K), g).to(dt)
    y = linear_forward(xi, wsub)
    assert bool(((y != 0) & (y.abs() < 2.0 ** -14)).any())
    _same(y, F.linear(xi, wsub), 'subnormal weights')


# ---- degenerate shapes ---------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_m0_returns_empty_without_a_launch(dtype):
    lib = load()
    K, N = 256, 264
    w = torch.ones(N, K, dtype=dtype, device='cuda')
    b = torch.ones(N, dtype=dtype, device='cuda')
    wg = WGrid(1, N, K, 4, 128, False, dtype, True, key='m0')
    wg8 = WGrid(1, N, K, 8, 128, True, dtype, False, key='m0')
    for shape in ((0, K), (2, 0, K)):
        x = torch.empty(shape, dtype=dtype, device='cuda')
        torch.cuda.synchronize()
        before = lib.llmc_b200_launch_count()
        outs = [linear_forward(x, w, b), wg.run(False, False, x=x), wg8.run(True, True, x=x)]
        assert lib.llmc_b200_launch_count() == before
        for y in outs:
            assert y.shape == shape[:-1] + (N,) and y.dtype == dtype
