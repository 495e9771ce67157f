"""GPU: the grouped sparse-MoE kernels bit for bit against an exact oracle at every segment, tile and
routing edge: the dense grouped GEMM (`llmc_moe_gemm_swiglu`, `llmc_moe_gemm_down`, csrc/gemm.cu),
the grouped dequant GEMM on packed W4 / W8 experts (`llmc_moe_gemm_packed_swiglu`,
`llmc_moe_gemm_packed_down`, csrc/gemm_w4.cu) and the combine (`llmc_moe_combine`).

Inputs are built at the C entry points: hand-made int32 segment offsets, routing weights and host
arrays of expert pointers, so that the routing code (moe_routing, MixtralSparseMoe) is no part of the
oracle.  test_gpu_moe_grouped.py and test_gpu_moe_packed.py compare moe_forward with the per-expert
loop, which stays the definition of the routing.

The oracle is test_gpu_gemm_paths.py's integer grid: integer activations and weights (packed: codes
and zero-points in [0, 2^bits), power-of-two scales) keep every partial sum exact in fp32, so a
GEMM's accumulator is the fp64 product.  On top of it the header's arithmetic:
  gate/up  act = F.silu(rT(G)) * rT(U), evaluated by torch on the GPU (silu_mul_f32 is F.silu's
           formula; expf differs between CPU and GPU);
  down     y = rT(rT(S) * w): the product of two 16-bit values is exact in fp64, so rounding it once
           gives the kernel's fp32 product rounded once;
  combine  out[t] = rT(... rT(rT(0 + y[rows[t, 0]]) + y[rows[t, 1]]) ...), sequential fp32 adds on
           the CPU, in slot order.
Every output is allocated with guard rows after its last row, all filled with a NaN bit pattern no
kernel writes (SENTINEL): every real row must be written, and no guard row touched.

Each path-table entry names the cases its segments and shapes reach and asserts that it reaches
them, from a restatement of the launch plans: moe_tiles (tc::moe_segment_tile) and moe_plan
(launch_moe in gemm.cu, launch_moe_packed in gemm_w4.cu).  That check needs no GPU."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from llmc_b200._lib import call, dtype_enum, stream_ptr
from test_gpu_gemm_paths import (EXACT_LIMIT, _cdiv, _gen, _int_range, _nontrivial, _randint, _same,
                                 l2_group_width, pack_codes)

gpu = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
NUM_SMS = 132                   # persistent kernels run min(units, 132) CTAs
BM = 128                        # m-tile of both grouped GEMMs
SENTINEL = 0x7FA5               # a NaN in fp16 and bf16 alike; kernels write the canonical 0x7FFF
GUARD = 3                       # guard rows after every output
COMBINE_THREADS = NUM_SMS * 32 * 256    # llmc_moe_combine's grid-stride pass, in 8-column chunks


# ---- the launch plans, restated -------------------------------------------------------------------
def grouped_tile(u, m_tiles, n_tiles, gn):
    """tc::grouped_tile: (m_blk, n_blk) of unit u, groups of gn n-tiles, n fastest in a group."""
    g, rem = divmod(u, gn * m_tiles)
    gsz = min(gn, n_tiles - g * gn)
    m_blk, n_in = divmod(rem, gsz)
    return m_blk, g * gn + n_in


def moe_tiles(offsets, n_tiles, gn):
    """tc::moe_segment_tile for every unit that has a tile: (expert, m_blk, n_blk, row0, row_end)
    in unit order; units past the last one exit."""
    tiles = []
    for e in range(len(offsets) - 1):
        r0, r1 = offsets[e], offsets[e + 1]
        m_tiles = _cdiv(r1 - r0, BM)
        for u in range(m_tiles * n_tiles):
            m_blk, n_blk = grouped_tile(u, m_tiles, n_tiles, gn)
            tiles.append((e, m_blk, n_blk, r0 + m_blk * BM, r1))
    return tiles


def moe_plan(kernel, rows, E, N, K, bits=16):
    """(n_tiles, gn, units, grid) of one grouped launch: launch_moe for 'dense-swiglu' / 'dense-down'
    (BN = 256 output columns; gate/up tiles are 128 act columns), launch_moe_packed for
    'packed-swiglu' / 'packed-down' (BN = 128; gate/up tiles are 64 act columns).  N is the output
    width (inter for gate/up), K the reduction depth."""
    n_tiles, div = {
        'dense-swiglu': (N // 128, 256 * K * 2),
        'dense-down': (_cdiv(N, 256), 256 * K * 2),
        'packed-swiglu': (N // 64, 128 * K * bits // 8 + 1),
        'packed-down': (_cdiv(N, 128), 128 * K * bits // 8 + 1),
    }[kernel]
    units = (_cdiv(rows, BM) + E) * n_tiles
    return n_tiles, l2_group_width(div, n_tiles), units, min(units, NUM_SMS)


def kernel_cases(kernel, offsets, N, K, bits=16):
    """The cases one grouped launch reaches.  Also checks the restated plan: every tile of every
    expert comes exactly once, within the launched units."""
    rows, E = offsets[-1], len(offsets) - 1
    n_tiles, gn, units, grid = moe_plan(kernel, rows, E, N, K, bits)
    tiles = moe_tiles(offsets, n_tiles, gn)
    assert len(tiles) <= units, (kernel, offsets, len(tiles), units)
    for e in range(E):
        m_tiles = _cdiv(offsets[e + 1] - offsets[e], BM)
        assert sorted(t[1:3] for t in tiles if t[0] == e) == \
            [(m, n) for m in range(m_tiles) for n in range(n_tiles)], (kernel, e)
    sizes = [offsets[e + 1] - offsets[e] for e in range(E)]
    cases = {'E1'} if E == 1 else set()
    if E < 8:
        cases.add('E<8')
    if 0 in sizes:
        cases.add('empty-expert')
    if sizes[0] == 0:
        cases.add('leading-empty')
    if sizes[-1] == 0:
        cases.add('trailing-empty')
    if 1 in sizes:
        cases.add('one-row-segment')
    if E > 1 and rows in sizes:
        cases.add('all-rows-one-expert')
    if max(sizes) > BM:
        cases.add('multi-m-tile')
    for e, m_blk, n_blk, row0, row_end in tiles:
        if row0 + BM > row_end and row_end < rows:
            cases.add('straddle')         # the tile's last A rows are the next expert's
        if row0 + BM > rows:
            cases.add('tail-past-rows')   # TMA zero-fills A rows past `rows`
        if row_end - row0 <= 64:
            cases.add('wg1-empty')        # the second consumer warpgroup stores nothing
    if len(tiles) > NUM_SMS:
        cases.add('persistent')
    if len(tiles) < grid:
        cases.add('idle-ctas')
    if n_tiles % gn:
        cases.add('partial-group')
    elif n_tiles // gn >= 2:
        cases.add('full-groups')
    kb = _cdiv(K, 64)
    if kb == 1:
        cases.add('one-kb')
    if kernel.startswith('dense'):
        if K % 64:
            cases.add('k-tail')
        if kernel == 'dense-down' and N % 256:
            cases.add('partial-n')
    else:
        if kernel == 'packed-down' and N % 128:
            cases.add('partial-n')
        # the two dequant groups take alternate K steps counted across a CTA's tiles: with an odd
        # step count the next tile, here another expert's, starts on the other group
        if kb % 2 and any(a[0] != b[0] for c in range(grid) for a, b in
                          zip(tiles[c::grid], tiles[c + grid::grid])):
            cases.add('odd-kb')
    return cases


def offsets_of(sizes):
    out = [0]
    for s in sizes:
        out.append(out[-1] + s)
    return out


def dense_cases(sizes, hidden, inter):
    o = offsets_of(sizes)
    return kernel_cases('dense-swiglu', o, inter, hidden) | kernel_cases('dense-down', o, hidden, inter)


def packed_cases(sizes, hidden, inter, bits):
    o = offsets_of(sizes)
    return (kernel_cases('packed-swiglu', o, inter, hidden, bits)
            | kernel_cases('packed-down', o, hidden, inter, bits))


def combine_cases(T, k, N):
    chunks = T * (N // 8)
    cases = {'top_k>=3'} if k >= 3 else set()
    if k == 1:
        cases.add('top_k1')
    if chunks > COMBINE_THREADS:
        cases.add('grid-stride')
    if chunks % 256:
        cases.add('partial-block')
    return cases


SEGMENT_CASES = {'empty-expert', 'leading-empty', 'trailing-empty', 'one-row-segment',
                 'all-rows-one-expert', 'multi-m-tile', 'straddle', 'tail-past-rows', 'wg1-empty',
                 'persistent', 'idle-ctas', 'partial-group', 'full-groups', 'partial-n', 'one-kb',
                 'E1', 'E<8'}

# ---- path tables ---------------------------------------------------------------------------------
DENSE_PATHS = [
    # name, segment sizes (one per expert), hidden, inter, cases: gate/up is [rows, hidden] ->
    # [rows, inter], down [rows, inter] -> [rows, hidden]
    ('e1-one-row-one-kb', [1], 64, 128,
     {'E1', 'one-row-segment', 'one-kb', 'wg1-empty', 'tail-past-rows', 'idle-ctas', 'partial-n'}),
    ('e1-k8', [200], 8, 256, {'E1', 'multi-m-tile', 'one-kb', 'k-tail', 'partial-n'}),
    ('e3-leading-empty-k-tail', [0, 130, 5], 264, 128,
     {'E<8', 'leading-empty', 'empty-expert', 'multi-m-tile', 'straddle', 'wg1-empty', 'k-tail',
      'partial-n'}),
    ('e5-trailing-empty-k56', [64, 65, 1, 200, 0], 56, 384,
     {'trailing-empty', 'one-row-segment', 'straddle', 'one-kb', 'k-tail', 'partial-n'}),
    ('e4-all-rows-one-expert', [0, 0, 517, 0], 520, 384,
     {'all-rows-one-expert', 'leading-empty', 'trailing-empty', 'tail-past-rows', 'k-tail',
      'partial-n'}),
    ('e8-mixtral-sizes-partial-group', [0, 1, 63, 64, 127, 128, 129, 300], 4096, 2176,
     {'partial-group', 'persistent', 'straddle', 'wg1-empty', 'leading-empty'}),
    ('e3-down-partial-group-partial-n', [300, 0, 700], 4104, 14336,
     {'partial-group', 'partial-n', 'k-tail', 'persistent', 'empty-expert'}),
    ('e2-full-groups', [129, 1000], 4096, 14336, {'full-groups', 'persistent', 'straddle'}),
]

PACKED_PATHS = [
    # name, bits, group (negative: qparams [ng, N]; at least K: per channel), g_idx, zeros, native
    # qparams, sizes, hidden, inter, cases
    ('w4-e1-inter64-one-kb', 4, 64, False, True, True, [60], 192, 64,
     {'E1', 'one-kb', 'partial-n', 'wg1-empty', 'tail-past-rows', 'idle-ctas'}),
    ('w8-e5-odd-kb-persistent', 8, -64, False, True, False, [300, 1, 257, 0, 64], 320, 2048,
     {'odd-kb', 'persistent', 'one-row-segment', 'empty-expert', 'straddle', 'partial-n'}),
    ('w4-gidx-odd-kb', 4, 64, True, False, False, [1, 150, 0, 99, 200, 3, 64], 448, 1152,
     {'odd-kb', 'persistent', 'E<8', 'straddle', 'wg1-empty', 'partial-n'}),
    ('w8-gidx-leading-trailing-empty', 8, -128, True, True, True, [0, 129, 0, 0], 256, 128,
     {'leading-empty', 'trailing-empty', 'all-rows-one-expert', 'multi-m-tile', 'tail-past-rows'}),
    ('w4-e8-mixtral-sizes', 4, -64, False, False, True, [0, 1, 63, 64, 127, 128, 129, 300], 704, 1216,
     {'leading-empty', 'one-row-segment', 'straddle', 'partial-n', 'odd-kb', 'persistent'}),
    ('w4-partial-group', 4, 128, False, True, True, [129, 200], 4096, 14336,
     {'partial-group', 'persistent', 'multi-m-tile'}),
    ('w4-full-groups-per-channel', 4, 1 << 20, False, False, False, [300, 41], 4096, 16256,
     {'full-groups', 'persistent', 'straddle'}),
]

COMBINE_PATHS = [
    # name, T, top_k, N, rows of y, cases
    ('t1-k1-n8', 1, 1, 8, 1, {'top_k1', 'partial-block'}),
    ('t77-k2-n264', 77, 2, 264, 200, {'partial-block'}),
    ('t300-k3-n520', 300, 3, 520, 900, {'top_k>=3', 'partial-block'}),
    ('t129-k8-n4096', 129, 8, 4096, 1032, {'top_k>=3'}),
    ('t2200-k2-grid-stride', 2200, 2, 4096, 4400, {'grid-stride'}),
    ('t2200-k5-grid-stride', 2200, 5, 4096, 11000, {'grid-stride', 'top_k>=3'}),
]


def test_path_tables_reach_their_cases():
    """No GPU: every entry reaches the cases it names, and the tables together claim every case."""
    for name, sizes, hidden, inter, want in DENSE_PATHS:
        assert want <= dense_cases(sizes, hidden, inter), (name, want - dense_cases(sizes, hidden, inter))
    for name, bits, group, gidx, zeros, native, sizes, hidden, inter, want in PACKED_PATHS:
        assert all(K % min(abs(group), K) == 0 for K in (hidden, inter)), name
        got = packed_cases(sizes, hidden, inter, bits)
        assert want <= got, (name, want - got)
    for name, T, k, N, R, want in COMBINE_PATHS:
        assert want <= combine_cases(T, k, N), (name, want - combine_cases(T, k, N))
    claimed_dense = set().union(*(p[-1] for p in DENSE_PATHS))
    claimed_packed = set().union(*(p[-1] for p in PACKED_PATHS))
    assert SEGMENT_CASES | {'k-tail'} <= claimed_dense, SEGMENT_CASES | {'k-tail'} - claimed_dense
    assert SEGMENT_CASES | {'odd-kb'} <= claimed_packed, SEGMENT_CASES | {'odd-kb'} - claimed_packed
    assert {'top_k>=3', 'top_k1', 'grid-stride'} <= set().union(*(p[-1] for p in COMBINE_PATHS))


def test_restated_plan_at_mixtral_widths():
    """No GPU: the raster widths the launch plans give at Mixtral-8x7B's widths."""
    assert moe_plan('dense-swiglu', 1000, 8, 2176, 4096)[:2] == (17, 16)
    assert moe_plan('dense-swiglu', 1000, 8, 14336, 4096)[:2] == (112, 16)
    assert moe_plan('dense-down', 1000, 8, 4104, 14336)[:2] == (17, 4)
    assert moe_plan('packed-swiglu', 1000, 8, 14336, 4096, 4)[:2] == (224, 127)
    # the units bound: ceil(rows / 128) + E m-tiles per column of n-tiles, grid at most 132
    assert moe_plan('packed-down', 1, 1, 8, 64, 8) == (1, 1, 2, 2)
    assert moe_plan('dense-down', 300, 3, 264, 128)[2:] == (12, 12)
    assert moe_plan('dense-swiglu', 10000, 8, 14336, 4096)[2:] == ((79 + 8) * 112, 132)


# ---- helpers -------------------------------------------------------------------------------------
def _ptrs(ts):
    """A host array of device pointers, as the grouped entry points take them."""
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _ptrs_or_null(ts):
    return None if ts is None else _ptrs(ts)


def _guarded(rows, N, dtype):
    """[rows + GUARD, N] of SENTINEL."""
    return torch.full((rows + GUARD, N), SENTINEL, dtype=torch.int16, device='cuda').view(dtype)


def _check_guarded(buf, rows, exp, what, sample=None):
    """Rows 0 .. rows - 1 (or those in `sample`) all written and equal to exp bit for bit, the
    guard rows untouched."""
    bits = buf.view(torch.int16)
    assert bool((bits[rows:] == SENTINEL).all()), f'{what}: a guard row was written'
    got = buf[:rows] if sample is None else buf[sample]
    assert not bool((got.view(torch.int16) == SENTINEL).any()), f'{what}: a row was not written'
    _same(got, exp, what)


def _seg_of(offsets, rows=None):
    """The expert of each row (of `rows`, default all), as a CPU int64 tensor."""
    o = torch.tensor(offsets)
    r = torch.arange(offsets[-1]) if rows is None else rows.cpu()
    return torch.searchsorted(o, r, right=True) - 1


def _swiglu_ref(G, U, dtype):
    """act = F.silu(rT(G)) * rT(U) on the GPU, as silu_mul_f32<DT, true> computes it."""
    return F.silu(G.to(dtype)) * U.to(dtype)


def _routed_ref(S, w, dtype):
    """y = rT(rT(S) * w[row]): the fp64 product of two 16-bit values is exact."""
    return (S.to(dtype).double() * w.double()[:, None]).to(dtype)


def _swiglu_range(K, dtype):
    """Activation / weight magnitude of the gate/up grid: test_gpu_gemm_paths' for bf16; for fp16
    a typical |G|, |U| ~ 40, so that silu(G) * U stays mostly finite."""
    if dtype == torch.bfloat16:
        return _int_range(K, dtype)
    r = 1
    while (r + 1) * (r + 2) / 3 <= 40 / math.sqrt(K):
        r += 1
    return r


def route_weights(rows, dtype, g):
    """Routing weights [rows]: random fractions, with every 5th row a value edge in turn: 1, powers
    of two, 0, -0, negative values, the smallest subnormal, the largest finite value (fp16: its
    products overflow), inf and NaN."""
    fi = torch.finfo(dtype)
    edges = [1.0, 0.5, 2.0, 0.0, -0.0, -1.0, -0.625, 0.125, fi.tiny * fi.eps, -fi.tiny * fi.eps,
             fi.max, -fi.max, 4.0, float('inf'), float('nan'), 1.0 / 3]
    w = (torch.rand(rows, generator=g, device='cuda') * 1.5 - 0.25).double()
    idx = torch.arange(0, rows, 5, device='cuda')
    e = torch.tensor(edges, dtype=torch.float64, device='cuda')
    w[idx] = e[torch.arange(idx.numel(), device='cuda') % len(edges)]
    return w.to(dtype)


def _distinguishes_experts(ref_fn, E, what):
    """The expected output with every segment on its neighbour's weight differs almost everywhere:
    a tile that takes another expert's weight cannot pass."""
    if E < 2:
        return
    same, total = 0, 0
    for e in range(E):
        a, b = ref_fn(e, e), ref_fn(e, (e + 1) % E)
        same += int((a == b).sum())
        total += a.numel()
    assert total == 0 or same < 0.1 * total, (what, same, total)


# ---- the dense grouped GEMM ----------------------------------------------------------------------
class DenseExperts:
    """E experts on the integer grid: w1 / w3 [inter, hidden], w2 [hidden, inter] in dtype."""

    def __init__(self, E, hidden, inter, dtype, key=()):
        g = _gen('moe-dense', E, hidden, inter, str(dtype), key)
        r1 = _swiglu_range(hidden, dtype)
        r2 = _int_range(inter, dtype)
        self.r1, self.r2 = r1, r2
        self.w1 = [_randint(-r1, r1, (inter, hidden), g).to(dtype) for _ in range(E)]
        self.w3 = [_randint(-r1, r1, (inter, hidden), g).to(dtype) for _ in range(E)]
        self.w2 = [_randint(-r2, r2, (hidden, inter), g).to(dtype) for _ in range(E)]
        self.g, self.E, self.hidden, self.inter, self.dtype = g, E, hidden, inter, dtype


def dense_swiglu(xp, w1, w3, offsets, act, inter):
    rows, K = xp.shape
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    call('llmc_moe_gemm_swiglu', ctypes.c_void_p(xp.data_ptr()), _ptrs(w1), _ptrs(w3),
         ctypes.c_void_p(off.data_ptr()), ctypes.c_void_p(act.data_ptr()), rows, inter, K, len(w1),
         dtype_enum(xp.dtype), stream_ptr())


def dense_down(act, w2, offsets, w_route, y, N):
    rows, inter = act.shape
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    call('llmc_moe_gemm_down', ctypes.c_void_p(act.data_ptr()), _ptrs(w2), ctypes.c_void_p(off.data_ptr()),
         ctypes.c_void_p(w_route.data_ptr()), ctypes.c_void_p(y.data_ptr()), rows, N, inter, len(w2),
         dtype_enum(act.dtype), stream_ptr())


def check_dense(ex, offsets, what):
    """Both dense grouped GEMMs over the segments `offsets` against the oracle."""
    rows, E, dt = offsets[-1], ex.E, ex.dtype
    hidden, inter = ex.hidden, ex.inter
    xp = _randint(-ex.r1, ex.r1, (rows, hidden), ex.g)
    act_in = _randint(-ex.r2, ex.r2, (rows, inter), ex.g)
    w_route = route_weights(rows, dt, ex.g)

    def seg(e):
        return slice(offsets[e], offsets[e + 1])

    def G(e, f):
        return xp[seg(e)] @ ex.w1[f].double().t() + 0.0

    def U(e, f):
        return xp[seg(e)] @ ex.w3[f].double().t() + 0.0

    def S(e, f):
        return act_in[seg(e)] @ ex.w2[f].double().t() + 0.0

    _distinguishes_experts(G, E, what + ' w1')
    _distinguishes_experts(S, E, what + ' w2')
    act_ref = torch.cat([_swiglu_ref(G(e, e), U(e, e), dt) for e in range(E)])
    S_all = torch.cat([S(e, e) for e in range(E)])
    _nontrivial(S_all, dt, what)
    y_ref = _routed_ref(S_all, w_route, dt)
    fused = (S_all * w_route.double()[:, None]).to(dt)
    differs = ~((y_ref == fused) | (torch.isnan(y_ref) & torch.isnan(fused)))
    assert rows < 64 or bool(differs.any()), f'{what}: rT(rT(S) w) and rT(S w) agree everywhere'

    act = _guarded(rows, inter, dt)
    dense_swiglu(xp.to(dt), ex.w1, ex.w3, offsets, act[:rows], inter)
    _check_guarded(act, rows, act_ref, what + ' gate/up')
    y = _guarded(rows, hidden, dt)
    dense_down(act_in.to(dt), ex.w2, offsets, w_route, y[:rows], hidden)
    _check_guarded(y, rows, y_ref, what + ' down')


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,sizes,hidden,inter,want', DENSE_PATHS, ids=[p[0] for p in DENSE_PATHS])
def test_dense_path_table(name, sizes, hidden, inter, want, dtype):
    assert want <= dense_cases(sizes, hidden, inter)
    ex = DenseExperts(len(sizes), hidden, inter, dtype, key=name)
    check_dense(ex, offsets_of(sizes), name)
    del ex
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_dense_grid_sweep(dtype):
    """hidden 8 .. 520 (one k-step, K tails, partial n-tiles of the down projection) x inter
    128 / 256 / 384 x expert counts 1 .. 8 with random segment sizes, empty ones included."""
    g = torch.Generator().manual_seed(11)
    i = 0
    for hidden in (8, 56, 64, 72, 264, 520):
        for inter in (128, 256, 384):
            E = 1 + i % 8
            i += 1
            sizes = torch.randint(0, 150, (E,), generator=g)
            sizes[torch.rand(E, generator=g) < 0.25] = 0
            sizes = [int(s) for s in sizes]
            if sum(sizes) == 0:
                sizes[-1] = 1
            ex = DenseExperts(E, hidden, inter, dtype, key=('sweep', i))
            check_dense(ex, offsets_of(sizes), f'hidden={hidden} inter={inter} sizes={sizes}')


# ---- the grouped dequant GEMM on packed experts --------------------------------------------------
class PackedLinear:
    """One expert linear [N, K] on test_gpu_gemm_paths.WGrid's grid: codes and zero-points in
    [0, 2^bits), scales 2^-3 .. 2^1, so every dequantised weight is exact in bf16 / fp16.  Groups of
    `group` columns, contiguous or (gidx) scattered by the linear's own random permutation; zeros
    False: symmetric (the kernel's 2^(bits-1))."""

    def __init__(self, N, K, bits, group, gidx, zeros, dtype, g):
        qmax = (1 << bits) - 1
        assert K % group == 0, (K, group)
        ng = K // group
        codes = _randint(0, qmax, (N, K), g)
        self.scales = torch.pow(2.0, _randint(-3, 1, (N, ng), g))
        self.zeros = _randint(0, qmax, (N, ng), g) if zeros else None
        cg = (torch.randperm(K, generator=g, device='cuda') if gidx
              else torch.arange(K, device='cuda')) // group
        z = self.zeros if zeros else torch.full((N, ng), float(1 << (bits - 1)), device='cuda',
                                                dtype=torch.float64)
        self.w = ((codes - z[:, cg]) * self.scales[:, cg]).to(dtype)     # exact
        self.wq = pack_codes(codes, bits)
        self.g_idx = cg.to(torch.int32) if gidx else None
        self.ng = ng

    def qparams(self, qdt, transposed):
        s = self.scales.to(qdt)
        z = self.zeros.to(qdt) if self.zeros is not None else None
        if transposed:
            s = s.t().contiguous()
            z = z.t().contiguous() if z is not None else None
        return s, z


class PackedExperts:
    """E experts of one form: w1 / w3 [inter, hidden], w2 [hidden, inter].  group < 0: qparams
    stored [ng, N]; per-channel: group = K of each linear."""

    def __init__(self, E, hidden, inter, bits, group, gidx, zeros, native, dtype, key=()):
        g = _gen('moe-packed', E, hidden, inter, bits, group, gidx, zeros, native, str(dtype), key)
        self.transposed = group < 0
        ag = abs(group)
        self.group1, self.group2 = min(ag, hidden), min(ag, inter)

        def lin(N, K, grp):
            return PackedLinear(N, K, bits, grp, gidx, zeros, dtype, g)
        self.w1 = [lin(inter, hidden, self.group1) for _ in range(E)]
        self.w3 = [lin(inter, hidden, self.group1) for _ in range(E)]
        self.w2 = [lin(hidden, inter, self.group2) for _ in range(E)]
        self.qdt = dtype if native else torch.float32
        wmax = ((1 << bits) - 1) * 2
        # every partial sum below 2^24 units of 2^-3 (checked where the range is used)
        self.r1 = min(64, (EXACT_LIMIT // 8 - 256) // (hidden * wmax))
        self.r2 = min(64, (EXACT_LIMIT // 8 - 256) // (inter * wmax))
        self.g, self.E, self.bits, self.hidden, self.inter, self.dtype = g, E, bits, hidden, inter, dtype

    def operands(self, lins, group):
        """(qparam copies, (wq, scales, zeros, g_idx) host pointer arrays, (qparam dtype, group,
        ng)).  The caller holds the copies until the launch is queued: freed earlier, the caching
        allocator hands their memory to the next copies while the pointer arrays still name it."""
        qp = [lin.qparams(self.qdt, self.transposed) for lin in lins]
        arrs = (_ptrs([lin.wq for lin in lins]), _ptrs([s for s, _ in qp]),
                _ptrs_or_null(None if qp[0][1] is None else [z for _, z in qp]),
                _ptrs_or_null(None if lins[0].g_idx is None else [lin.g_idx for lin in lins]))
        return qp, arrs, (dtype_enum(self.qdt), -group if self.transposed else group, lins[0].ng)


def packed_swiglu(ex, xp, offsets, act):
    rows = xp.shape[0]
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    q1, (wq1, s1, z1, g1), (qd, grp, ng) = ex.operands(ex.w1, ex.group1)
    q3, (wq3, s3, z3, g3), _ = ex.operands(ex.w3, ex.group1)
    call('llmc_moe_gemm_packed_swiglu', ctypes.c_void_p(xp.data_ptr()), ex.bits, wq1, wq3, s1, s3, z1,
         z3, g1, g3, qd, grp, ng, ctypes.c_void_p(off.data_ptr()), ctypes.c_void_p(act.data_ptr()),
         rows, ex.inter, ex.hidden, ex.E, dtype_enum(xp.dtype), stream_ptr())


def packed_down(ex, act_in, offsets, w_route, y):
    rows = act_in.shape[0]
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    q2, (wq2, s2, z2, g2), (qd, grp, ng) = ex.operands(ex.w2, ex.group2)
    call('llmc_moe_gemm_packed_down', ctypes.c_void_p(act_in.data_ptr()), ex.bits, wq2, s2, z2, g2, qd,
         grp, ng, ctypes.c_void_p(off.data_ptr()), ctypes.c_void_p(w_route.data_ptr()),
         ctypes.c_void_p(y.data_ptr()), rows, ex.hidden, ex.inter, ex.E, dtype_enum(act_in.dtype),
         stream_ptr())


def check_packed(ex, offsets, what):
    """Both grouped dequant GEMMs over the segments `offsets` against the oracle."""
    rows, E, dt = offsets[-1], ex.E, ex.dtype
    assert ex.r1 >= 1 and ex.r2 >= 1, (what, ex.r1, ex.r2)
    xp = _randint(-ex.r1, ex.r1, (rows, ex.hidden), ex.g)
    act_in = _randint(-ex.r2, ex.r2, (rows, ex.inter), ex.g)
    w_route = route_weights(rows, dt, ex.g)

    def seg(e):
        return slice(offsets[e], offsets[e + 1])

    def G(e, f):
        return xp[seg(e)] @ ex.w1[f].w.double().t() + 0.0

    def U(e, f):
        return xp[seg(e)] @ ex.w3[f].w.double().t() + 0.0

    def S(e, f):
        return act_in[seg(e)] @ ex.w2[f].w.double().t() + 0.0

    _distinguishes_experts(G, E, what + ' w1')
    _distinguishes_experts(S, E, what + ' w2')
    e = next(e for e in range(E) if offsets[e + 1] > offsets[e])
    assert (G(e, e) != U(e, e)).double().mean() > 0.9, what      # w1 and w3 tell apart too
    act_ref = torch.cat([_swiglu_ref(G(e, e), U(e, e), dt) for e in range(E)])
    y_ref = _routed_ref(torch.cat([S(e, e) for e in range(E)]), w_route, dt)

    act = _guarded(rows, ex.inter, dt)
    packed_swiglu(ex, xp.to(dt), offsets, act[:rows])
    _check_guarded(act, rows, act_ref, what + ' gate/up')
    y = _guarded(rows, ex.hidden, dt)
    packed_down(ex, act_in.to(dt), offsets, w_route, y[:rows])
    _check_guarded(y, rows, y_ref, what + ' down')


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,bits,group,gidx,zeros,native,sizes,hidden,inter,want', PACKED_PATHS,
                         ids=[p[0] for p in PACKED_PATHS])
def test_packed_path_table(name, bits, group, gidx, zeros, native, sizes, hidden, inter, want, dtype):
    assert want <= packed_cases(sizes, hidden, inter, bits)
    ex = PackedExperts(len(sizes), hidden, inter, bits, group, gidx, zeros, native, dtype, key=name)
    check_packed(ex, offsets_of(sizes), name)
    del ex
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('bits', [4, 8])
def test_packed_form_sweep(bits, dtype):
    """Every form: groups of 64 / 128 / K (per channel) / g_idx x fp32 or native qparams x [N, ng] or
    [ng, N] x zero-points or symmetric, on segments that rotate through the edges."""
    hidden, inter = 256, 128
    layouts = ([3, 0, 130], [0, 64, 65, 1], [200], [0, 0, 1, 70, 0, 129, 2, 0], [129, 0, 0, 0, 0])
    i = 0
    for group in (64, 128, 1 << 20, 'gidx'):
        for native in (False, True):
            for transposed in (False, True):
                for zeros in (True, False):
                    sizes = layouts[i % len(layouts)]
                    i += 1
                    gidx = group == 'gidx'
                    grp = 64 if gidx else group
                    ex = PackedExperts(len(sizes), hidden, inter, bits, -grp if transposed else grp,
                                       gidx, zeros, native, dtype, key=('sweep', i))
                    check_packed(ex, offsets_of(sizes), f'group={group} native={native} '
                                 f'transposed={transposed} zeros={zeros} sizes={sizes}')


# ---- the combine ---------------------------------------------------------------------------------
def combine_ref(y, rows, dtype):
    """out[t] = rT(... rT(rT(0 + y[rows[t, 0]]) + y[rows[t, 1]]) ...): sequential fp32 adds on the
    CPU, rounded after each, in slot order."""
    yc, rc = y.cpu().float(), rows.cpu()
    acc = torch.zeros(rc.shape[0], y.shape[1])
    for s in range(rc.shape[1]):
        acc = (acc + yc[rc[:, s]]).to(dtype).float()
    return acc.to(dtype)


def combine(y, rows, out):
    T, k = rows.shape
    call('llmc_moe_combine', ctypes.c_void_p(y.data_ptr()), ctypes.c_void_p(rows.data_ptr()),
         ctypes.c_void_p(out.data_ptr()), T, k, y.shape[1], dtype_enum(y.dtype), stream_ptr())


def combine_inputs(T, k, N, R, dtype, key=()):
    """y [R, N] and rows [T, k] (distinct rows of y in random order) whose chains meet every value
    edge: an all-(-0) token, inf + (-inf), overflow partway through a chain, subnormals, big + small
    - big, NaN; the rest of mixed magnitude so that the order of the adds matters."""
    g = _gen('combine', T, k, N, R, str(dtype), key)
    fi = torch.finfo(dtype)
    big = 2.0 ** (12 if dtype == torch.float16 else 40)
    mag = torch.pow(2.0, _randint(-4, int(math.log2(big)), (R, N), g))
    y = (_randint(-7, 7, (R, N), g) * mag).to(dtype)
    rows = torch.randperm(R, generator=g, device='cuda')[:T * k].view(T, k).contiguous()
    sub = fi.tiny * fi.eps
    specials = [
        [-0.0] * k,                                               # -> +0: the sum starts from 0.f
        [float('inf'), float('-inf')] + [1.0] * (k - 2),          # -> NaN
        [fi.max * 0.75, fi.max * 0.75, -fi.max * 0.75] + [0.0] * (k - 3),   # overflow, then stays inf
        [sub, -3 * sub, 0.5 * fi.tiny] + [sub] * (k - 3),         # subnormal sums
        [big, 1.0, -big] + [0.25] * (k - 3),                      # big + small - big
        [float('nan')] + [1.0] * (k - 1),
        [1.0] + [-0.0] * (k - 1),
    ]
    for t, vals in enumerate(specials[:T]):
        vals = vals[:k]
        for s, v in enumerate(vals):
            y[rows[t, s], : N // 2] = v
    return y, rows


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('name,T,k,N,R,want', COMBINE_PATHS, ids=[p[0] for p in COMBINE_PATHS])
def test_combine_path_table(name, T, k, N, R, want, dtype):
    assert want <= combine_cases(T, k, N)
    y, rows = combine_inputs(T, k, N, R, dtype, key=name)
    ref = combine_ref(y, rows, dtype).cuda()
    if k >= 3:                          # two slots commute: rT(0 + a) = a
        rev = combine_ref(y, rows.flip(1), dtype).cuda()
        differs = ~((rev == ref) | (torch.isnan(rev) & torch.isnan(ref)))
        assert bool(differs.any()), f'{name}: the slot order does not matter to this data'
    if T >= 7 and k >= 2:
        hb = N // 2
        assert bool((ref[0, :hb].view(torch.int16) == 0).all())            # +0, not -0
        assert bool(torch.isnan(ref[1, :hb]).all())
        if k >= 3:
            assert bool(torch.isinf(ref[2, :hb]).all())
    out = _guarded(T, N, dtype)
    combine(y, rows, out[:T])
    _check_guarded(out, T, ref, name)


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
def test_combine_top_k_sweep(dtype):
    """top_k 1 .. 8 at ragged T and N, each token's slots in shuffled order."""
    for k in range(1, 9):
        for T, N in ((1, 8), (7, 24), (300, 264)):
            y, rows = combine_inputs(T, k, N, T * k, dtype, key=('sweep', k))
            rows = rows[:, torch.randperm(k, generator=torch.Generator().manual_seed(k)).cuda()]
            rows = rows.contiguous()
            out = _guarded(T, N, dtype)
            combine(y, rows, out[:T])
            _check_guarded(out, T, combine_ref(y, rows, dtype).cuda(), f'k={k} T={T} N={N}')


# ---- argument edges ------------------------------------------------------------------------------
@gpu
def test_zero_rows_and_zero_tokens_launch_nothing():
    """rows == 0 (every segment empty) and T == 0 return without a launch or a write."""
    from llmc_b200._lib import load
    lib = load()
    dt = torch.bfloat16
    ex = DenseExperts(3, 64, 128, dt, key='zero')
    px = PackedExperts(2, 128, 64, 4, 64, False, True, True, dt, key='zero')
    empty = torch.empty(0, 128, dtype=dt, device='cuda')
    buf = _guarded(0, 128, dt)
    torch.cuda.synchronize()
    before = lib.llmc_b200_launch_count()
    dense_swiglu(torch.empty(0, 64, dtype=dt, device='cuda'), ex.w1, ex.w3, [0, 0, 0, 0], buf, 128)
    dense_down(empty, ex.w2, [0, 0, 0, 0], torch.empty(0, dtype=dt, device='cuda'), buf[:, :64], 64)
    packed_swiglu(px, empty, [0, 0, 0], buf[:, :64])
    packed_down(px, torch.empty(0, 64, dtype=dt, device='cuda'), [0, 0, 0],
                torch.empty(0, dtype=dt, device='cuda'), buf)
    combine(empty, torch.empty(0, 2, dtype=torch.int64, device='cuda'), buf)
    torch.cuda.synchronize()
    assert lib.llmc_b200_launch_count() == before
    assert bool((buf.view(torch.int16) == SENTINEL).all())


@gpu
def test_expert_count_outside_one_to_eight_is_refused():
    from llmc_b200._lib import MOE_MAX_EXPERTS, LlmcB200Error
    dt = torch.bfloat16
    ex = DenseExperts(MOE_MAX_EXPERTS + 1, 64, 128, dt, key='nine')
    xp = torch.zeros(4, 64, dtype=dt, device='cuda')
    act = _guarded(4, 128, dt)
    with pytest.raises(LlmcB200Error, match='experts outside'):
        dense_swiglu(xp, ex.w1, ex.w3, [0] * MOE_MAX_EXPERTS + [4, 4], act[:4], 128)
    with pytest.raises(LlmcB200Error, match='experts outside'):
        dense_swiglu(xp, [], [], [4], act[:4], 128)
    assert bool((act.view(torch.int16) == SENTINEL).all())


# ---- offsets past 2^31 elements ------------------------------------------------------------------
def _sample_rows(offsets, extra, g):
    """Every segment's first and last rows, the last row, and `extra` random ones."""
    rows = offsets[-1]
    picks = {rows - 1}
    for e in range(len(offsets) - 1):
        if offsets[e + 1] > offsets[e]:
            picks.update((offsets[e], offsets[e + 1] - 1))
    picks.update(torch.randint(0, rows, (extra,), generator=g).tolist())
    return torch.tensor(sorted(picks), device='cuda')


def _large_grid(shape, r, dtype, g):
    """An integer tensor in [-r, r] of dtype, filled in place (no fp64 / int64 copy of its size)."""
    t = torch.empty(shape, dtype=dtype, device='cuda')
    return t.random_(-r, r + 1, generator=g)


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


LARGE_SWIGLU = ([1, 80000, 0, 70015], 64, 14336)     # act: 150,016 x 14336 = 2.15e9 elements
LARGE_DOWN = ([65603, 65597], 16384, 128)            # y: 131,200 x 16384 = 2.15e9 elements


@gpu
@pytest.mark.parametrize('kind', ['dense', 'packed'])
def test_gate_up_output_past_2_31_elements(kind):
    sizes, hidden, inter = LARGE_SWIGLU
    offsets = offsets_of(sizes)
    rows = offsets[-1]
    assert rows * inter > 2 ** 31
    dt = torch.bfloat16
    g = _gen('large-swiglu', kind)
    if kind == 'dense':
        ex = DenseExperts(len(sizes), hidden, inter, dt, key='large')
        w1, w3 = [w.double() for w in ex.w1], [w.double() for w in ex.w3]
        r = ex.r1
    else:
        ex = PackedExperts(len(sizes), hidden, inter, 4, 64, False, True, True, dt, key='large')
        w1, w3 = [lin.w.double() for lin in ex.w1], [lin.w.double() for lin in ex.w3]
        r = ex.r1
    xp = _large_grid((rows, hidden), r, dt, g)
    act = _guarded(rows, inter, dt)
    if kind == 'dense':
        dense_swiglu(xp, ex.w1, ex.w3, offsets, act[:rows], inter)
    else:
        packed_swiglu(ex, xp, offsets, act[:rows])
    pick = _sample_rows(offsets, 64, torch.Generator().manual_seed(1))
    seg = _seg_of(offsets, pick).tolist()
    x = xp[pick].double()
    G = torch.stack([x[i] @ w1[e].t() for i, e in enumerate(seg)]) + 0.0
    U = torch.stack([x[i] @ w3[e].t() for i, e in enumerate(seg)]) + 0.0
    _check_guarded(act, rows, _swiglu_ref(G, U, dt), f'{kind} gate/up rows={rows}', sample=pick)
    del act, xp, ex
    _free()


@gpu
@pytest.mark.parametrize('kind', ['dense', 'packed'])
def test_down_output_past_2_31_elements(kind):
    sizes, hidden, inter = LARGE_DOWN
    offsets = offsets_of(sizes)
    rows = offsets[-1]
    assert rows * hidden > 2 ** 31
    dt = torch.bfloat16
    g = _gen('large-down', kind)
    if kind == 'dense':
        ex = DenseExperts(len(sizes), hidden, inter, dt, key='large')
        w2, r = [w.double() for w in ex.w2], ex.r2
    else:
        ex = PackedExperts(len(sizes), hidden, inter, 8, -128, True, True, False, dt, key='large')
        w2, r = [lin.w.double() for lin in ex.w2], ex.r2
        assert r >= 1
    act_in = _large_grid((rows, inter), r, dt, g)
    w_route = route_weights(rows, dt, g)
    y = _guarded(rows, hidden, dt)
    if kind == 'dense':
        dense_down(act_in, ex.w2, offsets, w_route, y[:rows], hidden)
    else:
        packed_down(ex, act_in, offsets, w_route, y[:rows])
    pick = _sample_rows(offsets, 64, torch.Generator().manual_seed(2))
    seg = _seg_of(offsets, pick).tolist()
    a = act_in[pick].double()
    S = torch.stack([a[i] @ w2[e].t() for i, e in enumerate(seg)]) + 0.0
    _check_guarded(y, rows, _routed_ref(S, w_route[pick], dt), f'{kind} down rows={rows}', sample=pick)
    del y, act_in, ex
    _free()


@gpu
def test_combine_output_past_2_31_elements():
    """131,200 tokens x 16384, top_k 2 over a 131,200-row y: both the y rows read and the out rows
    written lie past 2^31 elements."""
    T, k, N = 131200, 2, 16384
    assert T * N > 2 ** 31
    dt = torch.bfloat16
    g = _gen('large-combine')
    y = _large_grid((T, N), 64, dt, g)
    rows = torch.stack([torch.randperm(T, generator=g, device='cuda'),
                        torch.arange(T, device='cuda').flip(0)], 1).contiguous()
    out = _guarded(T, N, dt)
    combine(y, rows, out[:T])
    pick = torch.tensor(sorted({0, 1, (2 ** 31) // N, T // 2, T - 2, T - 1}
                               | set(torch.randint(0, T, (64,), generator=torch.Generator().manual_seed(3))
                                     .tolist())), device='cuda')
    used = rows[pick]                                  # y's rows the sample reads, gathered
    ref = combine_ref(y[used.reshape(-1)], torch.arange(used.numel()).view(used.shape), dt).cuda()
    _check_guarded(out, T, ref, 'combine T=131200', sample=pick)
    del y, out
    _free()
