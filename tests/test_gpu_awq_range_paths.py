"""GPU: AWQ's tensor-level kernels (csrc/awq.cu: llmc_absmean_cols, llmc_div_cols, llmc_mse,
llmc_awq_clip) and the range observers (csrc/range.cu: llmc_mse_range, llmc_histc) bit for bit
against the exact oracles of oracle/awq_range_oracle.py, on every branch of their host plans.

On the oracles' inputs every sum these kernels form is exact in any order, so a dropped row
split, token chunk or tail, a wrong divisor or a changed tie rule changes the output.  The mse
range search cannot be made order free; there the oracle certifies which rows' decisions no
rounding of the device can flip, and those rows must match exactly.  Each path-table entry
asserts, from a restatement of the host plan, that it reaches the case it is named for."""
import numpy as np
import pytest
import torch

from llmc_b200._lib import BF16, F16, F32, call, load, ptr, stream_ptr
from oracle import awq_range_oracle as ar

pytestmark = pytest.mark.gpu

DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def _same(got, exp, what):
    """Bit equality (NaN payloads aside: NaN must meet NaN)."""
    got, exp = got.cpu(), exp.cpu()
    assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, exp.shape, got.dtype)
    g, e = got.float(), exp.float()
    bad = ~((g == e) & (torch.signbit(g) == torch.signbit(e)) | (torch.isnan(g) & torch.isnan(e)))
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        first = [(i, got[tuple(i)].item(), exp[tuple(i)].item()) for i in idx]
        raise AssertionError(f'{what}: {int(bad.sum())}/{got.numel()} elements differ; first '
                             f'(index, got, expected): {first}')


# ---- absmean_cols ---------------------------------------------------------------------------------
ABSMEAN = [  # T, C, workspace floats (None: the wrapper's 256 * C), cases reached
    pytest.param(1, 8, None, {'one-split'}, id='T1'),
    pytest.param(63, 8, None, {'one-split'}, id='T63'),
    pytest.param(64, 8, None, {'one-split'}, id='T64'),
    pytest.param(65, 2056, None, {'one-split', 'grid2'}, id='T65-C2056'),
    pytest.param(1000, 2048, None, {'splits'}, id='T1000'),
    pytest.param(16448, 8, None, {'cap'}, id='T16448-cap'),
    pytest.param(16447, 16, None, {'cap', 'recount'}, id='T16447-recount'),
    pytest.param(4096, 64, 64 * 5, {'halved'}, id='T4096-halved'),
]


def _absmean_cases(T, C, wsf):
    p = ar.absmean_plan(T, C, wsf)
    c = set()
    c.add('one-split' if p['splits'] == 1 else 'splits')
    if p['first'] == 256:
        c.add('cap')
    if p['recount']:
        c.add('recount')
    if p['halved']:
        c.add('halved')
    if p['grid_x'] == 2:
        c.add('grid2')
    return c


@pytest.mark.parametrize('T,C,wsf,reached', ABSMEAN)
@pytest.mark.parametrize('dtype', DTYPES)
def test_absmean_cols(T, C, wsf, reached, dtype):
    assert reached <= _absmean_cases(T, C, wsf), (T, C, _absmean_cases(T, C, wsf))
    x = ar.absmean_input(T, C, dtype, seed=T + C, device='cuda')
    exp = ar.absmean_expected(x)
    nfl = 256 * C if wsf is None else wsf
    ws = torch.full((nfl,), float('nan'), device='cuda')
    out = torch.empty(C, dtype=dtype, device='cuda')
    call('llmc_absmean_cols', ptr(x), T, C, DT[dtype], ptr(out), ptr(ws), nfl, stream_ptr())
    _same(out, exp, f'absmean T={T} C={C}')
    if wsf is None:
        from llmc_b200.awq import absmean_cols
        _same(absmean_cols(x), exp, 'absmean wrapper')


def test_get_act_scale_with_several_chunks():
    """awq.py:74-85: the mean of per-_bs-chunk means."""
    from llmc_b200.awq import Awq
    a = Awq.__new__(Awq)
    x = ar.absmean_input(4 * 96, 64, torch.bfloat16, seed=3, device='cuda')
    a._bs = 96
    got = a.get_act_scale(x)
    means = [ar.absmean_expected(x[i * 96:(i + 1) * 96]).cuda() for i in range(4)]
    _same(got, sum(means) / 4, 'get_act_scale over 4 chunks')


# ---- div_cols -------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', DTYPES)
def test_div_cols(dtype):
    T, C = 1100, 8 * 1024          # T * C / 8 > 132 * 32 * 256: the grid-stride loop runs
    assert T * C // 8 > 132 * 32 * 256
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(T, C, generator=g) * 3).to(dtype)
    s = (torch.rand(C, generator=g) + 0.25).to(dtype)
    specials_x = [0.0, 1.0, float('inf'), -float('inf'), 0.0, 5.0, -7.0, 1.5]
    specials_s = [0.0, 0.0, float('inf'), 2.0, -0.0, 1e-3, 3.0, 7.0]
    x[0, :8] = torch.tensor(specials_x).to(dtype)
    s[:8] = torch.tensor(specials_s).to(dtype)
    if dtype == torch.float16:
        x[1, :8] = torch.tensor([6e-8, -6e-8, 1e-5, 3e-7, 1.0, 2.0, 3.0, 4.0]).half()    # subnormals
    if dtype == torch.bfloat16:
        x[2, 5] = 1e30                                # quotient beyond fp16's range
    xc, sc = x.cuda(), s.cuda()
    out = torch.full((T, C), float('nan'), dtype=dtype, device='cuda')
    call('llmc_div_cols', ptr(xc), ptr(sc), T, C, DT[dtype], ptr(out), stream_ptr())
    exp = ar.div_expected(x, s)
    _same(out, exp, f'div_cols {dtype}')
    if dtype == torch.bfloat16:
        assert float(exp[2, 5]) > 65504
    # T = 0 launches nothing
    lib = load()
    n0 = lib.llmc_b200_launch_count()
    call('llmc_div_cols', ptr(xc), ptr(sc), 0, C, DT[dtype], ptr(out), stream_ptr())
    assert lib.llmc_b200_launch_count() == n0


# ---- mse ------------------------------------------------------------------------------------------
MSE = [  # n, cases
    pytest.param(1, {'only-tail'}, id='1'), pytest.param(7, {'only-tail'}, id='7'),
    pytest.param(8, {'one-block'}, id='8'), pytest.param(2048 * 5 + 3, {'blocks', 'tail'}, id='10243'),
    pytest.param(1024 * 256 * 8 + 8 * 37 + 5, {'grid-stride', 'tail'}, id='grid-stride'),
]


def _mse_cases(n):
    p = ar.mse_plan(n)
    c = {'only-tail'} if p['only_tail'] else set()
    if p['tail'] and not p['only_tail']:
        c.add('tail')
    c.add('one-block' if p['blocks'] == 1 else 'blocks')
    if p['grid_stride']:
        c.add('grid-stride')
    return c


def _mse(a, b):
    out = torch.full((1,), float('nan'), device='cuda')
    ws = torch.full((1024,), float('nan'), device='cuda')
    call('llmc_mse', ptr(a), ptr(b), a.numel(), DT[a.dtype], ptr(out), ptr(ws), stream_ptr())
    return out


@pytest.mark.parametrize('n,reached', MSE)
@pytest.mark.parametrize('dtype', DTYPES)
def test_mse(n, reached, dtype):
    assert reached <= _mse_cases(n), (n, _mse_cases(n))
    a, b, S = ar.mse_pair(n, dtype, seed=n, device='cuda')
    assert ar.mse_premises(a, b) == S
    _same(_mse(a, b), torch.tensor([ar.mse_expected(S, n)]), f'mse n={n}')


def test_mse_rounds_the_mean_once():
    """S / n halfway between two fp32 values: t * (1 / n) rounds it the wrong way."""
    a, b, S, n = ar.mse_double_rounding_pair(device='cuda')
    _same(_mse(a, b), torch.tensor([ar.mse_expected(S, n)]), 'mse midpoint')


def test_calculate_loss_over_batches():
    from llmc_b200.awq import Awq
    a = Awq.__new__(Awq)
    a._bs = 64
    x, y, _ = ar.mse_pair(4 * 64 * 40, torch.float16, seed=9, device='cuda')
    x, y = x.view(4 * 64, 40), y.view(4 * 64, 40)
    parts = [torch.tensor(ar.mse_expected(ar.mse_premises(x[i * 64:(i + 1) * 64],
                                                          y[i * 64:(i + 1) * 64]), 64 * 40))
             for i in range(4)]
    tot = parts[0] + parts[1] + parts[2] + parts[3]       # fp32, left to right like sum()
    got = a.calculate_loss(x, y)
    _same(got.reshape(1), (tot / 4).reshape(1).float(), 'calculate_loss b_num=4')


# ---- auto-clip ------------------------------------------------------------------------------------
CLIP = [  # R, ng, group, ns, bit, sym, clip_sym, dtype, cases
    pytest.param(1, 1, 8, 1, 4, True, True, torch.float16, {'one-slice'}, id='R1-g8-ns1'),
    pytest.param(7, 2, 32, 2, 3, False, False, torch.bfloat16, {'one-slice'}, id='R7-g32-ns2'),
    pytest.param(8, 32, 36, 31, 2, True, False, torch.float32, {'one-slice', 'empty-lanes'}, id='R8-g36'),
    pytest.param(9, 112, 96, 33, 8, False, True, torch.float16, {'ragged-slice', 'empty-lanes'}, id='R9-g96'),
    pytest.param(201, 2, 128, 255, 4, True, True, torch.bfloat16, {'ragged-slice'}, id='R201-ns255'),
    pytest.param(200, 32, 128, 256, 4, False, False, torch.float16, {'ragged-slice'}, id='R200-ns256'),
    pytest.param(200, 1, 128, 257, 3, True, False, torch.float32, {'chunks'}, id='R200-ns257'),
    pytest.param(4100, 1, 128, 600, 4, False, True, torch.bfloat16, {'chunks', 'ragged-slice'}, id='R4100-ns600'),
    pytest.param(4096, 2, 64, 1023, 2, False, False, torch.float16, {'chunks'}, id='R4096-ns1023'),
    pytest.param(64, 112, 128, 512, 8, True, True, torch.float32, {'chunks'}, id='ng112-ns512'),
    pytest.param(33, 2, 128, 600, 4, True, False, torch.float16, {'chunks', 'ragged-slice'}, id='R33'),
]


def _clip_cases(R, ng, group, ns):
    p = ar.clip_plan(R, ng, ns)
    c = {'one-slice'} if p['slices'] == 1 else set()
    if R % p['rows_per_cta'] and p['slices'] > 1:
        c.add('ragged-slice')
    if p['chunks'] > 1:
        c.add('chunks')
    if group < 128:
        c.add('empty-lanes')            # lanes whose 4 weights lie (partly) past the group
    return c


def _clip_abi(w, x, group, bit, sym, clip_sym):
    R, C = w.shape
    ng = C // group
    nfl = R * ng * 10
    ws = torch.full((nfl,), float('nan'), device='cuda')
    bmax = torch.full((R, ng), float('nan'), dtype=w.dtype, device='cuda')
    bmin = torch.full_like(bmax, float('nan'))
    call('llmc_awq_clip', ptr(w), R, C, ptr(x), x.shape[0], DT[w.dtype], group, bit, int(sym),
         int(clip_sym), ptr(bmax), ptr(bmin), ptr(ws), nfl, stream_ptr())
    return bmax, bmin, ws.view(R, ng, 10)


@pytest.mark.parametrize('R,ng,group,ns,bit,sym,clip_sym,dtype,reached', CLIP)
def test_awq_clip_exact(R, ng, group, ns, bit, sym, clip_sym, dtype, reached):
    assert reached <= _clip_cases(R, ng, group, ns), (reached, _clip_cases(R, ng, group, ns))
    w, x, slots = ar.clip_inputs(R, ng, group, ns, dtype, seed=R * 7 + ng + ns, device='cuda')
    err, maxs, mins, om, on = ar.clip_reference(w, x, slots, bit, sym, group, clip_sym)
    bm, bn, ties, _ = ar.clip_select(err, maxs, mins, om, on, ns)
    if R * ng >= 64:
        assert ties > 0
    gmax, gmin, gerr = _clip_abi(w, x, group, bit, sym, clip_sym)
    _same(gerr, err, 'err workspace')
    _same(gmax, bm, 'best_max')
    _same(gmin, bn, 'best_min')


def test_awq_clip_wrapper_matches_abi():
    from llmc_b200.awq import AutoClipper
    from llmc_b200.quant import IntegerQuantizer
    w, x, slots = ar.clip_inputs(72, 4, 128, 300, torch.bfloat16, seed=11, device='cuda')
    q = IntegerQuantizer(4, False, 'per_group', group_size=128)
    ac = AutoClipper(True, q, None, 'v1', False, False, None)
    mx, mn = ac.auto_clip_layer(0, 'fc', w, [x], n_sample_token=300)
    err, maxs, mins, om, on = ar.clip_reference(w, x, slots, 4, False, 128, False)
    bm, bn, _, _ = ar.clip_select(err, maxs, mins, om, on, 300)
    _same(mx.squeeze(-1), bm, 'wrapper best_max')
    _same(mn.squeeze(-1), bn, 'wrapper best_min')


def test_awq_clip_refuses_wide_groups_without_launching():
    lib = load()
    w = torch.zeros(8, 256, dtype=torch.float16, device='cuda')
    x = torch.zeros(4, 256, dtype=torch.float16, device='cuda')
    bmax = torch.full((8, 1), 3.0, dtype=torch.float16, device='cuda')
    bmin = bmax.clone()
    ws = torch.full((80,), 5.0, device='cuda')
    torch.cuda.synchronize()
    n0 = lib.llmc_b200_launch_count()
    rc = lib.llmc_awq_clip(ptr(w), 8, 256, ptr(x), 4, F16, 256, 4, 1, 1, ptr(bmax), ptr(bmin),
                           ptr(ws), 80, stream_ptr())
    assert rc == -2 and b'group 256' in lib.llmc_b200_last_error()
    torch.cuda.synchronize()
    assert lib.llmc_b200_launch_count() == n0
    assert bool((bmax == 3).all()) and bool((bmin == 3).all()) and bool((ws == 5).all())


@pytest.mark.parametrize('R', [4096, 11008])
def test_awq_clip_random_data_is_deterministic(R):
    g = torch.Generator(device='cuda')
    g.manual_seed(R)
    w = torch.randn(R, 4096, device='cuda', generator=g).half()
    x = torch.randn(512, 4096, device='cuda', generator=g).half()
    a = _clip_abi(w, x, 128, 4, True, True)
    b = _clip_abi(w, x, 128, 4, True, True)
    for u, v in zip(a, b):
        assert torch.equal(u.view(-1).view(torch.int16 if u.element_size() == 2 else torch.int32),
                           v.view(-1).view(torch.int16 if v.element_size() == 2 else torch.int32))


# ---- mse range ------------------------------------------------------------------------------------
def _mse_range_abi(t, bit, sym, steps, grid):
    from oracle import quant_oracle as qo
    qmin, qmax = qo.int_range(bit, sym)
    rows, cols = t.shape
    mn = torch.full((rows,), float('nan'), device='cuda')
    mx = torch.full_like(mn, float('nan'))
    call('llmc_mse_range', ptr(t), rows, cols, DT[t.dtype], int(sym), int(qmin), int(qmax), steps,
         float(grid), 2.4, ptr(mn), ptr(mx), stream_ptr())
    return mn, mx


# undecided: the largest fraction of random rows the certificate may leave open.  Measured with
# these seeds: 0 everywhere except 24576 columns, where the summation bound (gamma_n ~ 1.5e-3)
# leaves 1 of 16 rows open.
MSE_RANGE = [  # rows, cols, bit, sym, maxshrink, mse_grid, dtype, undecided, cases
    pytest.param(64, 128, 4, True, 0.8, 100, torch.float32, 0.0, {'cached'}, id='128-sym4'),
    pytest.param(64, 128, 3, False, 0.8, 100, torch.bfloat16, 0.0, {'cached'}, id='128-asym3'),
    pytest.param(16, 24576, 7, False, 0.8, 100, torch.float16, 1 / 16, {'cached'}, id='24576-asym7'),
    pytest.param(8, 28672, 4, True, 0.8, 100, torch.bfloat16, 0.0, {'uncached'}, id='28672-sym4'),
    pytest.param(2200, 128, 2, False, 0.5, 40, torch.float16, 0.0, {'grid-stride'}, id='2200-asym2'),
    pytest.param(2200, 64, 6, True, 0.9, 30, torch.float32, 0.0, {'grid-stride'}, id='2200-sym6'),
]


def _mse_range_cases(rows, cols):
    p = ar.mse_range_plan(rows, cols)
    c = {'cached' if p['cached'] else 'uncached'}
    if p['grid_stride']:
        c.add('grid-stride')
    return c


@pytest.mark.parametrize('rows,cols,bit,sym,maxshrink,grid,dtype,undecided,reached', MSE_RANGE)
def test_mse_range_certified(rows, cols, bit, sym, maxshrink, grid, dtype, undecided, reached):
    assert reached <= _mse_range_cases(rows, cols)
    steps = int(maxshrink * grid)
    g = torch.Generator().manual_seed(rows + cols + bit)
    t = torch.randn(rows, cols, generator=g).to(dtype).cuda()
    emn, emx, dec = ar.mse_range_certified(t.float(), bit, sym, steps, grid)
    frac = 1 - float(dec.float().mean())
    print(f'{rows}x{cols} bit {bit} sym {sym}: undecided rows {frac:.4f}')
    assert frac <= undecided, frac
    mn, mx = _mse_range_abi(t, bit, sym, steps, grid)
    _same(mn[dec], emn.squeeze(1)[dec], 'min (decided rows)')
    _same(mx[dec], emx.squeeze(1)[dec], 'max (decided rows)')
    if cols > 4096:
        return                       # constructed rows are certified up to 4096 columns
    c = ar.constructed_mse_rows(rows if rows < 64 else 64, cols).to(dtype).cuda()
    cmn, cmx, cdec = ar.mse_range_certified(c.float(), bit, sym, steps, grid)
    assert bool(cdec.all())
    mn, mx = _mse_range_abi(c, bit, sym, steps, grid)
    _same(mn, cmn.squeeze(1), 'min (constructed rows)')
    _same(mx, cmx.squeeze(1), 'max (constructed rows)')


@pytest.mark.parametrize('sym', [True, False])
def test_mse_range_qparams_and_fake_quant_follow(sym):
    """Through IntegerQuantizer: decided rows' qparams and fake-quant output, and mse_b_num = 2
    gives what mse_b_num = 1 gives."""
    from llmc_b200.quant import IntegerQuantizer
    from oracle import quant_oracle as qo
    g = torch.Generator().manual_seed(5)
    w = torch.randn(96, 512, generator=g).to(torch.bfloat16).cuda()
    q = IntegerQuantizer(4, sym, 'per_group', group_size=128, calib_algo='mse')
    t = q.reshape_tensor(w)
    emn, emx, dec = ar.mse_range_certified(t.float(), 4, sym, 80, 100)
    mn, mx = q.get_mse_range(t)
    _same(mn[dec], emn[dec], 'min')
    _same(mx[dec], emx[dec], 'max')
    q2 = IntegerQuantizer(4, sym, 'per_group', group_size=128, calib_algo='mse', mse_b_num=2)
    mn2, mx2 = q2.get_mse_range(t)
    _same(mn2, mn, 'mse_b_num 2 min')
    _same(mx2, mx, 'mse_b_num 2 max')
    s, z, qmax, qmin = qo.qparams(emn, emx, 4, sym)
    ref = qo.dequant(qo.quant(t.float(), s, z, qmax, qmin), s, z).to(w.dtype)
    out = q.fake_quant_weight_dynamic(w).reshape(t.shape)
    _same(out[dec], ref[dec], 'fake quant (decided rows)')


# ---- histc ----------------------------------------------------------------------------------------
def _histc(x, bins, lo, hi):
    hist = torch.full((bins,), float('nan'), device='cuda')
    call('llmc_histc', ptr(x), x.numel(), DT[x.dtype], bins, lo, hi, ptr(hist), stream_ptr())
    return hist


HISTC = [  # n, bins, log2 width, dtype
    pytest.param(0, 2048, 3, torch.float32, id='n0'),
    pytest.param(1, 1, 0, torch.float16, id='n1-bins1'),
    pytest.param(5000, 2048, 3, torch.bfloat16, id='2048'),
    pytest.param(132 * 8 * 256 + 777, 8192, 1, torch.float32, id='grid-stride-8192'),
    pytest.param(132 * 8 * 256 + 1, 2048, 4, torch.float16, id='grid-stride-2048'),
]


@pytest.mark.parametrize('n,bins,lw,dtype', HISTC)
def test_histc_exact(n, bins, lw, dtype):
    p = ar.histc_plan(n)
    assert p['grid_stride'] == (n > 132 * 8 * 256)
    lo = -2.0
    hi = lo + 2.0 ** lw
    extras = () if n == 0 else (-3.0, hi + 1.0, float('nan'), float('inf'), -float('inf'))
    x = ar.histc_input(n, lo, lw, bins, dtype, seed=n + bins, extras=extras)
    exp, _ = ar.histc_expected(x, bins, lo, hi)
    _same(_histc(x.cuda(), bins, lo, hi), exp, f'histc n={n} bins={bins}')


def test_histc_degenerate_range():
    x = torch.full((300,), 0.5, dtype=torch.float16)
    exp, _ = ar.histc_expected(x, 2048, 0.5, 0.5)
    _same(_histc(x.cuda(), 2048, 0.5, 0.5), exp, 'lo == hi')


def test_histc_counts_beyond_2_24_exactly_and_deterministically():
    """2^25 - 2 values in one bin: the exact count 33554430 is an fp32 value, and a float sum of
    the blocks' counts would round in completion order."""
    n = 2 ** 25 - 2
    x = torch.full((n,), 0.25, dtype=torch.bfloat16, device='cuda')
    x[::97] = 0.75
    big = int((x == 0.25).sum())
    a = _histc(x, 4, 0.0, 1.0)
    b = _histc(x, 4, 0.0, 1.0)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert float(a[1]) == float(np.float32(big)) and float(a[3]) == float(np.float32(n - big))
    assert float(a[0]) == 0 and float(a[2]) == 0
    assert big > 2 ** 24
