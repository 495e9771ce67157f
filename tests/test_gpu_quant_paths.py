"""GPU: every dispatch path of the integer quantiser (csrc/quant.cu) against the oracle, bit for bit.

`llmc_quant_dynamic` picks one of eight kernels from dtype, group, cols, ld, ld_out, pointer
alignment, out_mode and bit.  The tests call the C ABI directly (the Python classes never pass
ld, ld_out, use_range, an unaligned base or a different QDQ out dtype) and record, with
torch.profiler, which kernel ran, so that a dispatch change cannot quietly leave a path untested.

The oracle (oracle/quant_oracle.py) is plain torch; the large sweeps run it on CUDA tensors, which
`test_cuda_oracle_equals_cpu_oracle` pins to the CPU oracle.  One documented divergence: torch's
clamp propagates NaN, the kernels' clamp (fmaxf, then fminf) maps it to qmin.  Where the reference
clamps a NaN — the code of an element whose quotient x / s is NaN (inf / inf), the zero-point of a
group whose minimum is -inf — its result cannot be stored as an integer anyway; the expected value
here is qmin (`_ref_dyn`).  The 16-bit divider (RecipDiv, DESIGN.md §3) is exact on finite
quotients; a finite x whose IEEE quotient is not finite (bf16 |x / s| beyond fp32 range, or
s = inf) gets NaN and so qmin, which `_ref_dyn` states too."""
import math

import pytest
import torch

from llmc_b200._lib import (BF16, F16, F32, OUT_CODES_I8, OUT_CODES_I32, OUT_CODES_U8, OUT_NONE,
                            OUT_PACK_VLLM, OUT_QDQ, call, ptr, stream_ptr)
from oracle import quant_oracle as qo

pytestmark = pytest.mark.gpu

DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
ZP_INSIDE = 0x100
SENTINEL = 0x5A5A5A5A


# ---- helpers -------------------------------------------------------------------------------------
def _same(got, exp, what):
    """Bit-exact equality; NaN matches NaN whatever its payload."""
    exp = exp.to(got.device)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert got.dtype == exp.dtype, (what, got.dtype, exp.dtype)
    if got.is_floating_point():
        gn, en = torch.isnan(got), torch.isnan(exp)
        iv = INT_VIEW[got.dtype]
        bad = (gn != en) | (~gn & (got.view(iv) != exp.view(iv)))
    else:
        bad = got != exp
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        n = int(bad.sum())
        first = [(i, got[tuple(i)].item(), exp[tuple(i)].item()) for i in idx]
        raise AssertionError(f'{what}: {n}/{got.numel()} elements differ; first (index, got, '
                             f'expected): {first}')


PROBE = 'llmc_quant_probe'


class _Recorder:
    """torch.profiler around a block; `call(fn)` runs fn inside a probe range and `.names` lists
    the llmc kernels launched inside the probes (spaces removed).  Kernels are attributed through
    the profiler's launch correlation, else by start time: activity records of an earlier session
    can arrive late, and must not count for this one."""

    def __enter__(self):
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        self.prof = torch.profiler.profile(activities=acts)
        self.prof.__enter__()
        return self

    def call(self, fn):
        with torch.profiler.record_function(PROBE):
            return fn()

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        evs = self.prof.events()
        probes = [e for e in evs if e.name == PROBE]
        names = [k.name for p in probes for k in p.kernels]
        if not names and probes:
            t0 = min(p.time_range.start for p in probes)
            names = [e.name for e in evs if e.device_type == torch.autograd.DeviceType.CUDA
                     and e.time_range.start >= t0]
        self.names = [n.replace(' ', '') for n in names if 'llmc' in n]
        return False


def _kernels(fn, tries=3):
    """Run fn under torch.profiler -> (its result, names of the llmc kernels it launched).  fn is
    run again (its outputs are fresh buffers) if the profiler delivered no kernel record."""
    for _ in range(tries):
        with _Recorder() as rec:
            res = rec.call(fn)
        if rec.names:
            break
    return res, rec.names


def _assert_ran(names, pattern, what):
    import re
    assert any(re.search(pattern, n) for n in names), \
        f'{what}: expected a kernel matching {pattern!r}, the profiler recorded {sorted(set(names))}'


def _view(w, ld=None, offset=0):
    """w [rows, cols] as a CUDA view with row stride `ld` starting `offset` elements into its
    buffer.  The padding holds a large finite value, so a kernel that reads it changes the scales."""
    rows, cols = w.shape
    ld = ld or cols
    pad = torch.finfo(w.dtype).max / 2 if w.dtype != torch.float32 else 1e30
    buf = torch.full((offset + rows * ld + 16,), pad, dtype=w.dtype, device='cuda')
    v = buf.narrow(0, offset, rows * ld).view(rows, ld)[:, :cols]
    v.copy_(w)
    return v


def _out_buf(mode, rows, cols, bit, dtype, ld_out=0):
    if mode == OUT_NONE:
        return None
    if mode == OUT_QDQ:
        return torch.full((rows, ld_out or cols), -3.0, dtype=dtype, device='cuda')
    if mode in (OUT_CODES_I8, OUT_CODES_U8):
        return torch.full((rows, cols), 0x5A, dtype=torch.uint8, device='cuda')
    if mode == OUT_CODES_I32:
        return torch.full((rows, cols), SENTINEL, dtype=torch.int32, device='cuda')
    return torch.full((rows, math.ceil(cols / (32 // bit))), SENTINEL, dtype=torch.int32,
                      device='cuda')


def dyn(wv, group, bit, sym, mode, qrange=None, col_scale=None, ld_out=0, out_dtype=None):
    """llmc_quant_dynamic on the view wv -> (scales, zeros | None, out buffer | None)."""
    rows, cols = wv.shape
    ld = wv.stride(0)
    dt = wv.dtype
    od = out_dtype or dt
    s = torch.full((rows * (cols // group),), -7.0, dtype=dt, device='cuda')
    z = None if sym else torch.full_like(s, -7.0)
    out = _out_buf(mode, rows, cols, bit, od, ld_out)
    qmin, qmax = qrange or (0, 0)
    call('llmc_quant_dynamic', ptr(wv), rows, cols, ld, DT[dt], group, bit, int(sym),
         int(qrange is not None), qmin, qmax, ptr(col_scale), ptr(s), ptr(z), mode, ptr(out),
         ld_out, DT[od], stream_ptr())
    return s, z, out


def _ref_dyn(w, group, bit, sym, qrange=None, col_scale=None):
    """The oracle's dynamic quantiser on w's device; col_scale as awq.py:147-164 (W * s, then
    fake-quant; oracle/awq_oracle.fake_quantize_weight)."""
    if col_scale is not None:
        w = w * col_scale.view(1, -1)
    t = w.reshape(-1, group)
    mn, mx = qo.minmax(t, 'per_group')
    s, z, qmax, qmin = qo.qparams(mn, mx, bit, sym, qrange=qrange)
    if not sym:
        z = torch.where(torch.isnan(z), torch.full_like(z, float(qmin)), z)
    q = qo.quant(t, s, z, qmax, qmin)
    if w.dtype != torch.float32:               # RecipDiv outside its domain: NaN
        ieee = t.float() / s.float()
        out = torch.isfinite(t) & (~torch.isfinite(ieee) | torch.isinf(s))
        q = torch.where(out, torch.full_like(q, float('nan')), q)
    q = torch.where(torch.isnan(q), torch.full_like(q, float(qmin)), q)
    y = qo.dequant(q, s, z).to(w.dtype)
    return dict(s=s.reshape(-1), z=None if sym else z.reshape(-1), q=q.reshape(w.shape),
                y=y.reshape(w.shape))


def _expected_out(ref, mode, bit, od):
    q = ref['q']
    if mode == OUT_QDQ:
        return ref['y'].to(od)
    if mode in (OUT_CODES_I8, OUT_CODES_U8):
        return (q.to(torch.int32) & 0xff).to(torch.uint8)
    if mode == OUT_CODES_I32:
        return q.to(torch.int32)
    packed, _ = qo.pack_vllm(q.to(torch.int32).cpu(), ref['s'].cpu(), bit)
    return packed


def _check_dyn(ref, got, mode, bit, cols, what, ld_out=0, od=None):
    s, z, out = got
    _same(s, ref['s'], f'{what} scales')
    if ref['z'] is not None:
        _same(z, ref['z'], f'{what} zeros')
    if mode == OUT_NONE:
        return
    if mode == OUT_QDQ:
        _same(out[:, :cols], _expected_out(ref, mode, bit, od), f'{what} qdq')
        if ld_out > cols:
            assert bool((out[:, cols:] == -3.0).all()), f'{what}: QDQ wrote into the ld_out padding'
        return
    _same(out, _expected_out(ref, mode, bit, od), f'{what} out_mode {mode}')


def _modes(bit, sym):
    m = [OUT_NONE, OUT_QDQ, OUT_CODES_I32, OUT_PACK_VLLM]
    if bit == 8:
        m.append(OUT_CODES_I8 if sym else OUT_CODES_U8)
    return m


# ---- the path table -------------------------------------------------------------------------------
# (id, kernel the entry must reach, arguments).  Kernel names as the profiler records them with the
# spaces removed; template arguments are <DT, G, MODE, BITS> (fast), <DT, MODE, BITS, CH> (row-fast),
# <DT, CH> (warp), DT = 0 fp32 / 1 fp16 / 2 bf16.
FAST128 = r'quant_group_fast_kernel<\d,128,'
FAST64 = r'quant_group_fast_kernel<\d,64,'
ROW2 = r'quant_row_fast_kernel<\d,\d,\d,2>'
ROW4 = r'quant_row_fast_kernel<\d,\d,\d,4>'
WARP = r'quant_dynamic_warp_kernel<\d,{}>'
BLOCK = r'quant_dynamic_block_kernel<'
GENERIC = r'qparams_generic_kernel<'
H, B, S = torch.float16, torch.bfloat16, torch.float32

PATHS = [
    ('fast128-partial-tile', FAST128, dict(dt=B, rows=333, cols=512, group=128, bit=4, sym=False, mode=OUT_PACK_VLLM)),
    ('fast128-persistent', FAST128, dict(dt=H, rows=1601, cols=4096, group=128, bit=4, sym=True, mode=OUT_QDQ)),
    ('fast128-rows1', FAST128, dict(dt=B, rows=1, cols=4096, group=128, bit=4, sym=False, mode=OUT_QDQ)),
    ('fast128-none', FAST128, dict(dt=H, rows=40, cols=1024, group=128, bit=3, sym=False, mode=OUT_NONE)),
    ('fast128-codes8', FAST128, dict(dt=B, rows=40, cols=1024, group=128, bit=8, sym=True, mode=OUT_CODES_I8)),
    ('fast64-partial-tile', FAST64, dict(dt=H, rows=7, cols=576, group=64, bit=8, sym=False, mode=OUT_CODES_U8)),
    ('fast64-persistent', FAST64, dict(dt=B, rows=1601, cols=4096, group=64, bit=8, sym=False, mode=OUT_PACK_VLLM)),
    ('fast64-qdq', FAST64, dict(dt=H, rows=100, cols=640, group=64, bit=4, sym=False, mode=OUT_QDQ)),
    ('row2-512-rows1', ROW2, dict(dt=B, rows=1, cols=512, group=512, bit=4, sym=True, mode=OUT_QDQ)),
    ('row2-4096-above-grid', ROW2, dict(dt=H, rows=1000, cols=4096, group=4096, bit=4, sym=False, mode=OUT_PACK_VLLM)),
    ('row2-ld-out', ROW2, dict(dt=B, rows=300, cols=4096, group=4096, bit=8, sym=False, mode=OUT_QDQ, ld_out=4160)),
    ('row4-4104-above-grid', ROW4, dict(dt=B, rows=600, cols=4104, group=4104, bit=8, sym=False, mode=OUT_CODES_U8)),
    ('row4-8192', ROW4, dict(dt=H, rows=3, cols=8192, group=8192, bit=4, sym=False, mode=OUT_QDQ)),
    ('row4-8192-codes8', ROW4, dict(dt=H, rows=20, cols=8192, group=8192, bit=8, sym=True, mode=OUT_CODES_I8)),
    ('row-narrow-64-ld', ROW2, dict(dt=B, rows=50, cols=64, group=64, bit=4, sym=False, mode=OUT_QDQ, ld=72)),
    ('row-narrow-128-ld', ROW2, dict(dt=H, rows=50, cols=128, group=128, bit=4, sym=True, mode=OUT_PACK_VLLM, ld=136)),
    ('warp-g8', WARP.format(1), dict(dt=H, rows=64, cols=256, group=8, bit=4, sym=False, mode=OUT_CODES_I32)),
    ('warp-g16', WARP.format(2), dict(dt=B, rows=64, cols=256, group=16, bit=4, sym=True, mode=OUT_PACK_VLLM)),
    ('warp-g32', WARP.format(4), dict(dt=H, rows=64, cols=256, group=32, bit=8, sym=False, mode=OUT_CODES_U8)),
    ('warp-g256', WARP.format(4), dict(dt=B, rows=64, cols=1024, group=256, bit=4, sym=False, mode=OUT_QDQ)),
    ('warp-g1024', WARP.format(4), dict(dt=H, rows=33, cols=2048, group=1024, bit=4, sym=False, mode=OUT_PACK_VLLM)),
    ('warp-fp32-g128', WARP.format(4), dict(dt=S, rows=50, cols=1024, group=128, bit=4, sym=False, mode=OUT_QDQ)),
    ('warp-codes-i32', WARP.format(4), dict(dt=B, rows=50, cols=1024, group=128, bit=4, sym=True, mode=OUT_CODES_I32)),
    ('warp-g128-ld', WARP.format(4), dict(dt=H, rows=50, cols=1024, group=128, bit=4, sym=False, mode=OUT_PACK_VLLM, ld=1032)),
    ('warp-qdq-out-fp32', WARP.format(4), dict(dt=B, rows=50, cols=1024, group=128, bit=4, sym=False, mode=OUT_QDQ, out_dtype=S)),
    ('block-14336', BLOCK, dict(dt=H, rows=4, cols=14336, group=14336, bit=4, sym=False, mode=OUT_QDQ)),
    ('block-14336-pack', BLOCK, dict(dt=B, rows=4, cols=14336, group=14336, bit=8, sym=True, mode=OUT_PACK_VLLM)),
    ('block-g2048', BLOCK, dict(dt=B, rows=10, cols=4096, group=2048, bit=4, sym=False, mode=OUT_QDQ)),
    ('block-fp32-4096', BLOCK, dict(dt=S, rows=10, cols=4096, group=4096, bit=8, sym=False, mode=OUT_CODES_U8)),
    ('warp-g24', WARP.format(4), dict(dt=H, rows=20, cols=96, group=24, bit=4, sym=False, mode=OUT_QDQ)),
    ('generic-g20', GENERIC, dict(dt=H, rows=20, cols=80, group=20, bit=4, sym=False, mode=OUT_QDQ)),
    ('generic-ld-plus-4', GENERIC, dict(dt=B, rows=20, cols=128, group=128, bit=4, sym=False, mode=OUT_CODES_I32, ld=132)),
    ('generic-offset-base', GENERIC, dict(dt=H, rows=20, cols=256, group=128, bit=4, sym=True, mode=OUT_PACK_VLLM, offset=1)),
    ('generic-fp32-offset', GENERIC, dict(dt=S, rows=20, cols=256, group=64, bit=8, sym=False, mode=OUT_QDQ, offset=1)),
] + [(f'generic-pack-b{b}', GENERIC, dict(dt=B, rows=9, cols=128, group=128, bit=b, sym=b % 2 == 0,
                                         mode=OUT_PACK_VLLM)) for b in (2, 3, 5, 6, 7)] + [
    ('generic-pack-b3-cols120', GENERIC, dict(dt=H, rows=9, cols=120, group=40, bit=3, sym=False, mode=OUT_PACK_VLLM)),
]


def _randw(rows, cols, dtype, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    w = torch.randn(rows, cols, generator=g, device='cuda') * 0.02
    w[:, ::97] *= 6
    w[::5] += 0.01                                  # rows with a positive offset (asym zero-point)
    return w.to(dtype)


@pytest.mark.parametrize('entry', PATHS, ids=[p[0] for p in PATHS])
def test_path_table(entry):
    """Each entry reaches the kernel it names and matches the oracle bit for bit."""
    name, kernel, a = entry
    w = _randw(a['rows'], a['cols'], a['dt'], seed=len(name))
    wv = _view(w, a.get('ld'), a.get('offset', 0))
    ld_out, od = a.get('ld_out', 0), a.get('out_dtype')
    got, names = _kernels(lambda: dyn(wv, a['group'], a['bit'], a['sym'], a['mode'],
                                      ld_out=ld_out, out_dtype=od))
    _assert_ran(names, kernel, name)
    if kernel == GENERIC and a['mode'] != OUT_NONE:
        _assert_ran(names, r'quant_static_kernel<', name)
    ref = _ref_dyn(w, a['group'], a['bit'], a['sym'])
    _check_dyn(ref, got, a['mode'], a['bit'], a['cols'], name, ld_out, od or a['dt'])


# ---- exhaustive 16-bit sweep ----------------------------------------------------------------------
# (group, groups per row, kernel): one layout per 16-bit path.  cols = group * groups per row.
LAYOUTS = {
    'fast128': (128, 4, FAST128),
    'fast64': (64, 4, FAST64),
    'row2': (4096, 1, ROW2),
    'row4': (8192, 1, ROW4),
    'warp': (256, 4, WARP.format(4)),
    'block': (2048, 2, BLOCK),
    'generic': (20, 4, GENERIC),
}


def _finite_sorted(dtype):
    """Every finite value of a 16-bit dtype, ascending (one zero)."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    return torch.unique(v[torch.isfinite(v)].float())


def _anchors(dtype, sym):
    """The ladder: one or more group maxima per binade of the dtype, subnormals included, so the
    scales cover every reachable binade (down to the 1e-5 clamp).  Asymmetric groups get a minimum
    -c * max with c cycling through 1, 1/4, 3 and -1/2 (a positive minimum: the zero-point clamps)."""
    fi = torch.finfo(dtype)
    lo_e = -24 if dtype == torch.float16 else -133
    hi_e = 15 if dtype == torch.float16 else 127
    per = (0, 5, 11, 17) if dtype == torch.float16 else (0,)
    mant = 1024 if dtype == torch.float16 else 128
    tops = []
    for e in range(lo_e, hi_e + 1):
        for k in per:
            m = ((e * 37 + k * 101) % mant) / mant
            tops.append(min(2.0 ** e * (1 + m), fi.max))
    tops.append(fi.max)
    hi = torch.tensor(tops).to(dtype).float()
    if sym:
        return -hi, hi
    c = torch.tensor([1.0, 0.25, 3.0, -0.5]).repeat(len(tops) // 4 + 1)[:len(tops)]
    lo = (-c * hi).clamp(-fi.max, fi.max).to(dtype).float()
    return lo, hi


def _ladder(dtype, sym, group, per_row):
    """Groups of `group` values: the two anchors plus every finite value between them, in as many
    groups as that takes (the last one padded with the maximum), rotated so that the anchors sit
    at varying lanes.  -> [rows, group * per_row] CUDA tensor."""
    vals = _finite_sorted(dtype).cuda()
    lo, hi = (t.cuda() for t in _anchors(dtype, sym))
    i0 = torch.searchsorted(vals, lo)
    i1 = torch.searchsorted(vals, hi, right=True)
    f = group - 2
    cnt = i1 - i0
    ng = (cnt + f - 1) // f
    ga = torch.repeat_interleave(torch.arange(len(lo), device='cuda'), ng)
    start = torch.cumsum(ng, 0) - ng
    local = torch.arange(len(ga), device='cuda') - start[ga]
    pos = local[:, None] * f + torch.arange(f, device='cuda')[None, :]
    idx = (i0[ga][:, None] + pos).clamp(max=len(vals) - 1)
    fill = torch.where(pos < cnt[ga][:, None], vals[idx], hi[ga][:, None])
    grp = torch.cat([lo[ga][:, None], hi[ga][:, None], fill], 1)
    shift = (torch.arange(len(ga), device='cuda') * 7) % group
    grp = torch.gather(grp, 1, (torch.arange(group, device='cuda')[None, :] - shift[:, None]) % group)
    pad = (-len(ga)) % per_row
    if pad:
        grp = torch.cat([grp, grp[-1:].expand(pad, group)], 0)
    return grp.to(dtype).reshape(-1, group * per_row)


def _run_all(w, group, bits, syms, what, kernel=None, qrange=None, col_scale=None, wv=None):
    """Every output mode of every (bit, sym) on w (or its view wv) against the oracle; the kernel
    pattern must be among those that ran."""
    wv = w if wv is None else wv
    with _Recorder() as rec:
        for sym in syms:
            for bit in bits:
                ref = _ref_dyn(w, group, bit, sym, qrange, col_scale)
                for mode in _modes(bit, sym):
                    got = rec.call(lambda: dyn(wv, group, bit, sym, mode, qrange, col_scale))
                    _check_dyn(ref, got, mode, bit, w.shape[1], f'{what} bit {bit} sym {sym}', 0,
                               w.dtype)
    if kernel is not None:
        _assert_ran(rec.names, kernel, what)


@pytest.mark.parametrize('path', list(LAYOUTS))
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16], ids=['fp16', 'bf16'])
def test_exhaustive_16bit(dtype, path):
    """Every finite fp16 / bf16 value inside a ladder of group ranges, through each 16-bit path:
    scales, zeros, codes, QDQ and packed words equal the oracle for bits 2, 3, 4, 8, sym and asym."""
    group, per_row, kernel = LAYOUTS[path]
    for sym in (True, False):
        w = _ladder(dtype, sym, group, per_row)
        _run_all(w, group, (2, 3, 4, 8), (sym,), f'{path} {dtype}', kernel)


# ---- degenerate groups ----------------------------------------------------------------------------
def _special_groups(dtype, group):
    """One group per row of degenerate content -> [n, group] CUDA tensor of dtype."""
    iv = INT_VIEW[dtype]
    G = group
    g = torch.Generator().manual_seed(7)
    rows = []

    def const(v):
        rows.append(torch.full((G,), v, dtype=torch.float32).to(dtype))

    const(0.0)
    const(-0.0)
    rows.append(torch.tensor([0.0, -0.0]).repeat(G // 2).to(dtype))
    for v in (0.37, -2.5, 1e-3, -1e-3, 7.0, torch.finfo(dtype).max, -torch.finfo(dtype).max):
        const(v)
    for v in (0.7, -0.7, 1e-6):
        r = torch.zeros(G, dtype=dtype)
        r[G // 3] = v
        rows.append(r)
    # spreads around the 1e-5 clamp: b and b + k ulp (asym), and maxima next to 1e-5 (sym)
    b = torch.tensor(1e-3, dtype=dtype)
    for k in (1, 2, 3, 10, 11, 12):
        r = b.repeat(G)
        r[G // 2] = (b.view(iv) + k).view(dtype)
        rows.append(r)
    e5 = torch.tensor(1e-5, dtype=dtype)
    for k in (-2, -1, 0, 1, 2):
        r = torch.zeros(G, dtype=dtype)
        r[1] = (e5.view(iv) + k).view(dtype)
        r[2] = -r[1] / 2
        rows.append(r)
    # subnormals
    nsub = {torch.float16: 1023, torch.bfloat16: 127, torch.float32: 2 ** 23 - 1}[dtype]
    for sign in (1, -1, 0):
        bits = torch.randint(1, nsub + 1, (G,), generator=g)
        if sign == 0:
            bits = bits * torch.where(torch.rand(G, generator=g) < 0.5, -1, 1)
        r = (bits.abs().to(torch.int32 if dtype == torch.float32 else torch.int16)).view(dtype)
        rows.append(r if sign >= 0 else -r)
        if sign == 0:
            rows[-1] = torch.where(bits < 0, -r, r)
    # infinities
    for spec in ('+', '-', '+-'):
        r = (torch.randn(G, generator=g) * 0.1).to(dtype)
        if '+' in spec:
            r[3] = float('inf')
        if '-' in spec:
            r[G - 2] = -float('inf')
        rows.append(r)
    # huge magnitudes with a spread under the clamp: constant groups (bf16 quotients overflow fp32)
    huge = (1e31, 1e33, 1e35, 1e37, 3e38) if dtype != torch.float16 else (3e4, 6e4)
    for v in huge:
        const(v)
        const(-v)
    return torch.stack(rows).cuda()


DEGENERATE = [(dt, p) for dt in (torch.float16, torch.bfloat16) for p in LAYOUTS] + \
             [(torch.float32, p) for p in ('warp', 'block', 'generic')]


@pytest.mark.parametrize('dtype,path', DEGENERATE, ids=[f'{str(d)[6:]}-{p}' for d, p in DEGENERATE])
def test_degenerate_groups(dtype, path):
    """All +-0, constant, single non-zero, spreads at the 1e-5 clamp, subnormal, +-inf and (bf16)
    |x| ~ 1e31-1e38 groups whose quotients overflow fp32 (qmin on the 16-bit paths, the divider's
    documented domain; the IEEE code on fp32)."""
    group, per_row, kernel = LAYOUTS[path]
    if dtype == torch.float32:
        kernel = kernel.replace(r'<\d', '<0')
    rows = _special_groups(dtype, group)
    pad = (-rows.shape[0]) % per_row
    rows = torch.cat([rows, rows[:pad]]) if pad else rows
    w = rows.reshape(-1, group * per_row)
    _run_all(w, group, (4, 8), (True, False), f'{path} {dtype}', kernel)


def test_bf16_overflowing_quotient_gives_qmin():
    """The documented domain of the 16-bit divider: a bf16 asymmetric group at +-1e35 with no spread
    has x / s = 1e35 / (1e-5 / 15), beyond fp32.  The reference's quotient is +-inf (codes qmax for
    +1e35 after its zero-point clamps at qmin, qmin for -1e35); the divider's is NaN, so every code
    is qmin — on every path, the fast kernels' packed tail included."""
    w = torch.full((4, 128), 1e35, dtype=torch.bfloat16, device='cuda')
    w[1] = -1e35
    for ld in (None, 136):                          # the G=128 fast kernel, then the row kernel
        for mode in (OUT_CODES_I32, OUT_QDQ, OUT_PACK_VLLM):
            _, _, out = dyn(_view(w, ld), 128, 4, False, mode)
            ref = _ref_dyn(w, 128, 4, False)
            _same(out, _expected_out(ref, mode, 4, w.dtype), f'ld {ld} mode {mode}')
        _, _, codes = dyn(_view(w, ld), 128, 4, False, OUT_CODES_I32)
        assert bool((codes == 0).all())


# ---- cross-path identity --------------------------------------------------------------------------
def _variants(w, group):
    """The same logical tensor laid out for every path that can serve it."""
    rows, cols = w.shape
    ones = torch.ones(cols, dtype=w.dtype, device='cuda')
    return {'dense': (_view(w), None), 'ld+8': (_view(w, cols + 8), None),
            'ld+4': (_view(w, cols + 4), None), 'offset1': (_view(w, None, 1), None),
            'col_scale=1': (_view(w), ones)}


CROSS = [(128, 4096), (64, 1024), (4096, 4096), (8192, 8192), (1024, 4096), (2048, 4096), (32, 256)]


@pytest.mark.parametrize('group,cols', CROSS, ids=[f'g{g}-c{c}' for g, c in CROSS])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32],
                         ids=['fp16', 'bf16', 'fp32'])
def test_cross_path_identity(dtype, group, cols):
    """One tensor (random rows plus degenerate groups) through every path that accepts it — fast,
    row-fast, warp, block and generic — gives identical scales, zeros and output bytes."""
    w = _randw(40, cols, dtype, seed=group)
    sp = _special_groups(dtype, group).reshape(-1)
    n = (sp.numel() // cols) * cols
    if n:
        w = torch.cat([w, sp[:n].reshape(-1, cols)])
    _cross(w, group)


def _cross(w, group):
    rows, cols = w.shape
    for sym in (True, False):
        for bit in (3, 4, 8):
            for mode in _modes(bit, sym):
                outs = {}
                for name, (wv, cs) in _variants(w, group).items():
                    if cs is not None and mode == OUT_PACK_VLLM and bit not in (4, 8):
                        continue                   # col_scale needs the vectorised path
                    s, z, o = dyn(wv, group, bit, sym, mode, col_scale=cs)
                    outs[name] = (s, z, None if o is None else o[:, :cols])
                base = outs['dense']
                for name, (s, z, o) in outs.items():
                    what = f'{name} vs dense, group {group} bit {bit} sym {sym} mode {mode}'
                    _same(s, base[0], what + ' scales')
                    if z is not None:
                        _same(z, base[1], what + ' zeros')
                    if o is not None:
                        _same(o, base[2], what + ' out')


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32],
                         ids=['fp16', 'bf16', 'fp32'])
def test_nan_inputs_agree_across_paths(dtype):
    """NaN inputs.  The reference's amin / amax propagate NaN (every output of the group is NaN);
    every path here drops NaN in its min / max (fminf / __hmin2) and clamps a NaN quotient to qmin.
    So only agreement between the paths is asserted, not agreement with the oracle."""
    for group, cols in ((128, 4096), (64, 1024), (4096, 4096), (2048, 4096), (256, 1024)):
        w = _randw(24, cols, dtype, seed=3).float()
        w[0, 5] = float('nan')
        w[1, :group] = float('nan')
        w[2, 7::group] = float('nan')
        w[3, 9] = float('nan')
        w[3, 10] = float('inf')
        _cross(w.to(dtype), group)


# ---- non-default ranges and AWQ col_scale -------------------------------------------------------------
RANGES = [(False, (-8, 7)), (True, (-7, 7)), (True, (-127, 127))]
RANGE_LAYOUTS = [('fast128', 128, 1024, None, FAST128), ('row2', 4096, 4096, None, ROW2),
                 ('warp', 128, 1024, 1032, WARP.format(4)), ('warp-g256', 256, 1024, None, WARP.format(4))]


@pytest.mark.parametrize('layout', RANGE_LAYOUTS, ids=[r[0] for r in RANGE_LAYOUTS])
@pytest.mark.parametrize('sym,qrange', RANGES, ids=['asym-8..7', 'sym-7..7', 'sym-127..127'])
@pytest.mark.parametrize('bit', [4, 8])
def test_use_range(bit, sym, qrange, layout):
    """use_range: QDQ, codes and packed words with an explicit [qmin, qmax].  An asymmetric range
    with negative codes cannot use the fast kernels' plain-code packing (it borrows across
    fields); those calls must still give the reference's bytes."""
    name, group, cols, ld, kernel = layout
    for dtype in (torch.float16, torch.bfloat16):
        w = _randw(64, cols, dtype, seed=bit)
        wv = _view(w, ld)
        ref = _ref_dyn(w, group, bit, sym, qrange)
        names = []
        for mode in (OUT_QDQ, OUT_CODES_I32, OUT_PACK_VLLM, OUT_CODES_I8 if sym else OUT_CODES_U8):
            if mode in (OUT_CODES_I8, OUT_CODES_U8) and bit != 8:
                continue
            got, n = _kernels(lambda: dyn(wv, group, bit, sym, mode, qrange))
            names += n
            _check_dyn(ref, got, mode, bit, cols, f'{name} {dtype} mode {mode}', 0, dtype)
        _assert_ran(names, kernel, name)


AWQ = [('fast64', 64, 1024, FAST64), ('fast128', 128, 1024, FAST128), ('warp-g32', 32, 1024, WARP.format(4)),
       ('warp-g256', 256, 1024, WARP.format(4)), ('block-perchannel', 4096, 4096, BLOCK)]


@pytest.mark.parametrize('layout', AWQ, ids=[a[0] for a in AWQ])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32], ids=['fp16', 'bf16', 'fp32'])
def test_awq_col_scale(dtype, layout):
    """col_scale: the kernels quantise rT(w * s[c]) (awq.py:147-164) without touching w."""
    name, group, cols, kernel = layout
    if dtype == torch.float32:
        kernel = {FAST64: WARP.format(4), FAST128: WARP.format(4)}.get(kernel, kernel)
    w = _randw(48, cols, dtype, seed=group)
    g = torch.Generator(device='cuda').manual_seed(group)
    cs = torch.exp(torch.randn(cols, generator=g, device='cuda') * 0.7).to(dtype)
    w0 = w.clone()
    _run_all(w, group, (4, 8), (True, False), name, kernel, col_scale=cs)
    _same(w, w0, 'weights after col_scale')


# ---- static qparams -----------------------------------------------------------------------------------
# (compute dtype, weight dtype, qparam dtype): the 11 combinations llmc_quant_static dispatches.
COMBOS = [(S, S, S), (H, H, H), (B, B, B), (S, S, H), (S, S, B), (S, H, S), (S, B, S), (S, H, B),
          (S, B, H), (H, H, S), (B, B, S)]


def stat(wv, scales, zeros, round_dtype, q_row_stride, group, gmap, bit, qmin, qmax, mode,
         out_dtype, ld_out=0, zp_inside=False):
    rows, cols = wv.shape
    out = _out_buf(mode, rows, cols, bit, out_dtype, ld_out)
    call('llmc_quant_static', ptr(wv), rows, cols, wv.stride(0), DT[wv.dtype], ptr(scales),
         ptr(zeros), DT[scales.dtype], round_dtype, q_row_stride, group, ptr(gmap), bit, qmin, qmax,
         mode | (ZP_INSIDE if zp_inside else 0), ptr(out), ld_out, DT[out_dtype], stream_ptr())
    return out


def _static_qparams(w, group, bit, sym, qt, real_zeros=False):
    t = w.float().reshape(w.shape[0], -1, group)
    qmax = 2 ** (bit - 1) - 1 if sym else 2 ** bit - 1
    s = (t.abs().amax(-1) / qmax * (1.3 if not sym else 1.0)).clamp(min=1e-5).to(qt)
    if sym:
        return s, None
    g = torch.Generator(device='cuda').manual_seed(5)
    z = torch.rand(s.shape, generator=g, device='cuda') * qmax
    return s, (z if real_zeros else z.round()).to(qt)


def _check_static(w, wv, s, z, ref_q, ref_y, ct, round_dtype, stride, group, gmap, bit, qmin, qmax,
                  what, zp_inside=False, vec=True):
    """QDQ (with ld_out > cols), codes and packed words of one static call against (ref_q, ref_y)."""
    rows, cols = w.shape
    ld_out = cols + (8 if vec else 3)
    names = []
    for mode in (OUT_QDQ, OUT_CODES_I32, OUT_PACK_VLLM):
        if mode == OUT_PACK_VLLM and (bit not in (4, 8) and vec):
            continue
        lo = ld_out if mode == OUT_QDQ else 0
        out, n = _kernels(lambda: stat(wv, s, z, round_dtype, stride, group, gmap, bit, qmin, qmax, mode,
                                       ct, lo, zp_inside))
        names += n
        if mode == OUT_QDQ:
            _same(out[:, :cols], ref_y.to(ct), f'{what} qdq')
            assert bool((out[:, cols:] == -3.0).all()), f'{what}: QDQ wrote into the ld_out padding'
        elif mode == OUT_CODES_I32:
            _same(out, ref_q.to(torch.int32), f'{what} codes')
        else:
            _same(out, qo.pack_vllm(ref_q.to(torch.int32).cpu(), s.cpu(), bit)[0], f'{what} packed')
    return names


@pytest.mark.parametrize('vec', [True, False], ids=['vec8', 'scalar'])
@pytest.mark.parametrize('combo', COMBOS, ids=['-'.join(str(d)[6:] for d in c) for c in COMBOS])
def test_static_combos(combo, vec):
    """Static qparams for every (compute, weight, qparam) dtype combination on both kernels.  The
    last two are torch's CPU scalar-operand path: a 0-dim fp32 scale with results rounded to the
    tensor dtype (round_dtype), so their oracle runs on CPU."""
    ct, wt, qt = combo
    rows, cols, group = 24, 512, 128
    w = _randw(rows, cols, wt, seed=11)
    wv = _view(w, None if vec else cols + 1)
    for sym in (True, False):
        bit = 4
        qmin, qmax = qo.int_range(bit, sym)
        if qt == S and ct == wt != S:              # 0-dim fp32 qparams, round_dtype = w dtype
            sval = float(w.float().abs().max()) / 7
            s = torch.tensor([sval], dtype=torch.float32, device='cuda')
            z = None if sym else torch.tensor([3.0], device='cuda')
            s0, z0 = torch.tensor(sval), (torch.tensor(0.0) if sym else torch.tensor(3.0))
            q = qo.quant(w.cpu(), s0, z0, qmax, qmin)
            y = qo.dequant(q, s0, z0)
            stride, grp, rd = 0, cols, DT[wt]
        else:
            s, z = _static_qparams(w, group, bit, sym, qt)
            t = w.reshape(-1, group)
            zz = torch.tensor(0.0) if z is None else z.reshape(-1, 1)
            q = qo.quant(t, s.reshape(-1, 1), zz, qmax.cuda(), qmin.cuda())
            y = qo.dequant(q, s.reshape(-1, 1), zz)
            q, y = q.reshape(rows, cols), y.reshape(rows, cols)
            stride, grp, rd = cols // group, group, -1
        assert y.dtype == ct
        names = _check_static(w, wv, s, z, q, y, ct, rd, stride, grp, None, bit, int(qmin), int(qmax),
                              f'{combo} sym {sym}', vec=vec)
        kern = 'quant_static_vec8_kernel' if vec else 'quant_static_kernel'
        _assert_ran(names, rf'{kern}<{DT[ct]},{DT[wt]},{DT[qt]}>', f'{combo} {kern}')


GMAP = [(S, S, S), (B, B, B), (S, H, S), (S, S, H)]


@pytest.mark.parametrize('zp_inside', [False, True], ids=['round_zp', 'zp_inside'])
@pytest.mark.parametrize('vec', [True, False], ids=['vec8', 'scalar'])
@pytest.mark.parametrize('combo', GMAP, ids=['-'.join(str(d)[6:] for d in c) for c in GMAP])
def test_static_gmap_and_zp_inside(combo, vec, zp_inside):
    """Act-order: column c uses group invperm[c] // group (gptq.py:424-452), a real permutation, so
    the eight columns of one vector belong to different groups.  zp_inside: round_zp False
    (quant.py:702-707) with real-valued zero-points added before the rounding."""
    ct, wt, qt = combo
    rows, cols, group = 32, 1024, 128
    w = _randw(rows, cols, wt, seed=13)
    wv = _view(w, None if vec else cols + 1)
    g = torch.Generator(device='cuda').manual_seed(17)
    perm = torch.randperm(cols, generator=g, device='cuda')
    gmap = (torch.argsort(perm) // group).to(torch.int32)
    for sym in ((False,) if zp_inside else (True, False)):
        for bit in (4, 8):
            qmin, qmax = qo.int_range(bit, sym)
            s, z = _static_qparams(w[:, perm], group, bit, sym, qt, real_zeros=zp_inside)
            zz = torch.tensor(0.0) if z is None else z
            q, y = qo.quant_static_gmap(w, s, zz, gmap.long(), qmax.cuda(), qmin.cuda(),
                                        round_zp=not zp_inside)
            names = _check_static(w, wv, s, z, q, y, ct, -1, cols // group, group, gmap, bit, int(qmin),
                                  int(qmax), f'{combo} bit {bit} sym {sym}', zp_inside, vec)
            _assert_ran(names, 'quant_static_vec8_kernel' if vec else 'quant_static_kernel<', str(combo))


def test_static_ungrouped_zp_inside():
    """zp_inside without a column map on both static kernels, fp16 qparams with an fp32 weight."""
    rows, cols, group = 16, 256, 64
    w = _randw(rows, cols, torch.float32, seed=19)
    s, z = _static_qparams(w, group, 4, False, torch.float16, real_zeros=True)
    qmin, qmax = qo.int_range(4, False)
    t = w.reshape(-1, group)
    q = qo.quant(t, s.reshape(-1, 1), z.reshape(-1, 1), qmax.cuda(), qmin.cuda(), round_zp=False)
    y = qo.dequant(q, s.reshape(-1, 1), z.reshape(-1, 1))
    for vec in (True, False):
        _check_static(w, _view(w, None if vec else cols + 1), s, z, q.reshape(rows, cols),
                      y.reshape(rows, cols), torch.float32, -1, cols // group, group, None, 4, 0, 15,
                      f'vec {vec}', True, vec)


# ---- minmax_tensor and pack_vllm_codes ------------------------------------------------------------------
@pytest.mark.parametrize('n', [13, 1000003, 1024 * 256 * 8 * 2 + 7])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32], ids=['fp16', 'bf16', 'fp32'])
def test_minmax_tensor(dtype, n):
    """Per-tensor range: the tail past the last multiple of 8 (read by block 0), the grid-stride loop
    beyond 1024 blocks x 256 threads x 8, +-inf and -0.  Compared by value (-0 == +0)."""
    g = torch.Generator(device='cuda').manual_seed(n)
    base = (torch.randn(n, generator=g, device='cuda') * 0.5).to(dtype)
    ws = torch.empty(2048, dtype=torch.float32, device='cuda')
    n8 = (n // 8) * 8
    cases = {'random': base}
    x = base.clone()
    x[n - 1] = 50.0
    x[max(n - 2, 0)] = -50.0
    cases['extremes in tail'] = x
    x = base.clone()
    x[n8 - 1] = 60.0
    x[min(1024 * 256 * 8 + 3, n8 - 2)] = -60.0
    cases['extremes late in the stride'] = x
    x = base.clone()
    x[n // 3] = float('inf')
    x[n // 2] = -float('inf')
    cases['+-inf'] = x
    cases['all -0'] = torch.full((n,), -0.0, dtype=dtype, device='cuda')
    x = torch.full((n,), -0.0, dtype=dtype, device='cuda')
    x[::3] = 0.0
    cases['mixed zeros'] = x
    for what, x in cases.items():
        names = []
        mm = torch.empty(2, dtype=dtype, device='cuda')
        _, names = _kernels(lambda: call('llmc_minmax_tensor', ptr(x), n, DT[dtype], ptr(mm), ptr(ws),
                                         stream_ptr()))
        _assert_ran(names, 'minmax_stage1<', what)
        _assert_ran(names, 'minmax_stage2<', what)
        assert float(mm[0]) == float(x.min()) and float(mm[1]) == float(x.max()), \
            (what, mm.tolist(), float(x.min()), float(x.max()))


@pytest.mark.parametrize('code_dtype', [torch.int8, torch.int32])
@pytest.mark.parametrize('bit', [2, 3, 4, 5, 6, 7, 8])
def test_pack_vllm_codes(bit, code_dtype):
    """Packing precomputed codes, including codes outside the bit's range (the reference's
    (code + 2^(bit-1)).to(uint8) keeps the low byte) and widths that leave a partial last word."""
    g = torch.Generator().manual_seed(bit)
    for rows, cols in ((33, 128), (5, 100), (3, 7), (17, 4096)):
        hi = 128 if code_dtype == torch.int8 else 1000
        codes = torch.randint(-hi, hi, (rows, cols), generator=g).to(code_dtype)
        lim = 2 ** (bit - 1)
        codes[::2] = codes[::2].clamp(-lim, lim - 1)
        cuda = codes.cuda()
        out = torch.full((rows, math.ceil(cols / (32 // bit))), SENTINEL, dtype=torch.int32, device='cuda')
        _, names = _kernels(lambda: call('llmc_pack_vllm_codes', ptr(cuda), cuda.element_size(), rows, cols,
                                         bit, ptr(out), stream_ptr()))
        _assert_ran(names, 'pack_vllm_codes_kernel<', f'{rows}x{cols}')
        _same(out, qo.pack_vllm(codes, torch.ones(rows), bit)[0], f'{rows}x{cols} {code_dtype}')


# ---- the CUDA-run oracle ------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32], ids=['fp16', 'bf16', 'fp32'])
def test_cuda_oracle_equals_cpu_oracle(dtype):
    """The sweeps above run the oracle on CUDA tensors.  That rests on torch's CUDA division,
    rounding and reductions being the IEEE operations of its CPU kernels: checked here bit for bit
    on a subsample of ladder, degenerate and scaled random groups, sym and asym."""
    parts = [_special_groups(dtype, 128).float()]
    for scale in (1e-6, 1e-3, 1.0, 300.0):
        parts.append((torch.randn(64, 128, device='cuda') * scale))
    if dtype != torch.float32:
        lad = _ladder(dtype, False, 128, 1).float()
        parts.append(lad[torch.randperm(lad.shape[0], device='cuda')[:2000]])
    w = torch.cat(parts).to(dtype)
    for sym in (True, False):
        for bit in (3, 4, 8):
            for qrange in (None, (-8, 7)):
                c = _ref_dyn(w, 128, bit, sym, qrange)
                h = _ref_dyn(w.cpu(), 128, bit, sym, qrange)
                for k in ('s', 'z', 'q', 'y'):
                    if c[k] is not None:
                        _same(c[k].cpu(), h[k], f'{k} bit {bit} sym {sym} range {qrange}')
