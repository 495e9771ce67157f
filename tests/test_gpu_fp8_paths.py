"""GPU: every path of the FP8 quantiser (csrc/fp8.cu: llmc_fp8_quant, llmc_fp8_block_quant,
llmc_fp8_block_dequant) and of FloatQuantizer against the oracle (oracle/fp8_oracle.py, run on the
CPU), bit for bit.

The kernels are called through the C ABI where the Python classes cannot reach a path (out_mode 0 of
the dynamic kernel, raw scales, oversized output buffers), and torch.profiler records which kernel
each entry point runs for each dtype (`test_kernels_ran`, in a child process), so that a dispatch change cannot quietly
leave a path untested.  The rounding itself is IEEE
round-to-nearest-even onto the e4m3fn / e5m2 grid with saturation (PARITY UNPINNED w.r.t. qtorch,
see the oracle's header); everything around it follows the reference's dtype and object flow.

NaN: the kernels' absmax propagates NaN as the reference's amax / clamp do, so a NaN (or an inf,
through inf / inf and 0 * inf) anywhere in a group makes the whole group NaN.  A NaN result matches
any NaN, whatever its payload and sign: the CPU's division gives a negative default NaN where the
GPU gives a positive one.  Likewise any NaN byte (0x7f / 0xff on either grid) matches any other."""
import pytest
import torch

from llmc_b200._lib import BF16, F16, F32, call, ptr, stream_ptr
from oracle import fp8_oracle as fo

pytestmark = pytest.mark.gpu

DT = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
E5M2 = {'e4m3': 0, 'e5m2': 1}
FMAX = {'e4m3': 448.0, 'e5m2': 57344.0}
SCALE_SENTINEL = -7.0
OUT_SENTINEL = -3.0
BYTE_SENTINEL = 0x5A


# ---- helpers (as in test_gpu_quant_paths.py) -------------------------------------------------------
def _same(got, exp, what):
    """Bit-exact equality; NaN matches NaN whatever its payload."""
    got, exp = got.cpu(), exp.cpu()
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


def _same_codes(got, exp, bit, what):
    """fp8 bytes equal; a NaN code matches any NaN code."""
    got, exp = got.cpu().view(torch.uint8), exp.cpu().view(torch.uint8)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    gn = got.view(fo.FP8[bit]).float().isnan()
    en = exp.view(fo.FP8[bit]).float().isnan()
    bad = (gn != en) | (~gn & (got != exp))
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        first = [(i, hex(got[tuple(i)].item()), hex(exp[tuple(i)].item())) for i in idx]
        raise AssertionError(f'{what}: {int(bad.sum())}/{got.numel()} codes differ; first (index, got, '
                             f'expected): {first}')


PROBE = 'llmc_fp8_probe'


class _Recorder:
    """torch.profiler around a block; `call(fn)` runs fn inside a probe range and `.names` lists
    the llmc kernels launched inside the probes (spaces removed).  Kernels are attributed through
    the profiler's launch correlation, else by start time."""

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
        self.names = [n.replace(' ', '') for n in names if 'fp8' in n]
        return False


def _kernels(fn, tries=3):
    """Run fn under torch.profiler -> (its result, names of the fp8 kernels it launched).  fn is
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


def _run(fn, pattern, what):
    res, names = _kernels(fn)
    _assert_ran(names, pattern, what)
    return res


# ---- C ABI -----------------------------------------------------------------------------------------
def fp8_quant(w2d, group, bit, dynamic, scales, mode, q_row_stride=0, scale_f32=0):
    """llmc_fp8_quant on a contiguous CUDA [rows, cols] -> the output buffer (None for mode 0)."""
    rows, cols = w2d.shape
    out = None
    if mode == 1:
        out = torch.full_like(w2d, OUT_SENTINEL)
    elif mode == 2:
        out = torch.full(w2d.shape, BYTE_SENTINEL, dtype=torch.uint8, device=w2d.device)
    call('llmc_fp8_quant', ptr(w2d), rows, cols, DT[w2d.dtype], int(group), E5M2[bit], int(dynamic),
         ptr(scales), int(q_row_stride), int(scale_f32), mode, ptr(out), stream_ptr(w2d.device))
    return out


def _randw(shape, dtype, seed):
    """randn * 0.05 with outlier columns; with four rows or more also an all-zero row, a row of
    absmax ~4e-4 (its fp16 e5m2 scale underflows to 0) and a row of -0.0 / +-values."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(shape, generator=g) * 0.05
    w2 = w.view(-1, shape[-1])
    w2[:, ::37] *= 7
    if w2.shape[0] >= 4:
        w2[0].zero_()
        w2[1] *= 0.002
        w2[2, ::3] = -0.0
    return w.to(dtype)


def _eff(s):
    """The scale quant() divides and multiplies by: zero replaced by 1 (quant.py:1062)."""
    return torch.where(s == 0, torch.ones_like(s), s)


# ---- which kernel each entry point runs ------------------------------------------------------------
def _check_kernels_ran():
    """Each entry point has one kernel per input dtype; the profiler records it once per dtype."""
    for dtype in DTYPES:
        w = _randw((64, 256), dtype, seed=1).cuda()
        s = torch.ones((64 * 4, 1), dtype=dtype, device='cuda')
        t = DT[dtype]
        _run(lambda: fp8_quant(w, 64, 'e4m3', 1, s, 2), rf'fp8_dynamic_kernel<{t}>', f'{dtype} dynamic')
        _run(lambda: fp8_quant(w, 64, 'e5m2', 0, s, 1, 4, 0), rf'fp8_static_kernel<{t}>', f'{dtype} static')
        sc = torch.empty(2, dtype=torch.float32, device='cuda')
        q = torch.empty((64, 256), dtype=torch.uint8, device='cuda')
        _run(lambda: call('llmc_fp8_block_quant', ptr(w), 64, 256, t, 128, 0, ptr(sc), 2, ptr(q),
                          stream_ptr(w.device)), rf'fp8_block_quant_kernel<{t}>', f'{dtype} block quant')
        back = torch.empty((64, 256), dtype=torch.bfloat16, device='cuda')
        _run(lambda: call('llmc_fp8_block_dequant', ptr(q), 64, 256, 128, 0, ptr(sc), ptr(back),
                          stream_ptr(w.device)), r'fp8_block_dequant_kernel', f'{dtype} block dequant')


def test_kernels_ran():
    """_check_kernels_ran in a child process: profiling in the test process left later
    torch.profiler sessions (test_gpu_quant_paths) without kernel records, so this file keeps its
    sessions out of it."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    path = os.pathsep.join([root, here, os.environ.get('PYTHONPATH', '')])
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE='1', PYTHONPATH=path)
    r = subprocess.run([sys.executable, '-c', 'import test_gpu_fp8_paths as t; t._check_kernels_ran()'],
                       cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


# ---- llmc_fp8_quant, dynamic -----------------------------------------------------------------------
LAYOUTS = {   # name: (shape, granularity, group_size)
    'per_channel': ((96, 512), 'per_channel', None),
    'group32': ((96, 512), 'per_group', 32),
    'group64': ((96, 512), 'per_group', 64),
    'group128': ((96, 512), 'per_group', 128),
    'group2048': ((6, 4096), 'per_group', 2048),          # wider than the 256-thread block
    'short_rows': ((2, 5, 96), 'per_group', 128),         # a row shorter than the group is one group
    'per_token_3d': ((3, 7, 256), 'per_token', None),
    'one_row': ((1, 384), 'per_channel', None),
}


def _dyn_case(w, gran, gs, bit):
    """-> (w2d on CUDA, group, oracle view t, oracle scales of t as get_qparams returns them)."""
    C = w.shape[-1]
    group = gs if gran == 'per_group' and C >= gs else C
    t = fo.reshape(w, gran, gs).reshape(-1, group)
    return w.reshape(-1, C).contiguous().cuda(), group, t, fo.qparams(t, bit, gran)


def _check_dynamic(w, gran, gs, bit, what):
    w2d, group, t, s_o = _dyn_case(w, gran, gs, bit)
    rows, cols = w2d.shape
    n = rows * (cols // group)
    y_o = fo.quant_dequant(t, s_o.clone(), bit).reshape(w2d.shape).to(w.dtype)
    q_o = fo.quant(t, s_o.clone(), bit).reshape(w2d.shape).to(fo.FP8[bit])
    outs = {}
    for mode in (0, 1, 2):
        s = torch.full((n + 32, 1), SCALE_SENTINEL, dtype=w.dtype, device='cuda')
        out = fp8_quant(w2d, group, bit, 1, s, mode)
        # the kernel writes get_qparams' scales, zeros included; FloatQuantizer maps them for export
        _same(s[:n], s_o.reshape(n, 1), f'{what} mode {mode} scales')
        assert bool((s[n:] == SCALE_SENTINEL).all()), f'{what}: scales written past {n}'
        outs[mode] = out
    _same(outs[1], y_o, f'{what} QDQ')
    _same_codes(outs[2], q_o, bit, f'{what} codes')
    # the bytes with their (zero -> 1) scales rebuild the QDQ output exactly
    s_full = _eff(s_o).reshape(rows, cols // group).repeat_interleave(group, 1).cuda()
    rebuilt = (outs[2].view(fo.FP8[bit]).float() * s_full).to(w.dtype)
    _same(rebuilt, outs[1], f'{what} bytes * scales vs QDQ')


@pytest.mark.parametrize('layout', list(LAYOUTS))
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_dynamic_paths(dtype, bit, layout):
    shape, gran, gs = LAYOUTS[layout]
    w = _randw(shape, dtype, seed=len(layout) * 31 + shape[-1])
    _check_dynamic(w, gran, gs, bit, f'{layout} {dtype} {bit}')


@pytest.mark.parametrize('case', ['per_channel_8192x512', 'group64_4096x4096'])
def test_dynamic_grid_stride(case):
    """More groups than the kNumSMs * 32 CTAs launched: every CTA loops."""
    if case == 'per_channel_8192x512':
        w, gran, gs, bit = _randw((8192, 512), torch.bfloat16, 1), 'per_channel', None, 'e4m3'
    else:
        w, gran, gs, bit = _randw((4096, 4096), torch.float16, 2), 'per_group', 64, 'e5m2'
    _check_dynamic(w, gran, gs, bit, case)


# ---- llmc_fp8_quant, static ------------------------------------------------------------------------
STATIC = {   # name: (shape, granularity, group_size)
    'per_tensor': ((64, 384), 'per_tensor', None),
    'per_channel': ((64, 384), 'per_channel', None),
    'group64': ((64, 384), 'per_group', 64),
    'group2048': ((4, 4096), 'per_group', 2048),
    'one_row': ((1, 384), 'per_channel', None),
    'grid_stride': ((2048, 2048), 'per_group', 128),      # rows * cols / 256 > kNumSMs * 32 blocks
}


def _static_scales(w, gran, gs, bit, seed):
    """Calibrated-looking scales: get_qparams' times a factor in [0.4, 1.6) (so some quotients
    saturate), one of them 0.  per_tensor: a 0-dim fp32 scalar."""
    t = fo.reshape(w, gran, gs)
    s = fo.qparams(t, bit, gran)
    g = torch.Generator().manual_seed(seed)
    f = 0.4 + 1.2 * torch.rand(s.shape, generator=g)
    s = (s.float() * f).to(s.dtype)
    if gran != 'per_tensor':
        s.view(-1)[min(3, s.numel() - 1)] = 0
    return t, s


@pytest.mark.parametrize('layout', list(STATIC))
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_static_paths(dtype, bit, layout):
    shape, gran, gs = STATIC[layout]
    what = f'static {layout} {dtype} {bit}'
    w = _randw(shape, dtype, seed=7 + shape[0])
    t, s_o = _static_scales(w, gran, gs, bit, seed=shape[1])
    w2d = w.cuda()
    rows, cols = w2d.shape
    if gran == 'per_tensor':
        s_dev, group, stride, f32 = s_o.reshape(1).float().cuda(), cols, 0, 1
    else:
        group = gs if gran == 'per_group' else cols
        s_dev, stride, f32 = s_o.reshape(-1).cuda(), cols // group, 0
    y_o = fo.quant_dequant(t, s_o.clone(), bit).reshape(w.shape).to(dtype)
    q_o = fo.quant(t, s_o.clone(), bit).reshape(w.shape).to(fo.FP8[bit])
    y = fp8_quant(w2d, group, bit, 0, s_dev, 1, stride, f32)
    _same(y, y_o, f'{what} QDQ')
    _same_codes(fp8_quant(w2d, group, bit, 0, s_dev, 2, stride, f32), q_o, bit, f'{what} codes')


@pytest.mark.parametrize('sdtype', DTYPES + ['0-dim'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_static_scale_dtypes_and_mutation(dtype, sdtype):
    """FloatQuantizer's static paths with scales of another dtype than the weight: the division
    follows torch's promotion (a dimensioned fp32 / other-16-bit scale gives an fp32 quotient), and
    args['scales'] comes back with its zeros set to 1, as quant.py:1062 leaves it."""
    from llmc_b200.quant_float import FloatQuantizer
    for bit in ('e4m3', 'e5m2'):
        what = f'{dtype} scales {sdtype} {bit}'
        w = _randw((48, 256), dtype, seed=5)
        if sdtype == '0-dim':
            gran, s0 = 'per_tensor', (w.float().abs().max() / FMAX[bit] * 0.5)
        else:
            gran = 'per_channel'
            s0 = (fo.qparams(w.float(), bit, gran) * 0.8).to(sdtype)
            s0[5] = 0
        q = FloatQuantizer(bit, True, gran, use_qtorch=True)
        args = {'scales': s0.clone().cuda()}
        y = q.fake_quant_weight_static(w.cuda(), args)
        s_ref = s0.clone()
        y_o = fo.fake_quant_static(w, s_ref, bit, gran)
        _same(y, y_o, f'{what} fake_quant_weight_static')
        _same(args['scales'], s_ref, f'{what} args[scales] after fake quant')

        args = {'scales': s0.clone().cuda()}
        ya = q.fake_quant_act_static(w.cuda(), args)
        _same(ya, y_o, f'{what} fake_quant_act_static')
        _same(args['scales'], s_ref, f'{what} args[scales] after act fake quant')

        args = {'scales': s0.clone().cuda()}
        fw, fs, z = q.real_quant_weight_static(w.cuda(), args)
        s_ref = s0.clone()
        q_o, fs_o = fo.real_quant_static(w, s_ref, bit, gran)
        assert z is None and fw.dtype == fo.FP8[bit]
        _same_codes(fw, q_o, bit, f'{what} real_quant_weight_static codes')
        _same(fs, fs_o, f'{what} real_quant_weight_static scales')
        _same(args['scales'], s_ref, f'{what} args[scales] after real quant')


# ---- llmc_fp8_block_quant / llmc_fp8_block_dequant -------------------------------------------------
@pytest.mark.parametrize('M,N', [(1, 1), (127, 129), (300, 127), (129, 300)])
@pytest.mark.parametrize('bs', [64, 128, 256])
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
def test_block_paths(bit, bs, M, N):
    """Scales, QDQ and bytes of every ragged block, and nothing written past M x N or past the
    ceil(M/bs) x ceil(N/bs) scales (oversized sentinel-filled buffers)."""
    mb, nb = -(-M // bs), -(-N // bs)
    for dtype in DTYPES:
        what = f'block {bs} {M}x{N} {dtype} {bit}'
        w = _randw((M, N), dtype, seed=M * 7 + N)
        wd = w.cuda()
        q_o, s_o = fo.block_quant(w, bit, bs)
        y_o, _ = fo.block_fake_quant(w, bit, bs)
        outs = {}
        for mode in (0, 1, 2):
            sc = torch.full((mb * nb + 64,), SCALE_SENTINEL, dtype=torch.float32, device='cuda')
            out = None
            if mode == 1:
                out = torch.full((M * N + 1024,), OUT_SENTINEL, dtype=dtype, device='cuda')
            elif mode == 2:
                out = torch.full((M * N + 1024,), BYTE_SENTINEL, dtype=torch.uint8, device='cuda')
            call('llmc_fp8_block_quant', ptr(wd), M, N, DT[dtype], bs, E5M2[bit], ptr(sc), mode, ptr(out),
                 stream_ptr(wd.device))
            _same(sc[:mb * nb].view(mb, nb), s_o, f'{what} mode {mode} scales')
            assert bool((sc[mb * nb:] == SCALE_SENTINEL).all()), f'{what}: scales written past the blocks'
            if out is not None:
                tail = out[M * N:]
                assert bool((tail == (OUT_SENTINEL if mode == 1 else BYTE_SENTINEL)).all()), \
                    f'{what} mode {mode}: written past M x N'
                outs[mode] = out[:M * N].view(M, N)
        _same(outs[1], y_o, f'{what} QDQ')
        _same_codes(outs[2], q_o, bit, f'{what} codes')
        # weight_cast_to_bf16's kernel on either grid, with the same sentinel tail
        back = torch.full((M * N + 1024,), OUT_SENTINEL, dtype=torch.bfloat16, device='cuda')
        s_dev = s_o.cuda()
        call('llmc_fp8_block_dequant', ptr(outs[2]), M, N, bs, E5M2[bit], ptr(s_dev), ptr(back),
             stream_ptr(wd.device))
        _same(back[:M * N].view(M, N), fo.block_dequant(q_o, s_o, bs), f'{what} dequant')
        assert bool((back[M * N:] == OUT_SENTINEL).all()), f'{what}: dequant written past M x N'


@pytest.mark.parametrize('bs', [64, 128, 256])
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_per_block_quantizer(dtype, bit, bs):
    """FloatQuantizer(per_block): fake quant, get_tensor_qparams and real quant, then
    weight_cast_to_bf16 of the real-quant output (M ragged, N a multiple of every block)."""
    from llmc_b200.quant_float import FloatQuantizer, weight_cast_to_bf16
    what = f'per_block {bs} {dtype} {bit}'
    w = _randw((300, 512), dtype, seed=bs)
    wd = w.cuda()
    q = FloatQuantizer(bit, True, 'per_block', block_size=bs, use_qtorch=True)
    y_o, s_o = fo.block_fake_quant(w, bit, bs)
    _same(q.fake_quant_weight_dynamic(wd), y_o, f'{what} fake quant')
    t, s, z, qmax, qmin = q.get_tensor_qparams(wd)
    tv = fo._block_view(w, bs)
    _same(t, tv, f'{what} reshaped')
    _same(s, fo.block_qparams(tv, bit), f'{what} get_tensor_qparams scales')
    assert float(qmax) == FMAX[bit] and float(qmin) == -FMAX[bit] and float(z) == 0
    fw, fs, _ = q.real_quant_weight_dynamic(wd)
    q_o, fs_o = fo.block_quant(w, bit, bs)
    _same_codes(fw, q_o, bit, f'{what} real quant codes')
    _same(fs, fs_o, f'{what} real quant scales')
    _same(weight_cast_to_bf16(fw, fs, bs), fo.block_dequant(q_o, fs_o, bs), f'{what} weight_cast_to_bf16')


# ---- value edges -----------------------------------------------------------------------------------
def _all_16bit(dtype):
    """Every bit pattern of a 16-bit dtype as a [256, 256] tensor: ties, subnormals of both the input
    and the fp8 grid, saturation, +-0, +-inf and NaN, one row per 256 consecutive patterns."""
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype).reshape(256, 256)


def _fp32_edges():
    """fp32: every finite value of both fp8 grids, the midpoints between neighbours and one fp32 ulp
    either side of them, values beyond finfo.max, fp32 subnormals, +-0, +-inf and NaN."""
    vals = []
    for fp8 in (torch.float8_e4m3fn, torch.float8_e5m2):
        g = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(fp8).float()
        g = g[torch.isfinite(g)].unique()
        mid = (g[1:] + g[:-1]) / 2
        vals += [g, mid, torch.nextafter(mid, torch.tensor(float('inf'))),
                 torch.nextafter(mid, torch.tensor(-float('inf')))]
    vals.append(torch.tensor([0.0, -0.0, 1e-45, -1e-45, 1e-40, 448.5, 464.0, -500.0, 61440.0, 65536.0,
                              -1e38, 3e38, float('inf'), -float('inf'), float('nan')]))
    v = torch.cat(vals)
    v = torch.cat([v, torch.zeros((-v.numel()) % 256)])
    return v.reshape(-1, 256)


def _edge_tensor(dtype):
    return _fp32_edges() if dtype == torch.float32 else _all_16bit(dtype)


@pytest.mark.parametrize('path', ['static_1', 'static_0.3', 'static_2^-12', 'dynamic_rows',
                                  'dynamic_g32'])
@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_value_edges(dtype, bit, path):
    """Static per-tensor scale 1 puts the input values on the grid's rounding boundaries themselves;
    0.3 overflows fp16 quotients to inf (which must give +-fmax); 2^-12 pushes most values into
    saturation.  The dynamic paths put inf and NaN into groups of finite values."""
    w = _edge_tensor(dtype)
    what = f'edges {path} {dtype} {bit}'
    if path.startswith('dynamic'):
        _check_dynamic(w, 'per_group' if path == 'dynamic_g32' else 'per_channel', 32, bit, what)
        return
    s = torch.tensor({'static_1': 1.0, 'static_0.3': 0.3, 'static_2^-12': 2.0 ** -12}[path])
    wd = w.cuda()
    s_dev = s.reshape(1).cuda()
    y_o = fo.quant_dequant(w, s.clone(), bit).to(dtype)
    q_o = fo.quant(w, s.clone(), bit).to(fo.FP8[bit])
    _same(fp8_quant(wd, w.shape[1], bit, 0, s_dev, 1, 0, 1), y_o, f'{what} QDQ')
    _same_codes(fp8_quant(wd, w.shape[1], bit, 0, s_dev, 2, 0, 1), q_o, bit, f'{what} codes')


@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_zero_static_scale(dtype, bit):
    """A static scale of 0 quantises with 1 (quant.py:1062), per tensor and per channel."""
    w = _randw((8, 128), dtype, seed=3) * 40
    wd = w.cuda()
    y_o = fo.quant_dequant(w, torch.tensor(1.0), bit).to(dtype)
    _same(fp8_quant(wd, 128, bit, 0, torch.zeros(1, device='cuda'), 1, 0, 1), y_o, f'{dtype} {bit} per-tensor 0')
    s = torch.zeros(8, dtype=dtype, device='cuda')
    _same(fp8_quant(wd, 128, bit, 0, s, 1, 1, 0), y_o, f'{dtype} {bit} per-channel 0')
    _same_codes(fp8_quant(wd, 128, bit, 0, s, 2, 1, 0), fo.quant(w, torch.tensor(1.0), bit).to(fo.FP8[bit]),
                bit, f'{dtype} {bit} per-channel 0 codes')


# ---- the defects this file pins ---------------------------------------------------------------------
@pytest.mark.parametrize('gran,gs', [('per_channel', None), ('per_group', 64)])
def test_fp16_underflow_exports_scale_one(gran, gs):
    """fp16 / e5m2: a group of absmax 1e-3 gets the scale 1e-3 / 57344, which underflows to 0 in fp16;
    e4m3: an all-zero group does too.  The kernel quantises such a group with scale 1, so the export
    must say 1: real_quant_weight_dynamic returns scale 1 and codes fp8(x), dequantising its output
    gives the fake-quant output, and the fp8 dequant GEMM is handed the same bytes and scales."""
    from llmc_b200.blockwise import BaseBlockwiseQuantization
    from llmc_b200.quant_float import FloatQuantizer
    for bit in ('e5m2', 'e4m3'):
        g = torch.Generator().manual_seed(11)
        w = torch.randn(16, 256, generator=g) * 0.05
        w[3] = torch.linspace(-1e-3, 1e-3, 256)
        w[7] = 0
        w = w.half()
        small = [3, 7] if bit == 'e5m2' else [7]
        kw = {'group_size': gs} if gs else {}
        q = FloatQuantizer(bit, True, gran, use_qtorch=True, **kw)
        fw, fs, _ = q.real_quant_weight_dynamic(w.cuda())
        q_o, fs_o = fo.real_quant_dynamic(w, bit, gran, gs)
        _same_codes(fw, q_o, bit, f'{bit} {gran} codes')
        _same(fs, fs_o, f'{bit} {gran} scales')
        for r in small:
            assert bool((fs[r] == 1).all()), (bit, gran, r, fs[r])
            _same_codes(fw[r], w[r].float().to(fo.FP8[bit]), bit, f'{bit} row {r}: codes are fp8(x)')
        group = gs or 256
        deq = (fw.float() * fs.repeat_interleave(group, 1)).half()
        _same(deq, q.fake_quant_weight_dynamic(w.cuda()), f'{bit} {gran} dequant(real) vs fake')
        lin = torch.nn.Linear(256, 16, bias=False).half().cuda()
        lin.weight.data.copy_(w)
        packed = BaseBlockwiseQuantization._fp8_packed(lin, q)
        _same_codes(packed['qweight'], fw, bit, f'{bit} {gran} _fp8_packed bytes')
        _same(packed['scales'], fs, f'{bit} {gran} _fp8_packed scales')


@pytest.mark.parametrize('gran,gs', [('per_tensor', None), ('per_channel', None), ('per_group', 128)])
def test_fp8_packed_is_real_quant(gran, gs):
    """The dequant GEMM's operands (blockwise._fp8_packed) are the real-quant export's bytes and
    scales, per-tensor's scalar expanded to one fp32 scale per row."""
    from llmc_b200.blockwise import BaseBlockwiseQuantization
    from llmc_b200.quant_float import FloatQuantizer
    w = _randw((64, 512), torch.bfloat16, seed=9).cuda()
    kw = {'group_size': gs} if gs else {}
    for bit in ('e4m3', 'e5m2'):
        q = FloatQuantizer(bit, True, gran, use_qtorch=True, **kw)
        lin = torch.nn.Linear(512, 64, bias=False).bfloat16().cuda()
        lin.weight.data.copy_(w)
        packed = BaseBlockwiseQuantization._fp8_packed(lin, q)
        fw, fs, _ = q.real_quant_weight_dynamic(w)
        _same_codes(packed['qweight'], fw, bit, f'{gran} {bit} bytes')
        exp = fs.reshape(1).float().expand(64, 1) if gran == 'per_tensor' else fs
        _same(packed['scales'], exp.contiguous(), f'{gran} {bit} scales')


@pytest.mark.parametrize('dtype', DTYPES)
def test_quant_dequant_returns_fp32(dtype):
    """quant.py:1078-1081: the fp32 grid values times the scales is fp32, whatever the tensor's dtype."""
    from llmc_b200.quant_float import FloatQuantizer
    w = _randw((32, 256), dtype, seed=4)
    q = FloatQuantizer('e4m3', True, 'per_channel', use_qtorch=True)
    t, s, z, qmax, qmin = q.get_tensor_qparams(w.cuda())
    y = q.quant_dequant(t, s.clone(), z, qmax, qmin)
    assert y.dtype == torch.float32
    _same(y, fo.quant_dequant(w, fo.qparams(w, 'e4m3', 'per_channel'), 'e4m3'), f'{dtype} quant_dequant')
    s_o = fo.qparams(w, 'e4m3', 'per_channel')
    _same(q.quant(t, s, z, qmax, qmin), fo.quant(w, s_o, 'e4m3'), f'{dtype} quant')
    _same(s, s_o, f'{dtype} scales after quant')          # fp16: the all-zero row's 0 is now 1


@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
def test_per_head_is_per_head(bit):
    """quant.py:633-634: per_head reshapes to (head_num, -1); 8 rows in 4 heads give 4 scales, each
    over two rows of different ranges (per-row scales would differ)."""
    from llmc_b200.quant_float import FloatQuantizer
    g = torch.Generator().manual_seed(2)
    w = (torch.randn(8, 64, generator=g) * torch.tensor([1.0, 8.0] * 4).unsqueeze(1)).bfloat16()
    q = FloatQuantizer(bit, True, 'per_head', head_num=4, use_qtorch=True)
    y_o, s_o = fo.fake_quant_dynamic(w, bit, 'per_head', head_num=4)
    _same(q.fake_quant_weight_dynamic(w.cuda()), y_o, f'per_head {bit} fake quant')
    _, s, _, _, _ = q.get_tensor_qparams(w.cuda())
    assert s.shape == (4, 1)
    _same(s, s_o, f'per_head {bit} scales')


@pytest.mark.parametrize('bit', ['e4m3', 'e5m2'])
@pytest.mark.parametrize('dtype', DTYPES)
def test_nan_poisons_its_group(dtype, bit):
    """torch's amax propagates NaN (quant.py:137-140, 550-551): a group holding a NaN gets a NaN
    scale and all-NaN output, the other groups are untouched.  Dynamic per-group and per-block."""
    from llmc_b200.quant_float import FloatQuantizer
    w = _randw((16, 256), dtype, seed=8)
    w[5, 70] = float('nan')
    q = FloatQuantizer(bit, True, 'per_group', group_size=64, use_qtorch=True)
    y = q.fake_quant_weight_dynamic(w.cuda())
    y_o, _ = fo.fake_quant_dynamic(w, bit, 'per_group', 64)
    _same(y, y_o, f'{dtype} {bit} per_group')
    assert bool(y[5, 64:128].isnan().all()) and not bool(y[5, :64].isnan().any())
    _, s, _, _, _ = q.get_tensor_qparams(w.cuda())
    assert bool(s.reshape(16, 4)[5, 1].isnan()) and int(s.isnan().sum()) == 1

    qb = FloatQuantizer(bit, True, 'per_block', block_size=64, use_qtorch=True)
    yb = qb.fake_quant_weight_dynamic(w.cuda())
    _same(yb, fo.block_fake_quant(w, bit, 64)[0], f'{dtype} {bit} per_block')
    assert bool(yb[:16, 64:128].isnan().all()) and not bool(yb[:, :64].isnan().any())
