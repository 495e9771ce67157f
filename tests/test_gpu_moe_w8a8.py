"""GPU: Mixtral sparse-MoE layers with W8A8 experts (exported VllmRealQuantLinear int8 / e4m3 linears) on
the grouped W8A8 GEMMs (`llmc_moe_gemm_w8a8_swiglu`, `llmc_moe_gemm_w8a8_down`, csrc/gemm_8bit.cu).

1. The C entry points bit for bit against an exact oracle at every segment, tile and shape edge, in
   the style of test_gpu_moe_paths.py: hand-made int32 segment offsets and host pointer arrays,
   outputs with guard rows of SENTINEL.  The oracle is w8a8_oracle's exact sum and epilogue per
   segment (fp8: operands whose 128-deep partial sums are exact, fp8_exact_operands), then
   F.silu(rT(G)) * rT(U) on the GPU for gate/up and rT(rT(S) * w) for down.  Every argument error is
   returned without a launch.
2. MixtralSparseMoe with W8A8 experts gives the bits of the per-expert loop (expert_loop), with no
   host sync after the first call; experts the grouped form cannot run take the loop.
3. End to end: the Mixtral FP8 static recipe and the shipped vLLM W8A8 / FP8 recipes export models
   whose perplexity is the same with the grouped path and with the loop."""
import copy
import ctypes
import json
import os
import zlib

import pytest
import torch
import yaml

from llmc_b200 import module_utils, synth
from llmc_b200._lib import CONSTANTS, MOE_MAX_EXPERTS, call, dtype_enum, load, stream_ptr
from llmc_b200.module_utils import VllmRealQuantLinear, W8A8Operands, moe_forward
from llmc_b200.synth import MixtralSparseMoe
from test_gpu_gemm_paths import _cdiv, _gen, l2_group_width
from test_gpu_moe_paths import (BM, DTYPES, NUM_SMS, _check_guarded, _guarded, _ptrs, _routed_ref, _swiglu_ref,
                                moe_tiles, offsets_of, route_weights)
from w8a8_oracle import E4M3, epilogue, exact_sum, fp8_exact_operands

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_K_INT8 = ((1 << 17) - 1) // 16 * 16


# ---- the launch plan, restated (moe_w8a8 in gemm_8bit.cu) -----------------------------------------
def w8a8_plan(kernel, rows, E, N, K):
    """(n_tiles, gn, units) of one grouped W8A8 launch: gate/up tiles are 64 act columns (64 rows of
    w1 and of w3), down tiles 128 output columns; gn from one n-tile's 128 x K weight bytes."""
    n_tiles = N // 64 if kernel == 'swiglu' else _cdiv(N, 128)
    return n_tiles, l2_group_width(128 * K, n_tiles), (_cdiv(rows, BM) + E) * n_tiles


def w8a8_cases(sizes, hidden, inter):
    """The cases both launches over segments `sizes` reach; also checks that every tile of every
    expert comes exactly once within the launched units."""
    offsets = offsets_of(sizes)
    rows, E = offsets[-1], len(sizes)
    cases = {'E1'} if E == 1 else ({'E8'} if E == 8 else set())
    if sizes[0] == 0:
        cases.add('empty-first')
    if sizes[-1] == 0:
        cases.add('empty-last')
    if any(s == 0 for s in sizes[1:-1]):
        cases.add('empty-middle')
    cases |= {f'seg{s}' for s in sizes if s in (1, 127, 128, 129)}
    if rows % BM:
        cases.add('rows%128')
    if hidden % 128 or inter % 128:
        cases.add('k-tail')
    if inter % 128:
        cases.add('inter%128')
    if hidden % 128:
        cases.add('partial-n')
    for kernel, N, K in (('swiglu', inter, hidden), ('down', hidden, inter)):
        n_tiles, gn, units = w8a8_plan(kernel, rows, E, N, K)
        tiles = moe_tiles(offsets, n_tiles, gn)
        assert len(tiles) <= units
        for e in range(E):
            assert sorted(t[1:3] for t in tiles if t[0] == e) == \
                [(m, n) for m in range(_cdiv(sizes[e], BM)) for n in range(n_tiles)]
        if len(tiles) > NUM_SMS:
            cases.add('persistent')
        if any(row0 + BM > row_end and row_end < rows for _, _, _, row0, row_end in tiles):
            cases.add('straddle')
    return cases


PATHS = [
    # name, segment sizes, hidden, inter, cases
    ('e1-one-row', [1], 64, 64, {'E1', 'seg1', 'rows%128', 'k-tail', 'inter%128', 'partial-n'}),
    ('e4-empty-first', [0, 127, 129, 3], 272, 192,
     {'empty-first', 'seg127', 'seg129', 'rows%128', 'k-tail', 'inter%128', 'partial-n', 'straddle'}),
    ('e8-empty-middle-last', [5, 1, 0, 127, 128, 129, 300, 0], 528, 1024,
     {'E8', 'empty-middle', 'empty-last', 'seg1', 'seg127', 'seg128', 'seg129', 'rows%128', 'k-tail',
      'partial-n', 'persistent', 'straddle'}),
    ('e8-empty-first', [0, 64, 65, 1, 200, 3, 0, 40], 256, 128, {'E8', 'empty-first', 'empty-middle'}),
    ('e2-persistent', [129, 1000], 512, 1088, {'persistent', 'seg129', 'straddle', 'inter%128'}),
]
ALL_CASES = {'E1', 'E8', 'empty-first', 'empty-middle', 'empty-last', 'seg1', 'seg127', 'seg128', 'seg129',
             'rows%128', 'k-tail', 'inter%128', 'partial-n', 'persistent'}


def test_path_table_reaches_its_cases():
    """No GPU: every entry reaches the cases it names, and the table claims every case."""
    for name, sizes, hidden, inter, want in PATHS:
        got = w8a8_cases(sizes, hidden, inter)
        assert want <= got, (name, want - got)
    assert ALL_CASES <= set().union(*(p[-1] for p in PATHS))


# ---- the C entry points against the oracle --------------------------------------------------------
def _codes(shape, fp8, g):
    """int8: any codes; e4m3: fp8_exact_operands' weights (x comes from _acts)."""
    if fp8:
        return fp8_exact_operands(1, shape[0], shape[1], g)[1].cuda()
    return torch.randint(-128, 128, shape, generator=g).to(torch.int8).cuda()


def _acts(rows, K, fp8, g):
    if fp8:
        return fp8_exact_operands(rows, 1, K, g)[0].cuda()
    return torch.randint(-128, 128, (rows, K), generator=g).to(torch.int8).cuda()


def _scales(n, g, lo=2.0 ** -12, hi=2.0 ** -8):
    return (torch.rand(n, generator=g) * (hi - lo) + lo).float().cuda()


def swiglu_call(xq, sx, fp8, w1, w3, s1, s3, stride, offsets, act, inter, dtype):
    rows, K = xq.shape
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    call('llmc_moe_gemm_w8a8_swiglu', ctypes.c_void_p(xq.data_ptr()), ctypes.c_void_p(sx.data_ptr()), int(fp8),
         _ptrs(w1), _ptrs(w3), _ptrs(s1), _ptrs(s3), stride, ctypes.c_void_p(off.data_ptr()),
         ctypes.c_void_p(act.data_ptr()), rows, inter, K, len(w1), dtype_enum(dtype), stream_ptr())


def down_call(aq, sx, fp8, w2, s2, stride, offsets, w_route, y, N):
    rows, inter = aq.shape
    off = torch.tensor(offsets, dtype=torch.int32, device='cuda')
    call('llmc_moe_gemm_w8a8_down', ctypes.c_void_p(aq.data_ptr()), ctypes.c_void_p(sx.data_ptr()), int(fp8),
         _ptrs(w2), _ptrs(s2), stride, ctypes.c_void_p(off.data_ptr()), ctypes.c_void_p(w_route.data_ptr()),
         ctypes.c_void_p(y.data_ptr()), rows, N, inter, len(w2), dtype_enum(w_route.dtype), stream_ptr())


def check_entry_points(sizes, hidden, inter, fp8, dtype, per_channel, what):
    g = torch.Generator().manual_seed(zlib.crc32(repr((sizes, hidden, inter, fp8, str(dtype), per_channel)).encode()))
    offsets = offsets_of(sizes)
    rows, E = offsets[-1], len(sizes)
    w1 = [_codes((inter, hidden), fp8, g) for _ in range(E)]
    w3 = [_codes((inter, hidden), fp8, g) for _ in range(E)]
    w2 = [_codes((hidden, inter), fp8, g) for _ in range(E)]
    ns = (inter, inter, hidden) if per_channel else (1, 1, 1)
    s1, s3, s2 = ([_scales(n, g) for _ in range(E)] for n in ns)
    xq, aq = _acts(rows, hidden, fp8, g), _acts(rows, inter, fp8, g)
    sx, sa = _scales(rows, g), _scales(rows, g)
    w_route = route_weights(rows, dtype, _gen('w8a8-route', what))
    f32 = torch.float32

    def seg(e):
        return slice(offsets[e], offsets[e + 1])

    # the oracle per segment: the exact sums, the scaling in fp32, then the grouped epilogues
    G = torch.cat([epilogue(exact_sum(xq[seg(e)], w1[e]), sx[seg(e)], s1[e], None, f32) for e in range(E)])
    U = torch.cat([epilogue(exact_sum(xq[seg(e)], w3[e]), sx[seg(e)], s3[e], None, f32) for e in range(E)])
    S = torch.cat([epilogue(exact_sum(aq[seg(e)], w2[e]), sa[seg(e)], s2[e], None, f32) for e in range(E)])
    act_ref = _swiglu_ref(G.cuda(), U.cuda(), dtype)
    y_ref = _routed_ref(S.cuda(), w_route, dtype)
    assert float((G != U).double().mean()) > 0.5, what                  # w1 and w3 tell apart

    stride = int(per_channel)
    act = _guarded(rows, inter, dtype)
    swiglu_call(xq, sx, fp8, w1, w3, s1, s3, stride, offsets, act[:rows], inter, dtype)
    _check_guarded(act, rows, act_ref, what + ' gate/up')
    y = _guarded(rows, hidden, dtype)
    down_call(aq, sa, fp8, w2, s2, stride, offsets, w_route, y[:rows], hidden)
    _check_guarded(y, rows, y_ref, what + ' down')


@gpu
@pytest.mark.parametrize('per_channel', [True, False], ids=['s_w-channel', 's_w-tensor'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('fp8', [False, True], ids=['int8', 'e4m3'])
@pytest.mark.parametrize('name,sizes,hidden,inter,want', PATHS, ids=[p[0] for p in PATHS])
def test_entry_points_path_table(name, sizes, hidden, inter, want, fp8, dtype, per_channel):
    assert want <= w8a8_cases(sizes, hidden, inter)
    check_entry_points(sizes, hidden, inter, fp8, dtype, per_channel, name)


@gpu
def test_argument_errors_launch_nothing():
    """Every refusal returns before any CUDA call; rows == 0 is a no-op."""
    lib = load()
    EALIGN = CONSTANTS['LLMC_EALIGN']
    dt, bf = torch.bfloat16, dtype_enum(torch.bfloat16)
    rows, K, inter, N = 8, 64, 64, 64
    xq = torch.zeros(rows + 16, K, dtype=torch.int8, device='cuda')
    sx = torch.ones(rows, device='cuda')
    w = [torch.zeros(inter, K, dtype=torch.int8, device='cuda') for _ in range(MOE_MAX_EXPERTS + 1)]
    s = [torch.ones(inter, device='cuda') for _ in range(MOE_MAX_EXPERTS + 1)]
    act = _guarded(rows, inter, dt)
    w_route = torch.ones(rows, dtype=dt, device='cuda')
    off = torch.zeros(MOE_MAX_EXPERTS + 2, dtype=torch.int32, device='cuda')
    p = ctypes.c_void_p

    def sw(x=xq.data_ptr(), scale=sx.data_ptr(), fp8=0, w1=None, w3=None, s1=None, s3=None, stride=1,
           offsets=off.data_ptr(), out=act.data_ptr(), n_rows=rows, n_inter=inter, k=K, E=2, dtype=bf):
        return lib.llmc_moe_gemm_w8a8_swiglu(
            p(x), p(scale), fp8, _ptrs(w[:E]) if w1 is None else w1, _ptrs(w[:E]) if w3 is None else w3,
            _ptrs(s[:E]) if s1 is None else s1, _ptrs(s[:E]) if s3 is None else s3, stride, p(offsets), p(out),
            n_rows, n_inter, k, E, dtype, stream_ptr())

    def dn(x=xq.data_ptr(), fp8=0, w2=None, stride=1, route=w_route.data_ptr(), n=N, k=inter, E=2, n_rows=rows):
        return lib.llmc_moe_gemm_w8a8_down(
            p(x), p(sx.data_ptr()), fp8, _ptrs(w[:E]) if w2 is None else w2, _ptrs(s[:E]), stride,
            p(off.data_ptr()), p(route), p(act.data_ptr()), n_rows, n, k, E, bf, stream_ptr())

    def null_at(i, E=2):
        return (ctypes.c_void_p * E)(*[None if j == i else w[j].data_ptr() for j in range(E)])

    torch.cuda.synchronize()
    before = lib.llmc_b200_launch_count()
    refusals = [
        (lambda: sw(E=MOE_MAX_EXPERTS + 1), -1, 'experts outside'),
        (lambda: sw(E=0), -1, 'experts outside'),
        (lambda: sw(k=24), -1, 'multiple of 16'),
        (lambda: sw(n_inter=96), -1, 'multiple of 64'),
        (lambda: dn(n=12), -1, 'multiple of 8'),
        (lambda: sw(k=MAX_K_INT8 + 16), -1, 'overflows the int32 sum'),
        (lambda: dn(k=MAX_K_INT8 + 16), -1, 'overflows the int32 sum'),
        (lambda: sw(stride=2), -1, 's_w_stride'),
        (lambda: sw(dtype=dtype_enum(torch.float32)), -1, 'bf16 or fp16'),
        (lambda: sw(n_rows=-1), -1, 'bad shape'),
        (lambda: sw(x=0), -1, 'null pointer'),
        (lambda: sw(scale=0), -1, 'null pointer'),
        (lambda: sw(offsets=0), -1, 'null pointer'),
        (lambda: sw(w3=null_at(1)), -1, 'null codes or scales of expert 1'),
        (lambda: sw(s1=(ctypes.c_void_p * 2)(s[0].data_ptr(), None)), -1, 'null codes or scales of expert 1'),
        (lambda: dn(route=0), -1, 'null pointer'),
        (lambda: dn(w2=null_at(0)), -1, 'null codes or scales of expert 0'),
        (lambda: sw(x=xq.data_ptr() + 8), EALIGN, '16-byte aligned'),
        (lambda: sw(out=act.data_ptr() + 2), EALIGN, '16-byte aligned'),
        (lambda: sw(w1=(ctypes.c_void_p * 2)(w[0].data_ptr(), w[1].data_ptr() + 8)), EALIGN, 'expert 1 not 16-byte'),
        (lambda: dn(w2=(ctypes.c_void_p * 2)(w[0].data_ptr() + 4, w[1].data_ptr())), EALIGN, 'expert 0 not 16-byte'),
    ]
    for i, (fn, want, msg) in enumerate(refusals):
        rc = fn()                                      # the last error is the latest call's
        assert rc == want, (i, rc, msg, lib.llmc_b200_last_error())
        assert msg in lib.llmc_b200_last_error().decode(), (i, msg, lib.llmc_b200_last_error())
    assert sw(n_rows=0) == 0 and dn(n_rows=0) == 0                    # rows == 0: nothing to do
    assert sw(n_rows=0, x=0, out=0, offsets=0) == 0
    torch.cuda.synchronize()
    assert lib.llmc_b200_launch_count() == before
    assert bool((act.view(torch.int16) == 0x7FA5).all())


# ---- the module against the loop -----------------------------------------------------------------
def _ref_act(rel):
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[rel]['quant']['act']


def _act_cfg(kind, static):
    """The act section of the shipped vLLM W8A8 / FP8 recipes, or its per-tensor static form."""
    act = dict(_ref_act('backend/vllm/rtn_w8a8.yml' if kind == 'int8' else 'backend/vllm/fp8/rtn_fp8.yml'))
    if static:
        act.update(granularity='per_tensor', static=True, calib_algo='static_minmax')
    return act


# kind, static, per-channel weight scales
FORMS = {'int8-dynamic': ('int8', False, True), 'int8-static': ('int8', True, True),
         'e4m3-dynamic': ('e4m3', False, True), 'e4m3-static': ('e4m3', True, False)}


def _w8a8_linear(N, K, kind, static, per_channel, g, input_scale=None):
    if kind == 'int8':
        w = torch.randint(-127, 128, (N, K), generator=g, device='cuda').to(torch.int8)
        s = torch.rand(N if per_channel else 1, 1, generator=g, device='cuda') * 2e-4 + 5e-5
    else:
        w = (torch.randn(N, K, generator=g, device='cuda') * 2).to(E4M3)
        s = torch.rand(N if per_channel else 1, 1, generator=g, device='cuda') * 0.01 + 0.002
    if static and input_scale is None:
        input_scale = torch.rand(1, generator=g, device='cuda') * (0.03 if kind == 'int8' else 0.01) + 1e-3
    m = VllmRealQuantLinear(w, None, s.reshape(-1) if not per_channel else s, input_scale if static else None,
                            False, 'weight_scale')
    m.in_features, m.out_features = K, N
    m.act_cfg = _act_cfg(kind, static)
    return m


def _moe(hidden, inter, E, k, dtype, form, seed=0):
    kind, static, per_channel = FORMS[form]
    g = torch.Generator(device='cuda').manual_seed(seed)
    with torch.device('meta'):
        moe = MixtralSparseMoe(hidden, inter, E, k)
    moe.gate = moe.gate.to_empty(device='cuda').to(dtype)
    moe.gate.weight.data.normal_(0, 0.02, generator=g)
    for ex in moe.experts:
        ex.w1 = _w8a8_linear(inter, hidden, kind, static, per_channel, g)
        # static minmax calibration gives w1 and w3 one input, hence one scale (a copy, not the same tensor)
        ex.w3 = _w8a8_linear(inter, hidden, kind, static, per_channel, g,
                             input_scale=ex.w1.input_scale.clone() if static else None)
        ex.w2 = _w8a8_linear(hidden, inter, kind, static, per_channel, g)
    return moe


def _x(T, hidden, dtype, seed=1):
    return torch.randn(T, hidden, device='cuda', generator=torch.Generator(device='cuda').manual_seed(seed)).to(dtype)


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _check(moe, x):
    sel, w = moe.route(x)
    assert moe.grouped_weights(x) is None and moe.grouped_packed_operands(x) is None
    ops = moe.grouped_w8a8_operands(x)
    assert ops is not None and all(isinstance(o, W8A8Operands) for t in ops for o in t)
    got = moe_forward(x, sel, w, ops)
    assert _same_bits(got, moe.expert_loop(x, sel, w))
    return got


@gpu
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'fp16'])
@pytest.mark.parametrize('form', list(FORMS))
def test_tiny_mixtral_forms(form, dtype):
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype, form)
    T = 300
    x = _x(T, s['hidden'], dtype)
    _check(moe, x)
    sel, w = moe.route(x)
    out = moe(x.view(2, T // 2, -1))                   # the module forward takes the grouped path
    assert _same_bits(out.view(T, -1), moe.expert_loop(x, sel, w))


@gpu
@pytest.mark.parametrize('form', list(FORMS))
def test_mixtral_8x7b_layer(form):
    s = synth.SHAPES['mixtral-8x7b']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16, form)
    _check(moe, _x(1024, s['hidden'], torch.bfloat16))
    del moe
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize('form', list(FORMS))
def test_zero_tokens_launch_nothing(form):
    dtype, s = torch.bfloat16, synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], dtype, form)
    x = torch.empty(0, s['hidden'], dtype=dtype, device='cuda')
    ops = moe.grouped_w8a8_operands(x)
    assert ops is not None
    torch.cuda.synchronize()
    before = load().llmc_b200_launch_count()
    out = moe_forward(x, torch.empty(0, 2, dtype=torch.int64, device='cuda'),
                      torch.empty(0, 2, dtype=dtype, device='cuda'), ops)
    torch.cuda.synchronize()
    assert load().llmc_b200_launch_count() == before
    assert out.shape == (0, s['hidden']) and out.dtype == dtype


@gpu
@pytest.mark.parametrize('form', list(FORMS))
def test_no_host_sync_after_the_first_call(form):
    s = synth.SHAPES['tiny-mixtral']
    moe = _moe(s['hidden'], s['inter'], s['experts'], s['top_k'], torch.bfloat16, form)
    hs = _x(256, s['hidden'], torch.bfloat16).view(2, 128, -1)
    ref = moe(hs)                                      # warm-up: library load, kernel attributes, caches
    torch.cuda.synchronize()
    assert not module_utils.TIMER.enabled
    calls = []
    real = synth.moe_forward
    synth.moe_forward = lambda *a: calls.append(isinstance(a[3][0][0], W8A8Operands)) or real(*a)
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = moe(hs)
    finally:
        torch.cuda.set_sync_debug_mode('default')
        synth.moe_forward = real
    assert calls == [True]
    assert torch.equal(out, ref)


@gpu
@pytest.mark.parametrize('case', ['w13-scales-differ', 'bias', 'expert-hook', 'linear-hook', 'mixed-int8-e4m3',
                                  'weight-packed', 'nine-experts'])
def test_fallbacks_take_the_loop(case, monkeypatch):
    s = synth.SHAPES['tiny-mixtral']
    dtype = torch.bfloat16
    form = 'e4m3-static' if case == 'w13-scales-differ' else 'int8-dynamic'
    E = MOE_MAX_EXPERTS + 1 if case == 'nine-experts' else s['experts']
    moe = _moe(s['hidden'], s['inter'], E, s['top_k'], dtype, form)
    g = torch.Generator(device='cuda').manual_seed(9)
    ex = moe.experts[1]
    seen = []
    T = 300
    x = _x(T, s['hidden'], dtype)
    if case == 'w13-scales-differ':
        assert moe.grouped_w8a8_operands(x) is not None          # cached as equal first
        ex.w3.input_scale.mul_(1.5)                              # a new buffer version: read again
    elif case == 'bias':
        ex.w2.bias = torch.randn(s['hidden'], generator=g, device='cuda').to(dtype)
    elif case == 'expert-hook':
        ex.register_forward_hook(lambda m, i, o: seen.append(i[0].clone()))
    elif case == 'linear-hook':
        ex.w1.register_forward_pre_hook(lambda m, i: seen.append(i[0].clone()))
    elif case == 'mixed-int8-e4m3':
        ex.w1, ex.w3, ex.w2 = (_w8a8_linear(n, k, 'e4m3', False, True, g)
                               for n, k in ((s['inter'], s['hidden']), (s['inter'], s['hidden']),
                                            (s['hidden'], s['inter'])))
    elif case == 'weight-packed':
        for name, (n, k) in (('w1', (s['inter'], s['hidden'])), ('w3', (s['inter'], s['hidden'])),
                             ('w2', (s['hidden'], s['inter']))):
            words = torch.randint(-2**31, 2**31 - 1, (n, k // 8), generator=g, device='cuda', dtype=torch.int32)
            sc = (torch.rand(n, k // 128, generator=g, device='cuda') * 0.01 + 1e-3).to(torch.float16)
            m = VllmRealQuantLinear(words, None, sc, None, True, 'weight_scale')
            m.in_features, m.out_features = k, n
            setattr(ex, name, m)
    sel, w = moe.route(x)
    assert moe.grouped_w8a8_operands(x) is None
    calls = []
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(1) or moe_forward(*a))
    out = moe(x.view(1, T, -1)).view(T, -1)
    assert not calls
    assert _same_bits(out, moe.expert_loop(x, sel, w))
    if case == 'expert-hook':
        assert torch.equal(seen[0], x[torch.where(sel == 1)[0]])


# ---- end to end ----------------------------------------------------------------------------------
def _recipe(name):
    if name == 'rtn_fp8_static_mixtral':
        with open(os.path.join(ROOT, 'configs', 'rtn_fp8_static_mixtral.yml')) as fh:
            return yaml.safe_load(fh)
    with open(os.path.join(ROOT, 'tests', 'golden', 'ref_yamls.json')) as fh:
        return json.load(fh)[name]


def _loop_forward(self, hidden_states):
    B, S, H = hidden_states.shape
    x = hidden_states.reshape(-1, H)
    sel, w = self.route(x)
    return self.expert_loop(x, sel, w).reshape(B, S, H)


@gpu
@pytest.mark.parametrize('name', ['rtn_fp8_static_mixtral', 'backend/vllm/rtn_w8a8.yml',
                                  'backend/vllm/fp8/rtn_fp8.yml'])
def test_exported_mixtral_perplexity_grouped_equals_loop(name, monkeypatch):
    from llmc_b200.__main__ import adapt_reference_config, main
    cfg = adapt_reference_config(copy.deepcopy(_recipe(name)), 'tiny-mixtral', n_samples=8, seq_len=128,
                                 eval_seq_len=128)
    cfg['model']['type'] = 'Mixtral'
    cfg['save'].pop('save_path', None)                 # deploy in memory
    cfg['eval']['eval_pos'] = []
    _, model, report = main(cfg, quiet=True)
    assert report['exported'] == 'vllm_quant'
    hidden = model.shape['hidden']
    x = torch.zeros(1, hidden, dtype=model.shape['dtype'], device='cuda')
    for blk in model.get_blocks():
        assert blk.block_sparse_moe.grouped_w8a8_operands(x) is not None
    tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 4), generator=torch.Generator().manual_seed(5))
    calls = []
    real = module_utils.moe_forward
    monkeypatch.setattr(synth, 'moe_forward', lambda *a: calls.append(isinstance(a[3][0][0], W8A8Operands))
                        or real(*a))
    ppl_grouped = synth.perplexity(model, tokens, 128)
    assert calls and all(calls)
    monkeypatch.setattr(MixtralSparseMoe, 'forward', _loop_forward)
    ppl_loop = synth.perplexity(model, tokens, 128)
    assert ppl_grouped == ppl_loop and ppl_grouped == ppl_grouped
