"""CPU: the premises of the exact AWQ / range-observer oracles (oracle/awq_range_oracle.py) that
tests/test_gpu_awq_range_paths.py relies on, checked on the generated inputs themselves, and the
oracles pinned to the plain restatements they replace: oracle/awq_oracle.auto_clip_layer for the
clip search, oracle/quant_oracle.mse_range for the mse search and torch.histc for the counts."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import awq_oracle as ao
from oracle import awq_range_oracle as ar
from oracle import quant_oracle as qo

DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def test_round_f32_is_one_rounding():
    assert ar.round_f32(Fraction(1, 3)) == np.float32(1 / 3)
    assert ar.round_f32(Fraction(2 ** 24 + 1)) == np.float32(2 ** 24)       # halfway: to even
    assert ar.round_f32(Fraction(2 ** 24 + 3)) == np.float32(2 ** 24 + 4)
    assert ar.round_f32(Fraction(-5, 7)) == np.float32(-5 / 7)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('T', [1, 63, 64, 65, 1000, 16448])
def test_absmean_sums_are_exact(dtype, T):
    x = ar.absmean_input(T, 16, dtype, seed=T)
    exp = ar.absmean_expected(x)                     # asserts the exact-range premise
    S = x.double().abs().sum(0)
    for splits in (1, 3, 64):                        # any split order gives the same fp32 sum
        parts = [x[i::splits].float().abs().sum(0) for i in range(splits)]
        tot = torch.zeros(16)
        for p in parts:
            tot += p
        assert torch.equal(tot.double(), S)
    assert torch.equal(exp, ((S.float() / np.float32(T)).to(dtype)))


def test_absmean_plan_reaches_its_paths():
    assert ar.absmean_plan(63, 8)['splits'] == 1
    assert ar.absmean_plan(64, 8)['splits'] == 1
    assert ar.absmean_plan(16384 + 64, 8)['first'] == 256
    assert ar.absmean_plan(129, 8)['splits'] == 2 and ar.absmean_plan(129, 8)['rows_per_split'] == 65
    p = ar.absmean_plan(4096, 64, workspace_floats=64 * 5)
    assert p['halved'] and p['splits'] == 4
    p = ar.absmean_plan(1000, 8)                     # 15 splits of 67 rows cover 1000 rows
    assert p['first'] == 15 and p['rows_per_split'] == 67 and p['splits'] == 15
    p = ar.absmean_plan(4000, 8)                     # 62 splits of 65 rows: 4000 needs only 62
    assert p['first'] == 62 and p['splits'] == 62
    p = ar.absmean_plan(16447, 8)                    # 256 splits of 65 rows: 254 suffice
    assert p['recount'] and p['splits'] == 254
    assert ar.absmean_plan(10, 2056)['grid_x'] == 2 and ar.absmean_plan(10, 2048)['grid_x'] == 1


def test_div_expected_special_values():
    x = torch.tensor([[0.0, 1.0, float('inf'), -3.0, 6e-8, 60000.0, 1.0, -0.0]])
    s = torch.tensor([0.0, 0.0, float('inf'), 2.0, 4.0, 1e-3, 3.0, 5.0])
    e = ar.div_expected(x, s)
    assert torch.isnan(e[0, 0]) and torch.isnan(e[0, 2])
    assert e[0, 1] == float('inf') and e[0, 3] == -1.5
    assert e[0, 6] == np.float32(1.0) / np.float32(3.0)
    torch.testing.assert_close(ar.div_expected(x.half(), s.half()),
                               (x.half().float() / s.half().float()).half(), rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize('n', [1, 7, 8, 9, 2047, 2048 * 3 + 5, 1024 * 256 * 8 + 8 * 37 + 3])
def test_mse_partials_are_exact(n):
    for dt in DTYPES:
        a, b, S = ar.mse_pair(n, dt, seed=n)
        assert ar.mse_premises(a, b) == S
    plan = ar.mse_plan(n)
    assert plan['only_tail'] == (n < 8)
    assert plan['grid_stride'] == (n >= 1024 * 256 * 8 + 8)


def test_mse_double_rounding_pair_separates_the_two_formulas():
    a, b, S, n = ar.mse_double_rounding_pair()
    assert ar.mse_premises(a, b) == S and a.numel() == n
    one = ar.mse_expected(S, n)
    assert one == np.float32(S / n)                  # 53 >= 2 * 24 + 2: rounding via fp64 is exact
    assert np.float32(S * (1.0 / n)) != one          # the old kernel's t * (1 / n)
    assert ar.mse_plan(n)['blocks'] > 1


CLIP_CASES = [  # R, ng, group, ns, bit, sym, clip_sym
    (64, 2, 128, 300, 4, True, True), (64, 4, 64, 600, 4, False, False),
    (7, 2, 32, 33, 3, False, True), (1, 1, 8, 1, 8, True, False),
    (9, 2, 128, 257, 2, False, False), (64, 3, 36, 600, 4, True, False),
    (200, 1, 96, 31, 4, False, True),
]


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('R,ng,group,ns,bit,sym,clip_sym', CLIP_CASES)
def test_clip_reference_is_the_plain_oracle(dtype, R, ng, group, ns, bit, sym, clip_sym):
    """The restatement on slot tokens (which also asserts that every product and k-sum is exact)
    equals auto_clip_layer on all ns tokens, ragged R included."""
    w, x, slots = ar.clip_inputs(R, ng, group, ns, dtype, seed=R + ng + group)
    assert all(len(t) <= 2 for t in slots)
    nz = (x.reshape(ns, ng, group) != 0).any(-1)
    for grp in range(ng):
        assert set(nz[:, grp].nonzero().flatten().tolist()) <= set(slots[grp])
    err, maxs, mins, om, on = ar.clip_reference(w, x, slots, bit, sym, group, clip_sym)
    bm, bn, ties, _ = ar.clip_select(err, maxs, mins, om, on, ns)
    rm, rn = ao.auto_clip_layer(w, x, bit, sym, 'per_group', group, clip_sym=clip_sym,
                                n_sample_token=ns)
    assert torch.equal(bm, rm.squeeze(-1)) and torch.equal(bn, rn.squeeze(-1))
    if R * ng >= 64:
        assert ties > 0                              # the earliest of tied levels must win


def test_clip_inputs_cover_one_signed_groups_and_chunk_edges():
    w, x, slots = ar.clip_inputs(64, 32, 128, 1023, torch.bfloat16, seed=5)
    wg = w.reshape(64, 32, 128)
    assert bool((wg >= 0).all(-1).any()) and bool((wg <= 0).all(-1).any())
    toks = {t for s in slots for t in s}
    assert {0, 255, 256, 1022} & toks and any(t >= 512 for t in toks)
    assert ar.clip_plan(4096, 1, 1023)['chunks'] == 4


def test_histc_expected_is_torch_histc():
    for dt in DTYPES:
        for bins, lw in ((1, 0), (2048, 3), (8192, 1)):
            x = ar.histc_input(5000, -2.0, lw, bins, dt, seed=bins,
                               extras=(-3.0, 2.0 ** lw, float('nan'), float('inf'), -float('inf')))
            lo, hi = -2.0, -2.0 + 2.0 ** lw
            exp, counts = ar.histc_expected(x, bins, lo, hi)
            ref = torch.histc(x.float()[torch.isfinite(x.float())], bins, min=lo, max=hi)
            assert torch.equal(exp, ref), (dt, bins)
            assert counts[-1] >= 1                               # v == hi lands in the last bin
    x = torch.full((5,), 0.5)
    assert torch.equal(ar.histc_expected(x, 2048, 0.5, 0.5)[0], torch.histc(x, 2048, min=0.5, max=0.5))


@pytest.mark.parametrize('sym,bit', [(True, 4), (False, 3), (False, 8), (True, 2)])
def test_mse_range_replay_is_the_plain_oracle(sym, bit):
    """On decided rows the certified replay picks the reference restatement's range."""
    g = torch.Generator().manual_seed(bit)
    t = torch.randn(64, 128, generator=g)
    mn, mx, dec = ar.mse_range_certified(t, bit, sym, 80, 100)
    rmn, rmx = qo.mse_range(t, bit, sym)
    assert float(dec.float().mean()) > 0.5
    assert torch.equal(mn[dec], rmn[dec]) and torch.equal(mx[dec], rmx[dec])
    c = ar.constructed_mse_rows(16, 128)
    mn, mx, dec = ar.mse_range_certified(c, bit, sym, 80, 100)
    assert bool(dec.all())
    rmn, rmx = qo.mse_range(c, bit, sym)
    assert torch.equal(mn, rmn) and torch.equal(mx, rmx)


def test_mse_range_refuses_unrounded_zero_points():
    from llmc_b200.quant import IntegerQuantizer
    q = IntegerQuantizer(4, False, 'per_group', group_size=128, calib_algo='mse', round_zp=False)
    with pytest.raises(NotImplementedError, match='round_zp'):
        q.get_mse_range(torch.zeros(4, 128))


def test_auto_clip_refuses_wide_groups_before_the_block_loop():
    from llmc_b200.awq import AutoClipper
    from llmc_b200.quant import IntegerQuantizer
    for kw in ({'granularity': 'per_group', 'group_size': 256}, {'granularity': 'per_channel'}):
        q = IntegerQuantizer(4, True, **kw)
        with pytest.raises(NotImplementedError, match='wider than 128'):
            AutoClipper(True, q, None, 'v1', True, False, None)


def test_histc_refuses_more_elements_than_its_counts_hold():
    """llmc_histc counts in 32-bit integers: n >= 2^32 is refused before any CUDA call."""
    import ctypes
    from llmc_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(256)
    assert lib.llmc_histc(p, 1 << 32, 0, 2048, 0.0, 1.0, p, None) == -1
    assert b'32-bit' in lib.llmc_b200_last_error()
