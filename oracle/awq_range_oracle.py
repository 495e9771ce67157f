"""Exact oracles for AWQ's tensor-level kernels (csrc/awq.cu, DESIGN.md §K8/K9) and the range
observers (csrc/range.cu, Q2-mse / Q7-hist): input generators whose arithmetic is exact in any
summation order, the expected outputs, and checks of those premises on the inputs themselves.

* absmean_cols: x = small integers * 2^-3, so every partial column sum is an exact fp32 value and
  the output is (S / fp32(T)) rounded once to fp32 and then to the dtype, for any split of the rows.
* div_cols: elementwise; the expected value is one IEEE fp32 division rounded to the dtype.
* mse: a - b are integers whose squares and every partial sum of a block stay below 2^24, so the
  device sum is exactly S = sum (a - b)^2 and the result must be S / n rounded once to fp32.
* awq_clip: weights are integers * 2^-6 (|k| <= 63), sampled tokens are sparse with +-2^j entries (j >= 0)
  and at most two tokens carry input in any one group.  Every rT(x * w), rT(x * q_w) and inner
  k-sum is then exact in fp32 and the per-(row, group, level) error sum has at most two nonzero
  terms, so the result does not depend on lanes, chunks or the order of any sum.
  `clip_reference` restates auto_clip.py:83-191 on the active tokens only; the CPU suite pins it
  to oracle/awq_oracle.auto_clip_layer, itself pinned to the reference's goldens.
* histc: lo, hi and the values are dyadic and hi - lo is a power of two, so the bin formula
  (v - lo) * bins / (hi - lo) is exact; counts come from integer binning.
* mse_range: the per-level error is an fp32 tree sum of powf(d, 2.4), which cannot be made order
  free.  `mse_range_certified` restates the elementwise arithmetic exactly in fp32, sums in fp64
  with a rigorous bound of the device's error, replays the aliased running range and reports a
  row as decided only if every comparison's margin exceeds the bound.
"""
import math
from fractions import Fraction

import numpy as np
import torch

from . import quant_oracle as qo

LEVELS = 10                      # int(max_shrink 0.5 * n_grid 20), auto_clip.py:127
CLIP_TOK = 256                   # tokens per llmc_awq_clip pass (kClipMaxTok)
NUM_SMS = 132

# powf's maximum error in ulp, CUDA C++ Programming Guide, "Mathematical Functions" appendix,
# single-precision table (powf(x, y): 4 ulp, full range)
POWF_ULP = 4
U32 = 2.0 ** -24                 # unit roundoff of fp32


def f32(x):
    return np.float32(x)


def round_f32(q):
    """A rational (Fraction) rounded once to fp32, nearest-even (normal range)."""
    q = Fraction(q)
    if q == 0:
        return np.float32(0.0)
    sign = -1 if q < 0 else 1
    a = abs(q)
    e = math.floor(math.log2(a.numerator) - math.log2(a.denominator))
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (e - 23)
    m = a / ulp
    n = math.floor(m)
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return np.float32(sign * float(n * ulp))


# ---- absmean_cols -------------------------------------------------------------------------------
def absmean_plan(T, C, workspace_floats=None):
    """llmc_absmean_cols's host plan (awq.cu:275-280): splits, rows per split, the grid."""
    if workspace_floats is None:
        workspace_floats = 256 * C
    splits = 1 if T < 64 else min(T // 64, 256)
    first = splits
    while splits * C > workspace_floats and splits > 1:
        splits //= 2
    halved = splits != first
    rows = -(-T // splits)
    final = -(-T // rows)
    return dict(splits=final, first=first, halved=halved, recount=final != splits,
                rows_per_split=rows, grid_x=-(-(C // 8) // 256))


def absmean_input(T, C, dtype, seed=0, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    k = torch.randint(-7, 8, (T, C), generator=g)
    return (k.double() / 8).to(dtype).to(device)


def absmean_expected(x):
    """(S_fp32 / fp32(T)).to(T) with S the exact column sum of |x|."""
    T = x.shape[0]
    S = (x.double().abs() * 8).sum(0).cpu().numpy()           # integers
    assert float(np.abs(S).max()) < 2 ** 24, 'absmean premise: a column sum leaves the exact range'
    S32 = (S / 8).astype(np.float32)
    assert np.array_equal(S32.astype(np.float64), S / 8)
    out = S32 / np.float32(T)
    return torch.from_numpy(out).to(x.dtype)


# ---- div_cols -----------------------------------------------------------------------------------
def div_expected(x, s):
    """One IEEE fp32 division per element, rounded to x's dtype."""
    xn = x.float().cpu().numpy()
    sn = s.float().cpu().numpy().reshape(1, -1)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        q = (xn / sn).astype(np.float32)
    return torch.from_numpy(q).to(x.dtype)


# ---- mse ----------------------------------------------------------------------------------------
def mse_plan(n):
    """llmc_mse's host plan (awq.cu:311-313)."""
    blocks = max(1, min(1024, ((n >> 3) + 255) // 256))
    n8 = n >> 3
    return dict(blocks=blocks, tail=n - 8 * n8, only_tail=n8 == 0,
                grid_stride=n8 > blocks * 256, per_block=-(-n8 // blocks) * 8)


def mse_pair(n, dtype, seed=0, dmax=16, device='cpu'):
    """(a, b, S): a - b integers in [-dmax, dmax], |a|, |b| <= 64, exact in every dtype."""
    g = torch.Generator().manual_seed(seed)
    b = torch.randint(-48, 49, (n,), generator=g)
    d = torch.randint(-dmax, dmax + 1, (n,), generator=g)
    a = b + d
    S = int((d * d).sum())
    return a.to(dtype).to(device), b.to(dtype).to(device), S


def mse_premises(a, b):
    """a - b are integers of magnitude <= 2^11 and each block's share of sum (a - b)^2 (octet o
    goes to block (o mod 256 * blocks) / 256, the tail to block 0) stays below 2^24, so every
    fp32 partial the kernel forms is exact."""
    n = a.numel()
    d = (a.double() - b.double()).cpu().reshape(-1)
    assert torch.equal(d, d.round()) and float(d.abs().max()) <= 2 ** 11
    plan = mse_plan(n)
    sq = (d * d).numpy()
    n8 = n >> 3
    blk = np.zeros(n, dtype=np.int64)
    blk[:8 * n8] = (np.arange(8 * n8) // 8 % (256 * plan['blocks'])) // 256
    per_block = np.bincount(blk, weights=sq, minlength=plan['blocks'])
    assert float(per_block.max()) < 2 ** 24, 'mse premise: a block partial leaves the exact range'
    return int(sq.sum())


def mse_expected(S, n):
    return round_f32(Fraction(S, n))


def mse_double_rounding_pair(device='cpu'):
    """fp32 (a, b) with n = 49 * 2^14 and S / n exactly halfway between two fp32 values, where
    fl32(S * fl64(1 / n)) != fl32(S / n): tells `t * (1 / n)` from `t / n` apart.  The squares
    are (41 + small)^2, spread so that every block's partial stays far below 2^24."""
    n = 49 * 2 ** 14
    K = 27982867                      # odd, in (2^24, 2^25): S / n = K * 2^-14 is a midpoint
    S = 49 * K
    d = np.full(n, 41, dtype=np.int64)
    rem = S - n * 41 * 41
    big = rem // (100 * 100 - 41 * 41)
    rem -= big * (100 * 100 - 41 * 41)
    # the remainder as four squares replacing four 41s
    target = rem + 4 * 41 * 41
    four = None
    r0 = int(math.isqrt(target))
    for x in range(r0, -1, -1):
        t1 = target - x * x
        for y in range(min(x, int(math.isqrt(t1))), -1, -1):
            t2 = t1 - y * y
            for z in range(min(y, int(math.isqrt(t2))), -1, -1):
                t3 = t2 - z * z
                w = int(math.isqrt(t3))
                if w * w == t3 and w <= z:
                    four = (x, y, z, w)
                    break
            if four:
                break
        if four:
            break
    idx = np.linspace(0, n - 1, big + 4).astype(np.int64)
    d[idx[:big]] = 100
    d[idx[big:]] = four
    assert int((d * d).sum()) == S
    g = np.random.default_rng(7)
    sign = g.choice(np.array([-1, 1]), n)
    b = g.integers(-1000, 1000, n)
    a = b + sign * d
    to = lambda v: torch.from_numpy(v.astype(np.float32)).to(device)
    return to(a), to(b), S, n


# ---- auto-clip ----------------------------------------------------------------------------------
def clip_plan(R, ng, ns):
    """llmc_awq_clip's host plan (awq.cu:347-357): row slices, rows per CTA, token chunks."""
    slices = -(-(4 * NUM_SMS) // ng)
    slices = max(1, min(slices, -(-R // 8)))
    rows_per_cta = -(-R // slices)
    chunks = -(-ns // CLIP_TOK)
    return dict(slices=slices, rows_per_cta=rows_per_cta, chunks=chunks,
                ragged_slice=R % rows_per_cta != 0, last_chunk=ns - (chunks - 1) * CLIP_TOK)


def clip_token_slots(ns, ng, seed):
    """For each group, the (at most two) tokens that carry input there: chunk edges, lane edges
    and random tokens."""
    g = np.random.default_rng(seed)
    special = sorted({t for t in (0, 1, 31, 32, 33, 63, 255, 256, 257, 511, 512, 513, 767, 768,
                                  ns - 2, ns - 1) if 0 <= t < ns})
    slots = []
    for grp in range(ng):
        k = 1 + (grp % 2) if ns > 1 else 1
        if grp % 3 == 0:
            toks = g.choice(special, size=min(k, len(special)), replace=False)
        else:
            toks = g.choice(ns, size=k, replace=False)
        slots.append(sorted(int(t) for t in toks))
    return slots


def clip_inputs(R, ng, group, ns, dtype, seed=0, device='cpu'):
    """(w [R, C], x [ns, C], slots): w = k * 2^-6 with |k| <= 63 and one-signed groups mixed in;
    x nonzero only on each group's slot tokens, with 1..3 entries of +-2^j (j in 0..2, so no product underflows); one for
    fp32, whose 24-bit q_w of different exponents need not sum exactly."""
    g = np.random.default_rng(seed)
    C = ng * group
    k = g.integers(-63, 64, (R, ng, group))
    sign_mode = g.integers(0, 6, (R, ng))            # 0: all >= 0, 1: all <= 0, else mixed
    k = np.where(sign_mode[..., None] == 0, np.abs(k), k)
    k = np.where(sign_mode[..., None] == 1, -np.abs(k), k)
    # rows of small dynamic range make coarse levels tie
    small = g.random((R, ng)) < 0.2
    k = np.where(small[..., None], np.clip(k, -3, 3), k)
    w = torch.from_numpy(k.reshape(R, C).astype(np.float64) / 64).to(dtype)
    slots = clip_token_slots(ns, ng, seed + 1)
    x = np.zeros((ns, C))
    for grp, toks in enumerate(slots):
        for t in toks:
            nnz = 1 if dtype == torch.float32 else g.integers(1, 4)
            ks = g.choice(group, size=nnz, replace=False)
            x[t, grp * group + ks] = g.choice([-1, 1], nnz) * 2.0 ** g.integers(0, 3, nnz)
    x = torch.from_numpy(x).to(dtype)
    return w.to(device), x.to(device), slots


def _exact_fp32_sum(terms, axis):
    """True where every partial sum of `terms` (fp64 values that are multiples of 2^-60) along
    `axis` is exact in fp32 in any order: sum |t| < 2^24 * the largest power of two dividing every
    term."""
    n = (terms.abs() * 2.0 ** 60).to(torch.int64)
    assert torch.equal(n.double() * 2.0 ** -60, terms.abs()), 'terms are not multiples of 2^-60'
    low = torch.where(n > 0, n & -n, torch.full_like(n, 1 << 62))
    q = low.amin(axis).double() * 2.0 ** -60
    return terms.abs().sum(axis) < q * 2.0 ** 24


def clip_reference(w, x, slots, bit, sym, group, clip_sym, check=True):
    """auto_clip.py:83-191 (v1, w_only) restated on each group's slot tokens, in the dtype of w.
    Returns (best_max [R, ng], best_min [R, ng], err [R, ng, 10] fp32 sums over tokens as the
    kernel accumulates them, ties: number of (row, group) where a later level ties the best)."""
    R, C = w.shape
    ng = C // group
    dt = w.dtype
    dev = w.device
    wg = w.reshape(R, ng, group)
    xa = torch.zeros(ng, 2, group, dtype=dt, device=dev)       # slot tokens of each group
    for grp, toks in enumerate(slots):
        for j, t in enumerate(toks):
            xa[grp, j] = x[t, grp * group:(grp + 1) * group]
    org_max = wg.abs().amax(-1) if clip_sym else wg.amax(-1)
    org_min = wg.amin(-1)

    def out(q):                      # (x * q).sum(-1) in T: [R, ng, 2]
        prod = xa.unsqueeze(0) * q.unsqueeze(2)
        if check:
            assert torch.equal(prod.double(), xa.double().unsqueeze(0) * q.double().unsqueeze(2)), \
                'clip premise: a product rT(x * w) is inexact'
            assert bool(_exact_fp32_sum(prod.double(), -1).all()), 'clip premise: inexact k-sum'
        return prod.sum(-1)
    org = out(wg)
    errs, maxs, mins = [], [], []
    for lvl in range(LEVELS):
        max_val = org_max * (1 - lvl / 20)
        min_val = -max_val if clip_sym else org_min * (1 - lvl / 20)
        cur = torch.clamp(wg, min_val.unsqueeze(-1), max_val.unsqueeze(-1))
        qw = qo.fake_quant_dynamic(cur.reshape(R, C), bit, sym, 'per_group', group).reshape(R, ng, group)
        d = out(qw) - org
        sq = (d * d).float()                                     # rT(d * d), then fp32
        if check:
            assert torch.equal((d.double() * d.double()).to(dt).double(), sq.double())
        errs.append(sq[..., 0] + sq[..., 1])                     # two terms: one rounding
        maxs.append(max_val)
        mins.append(min_val)
    err = torch.stack(errs, -1)
    return err, torch.stack(maxs, -1), torch.stack(mins, -1), org_max, org_min


def clip_select(err, maxs, mins, org_max, org_min, ns):
    """awq_clip_select_kernel / the reference's running argmin: e = rT(err / ns) in T, strict <,
    best starts at rT(1e9).  Returns (best_max, best_min, ties)."""
    dt = maxs.dtype
    e = (err / float(ns)).to(dt)             # fp32 division (err is fp32), then rounded to T
    best_e = torch.full(err.shape[:2], 1e9, device=err.device).to(dt)   # inf in fp16
    bmax, bmin = org_max.clone(), org_min.clone()
    for lvl in range(LEVELS):
        better = e[..., lvl] < best_e
        best_e = torch.where(better, e[..., lvl], best_e)
        bmax = torch.where(better, maxs[..., lvl], bmax)
        bmin = torch.where(better, mins[..., lvl], bmin)
    best_lvl = (e == best_e.unsqueeze(-1)).int().argmax(-1)
    ties = int(((e == best_e.unsqueeze(-1)).sum(-1) > 1).sum())
    return bmax, bmin, ties, best_lvl


# ---- histc --------------------------------------------------------------------------------------
def histc_plan(n):
    blocks = min(NUM_SMS * 8, max(1, -(-n // 256)))
    return dict(blocks=blocks, grid_stride=n > blocks * 256)


def histc_input(n, lo, width_log2, bins, dtype, seed=0, extras=(), device='cpu'):
    """Dyadic values on [lo, lo + 2^width_log2] (multiples of the bin width / 4 before rounding to
    the dtype), with hi itself, plus `extras` (out-of-range values, NaN, inf) mixed in."""
    g = np.random.default_rng(seed)
    width = 2.0 ** width_log2
    q = width / bins / 4
    k = g.integers(0, 4 * bins + 1, n)
    v = lo + k * q
    if n:
        v[g.integers(0, n)] = lo + width
    v = np.concatenate([v, np.array(extras, dtype=np.float64)]) if len(extras) else v
    g.shuffle(v)
    return torch.from_numpy(v).to(dtype).to(device)


def histc_expected(x, bins, lo, hi):
    """torch.histc counts by integer binning.  Premises: hi - lo and bins are powers of two and
    every v - lo is exact in fp32, so (v - lo) * bins / (hi - lo) is exact in fp32."""
    if hi == lo:
        lo, hi = lo - 1.0, hi + 1.0
    v = x.double().cpu().numpy()
    v = v[np.isfinite(v) & (v >= lo) & (v <= hi)]
    width = hi - lo
    assert math.frexp(width)[0] == 0.5 and math.frexp(bins)[0] == 0.5, \
        'histc premise: hi - lo or bins is not a power of two'
    assert np.array_equal((v - lo).astype(np.float32).astype(np.float64), v - lo), \
        'histc premise: some v - lo is inexact in fp32'
    pos = (v - lo) * bins / width
    b = np.minimum(np.floor(pos).astype(np.int64), bins - 1)
    counts = np.bincount(b, minlength=bins)
    return torch.from_numpy(counts.astype(np.float32)), counts


# ---- mse range ----------------------------------------------------------------------------------
def mse_range_plan(rows, cols):
    """llmc_mse_range's host plan (range.cu:143-147)."""
    grid = min(rows, NUM_SMS * 16)
    return dict(cached=cols <= 24 * 1024, grid_stride=rows > grid, grid=grid)


def mse_range_certified(t, bit, sym, steps, mse_grid, norm=2.4):
    """t [rows, cols] fp32 (any device).  The reference's search (quant.py:145-203) with every
    elementwise step in fp32 exactly as the kernel and the reference compute it, the per-level
    error E_i = sum |d|^norm in fp64, and a bound B_i on the device's fp32 value of it:

        |tot_i - E_i| <= (POWF_ULP * 2^-23 + gamma_(cols-1) * (1 + POWF_ULP * 2^-23)) * E_i
                         + cols * POWF_ULP * 2^-149         (subnormal terms, absolute)

    with gamma_k = k u / (1 - k u): powf within POWF_ULP ulp of d^norm, then any fp32 summation
    order of cols terms.  The aliased running range is replayed; a comparison `tot_i < best` is
    decided when |E_i - E_best| > B_i + B_best, or when level i's |d| equal the best level's in
    every column (then the device adds the same terms in the same order: a tie, kept by `<`).  Returns (min, max, decided [rows])."""
    t = t.float()
    rows, cols = t.shape
    mn = t.amin(-1, keepdim=True).clone()
    mx = t.amax(-1, keepdim=True).clone()
    best_e = torch.full((rows,), math.inf, dtype=torch.float64, device=t.device)
    best_b = torch.zeros(rows, dtype=torch.float64, device=t.device)
    decided = torch.ones(rows, dtype=torch.bool, device=t.device)
    rel = POWF_ULP * 2.0 ** -23
    gam = (cols - 1) * U32 / (1 - (cols - 1) * U32)
    for i in range(steps):
        p = 1 - i / mse_grid
        xmin, xmax = mn * float(f32(p)), mx * float(f32(p))   # fp32 multiply by fl32(p)
        s, z, qmx, qmn = qo.qparams(xmin, xmax, bit, sym)
        q = qo.dequant(qo.quant(t, s, z, qmx, qmn), s, z)  # two roundings: (q - z) * s
        d = (q - t).abs().double()
        E = d.pow(norm).sum(1)
        B = (rel + gam * (1 + rel) + 1e-12) * E + cols * POWF_ULP * 2.0 ** -149
        if i == 0:
            better = torch.ones(rows, dtype=torch.bool, device=t.device)
        else:
            margin = (E - best_e).abs()
            # the same |d| in every column: the device sums the same terms in the same order
            same = (d == best_d).all(1)
            decided &= (margin > B + best_b) | same
            better = (E < best_e) & ~same
        best_e = torch.where(better, E, best_e)
        best_b = torch.where(better, B, best_b)
        best_d = d if i == 0 else torch.where(better.unsqueeze(1), d, best_d)
        mn = torch.where(better.unsqueeze(1), xmin, mn)
        mx = torch.where(better.unsqueeze(1), xmax, mx)
    return mn, mx, decided


def constructed_mse_rows(rows, cols, seed=0):
    """Rows whose level errors are far apart: a few large values and a grid of small ones, so
    every comparison of the search is decided (asserted by the GPU test).  Includes a constant
    row (the 1e-5 floor) and an all-zero row."""
    g = np.random.default_rng(seed)
    base = np.round(g.standard_normal((rows, cols)) * 4) / 4
    base[:, 0] = 8 + g.integers(0, 8, rows)
    base[:, 1] = -8 - g.integers(0, 8, rows)
    base[0] = 0.0
    if rows > 1:
        base[1] = 0.375
    return torch.from_numpy(base.astype(np.float32))
