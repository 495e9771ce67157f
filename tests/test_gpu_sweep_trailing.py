"""The trailing updates of the GPTQ and SpQR column sweeps (`sweep_schedule` in
llmc_b200/csrc/gptq.cu) against the CPU oracle, bit for bit, through every schedule branch.

The sweep applies W[:, i2:] -= Err1 @ Hinv[i1:i2, i2:] lazily: rank-128 updates inside a 512-column
super-panel, one rank-512 update at its end, split by the look-ahead into a chain piece (the next
super-panel) and a bulk piece (everything beyond), with two error sets alternating by super-panel
parity; one-block super-panels when a group does not fit 512; the serial schedule for dynamic groups
wider than 512; the fp32 SIMT kernel when C % 8 != 0 or W is not 16-byte aligned.  These orders of
summation differ from the oracle's eager fp32 GEMM, so on a real Hinv they agree only to rounding.

Here Hinv keeps the 128 x 128 diagonal blocks of real upper factors, and every column j >= 128 gets
exactly ONE entry outside them, Hinv[k(j), j] = +-2^e with k(j) in an earlier block and
2^e <= Hinv[k, k] < 2^(e+3).  Every column then receives exactly one non-zero product from all its
trailing updates together, and that product is exact, so any schedule gives the same bits:
  * SIMT: fmaf(err, +-2^e, 0) is exact, and the oracle runs unchanged;
  * 3xTF32: the in-block kernel stores hi = tf32(err), lo = tf32(err - hi), the split of +-2^e is
    (+-2^e, 0), so the accumulator holds (hi + lo) * 2^e exactly (hi + lo fits an fp32
    significand) and the epilogue rounds once, W - acc.  The oracle models this with
    trailing_split=True.
k(j) cycles through three categories: an earlier block of the same super-panel (in-panel update),
the previous super-panel (look-ahead chain piece) and two or more super-panels back (bulk piece)."""
import functools
import math
import os
import zlib

import pytest
import torch

from oracle import gptq_oracle as go
from oracle import quant_oracle as qo
from oracle import spqr_oracle as so

BLOCK, PANEL = 128, 512


# ---- the structured Hinv ----------------------------------------------------------------------------
def _diag_blocks(C, g):
    """Block-diagonal [C, C]: each 128 x 128 block is the upper factor go.prepare makes from the
    Hessian of random bf16 activations of that block's columns."""
    U = torch.zeros(C, C)
    for b0 in range(0, C, BLOCK):
        n = min(BLOCK, C - b0)
        X = (torch.randn(1, 4 * BLOCK, n, generator=g) * torch.exp(torch.randn(n, generator=g))).bfloat16()
        H, _ = go.hessian([X], n)
        U[b0:b0 + n, b0:b0 + n] = go.prepare(torch.zeros(1, n), H, False, 0.01)[1]
    return U


def _structured_hinv(U, g):
    """U's 128 x 128 diagonal blocks plus one +-2^e entry per column j >= 128 (module docstring)."""
    C = U.shape[0]
    blk = torch.arange(C) // BLOCK
    Hinv = torch.where(blk[:, None] == blk[None, :], U, torch.zeros(()))
    diag = torch.diag(Hinv).tolist()
    u = torch.rand(C, generator=g, dtype=torch.float64).tolist()
    neg = torch.randint(0, 2, (C,), generator=g).tolist()
    shift = torch.randint(0, 3, (C,), generator=g).tolist()
    for j in range(BLOCK, C):
        p0 = j // PANEL * PANEL
        ranges = [(p0, j // BLOCK * BLOCK), (p0 - PANEL, p0), (0, p0 - PANEL)]
        ranges = [(max(lo, 0), hi) for lo, hi in ranges if hi > max(lo, 0)]
        lo, hi = ranges[j % len(ranges)]
        k = lo + int(u[j] * (hi - lo))
        e = math.frexp(diag[k])[1] - 1 - shift[j]            # floor(log2 Hinv[k, k]) - {0, 1, 2}
        Hinv[k, j] = (-1.0 if neg[j] else 1.0) * 2.0 ** e
    return Hinv


def _category(Hinv):
    """(k, category) of each column j >= 128: 0 same super-panel, 1 previous, 2 two or more back."""
    C = Hinv.shape[0]
    blk = torch.arange(C) // BLOCK
    off = torch.where(blk[:, None] == blk[None, :], torch.zeros(()), Hinv)
    k = (off != 0).to(torch.uint8).argmax(0)[BLOCK:]
    gap = torch.arange(BLOCK, C) // PANEL - k // PANEL
    return k, gap.clamp(max=2)


def _seed(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _diff(name, got, want):
    """None if bit-identical, else where they differ: for [R, C] the differing columns."""
    if torch.equal(got, want):
        return None
    bad = got != want
    if bad.dim() == 2:
        cols = bad.any(0).nonzero().flatten().tolist()
        return f'{name}: {int(bad.sum())} entries in {len(cols)} columns, first {cols[:8]}'
    return f'{name}: {int(bad.sum())} entries'


def _schedules(monkeypatch):
    """The default (look-ahead where it applies) and the serial schedule of sweep_schedule."""
    for sched in ('default', 'serial'):
        if sched == 'serial':
            monkeypatch.setenv('LLMC_B200_SWEEP_LOOKAHEAD', '0')
        else:
            monkeypatch.delenv('LLMC_B200_SWEEP_LOOKAHEAD', raising=False)
        yield sched


def _device_w(W, misalign):
    """W on the device; misalign: a contiguous view one float into a larger buffer (4-byte aligned)."""
    R, C = W.shape
    if misalign:
        Wd = torch.zeros(R * C + 1, device='cuda')[1:].view(R, C)
        assert Wd.is_contiguous() and Wd.data_ptr() % 16 == 4
    else:
        Wd = torch.empty(R, C, device='cuda')
    return Wd.copy_(W)


# ---- GPTQ cases: each reaches the schedule branch in its name -------------------------------------------
# group None: per-channel (static qparams from RTN on the weight, as GPTQ passes them)
GPTQ_CASES = {
    'g128-333x1152-lookahead-one-block-last-panel': dict(R=333, C=1152, bit=4, sym=False, group=128),
    'g128-1000x4096-out-perm-8-panels': dict(R=1000, C=4096, bit=4, sym=False, group=128, perm=True),
    'g16sym-333x1680-partial-last-panel-and-block': dict(R=333, C=1680, bit=4, sym=True, group=16),
    'g256w3-200x2560-search-reads-next-block': dict(R=200, C=2560, bit=3, sym=False, group=256),
    'g1024-200x2048-wide-group-serial': dict(R=200, C=2048, bit=4, sym=False, group=1024),
    'static-g128-520x2560-actorder-gmap-out-perm': dict(R=520, C=2560, bit=4, sym=False, group=128,
                                                        static=True, perm=True),
    'channel-w8sym-256x4096-lookahead': dict(R=256, C=4096, bit=8, sym=True, group=None),
    'channel-w4-96x1000-one-block-panels': dict(R=96, C=1000, bit=4, sym=False, group=None),
    'channel-w4-333x700-simt-c-not-mult-8': dict(R=333, C=700, bit=4, sym=False, group=None),
    'g128-333x1024-misaligned-w-simt': dict(R=333, C=1024, bit=4, sym=False, group=128, misalign=True),
}


@functools.lru_cache(maxsize=None)
def _gptq_problem(name):
    c = GPTQ_CASES[name]
    R, C, bit, sym = c['R'], c['C'], c['bit'], c['sym']
    g = _seed(name)
    W = torch.randn(R, C, generator=g) * 0.02 * torch.exp(0.3 * torch.randn(R, 1, generator=g))
    Hinv = _structured_hinv(_diag_blocks(C, g), g)
    perm = torch.randperm(C, generator=g) if c.get('perm') else None
    group = c['group'] or C
    gran = 'per_group' if c['group'] else 'per_channel'
    static = None
    if gran == 'per_channel' or c.get('static'):
        W_orig = W[:, torch.argsort(perm)] if perm is not None else W
        _, s, z, _, _ = qo.tensor_qparams(W_orig, bit, sym, gran, group)
        static = (s.reshape(R, -1), None if sym else z.reshape(R, -1))
    # the 3xTF32 trailing path needs C % 8 == 0 and 16-byte aligned W (gptq.cu, sweep_schedule)
    tensor_path = C % 8 == 0 and not c.get('misalign')
    return dict(c, W=W, Hinv=Hinv, perm=perm, group=group, gran=gran, static=static,
                tensor_path=tensor_path)


def _gptq_oracle(p, trailing_split):
    sq = None
    if p['static'] is not None:
        s, z = p['static']
        z = torch.zeros_like(s) if z is None else z
        sq = (s, z) if p['gran'] == 'per_channel' else \
            ([s[:, i:i + 1] for i in range(s.shape[1])], [z[:, i:i + 1] for i in range(s.shape[1])])
    return go.weight_transform(p['W'], p['Hinv'], p['bit'], p['sym'], p['gran'], p['group'],
                               static_qparams=sq, perm=p['perm'], trailing_split=trailing_split)


@functools.lru_cache(maxsize=None)
def _gptq_reference(name):
    p = _gptq_problem(name)
    return _gptq_oracle(p, p['tensor_path'])


def _lazy_sweep(W, Hinv, bit, sym, group):
    """go.weight_transform(..., trailing_split=True) for dynamic groups, on the library's schedule:
    each block's errors go onto the rest of its 512-column super-panel, and the super-panel's
    errors onto everything beyond it in one rank-512 update.  Groups are searched on W, not on the
    block's working copy, as in the reference."""
    W = W.clone()
    R, C = W.shape
    qmin, qmax = qo.int_range(bit, sym)
    tmp, Losses, groups = torch.zeros_like(W), torch.zeros_like(W), {}
    for p0 in range(0, C, PANEL):
        p1 = min(p0 + PANEL, C)
        E = torch.zeros(R, p1 - p0)
        for i1 in range(p0, p1, BLOCK):
            i2 = min(i1 + BLOCK, C)
            W1 = W[:, i1:i2].clone()
            for i in range(i2 - i1):
                idx = i1 + i
                if idx % group == 0:
                    groups[idx // group] = qo.tensor_qparams(W[:, idx:idx + group], bit, sym, 'per_group', group)[1:3]
                s, z = groups[idx // group]
                w, d = W1[:, i], Hinv[idx, idx]
                q = qo.dequant(qo.quant(w.unsqueeze(1), s, z, qmax, qmin), s, z).squeeze(1)
                tmp[:, idx], Losses[:, idx] = w, ((w - q) ** 2) / (2 * d ** 2)
                E[:, idx - p0] = (w - q) / d
                W1[:, i:] -= E[:, idx - p0].unsqueeze(1).matmul(Hinv[idx, idx:i2].unsqueeze(0))
            hi, lo = go.tf32_split(E[:, i1 - p0:i2 - p0])
            W[:, i2:p1] -= (hi + lo).matmul(Hinv[i1:i2, i2:p1])
        hi, lo = go.tf32_split(E)
        W[:, p1:] -= (hi + lo).matmul(Hinv[p0:p1, p1:])
    return tmp, Losses, [groups[k] for k in sorted(groups)]


@pytest.mark.parametrize('name', ['g16sym-333x1680-partial-last-panel-and-block',
                                  'g256w3-200x2560-search-reads-next-block'])
def test_structured_hinv_makes_every_schedule_exact(name):
    """CPU: the construction the GPU tests rest on.  One +-2^e entry per column outside the
    diagonal blocks, every category in every super-panel that can have it; hi + lo of the tf32
    split is exact in fp32 but not equal to x (so the split must be modelled); and the library's
    lazy super-panel schedule, emulated on the oracle, gives the eager oracle's bits."""
    p = _gptq_problem(name)
    Hinv, C = p['Hinv'], p['C']
    blk = torch.arange(C) // BLOCK
    off = torch.where(blk[:, None] == blk[None, :], torch.zeros(()), Hinv)
    per_col = (off != 0).sum(0)
    assert (per_col[:BLOCK] == 0).all() and (per_col[BLOCK:] == 1).all()
    k, cat = _category(Hinv)
    j = torch.arange(BLOCK, C)
    v = off[k, j]
    assert (blk[k] < blk[j]).all()
    assert (torch.frexp(v).mantissa.abs() == 0.5).all(), 'entries must be powers of two'
    ratio = torch.diag(Hinv)[k] / v.abs()
    assert ((ratio >= 1) & (ratio < 8)).all()
    panel = j // PANEL
    for sp in range(int(panel.max()) + 1):
        assert set(cat[panel == sp].tolist()) == set(range(min(sp, 2) + 1)), sp

    g = _seed('split')
    x = torch.randn(1 << 16, generator=g) * torch.exp2(torch.randint(-60, 20, (1 << 16,), generator=g).float())
    x[::4] = ((x[::4].view(torch.int32) & -0x2000) | 0x1000).view(torch.float32)     # exact ties
    hi, lo = go.tf32_split(x)
    assert ((hi.view(torch.int32) & 0x1fff) == 0).all() and ((lo.view(torch.int32) & 0x1fff) == 0).all()
    assert torch.equal((hi + lo).double(), hi.double() + lo.double()), 'hi + lo must be exact in fp32'
    assert ((hi + lo) != x).any()
    pw = torch.tensor([2.0 ** -20, -(2.0 ** -3), 2.0 ** 5])
    assert torch.equal(go.tf32_split(pw)[0], pw) and torch.equal(go.tf32_split(pw)[1], torch.zeros(3))

    ref = _gptq_reference(name)
    lazy = _lazy_sweep(p['W'], Hinv, p['bit'], p['sym'], p['group'])
    assert torch.equal(lazy[0], ref[0]) and torch.equal(lazy[1], ref[1])
    for (s, z), (s_o, z_o) in zip(lazy[2], ref[2], strict=True):
        assert torch.equal(s, s_o) and torch.equal(z, z_o)
    plain = _gptq_oracle(p, trailing_split=False)[0]
    assert float((plain != ref[0]).float().mean()) > 0.01, 'the split must be visible in tmp'


# ---- GPU ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_split_tf32_matches_oracle():
    """llmc_split_tf32 (the kernel that splits Hinv for every 3xTF32 trailing update) against
    go.tf32_split, bit for bit: random normals of both signs over a wide exponent range, exact ties
    (low 13 bits 0x1000, rounded away from zero), a tie that carries into the exponent, zero."""
    from llmc_b200._lib import call, ptr, stream_ptr
    g = _seed('split-gpu')
    x = torch.randn(64, 1000, generator=g) * torch.exp2(torch.randint(-60, 20, (64, 1), generator=g).float())
    x[:16] = ((x[:16].view(torch.int32) & -0x2000) | 0x1000).view(torch.float32)
    x[16, :4] = torch.tensor([0x3f7ff000, -0x40801000, 0, 0x3fc01000], dtype=torch.int32).view(torch.float32)
    xd = x.cuda()
    hi, lo = torch.empty_like(xd), torch.empty_like(xd)
    call('llmc_split_tf32', ptr(xd), 64, 1000, 1000, ptr(hi), ptr(lo), stream_ptr(xd.device))
    hi_o, lo_o = go.tf32_split(x)
    assert torch.equal(hi.cpu().view(torch.int32), hi_o.view(torch.int32))
    assert torch.equal(lo.cpu().view(torch.int32), lo_o.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(GPTQ_CASES))
def test_gptq_trailing_updates_bit_exact(name, monkeypatch):
    """ops.weight_transform on the structured Hinv, with the default and the serial schedule:
    tmp, scales and zeros bit-identical to the oracle (with the tf32 split on the 3xTF32 path,
    without it on the SIMT path), per-row losses within 1e-5 (the kernel sums a row in another
    order)."""
    from llmc_b200 import gptq_ops as ops
    p = _gptq_problem(name)
    tmp_o, L_o, groups = _gptq_reference(name)
    perm = p['perm']
    kw = {}
    if p['static'] is not None:
        s, z = p['static']
        kw['static_qparams'] = (s.reshape(-1).cuda(), None if z is None else z.reshape(-1).cuda())
        if perm is not None and p['gran'] == 'per_group':
            kw['gmap'] = (perm // p['group']).to(torch.int32).cuda()
    if perm is not None:
        kw['out_perm'] = perm.cuda()
    Hinv = p['Hinv'].cuda()
    bad = {}
    for sched in _schedules(monkeypatch):
        W = _device_w(p['W'], p.get('misalign'))
        tmp, losses, scales, zeros = (t.cpu() if t is not None else None for t in ops.weight_transform(
            W, Hinv, p['bit'], p['sym'], p['group'], **kw))
        if perm is not None:
            tmp = tmp[:, perm]
        msgs = [_diff('tmp', tmp, tmp_o)]
        if p['static'] is None:
            msgs.append(_diff('scales', scales, torch.cat([s for s, _ in groups], 1)))
            if not p['sym']:
                msgs.append(_diff('zeros', zeros, torch.cat([z for _, z in groups], 1)))
        if not torch.allclose(losses, L_o.sum(1), rtol=1e-5, atol=0):
            msgs.append('losses: max rel %.3g' % float(((losses - L_o.sum(1)).abs() / L_o.sum(1)).max()))
        msgs = [m for m in msgs if m]
        if msgs:
            bad[sched] = msgs
    assert not bad, bad


# ---- SpQR cases ------------------------------------------------------------------------------------------
SPQR_KAT = ['w4_g16_thr0.2', 'w3_g32_thr0.1_noorder', 'w4_g16_simplified', 'w4_g64_inf', 'w4_g16_roundzp']
SPQR_CASES = {
    **{f'kat-{n}': dict(kat=i) for i, n in enumerate(SPQR_KAT)},
    'g16-1000x2048-out-perm': dict(R=1000, C=2048, gs=16, perm=True),
    'g16-333x1680-partial-last-panel-and-block': dict(R=333, C=1680, gs=16),
    'g32-333x1024-misaligned-w-simt': dict(R=333, C=1024, gs=32, misalign=True),
}


@functools.lru_cache(maxsize=None)
def _spqr_problem(name, golden_dir):
    c = SPQR_CASES[name]
    g = _seed(name)
    if 'kat' in c:
        k = torch.load(os.path.join(golden_dir, 'spqr_kat.pt'), weights_only=False)[c['kat']]
        assert k['name'] == SPQR_KAT[c['kat']]
        W, U, perm = k['Wp'], k['Hinv'], None
        wkw, special, l2 = k['weight_kwargs'], k['special'], k['level2']
    else:
        R, C = c['R'], c['C']
        W = torch.randn(R, C, generator=g) * 0.02
        W[torch.rand(R, C, generator=g) < 0.01] *= 8
        U = _diag_blocks(C, g)
        perm = torch.randperm(C, generator=g) if c.get('perm') else None
        wkw = dict(bit=4, symmetric=False, round_zp=False, group_size=c['gs'])
        special = dict(relative_threshold=0.2, simplified_outliers=False)
        l2 = dict(bit=3, symmetric=False, round_zp=False)
    Hinv = _structured_hinv(U, g)
    thr = so.threshold_of(W, Hinv, special['relative_threshold'])
    tensor_path = W.shape[1] % 8 == 0 and not c.get('misalign')
    ref = so.weight_transform(W, Hinv, so.make_cfg(wkw, special, l2, l2, thr), trailing_split=tensor_path)
    wcfg = (wkw['bit'], wkw['symmetric'], wkw.get('round_zp', True), wkw['group_size'])
    l2c = (l2['bit'], l2['symmetric'], l2.get('round_zp', True))
    return dict(W=W, Hinv=Hinv, perm=perm, thr=thr, wcfg=wcfg, l2c=l2c,
                simplified=special['simplified_outliers'], misalign=c.get('misalign', False), ref=ref)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(SPQR_CASES))
def test_spqr_trailing_updates_bit_exact(name, golden_dir, monkeypatch):
    """ops.spqr_transform on the structured Hinv with the oracle's threshold, default and serial
    schedule: tmp, outlier mask, scales, zeros and per-row losses all bit-identical to the oracle
    (the SpQR kernel sums a row's loss in the oracle's order)."""
    from llmc_b200 import gptq_ops as ops
    p = _spqr_problem(name, golden_dir)
    tmp_o, mask_o, S_o, Z_o, loss_o = p['ref']
    perm = p['perm']
    thr = torch.tensor([p['thr']], dtype=torch.float32, device='cuda')
    Hinv = p['Hinv'].cuda()
    bad = {}
    for sched in _schedules(monkeypatch):
        W = _device_w(p['W'], p['misalign'])
        tmp, mask, losses, S, Z = (t.cpu() for t in ops.spqr_transform(
            W, Hinv, p['wcfg'], p['l2c'], p['l2c'], thr, p['simplified'],
            out_perm=perm.cuda() if perm is not None else None))
        if perm is not None:
            tmp, mask = tmp[:, perm], mask[:, perm]
        msgs = [_diff('tmp', tmp, tmp_o), _diff('mask', mask, mask_o), _diff('scales', S, S_o),
                _diff('zeros', Z, Z_o), _diff('losses', losses, loss_o)]
        msgs = [m for m in msgs if m]
        if msgs:
            bad[sched] = msgs
    assert not bad, bad
