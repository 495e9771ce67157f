"""CPU: oracle/glue_oracle.py — the block-forward glue and GPTQ's prepare restated in the kernels'
order — against exact sums, hand-derived reduction orders and the torch expressions the kernels
replace (llmc_b200/synth.py, oracle/block_oracle.py, oracle/gptq_oracle.py)."""
import os

import pytest
import torch

from oracle import block_oracle as bo
from oracle import glue_oracle as glo
from oracle import gptq_oracle as go

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


@pytest.mark.parametrize('cols', [8, 2048, 4096, 5120, 8192])
def test_rmsnorm_sumsq_is_exact_when_every_partial_sum_is(cols):
    g = torch.Generator().manual_seed(cols)
    x = torch.randint(-15, 16, (6, cols), generator=g).to(torch.bfloat16)
    x[0] = 0
    got = glo.rmsnorm_sumsq(x)
    exact = x.double().pow(2).sum(-1)
    assert exact.max() < 2 ** 24
    assert torch.equal(got.double(), exact)
    perm = torch.randperm(cols, generator=g)           # any order: every partial sum is an integer < 2^24
    assert torch.equal(glo.rmsnorm_sumsq(x[:, perm]), got)


def test_rmsnorm_sumsq_follows_the_kernel_order():
    """Thread 0 folds x[0] = 2^12 (square 2^24) and then fifteen ones, in chunks 0 and 256:
    every fmaf(1, 1, 2^24) ties back to 2^24.  Threads 1 .. 7 hold a single one each; in the
    warp butterfly lane 4's one meets lane 0's 2^24 at offset 4 and is lost too."""
    cols = 4096
    x = torch.zeros(2, cols, dtype=torch.float16)
    x[0, 0] = 4096
    x[0, 1:8] = 1
    x[0, 256 * 8:256 * 8 + 8] = 1
    assert float(glo.rmsnorm_sumsq(x[:1])) == 2.0 ** 24
    x[1, 0] = 4096
    for t in range(1, 8):
        x[1, t * 8] = 1
    # lanes: 0 -> 2^24, 1..7 -> 1.  offset 4: 2^24 + 1 -> 2^24, 1+1 three times; offset 2:
    # 2^24 + 2, 4; offset 1: 2^24 + 6.  The exact sum is 2^24 + 7.
    s = glo.rmsnorm_sumsq(x)
    assert float(s[1]) == 2.0 ** 24 + 6
    assert float(x[1].double().pow(2).sum()) == 2.0 ** 24 + 7
    ref = x.float().pow(2).sum(-1)                     # torch's own order keeps some of the ones
    assert float(ref[0]) != float(s[0])


def test_rmsnorm_sumsq_fma_rounds_once():
    """fp32 inputs: fmaf(v, v, acc) is one rounding of v*v + acc, not two."""
    v = 1.0 + 2.0 ** -12                               # v*v = 1 + 2^-11 + 2^-24: a tie at 1 ulp
    x = torch.zeros(1, 8, dtype=torch.float32)
    x[0, 0] = 2.0 ** -12
    x[0, 1] = v
    # acc = 2^-24, then fma(v, v, 2^-24) = 1 + 2^-11 + 2^-23 exactly (one rounding); two roundings
    # would give round(1 + 2^-11 + 2^-24) = 1 + 2^-11 (tie to even), then + 2^-24 -> 1 + 2^-11.
    got = float(glo.rmsnorm_sumsq(x)[0])
    assert got == 1 + 2.0 ** -11 + 2.0 ** -23
    two = (torch.tensor(v, dtype=torch.float32) ** 2 + torch.tensor(2.0 ** -24)).item()
    assert got != two


@pytest.mark.parametrize('dtype', DTYPES)
def test_rmsnorm_matches_the_module_at_the_correctly_rounded_inv(dtype):
    """With integer rows every order gives the same mean, so the module's expression (block_oracle,
    synth.RMSNorm's fallback) must be the oracle at torch's rsqrt, which is one of the candidates."""
    g = torch.Generator().manual_seed(1)
    x = torch.randint(-20, 21, (64, 512), generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(512, generator=g)).to(dtype)
    ref = bo.rmsnorm(x, w, 1e-5)
    s = glo.rmsnorm_sumsq(x)
    inv_t = torch.rsqrt(x.float().pow(2).mean(-1) + 1e-5)
    cand = glo.rmsnorm_inv_candidates(s, 512, 1e-5)
    assert bool((cand == inv_t[:, None]).any(-1).all())
    assert torch.equal(glo.rmsnorm(x, w, inv_t), ref)
    # a weight in fp32 under 16-bit activations: the product is promoted, as the module does
    wf = w.float()
    assert torch.equal(glo.rmsnorm(x, wf, inv_t), bo.rmsnorm(x, wf, 1e-5))


def test_rmsnorm_inv_candidates_edges():
    s = torch.tensor([0.0, float('inf'), 4.0 * 8])
    c = glo.rmsnorm_inv_candidates(s, 8, 1e-6)
    assert c.shape == (3, 5)
    assert float(c[0, 2]) == float((1.0 / torch.tensor(1e-6, dtype=torch.float32).double().sqrt()).float())
    assert float(c[1, 2]) == 0.0                        # rsqrt(inf) = 0, as torch gives
    assert float(c[2, 2]) == pytest.approx(0.5, rel=1e-6)
    assert bool((c[:, 1:] > c[:, :-1]).all())


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('heads,head_dim,S', [(1, 16, 1), (4, 64, 7), (2, 128, 33), (1, 256, 5)])
def test_rope_matches_the_module_expression(dtype, heads, head_dim, S):
    from llmc_b200.synth import _rot_half, rope_cos_sin
    g = torch.Generator().manual_seed(heads * head_dim + S)
    B = 2
    x = (torch.randn(B, S, heads * head_dim, generator=g) * 3).to(dtype)
    cos, sin = rope_cos_sin(S + 5, head_dim, 'cpu', dtype)
    cos, sin = cos[:S], sin[:S]
    q = x.view(B, S, heads, head_dim).transpose(1, 2)
    ref = (q * cos[None, None] + _rot_half(q) * sin[None, None]).transpose(1, 2).reshape(x.shape)
    assert torch.equal(glo.rope(x, cos, sin, heads, head_dim), ref)
    bc, bs = bo.rope(S, head_dim, dtype)
    ref2 = (q * bc + bo._rot(q) * bs).transpose(1, 2).reshape(x.shape)
    assert torch.equal(glo.rope(x, bc, bs, heads, head_dim), ref2)
    if dtype != torch.float32:                          # fp32 tables: torch promotes
        cf, sf = cos.float(), sin.float()
        ref3 = (q * cf + _rot_half(q) * sf).transpose(1, 2).reshape(x.shape)
        got = glo.rope(x, cf, sf, heads, head_dim)
        assert got.dtype == torch.float32 and torch.equal(got, ref3)


@pytest.mark.parametrize('dtype', DTYPES)
def test_add_matches_torch(dtype):
    g = torch.Generator().manual_seed(3)
    a = (torch.randn(4096, generator=g) * 100).to(dtype)
    b = (torch.randn(4096, generator=g) * 100).to(dtype)
    assert torch.equal(glo.add(a, b), a + b)


def test_diag_mean_order():
    """Exact when the partial sums are; 2^24 then ones held by other threads: the order decides."""
    C = 1000
    H = torch.diag(torch.arange(C, dtype=torch.float32) % 7)
    d = torch.diagonal(H)
    mean = float(torch.where(d == 0, torch.ones_like(d), d).double().sum()) / C
    assert float(glo.diag_mean(H, 1.0)) == float(torch.tensor(mean, dtype=torch.float32))
    H = torch.zeros(512, 512)
    H[0, 0] = 2.0 ** 24
    H[256, 256] = 3.0        # thread 0 again: 2^24 + 3 -> 2^24 + 4; the other 510 zeros become 1
    # thread 0: 2^24 + 3 -> 2^24 + 4 (tie to even); threads 1..255: 1 + 1 = 2 each
    lanes = [2.0 ** 24 + 4] + [2.0] * 255
    assert float(glo.diag_mean(H, 1.0) * 512) == pytest.approx(sum(lanes), rel=1e-7)
    assert float(glo.diag_mean(H, 0.01)) == float(torch.tensor(0.01, dtype=torch.float32)
                                                  * (glo.diag_mean(H, 1.0)))


def test_prepare_reproduces_the_golden_layers(golden_dir):
    """The four reference-generated GPTQ layers: Wp bit for bit, Hp off the diagonal bit for bit
    (pure gathers), the diagonal within the fp32 rounding of the damping's mean."""
    kat = torch.load(os.path.join(golden_dir, 'gptq_kat.pt'), weights_only=False)
    for c in kat:
        perm = c['perm'] if c['special']['actorder'] else None
        Wp, Hp = glo.prepare(c['W'], c['H'], perm, 0.01)
        assert torch.equal(Wp, c['Wp'])
        C = c['H'].shape[0]
        p = perm if perm is not None else torch.arange(C)
        ref = c['H'][p][:, p]
        off = ~torch.eye(C, dtype=torch.bool)
        assert torch.equal(Hp[off], ref[off])
        rd = torch.diagonal(ref).clone()
        rd[rd == 0] = 1
        rd = rd + 0.01 * torch.mean(rd)
        assert torch.allclose(torch.diagonal(Hp), rd, rtol=1e-6, atol=0)
        Wp2, _, _ = go.prepare(c['W'], c['H'], False, 0.01)      # dead columns, unpermuted
        assert torch.equal(glo.prepare(c['W'], c['H'], None, 0.01)[0], Wp2)


def test_prepare_dead_columns_follow_the_permutation():
    g = torch.Generator().manual_seed(5)
    C = 12
    X = torch.randn(64, C, generator=g)
    X[:, [2, 7]] = 0
    H = X.t() @ X
    W = torch.randn(3, C, generator=g).bfloat16()
    perm = torch.argsort(torch.diagonal(H), descending=True)
    Wp, Hp = glo.prepare(W, H, perm, 0.5)
    ref, _, rperm = go.prepare(W, H, True, 0.5)
    assert torch.equal(rperm, perm)
    assert torch.equal(Wp, ref)
    moved = [int(j) for j in range(C) if int(perm[j]) in (2, 7)]
    assert sorted(moved) == [10, 11]
    assert bool((Wp[:, moved] == 0).all())
    assert bool((torch.diagonal(Hp)[moved] == 1 + glo.diag_mean(H, 0.5)).all())


def test_division_is_correctly_rounded():
    """The kernels divide in IEEE fp32 (sum / cols, sum / C); the oracle must not divide through a
    reciprocal, which differs for divisors that are not powers of two (5120, 14336)."""
    import numpy as np
    g = torch.Generator().manual_seed(11)
    v = torch.rand(100000, generator=g) * 1e6
    for n in (7, 5120, 14336):
        ref = torch.from_numpy(v.numpy() / np.float32(n))
        assert torch.equal(glo._div32(v, n), ref)
