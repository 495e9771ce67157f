"""GPU: the blocked Cholesky inverse (`llmc_chol_inv_upper`, csrc/chol.cu, DESIGN.md §K4) bit for
bit against the exact integer oracle (oracle/chol_oracle.py) on every branch of its host schedule.

On the oracle's inputs every step of the factorisation and of the inverse is exact, in fp32 and in
3xTF32, in any order and under any cut of the lazy updates, so the output must equal U = J L^-1 J
exactly: a dropped or repeated rank-128 piece, a stale tf32 split or a read of unwritten workspace
changes it.  (Values are compared, so -0 equals +0.)  Each path-table entry asserts, from a
restatement of the host plan, that its C reaches the branches it is named for, and runs three ways:
through the wrapper out of place and in place, and through the C ABI with a workspace of 0xFF
bytes (NaN as fp32) and NaN in H's strict lower triangle, which the kernel does not read.

Around the table: a reused workspace left dirty by a wider call; the failure flag at chosen pivots
and for a NaN input; determinism across calls, streams and a concurrent GEMM; and accuracy on
damped Hessians against an fp64 Cholesky inverse, relative to cuSOLVER's fp32 one."""
import pytest
import torch

from llmc_b200 import gptq_ops as ops
from llmc_b200._lib import call, load, ptr, stream_ptr
from oracle import chol_oracle as co

pytestmark = pytest.mark.gpu

NB, SPW = 128, 512                   # diagonal block and super-panel widths of chol.cu


# ---- the host plan, restated ---------------------------------------------------------------------
def chol_cases(C):
    """The branches of llmc_chol_inv_upper's host plan that C reaches."""
    n = C
    nbk = -(-n // NB)
    cases = set()
    if n % NB:
        cases.add('partial-block')          # diag_kernel pads the last block with the identity
    if n <= SPW:
        cases.add('serial')
        cases.add('one-block' if nbk == 1 else 'multi-block')
        if n == SPW:
            cases.add('full-super-panel')
        return cases
    cases.add('look-ahead')
    if (nbk - 1) % 4 == 0:
        cases.add('last-sp-one-block')      # the last super-panel holds a single block
    for kb in range(nbk):
        k0 = kb * NB
        nb = min(NB, n - k0)
        sidx = k0 // SPW
        sp0 = sidx * SPW
        sp1 = min(sp0 + SPW, n)
        r0 = k0 + nb
        m = n - r0
        if k0 > sp0:
            cases.add('left-looking')       # rank-128*(j-j0) chain update inside a super-panel
            if sidx > 0 and k0 == sp0 + NB:
                cases.add('chain-waits-A′')  # columns written by the previous boundary's A' piece
        if m > 0 and r0 == sp1:
            cases.add('boundary')
            w1 = min(n - sp1, NB)
            cases.add('narrow-w1' if w1 < NB else 'full-w1')
            ca = sp1 + NB
            cb = min(ca + SPW, n)
            if ca < n:
                cases.add('A′')
                cases.add('A′-narrow' if cb - ca < SPW else 'A′-full')
            if cb < n:
                cases.add('B')
                if (n - cb) % NB:
                    cases.add('B-ragged')
        if m > 0 and r0 < sp1:
            cases.add('inverse-in-panel')
        elif m > 0:
            cases.add('inverse-boundary')
            if min(sp1 + SPW, n) < n:
                cases.add('s3')             # inverse rows beyond the next super-panel
    return cases


EVERY_LOOKAHEAD = {'look-ahead', 'left-looking', 'chain-waits-A′', 'boundary', 'full-w1', 'A′',
                   'A′-full', 'A′-narrow', 'B', 'inverse-in-panel', 'inverse-boundary', 's3'}
RAGGED = {'partial-block', 'narrow-w1', 'B-ragged', 'last-sp-one-block'}
SERIAL_PARTIAL = {'serial', 'one-block', 'partial-block'}

# (C, factors of L, seed, branches reached, branches not reached); factors = 0 is H = I.  Seed 2 at
# C = 14336 is the first whose rank-128 pieces are all nonzero (seed 0 leaves one zero there).
PATHS = [
    pytest.param(8, 0, 0, SERIAL_PARTIAL, set(), id='identity-8'),   # rsqrtf(1) == 1 exactly
    pytest.param(8, 3, 0, SERIAL_PARTIAL, set(), id='8'),
    pytest.param(120, 3, 0, SERIAL_PARTIAL, set(), id='120'),
    pytest.param(128, 3, 0, {'serial', 'one-block'}, {'partial-block'}, id='128'),
    pytest.param(136, 3, 0, {'serial', 'multi-block', 'partial-block'}, set(), id='136'),
    pytest.param(504, 3, 0, {'serial', 'multi-block', 'partial-block'}, set(), id='504'),
    pytest.param(512, 3, 0, {'serial', 'multi-block', 'full-super-panel'}, {'partial-block'}, id='512'),
    pytest.param(520, 3, 0, {'look-ahead', 'narrow-w1', 'last-sp-one-block', 'inverse-boundary'},
                 {'A′', 'B', 's3'}, id='520'),
    pytest.param(640, 3, 0, {'look-ahead', 'full-w1', 'left-looking'}, {'A′', 'B', 's3'}, id='640'),
    pytest.param(648, 3, 0, {'A′-narrow', 'chain-waits-A′'}, {'A′-full', 'B', 's3'}, id='648'),
    pytest.param(1024, 3, 0, {'A′-narrow', 'chain-waits-A′'}, {'A′-full', 'B', 's3'}, id='1024'),
    pytest.param(1032, 3, 0, {'s3', 'narrow-w1'}, {'B'}, id='1032'),
    pytest.param(1096, 3, 0, {'s3', 'narrow-w1'}, {'B'}, id='1096'),
    pytest.param(1160, 3, 0, {'B', 'B-ragged', 'A′-full', 's3'}, set(), id='1160'),
    pytest.param(1544, 3, 0, {'B', 'B-ragged', 'A′-narrow'}, set(), id='1544'),
    pytest.param(2056, 3, 0, {'B', 'B-ragged', 'last-sp-one-block'}, set(), id='2056'),
    pytest.param(4104, 3, 0, {'B', 'B-ragged', 'last-sp-one-block'}, set(), id='4104'),
    pytest.param(4096, 3, 0, EVERY_LOOKAHEAD, RAGGED, id='4096'),
    pytest.param(14336, 3, 2, EVERY_LOOKAHEAD, RAGGED, id='14336'),
]


# ---- helpers -------------------------------------------------------------------------------------
def _exact(got, exp, what):
    """Exact equality of values; NaN never matches."""
    assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, got.dtype)
    bad = ~(got == exp)
    if bool(bad.any()):
        idx = bad.nonzero()[:4].tolist()
        first = [(i, got[tuple(i)].item(), exp[tuple(i)].item()) for i in idx]
        raise AssertionError(f'{what}: {int(bad.sum())}/{got.numel()} elements differ; first '
                             f'(index, got, expected): {first}')


def _abi(H, info=None):
    """llmc_chol_inv_upper on a copy of H whose strict lower triangle is NaN, with a workspace of
    0xFF bytes; returns (U, info)."""
    C = H.shape[0]
    A = H.clone()
    A.masked_fill_(torch.ones(C, C, dtype=torch.bool, device=A.device).tril_(-1), float('nan'))
    nbytes = load().llmc_chol_workspace_bytes(C)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=A.device)
    if info is None:
        info = torch.full((1,), -7, dtype=torch.int32, device=A.device)
    call('llmc_chol_inv_upper', ptr(A), C, ptr(ws), nbytes, ptr(info), stream_ptr(A.device))
    return A, info


def _oracle(C, factors=3, seed=0):
    """(H, U) of the exact oracle, after asserting its exactness bounds and full coverage."""
    L, Y = co.unit_lower_pair(C, factors=factors, seed=seed, device='cuda')
    co.exactness_bounds(L, Y)
    for what, (got, total) in co.coverage(L, Y).items():
        assert got == total, (C, what, got, total)
    return co.chol_case(L, Y)


def _hessian(C, seed):
    """A damped Hessian of activations with log-normal column scales (as test_gpu_chol.py),
    symmetrised so that the kernel (upper triangle) and cuSOLVER (lower) see the same matrix."""
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    T = 4 * C
    X = torch.randn(T, C, device='cuda', generator=g) * torch.exp(
        torch.randn(C, device='cuda', generator=g) * 0.7)
    H = (2.0 / T) * (X.t() @ X)
    del X
    H = 0.5 * (H + H.t())
    H += 0.01 * torch.diag(H).mean() * torch.eye(C, device='cuda')
    return H


# ---- the path table ------------------------------------------------------------------------------
@pytest.mark.parametrize('C,factors,seed,reached,not_reached', PATHS)
def test_path_table(C, factors, seed, reached, not_reached):
    cases = chol_cases(C)
    assert reached <= cases, (C, reached - cases)
    assert not (not_reached & cases), (C, not_reached & cases)
    H, U = _oracle(C, factors, seed)
    H0 = H.clone()
    out, info = ops.chol_inv_upper(H, return_info=True)
    _exact(out, U, f'C={C} out of place')
    assert int(info.item()) == 0
    assert torch.equal(H, H0), 'out of place must not touch H'
    A = H.clone()
    out, info = ops.chol_inv_upper(A, inplace=True, return_info=True)
    assert out.data_ptr() == A.data_ptr()
    _exact(out, U, f'C={C} in place')
    assert int(info.item()) == 0
    out, info = _abi(H)
    _exact(out, U, f'C={C} C ABI, 0xFF workspace, NaN below the diagonal')
    assert int(info.item()) == 0


def test_dirty_workspace_from_a_wider_call():
    """The grow-only workspace cache hands a C = 4104 call's bytes to a C = 1544 call, which then
    sees them with another leading dimension."""
    ops.free_workspaces()
    for C in (4104, 1544):
        H, U = _oracle(C)
        out, info = ops.chol_inv_upper(H, return_info=True)
        _exact(out, U, f'C={C} after a wider call')
        assert int(info.item()) == 0
        ws = ops._workspace(0, H.device, 'chol')
        if C == 4104:
            first = ws.data_ptr()
    assert ws.data_ptr() == first, 'the second call must reuse the first call\'s workspace'


# ---- the failure flag ----------------------------------------------------------------------------
@pytest.mark.parametrize('C', [504, 1544, 4104])
def test_info_is_the_first_nonpositive_pivot(C):
    """G = L D L^T with D = I but d_k in {0, -1}: pivots 0 .. k-1 are exactly 1 and pivot k is d_k,
    so info = k + 1 (in the reversed order the kernel factors in)."""
    L, Y = co.unit_lower_pair(C, device='cuda')
    co.exactness_bounds(L, Y)            # |L| |D| |L|^T <= |L| |L|^T: the same bounds hold
    for k in [k for k in (0, 31, 32, 127, 128, 511, 512, 640, C - 1) if k < C]:
        for dk in (0.0, -1.0):
            d = torch.ones(C, dtype=torch.float64, device='cuda')
            d[k] = dk
            H, _ = co.chol_case(L, None, d)
            _, info = ops.chol_inv_upper(H, return_info=True)
            assert int(info.item()) == k + 1, (C, k, dk, int(info.item()))
    torch.cuda.synchronize()


@pytest.mark.parametrize('C', [504, 1544])
def test_info_for_a_nan_in_the_upper_triangle(C):
    """A NaN at H[p, q], p <= q, is G[C-1-p, C-1-q] on or below G's diagonal: it reaches only row
    C-1-p of L and the Schur columns right of it, so pivot C-1-p is the first non-positive one."""
    H, _ = _oracle(C)
    for p, q in [(0, 0), (0, C - 1), (C - 1, C - 1), (C - 129, C - 1), (C - 513, C - 2), (7, 300),
                 (C // 2, C // 2)]:
        if not 0 <= p <= q < C:
            continue
        A = H.clone()
        A[p, q] = float('nan')
        _, info = ops.chol_inv_upper(A, return_info=True)
        assert int(info.item()) == C - p, (C, p, q, int(info.item()))
        _, info = _abi(A)
        assert int(info.item()) == C - p, (C, p, q, int(info.item()))
    torch.cuda.synchronize()


def test_info_is_reset_by_the_next_call():
    C = 648
    L, Y = co.unit_lower_pair(C, device='cuda')
    d = torch.ones(C, dtype=torch.float64, device='cuda')
    d[200] = -1.0
    bad, _ = co.chol_case(L, None, d)
    good, U = co.chol_case(L, Y)
    info = torch.zeros(1, dtype=torch.int32, device='cuda')
    _abi(bad, info)
    assert int(info.item()) == 201
    out, _ = _abi(good, info)
    assert int(info.item()) == 0
    _exact(out, U, 'SPD call after a failed one')


# ---- determinism and accuracy on real Hessians ---------------------------------------------------
@pytest.mark.parametrize('C', [768, 1544, 4096, 14336])
def test_deterministic_across_calls_streams_and_load(C):
    """DESIGN §K4: every column block receives its updates in an order fixed by events, so the
    result does not depend on timing; the multi-GPU sweep relies on every rank getting the same
    bits.  Three calls, one on a non-default stream, one beside a bf16 GEMM on another stream."""
    H = _hessian(C, C)
    outs = [ops.chol_inv_upper(H) for _ in range(3)]
    cur = torch.cuda.current_stream()
    s = torch.cuda.Stream()
    s.wait_stream(cur)
    with torch.cuda.stream(s):
        outs.append(ops.chol_inv_upper(H))
    cur.wait_stream(s)
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        a = torch.randn(8192, 8192, device='cuda', dtype=torch.bfloat16)
        for _ in range(4 + C // 1024):
            b = a @ a
    outs.append(ops.chol_inv_upper(H))
    cur.wait_stream(side)
    del a, b
    for i, U in enumerate(outs[1:], 1):
        assert torch.equal(U.view(torch.int32), outs[0].view(torch.int32)), f'call {i} differs'


@pytest.mark.parametrize('C', [768, 1544, 4096, 14336])
def test_accuracy_against_fp64(C):
    """Per column, the relative 2-norm error against the fp64 Cholesky inverse of the same fp32 H
    is at most 16x cuSOLVER-fp32's error on that column, plus 2^-20.  3xTF32 carries its operands
    to about 2^-22 where fp32 rounds at 2^-24.  On an H100 80GB HBM3 (700 W limit), over three
    Hessians at each of these C, the median per-column ratio was 4.4-7 and the worst column needed
    a factor of 7.9-12.4 (the maximum error over all columns: 4.1-6.9x cuSOLVER's)."""
    H = _hessian(C, C + 1)
    U, info = ops.chol_inv_upper(H, return_info=True)
    assert int(info.item()) == 0
    Uc = ops.chol_inv_upper(H, backend='cusolver')
    Hd = H.double()
    Ud = torch.linalg.cholesky(torch.cholesky_inverse(torch.linalg.cholesky(Hd)), upper=True)
    del Hd
    norm = Ud.norm(dim=0)
    err = (U.double() - Ud).norm(dim=0) / norm
    err_c = (Uc.double() - Ud).norm(dim=0) / norm
    ratio = err / err_c
    bound = err / (16 * err_c + 2.0 ** -20)
    j = int(ratio.argmax())
    print(f'C={C}: worst err/err_cusolver {ratio[j].item():.3f} at column {j} '
          f'({err[j].item():.3e} vs {err_c[j].item():.3e}); max err {err.max().item():.3e}, '
          f'cuSOLVER {err_c.max().item():.3e}; worst err/bound {bound.max().item():.3f}')
    assert bool((bound <= 1).all()), (C, int(bound.argmax()), bound.max().item())
