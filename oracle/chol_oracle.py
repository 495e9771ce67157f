"""Exact integer oracle for the blocked Cholesky inverse (`llmc_chol_inv_upper`, DESIGN.md §K4).

The kernel factors the index-reversed matrix G = J H J = L L^T and returns U = J L^-1 J.  Here L
is built so that L^-1 is known in closed form and every step of any blocked schedule is exact:

    L = (I + N_1)(I + N_2)(I + N_3),    Y = L^-1 = (I - N_3)(I - N_2)(I - N_1),

where each N_t is strictly lower triangular with N_t^2 = 0: the indices are split at random into
two halves A_t and B_t, and each row i in B_t gets about k entries of +-1 at random columns j < i,
j in A_t.  N_t maps into B_t and reads only A_t, so N_t N_t = 0 and (I + N_t)^-1 = I - N_t.

With H = J G J the expected output is U = J Y J: upper triangular, unit diagonal, integer.  The
kernel's arithmetic on it is exact in any order and under any cut of the updates when

* every operand the 3xTF32 updates split (L panels, Schur complements, Y, the finished T' rows) is
  an integer of magnitude <= 2048, so its tf32 hi is exact, lo = 0 and the dropped lo*lo is 0;
  bounded elementwise by max(|L||L|^T) and max(|L||Y|);
* every accumulator stays below 2^24: partial sums of the factorisation, the panel solve, the
  inverse's T' and Y rows are bounded through absolute values by |L||L|^T, 128 |L||L|^T |Y|,
  |L||Y| and |Y||L||Y|;
* every pivot is 1, so `diag_kernel`'s rsqrt + Newton step is exact (rsqrtf(1) == 1).

`exactness_bounds` and `coverage` check these premises on the inputs themselves.  With this
sampler a 128 x 128 block of L holds only tens of nonzeros, so k trades coverage against the
bounds: k = 16 takes max(|L||L|^T) past 2048 from C = 512 on, k = 8 leaves rank-128 pieces zero
at C = 4104 and k = 10 at C = 14336.  The default k = 12 keeps max(|L||L|^T) near 1250 at
C = 14336; there a seed is chosen whose pieces are all nonzero.  The matrices
are built densely in fp64 (exact: every value is an integer far below 2^53) on any device; at
C = 14336 the products belong on a GPU.
"""
import zlib

import torch

NB = 128                  # diagonal block width of the kernel
TF32_EXACT = 2048         # integers up to here have an exact tf32 hi and lo = 0
EXACT_LIMIT = 1 << 24     # integers below this are exact in fp32


def _generator(*key):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


def nilpotent_factors(C, k=12, factors=3, seed=0):
    """The index form (rows, cols, signs) of N_1 .. N_factors, int64 CPU tensors, deterministic in
    (C, k, factors, seed).  Duplicate draws of one (row, col) collapse into one entry."""
    g = _generator('chol', C, k, factors, seed)
    out = []
    for _ in range(factors):
        perm = torch.randperm(C, generator=g)
        a = perm[:C // 2].sort().values
        b = perm[C // 2:]
        below = torch.searchsorted(a, b)               # |A ∩ [0, i)| for each row i in B
        b, below = b[below > 0], below[below > 0]
        pick = (torch.rand(len(b), k, generator=g, dtype=torch.float64) * below[:, None]).long()
        pick = torch.minimum(pick, below[:, None] - 1)
        key = torch.unique(b[:, None] * C + a[pick])
        signs = torch.randint(0, 2, (len(key),), generator=g) * 2 - 1
        out.append((key // C, key % C, signs))
    return out


def unit_lower_pair(C, k=12, factors=3, seed=0, device='cpu'):
    """(L, Y) fp64 [C, C] on `device` with L unit lower triangular and Y = L^-1 exactly.
    factors = 0 gives L = Y = I."""
    Ns = [torch.sparse_coo_tensor(torch.stack([r, c]), s.double(), (C, C)).to(device)
          for r, c, s in nilpotent_factors(C, k, factors, seed)]
    L = torch.eye(C, dtype=torch.float64, device=device)
    Y = L.clone()
    for N in reversed(Ns):            # L = (I + N_1)((I + N_2)((I + N_3) I))
        L += torch.sparse.mm(N, L)
    for N in Ns:                      # Y = (I - N_3)((I - N_2)((I - N_1) I))
        Y -= torch.sparse.mm(N, Y)
    return L, Y


def reverse(X):
    """J X J: X[C-1-i][C-1-j]."""
    return X.flip(0).flip(1)


def chol_case(L, Y, d=None):
    """(H fp32, U fp32): the kernel's input H = J G J with G = L diag(d) L^T (d = None: all ones)
    and, for d = None, its exact output U = J Y J (upper triangular, unit diagonal)."""
    G = (L @ L.t()) if d is None else (L * d) @ L.t()
    H = reverse(G).float()
    U = reverse(Y).float() if d is None else None
    return H, U


def exactness_bounds(L, Y):
    """The bounds behind exactness, in fp64 (all sums of absolute values, so they hold in any
    summation order); asserts them and returns them for reporting."""
    C = L.shape[0]
    aL, aY = L.abs(), Y.abs()
    LLt = (aL @ aL.t()).max().item()
    LYm = aL @ aY
    LY = LYm.max().item()
    YLY = (aY @ LYm).max().item()
    del LYm
    eye = torch.eye(C, dtype=torch.float64, device=L.device)
    stats = dict(maxL=aL.max().item(), maxY=aY.max().item(), LLt=LLt, LY=LY, YLY=YLY,
                 solve=min(NB, C) * LLt * aY.max().item())
    assert torch.equal(torch.tril(L), L) and torch.equal(torch.diagonal(L), eye.diagonal()), 'L unit lower'
    assert torch.equal(L @ Y, eye), 'L Y != I'
    assert stats['LLt'] <= TF32_EXACT and stats['LY'] <= TF32_EXACT, stats
    assert stats['YLY'] < EXACT_LIMIT and stats['solve'] < EXACT_LIMIT, stats
    return stats


def _block_any(mask, C):
    """[C, C] bool -> [nbk, nbk] bool: any element of each 128 x 128 block."""
    nbk = -(-C // NB)
    pad = nbk * NB - C
    m = torch.nn.functional.pad(mask, (0, pad, 0, pad))
    return m.reshape(nbk, NB, nbk, NB).any(3).any(1)


def coverage(L, Y):
    """Counts (nonzero, total) of the lower 128-block pairs (i >= j) of L and of Y, and of the
    rank-128 trailing pieces L[i-blk, k-blk] L[j-blk, k-blk]^T with i >= j > k: dropping any
    nonzero piece changes G's Schur complement and with it L and U."""
    C = L.shape[0]
    nbk = -(-C // NB)
    low = torch.tril(torch.ones(nbk, nbk, dtype=torch.bool, device=L.device))
    bl, by = _block_any(L != 0, C), _block_any(Y != 0, C)
    total = int(low.sum())
    out = dict(L=(int((bl & low).sum()), total), Y=(int((by & low).sum()), total))
    got = want = 0
    for kb in range(nbk - 1):
        r0 = (kb + 1) * NB
        Lk = L[r0:, kb * NB:r0]
        nz = _block_any((Lk @ Lk.t()) != 0, C - r0)
        lk = torch.tril(torch.ones_like(nz))
        got += int((nz & lk).sum())
        want += int(lk.sum())
    out['pieces'] = (got, want)
    return out
