"""CPU: the guarantees of the exact Cholesky-inverse oracle (oracle/chol_oracle.py) that
tests/test_gpu_chol_paths.py relies on: Y = L^-1 exactly, the exactness bounds, full block and
rank-128-piece coverage, the expected output satisfying U H U^T = I exactly, and the position of
the first non-positive pivot of G = L D L^T."""
import pytest
import torch

from oracle import chol_oracle as co

# the C of the GPU path table but 4096 and 14336, which the GPU test checks the same way
SIZES = [8, 120, 128, 136, 504, 512, 520, 640, 648, 1024, 1032, 1096, 1160, 1544, 2056, 4104]


def test_factors_are_strictly_lower_and_square_to_zero():
    C = 520
    for rows, cols, signs in co.nilpotent_factors(C):
        N = torch.zeros(C, C, dtype=torch.float64)
        N[rows, cols] = signs.double()
        assert bool((rows > cols).all())
        assert set(signs.tolist()) <= {-1, 1}
        assert torch.equal(N @ N, torch.zeros_like(N))
        assert len(set((rows * C + cols).tolist())) == len(rows)


def test_generator_is_deterministic():
    a = co.unit_lower_pair(648)
    b = co.unit_lower_pair(648)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(co.unit_lower_pair(648, seed=1)[0], a[0])


def test_identity_case():
    L, Y = co.unit_lower_pair(8, factors=0)
    H, U = co.chol_case(L, Y)
    assert torch.equal(H, torch.eye(8)) and torch.equal(U, torch.eye(8))


@pytest.mark.parametrize('C', SIZES)
def test_oracle_is_exact_and_covers_every_piece(C):
    L, Y = co.unit_lower_pair(C)
    stats = co.exactness_bounds(L, Y)
    cov = co.coverage(L, Y)
    print(C, stats, cov)
    for what, (got, total) in cov.items():
        assert got == total, (what, got, total)
    H, U = co.chol_case(L, Y)
    # H and U hold integers exactly in fp32; U is upper triangular with a unit diagonal
    assert torch.equal(H.double(), co.reverse(L @ L.t()))
    assert torch.equal(H, H.t())
    assert torch.equal(U, torch.triu(U)) and torch.equal(torch.diagonal(U), torch.ones(C))
    assert torch.equal(U.double(), co.reverse(Y))
    # the definition the kernel computes: U^T U = H^-1, i.e. U H U^T = I (integers: exact in fp64)
    Ud = U.double()
    assert torch.equal(Ud @ H.double() @ Ud.t(), torch.eye(C, dtype=torch.float64))


@pytest.mark.parametrize('C', [136, 648])
def test_first_nonpositive_pivot_of_ldl(C):
    """G = L D L^T with d_k in {0, -1}: the first k pivots are 1 and pivot k is d_k, so a Cholesky
    of G stops at leading minor k + 1."""
    L, _ = co.unit_lower_pair(C)
    for k in [0, 31, 128, C - 1]:
        for dk in [0.0, -1.0]:
            d = torch.ones(C, dtype=torch.float64)
            d[k] = dk
            H, U = co.chol_case(L, None, d)
            assert U is None
            G = co.reverse(H.double())
            assert int(torch.linalg.cholesky_ex(G).info) == k + 1, (k, dk)
