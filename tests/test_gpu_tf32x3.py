"""GPU: properties of the 3xTF32 update (llmc_gemm_f32x3) that the look-ahead schedules and the
epilogue paths rely on.

* A tile's value does not depend on how the call is cut: one call over N columns (or M rows) is
  bitwise equal to two calls that split the range at a multiple of 128.
* K that is not a multiple of the 32-deep ring stage (the last stage is partly zero-filled).
* M, N not multiples of 128 and an odd ldc: the ragged and misaligned store paths, which must not
  touch C outside [M, N].
Accuracy bound as in test_gpu_chol.py: fp32 level, 3xTF32 drops ~2^-22 relative per product."""
import pytest
import torch

pytestmark = pytest.mark.gpu

LAYOUTS = [(0, 0), (0, 1), (1, 0), (1, 1)]


def _split(x):
    from llmc_b200._lib import call, ptr, stream_ptr
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    call('llmc_split_tf32', ptr(x), x.shape[0], x.shape[1], x.shape[1], ptr(hi), ptr(lo),
         stream_ptr(x.device))
    return hi, lo


def _held(X, mn):
    """X [rows, K] split, K-major (ld K) or MN-major (ld rows rounded up to 4, TMA's 16 bytes)"""
    if not mn:
        return _split(X), X.shape[1]
    ld = (X.shape[0] + 3) // 4 * 4
    buf = torch.zeros(X.shape[1], ld, device=X.device)
    buf[:, :X.shape[0]] = X.t()
    return _split(buf), ld


class Operands:
    """A [M, K] and B [N, K] held split, in the requested layouts."""

    def __init__(self, M, N, K, a_mn, b_mn, seed):
        g = torch.Generator(device='cuda').manual_seed(seed)
        self.A = torch.randn(M, K, device='cuda', generator=g)
        self.B = torch.randn(N, K, device='cuda', generator=g)
        self.a_mn, self.b_mn, self.K = a_mn, b_mn, K
        self.a, self.lda = _held(self.A, a_mn)
        self.b, self.ldb = _held(self.B, b_mn)

    def a_at(self, m0):
        """(hi, lo) pointers of the operand starting at row m0 of A"""
        off = m0 if self.a_mn else m0 * self.lda
        return [t.view(-1)[off:] for t in self.a]

    def b_at(self, n0):
        off = n0 if self.b_mn else n0 * self.ldb
        return [t.view(-1)[off:] for t in self.b]

    def gemm(self, c_flat, ldc, m0, m1, n0, n1, mode):
        """C[m0:m1, n0:n1] of the matrix stored in c_flat with row stride ldc"""
        from llmc_b200._lib import call, ptr, stream_ptr
        ah, al = self.a_at(m0)
        bh, bl = self.b_at(n0)
        call('llmc_gemm_f32x3', ptr(ah), ptr(al), self.a_mn, self.lda, ptr(bh), ptr(bl), self.b_mn,
             self.ldb, ptr(c_flat[m0 * ldc + n0:]), ldc, m1 - m0, n1 - n0, self.K, mode, 0,
             stream_ptr(c_flat.device))


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('a_mn,b_mn', LAYOUTS)
def test_f32x3_cut_calls_bitwise_equal(a_mn, b_mn, mode):
    M, N, K = 640, 776, 96
    ops = Operands(M, N, K, a_mn, b_mn, seed=7 + 2 * a_mn + b_mn)
    C0 = torch.randn(M * N, device='cuda')
    whole = C0.clone()
    ops.gemm(whole, N, 0, M, 0, N, mode)
    cut_n = C0.clone()
    ops.gemm(cut_n, N, 0, M, 0, 384, mode)
    ops.gemm(cut_n, N, 0, M, 384, N, mode)
    cut_m = C0.clone()
    ops.gemm(cut_m, N, 0, 256, 0, N, mode)
    ops.gemm(cut_m, N, 256, M, 0, N, mode)
    assert torch.equal(whole, cut_n)
    assert torch.equal(whole, cut_m)


def _check(ops, c, C0, M, N, ldc, mode):
    """c: the flat result buffer with row stride ldc; C0 its contents before the call"""
    ref = ops.A.double() @ ops.B.double().t()
    want = ref if mode == 1 else C0.view(M, ldc)[:, :N].double() - ref
    got = c.view(M, ldc)[:, :N].double()
    err = (got - want).abs().max().item()
    assert err <= 2e-6 * ops.K ** 0.5 * ref.abs().max().item() + 1e-6, err
    # the columns between N and ldc are padding nobody may write
    assert torch.equal(c.view(M, ldc)[:, N:], C0.view(M, ldc)[:, N:])


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('a_mn,b_mn', LAYOUTS)
@pytest.mark.parametrize('K', [8, 40, 136])
def test_f32x3_partial_last_stage(K, a_mn, b_mn, mode):
    M, N = 256, 384
    ops = Operands(M, N, K, a_mn, b_mn, seed=K + 2 * a_mn + b_mn)
    C0 = torch.randn(M * N, device='cuda')
    c = C0.clone()
    ops.gemm(c, N, 0, M, 0, N, mode)
    _check(ops, c, C0, M, N, N, mode)


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('a_mn,b_mn', LAYOUTS)
def test_f32x3_ragged_tiles_odd_ldc(a_mn, b_mn, mode):
    M, N, K, ldc = 300, 203, 64, 211
    ops = Operands(M, N, K, a_mn, b_mn, seed=11 + 2 * a_mn + b_mn)
    C0 = torch.randn(M * ldc, device='cuda')
    c = C0.clone()
    ops.gemm(c, ldc, 0, M, 0, N, mode)
    _check(ops, c, C0, M, N, ldc, mode)
