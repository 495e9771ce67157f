"""GPU: the two kernels behind llmc_gemm_f32x3 give the same bits.

K-major x K-major operands run on the warpgroup kernel (wgmma m64n128k8 tf32); a call with either
operand MN-major runs on the warp-level mma.sync m16n8k8 kernel.  Both issue hi*hi, lo*hi, hi*lo
per k8 step, k ascending, into one zeroed fp32 accumulator, and round C - acc once, so the same
operands held in any of the four layouts must give bit-identical C.  Covered: ragged M and N, K
not a multiple of the 32-deep ring stage, an odd ldc, lower-triangle tiles, modes 0 and 1, and a
C larger than one wave of tiles (the persistent loop)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(x):
    from llmc_b200._lib import call, ptr, stream_ptr
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    call('llmc_split_tf32', ptr(x), x.shape[0], x.shape[1], x.shape[1], ptr(hi), ptr(lo),
         stream_ptr(x.device))
    return hi, lo


def _held(X, mn):
    """X [rows, K] split, K-major (ld K) or MN-major (ld rows rounded up to 4)"""
    if not mn:
        return _split(X), X.shape[1]
    ld = (X.shape[0] + 3) // 4 * 4
    buf = torch.zeros(X.shape[1], ld, device=X.device)
    buf[:, :X.shape[0]] = X.t()
    return _split(buf), ld


def _gemm(A, B, C0, ldc, a_mn, b_mn, mode, lower):
    from llmc_b200._lib import call, ptr, stream_ptr
    (ah, al), lda = _held(A, a_mn)
    (bh, bl), ldb = _held(B, b_mn)
    c = C0.clone()
    call('llmc_gemm_f32x3', ptr(ah), ptr(al), a_mn, lda, ptr(bh), ptr(bl), b_mn, ldb, ptr(c), ldc,
         A.shape[0], B.shape[0], A.shape[1], mode, lower, stream_ptr(c.device))
    return c


@pytest.mark.parametrize('lower', [0, 1])
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('M,N,K,ldc', [
    (256, 384, 128, 384),      # whole tiles, whole stages
    (300, 203, 40, 211),       # ragged tiles, a partial last stage, odd ldc (unfolded epilogue)
    (1000, 776, 136, 776),     # ragged M, K % 32 == 8
    (2048, 2048, 512, 2048),   # 256 tiles: more than one per CTA
])
def test_wgmma_matches_mma_sync(M, N, K, ldc, mode, lower):
    g = torch.Generator(device='cuda').manual_seed(M + N + K + 2 * mode + lower)
    # wide exponent range: the sums see cancellation and every rounding case
    A = torch.randn(M, K, device='cuda', generator=g) * torch.exp(torch.randn(M, 1, device='cuda', generator=g))
    B = torch.randn(N, K, device='cuda', generator=g) * torch.exp(torch.randn(1, K, device='cuda', generator=g))
    C0 = torch.randn(M * ldc, device='cuda', generator=g)
    ref = _gemm(A, B, C0, ldc, 0, 0, mode, lower)
    assert not torch.equal(ref, C0)
    for a_mn, b_mn in [(0, 1), (1, 0), (1, 1)]:
        got = _gemm(A, B, C0, ldc, a_mn, b_mn, mode, lower)
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), (a_mn, b_mn)
