"""GPU: the 3xTF32 update (llmc_gemm_f32x3), the fp32-accurate tensor-core GEMM behind the
Cholesky inverse and the GPTQ / SpQR column sweeps.

* Accuracy: fp32 level against an fp64 product (3xTF32 drops ~2^-22 relative per product), and
  exact on small integers, lower-triangle tiles included.
* A tile's value does not depend on how the call is cut: one call over N columns (or M rows) is
  bitwise equal to two calls that split the range at a multiple of 128.
* K that is not a multiple of the 32-deep ring stage (the last stage is partly zero-filled).
* M, N not multiples of 128 and an odd ldc: the ragged and misaligned store paths, which must not
  touch C outside [M, N].
* The bits themselves: per k8 step, k ascending, hi*hi, lo*hi, hi*lo into one zeroed fp32
  accumulator, then one rounding of C - acc.  Seeded inputs that are exact in fp32 go through the
  update and the SHA-256 of the whole C buffer is pinned, for ragged tiles, partial stages, an odd
  ldc, lower-triangle tiles and more tiles than CTAs."""
import hashlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(x):
    from llmc_b200._lib import call, ptr, stream_ptr
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    call('llmc_split_tf32', ptr(x), x.shape[0], x.shape[1], x.shape[1], ptr(hi), ptr(lo),
         stream_ptr(x.device))
    return hi, lo


class Operands:
    """A [M, K] and B [N, K] held split, K-major (ld K)."""

    def __init__(self, A, B):
        self.A, self.B, self.K = A, B, A.shape[1]
        self.a, self.b = _split(A), _split(B)

    @classmethod
    def randn(cls, M, N, K, seed):
        g = torch.Generator(device='cuda').manual_seed(seed)
        A = torch.randn(M, K, device='cuda', generator=g)
        return cls(A, torch.randn(N, K, device='cuda', generator=g))

    def gemm(self, c_flat, ldc, m0, m1, n0, n1, mode, lower=0):
        """C[m0:m1, n0:n1] of the matrix stored in c_flat with row stride ldc"""
        from llmc_b200._lib import call, ptr, stream_ptr
        ah, al = (t[m0:] for t in self.a)
        bh, bl = (t[n0:] for t in self.b)
        call('llmc_gemm_f32x3', ptr(ah), ptr(al), self.K, ptr(bh), ptr(bl), self.K,
             ptr(c_flat[m0 * ldc + n0:]), ldc, m1 - m0, n1 - n0, self.K, mode, lower,
             stream_ptr(c_flat.device))


def _check(ops, c, C0, M, N, ldc, mode):
    """c: the flat result buffer with row stride ldc; C0 its contents before the call"""
    ref = ops.A.double() @ ops.B.double().t()
    want = ref if mode == 1 else C0.view(M, ldc)[:, :N].double() - ref
    got = c.view(M, ldc)[:, :N].double()
    err = (got - want).abs().max().item()
    assert err <= 2e-6 * ops.K ** 0.5 * ref.abs().max().item() + 1e-6, err
    # the columns between N and ldc are padding nobody may write
    assert torch.equal(c.view(M, ldc)[:, N:], C0.view(M, ldc)[:, N:])


@pytest.mark.parametrize('M,N,K', [(128, 256, 32), (384, 512, 128), (1000, 776, 128), (4096, 2048, 64)])
def test_f32x3_accuracy(M, N, K):
    torch.manual_seed(M + N + K)
    ops = Operands(torch.randn(M, K, device='cuda'), torch.randn(N, K, device='cuda'))
    C0 = torch.randn(M * N, device='cuda')
    for mode in (1, 0):
        c = C0.clone()
        ops.gemm(c, N, 0, M, 0, N, mode)
        _check(ops, c, C0, M, N, N, mode)


def test_f32x3_exact_on_integers_and_lower_only():
    M = N = 512
    K = 128
    A = torch.randint(-8, 9, (M, K), device='cuda').float()
    c = torch.zeros(M * N, device='cuda')
    Operands(A, A).gemm(c, N, 0, M, 0, N, mode=0, lower=1)
    ref = -(A @ A.t())
    low = torch.tril(torch.ones(M, N, device='cuda', dtype=torch.bool))
    assert torch.equal(c.view(M, N)[low], ref[low]), 'lower triangle must be exact on small integers'


@pytest.mark.parametrize('mode', [0, 1])
def test_f32x3_cut_calls_bitwise_equal(mode):
    M, N, K = 640, 776, 96
    ops = Operands.randn(M, N, K, seed=7)
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


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('K', [8, 40, 136])
def test_f32x3_partial_last_stage(K, mode):
    M, N = 256, 384
    ops = Operands.randn(M, N, K, seed=K)
    C0 = torch.randn(M * N, device='cuda')
    c = C0.clone()
    ops.gemm(c, N, 0, M, 0, N, mode)
    _check(ops, c, C0, M, N, N, mode)


@pytest.mark.parametrize('mode', [0, 1])
def test_f32x3_ragged_tiles_odd_ldc(mode):
    M, N, K, ldc = 300, 203, 64, 211
    ops = Operands.randn(M, N, K, seed=11)
    C0 = torch.randn(M * ldc, device='cuda')
    c = C0.clone()
    ops.gemm(c, ldc, 0, M, 0, N, mode)
    _check(ops, c, C0, M, N, ldc, mode)


def pinned_inputs(M, N, K, ldc, mode, lower):
    """A [M, K], B [N, K] and the flat C [M * ldc] of one pinned case, as fp32 numpy arrays.

    Every value is a 24-bit integer times a power of two, so it is exact in fp32 and the inputs
    do not depend on any library's float conversions.  A's rows and B's k columns get scales
    2^-6 .. 2^6 and C's elements 2^-4 .. 2^8: the sums cancel, and the tf32 split, the three
    products and the final rounding all see every rounding case."""
    rng = np.random.Generator(np.random.PCG64(M + N + K + 2 * mode + lower))

    def exact(shape, exp):
        mant = rng.integers(-(1 << 24) + 1, 1 << 24, size=shape)
        return np.ldexp(mant.astype(np.float64), exp - 24).astype(np.float32)

    A = exact((M, K), rng.integers(-6, 7, size=(M, 1)))
    B = exact((N, K), rng.integers(-6, 7, size=(1, K)))
    C = exact((M * ldc,), rng.integers(-4, 9, size=M * ldc))
    return A, B, C


# sha256 of C's bytes (all M * ldc floats) after llmc_gemm_f32x3 on pinned_inputs, keyed by
# (M, N, K, ldc, mode, lower_only).  Taken on an H100 80GB HBM3 (700 W), where the warp-level
# m16n8k8 kernel that preceded the wgmma one gave the same bits for the same inputs.
PINNED = {
    (256, 384, 128, 384, 0, 0): 'fcda184b6d20549c3bad81f42c9c847b1fe5043397853aefa6df48e6d17240e2',
    (256, 384, 128, 384, 0, 1): 'ba19c1dd9f57633370c846ed6aa5dafec5b20eed5d5ba4baf9ae8f48357c28d6',
    (256, 384, 128, 384, 1, 0): 'fd875b894ee52f01e21b5c530baa8467faaa0585e3b3184c90dab8df6baa59ed',
    (256, 384, 128, 384, 1, 1): 'ed14c381b86e8fdbf67315fec60d15316b392d783f209f06bc4c879d12ca13c8',
    (300, 203, 40, 211, 0, 0): '88424d72ae7c70bfc5e5427501a230bab22746af309db72d99ae03162a015bb1',
    (300, 203, 40, 211, 0, 1): '6190e2b7adc681a3d6466213981a7a50f5130ced7ead60f8734455f384ddf823',
    (300, 203, 40, 211, 1, 0): '1cb73b265819dca4bcb657abe6a84c998f9649af260a8657df23a85971516684',
    (300, 203, 40, 211, 1, 1): '9dc05a8a43a12b10c5d9e6bf880fe11a2ee5d34e8149c142cbe9c2942b3a5c7c',
    (1000, 776, 136, 776, 0, 0): 'f8a2a0877ba8ed6fb6fc4497841e97d18d46fd3e36f9dcd7b614f8d1e63ee0bd',
    (1000, 776, 136, 776, 0, 1): '2ca7f4b824891d0513eb7ee0007a3bb6cc1fe356a415b8c58814414db555f8ab',
    (1000, 776, 136, 776, 1, 0): '136e00d769abdc0a2b3982b33c41debd7392ed28a96c8e252ea792b8bd3dfb6c',
    (1000, 776, 136, 776, 1, 1): '3c52c809ef7f70574fd129b04898f9fab2cf2d07207e1d21837c0283862c93cc',
    (2048, 2048, 512, 2048, 0, 0): '3dfcb9e2daf26f7f0da70d2c4a89530e18faee5e543907b6742e9461f1ddb7b7',
    (2048, 2048, 512, 2048, 0, 1): '8b13402fdd543dcc6805f5dcbd5994c84b37acf1e6d6d215b8cb3122df5302cd',
    (2048, 2048, 512, 2048, 1, 0): '206312ad65ae1ca4de113092d02bbb3b083982fde30cb042a59f4f298f3d88ec',
    (2048, 2048, 512, 2048, 1, 1): '1c2cf41c375afa42eadeb1dc14a4b868867f6f651051d6e469f7801e0a40144a',
}


@pytest.mark.parametrize('lower', [0, 1])
@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('M,N,K,ldc', [
    (256, 384, 128, 384),      # whole tiles, whole stages
    (300, 203, 40, 211),       # ragged tiles, a partial last stage, odd ldc (unfolded epilogue)
    (1000, 776, 136, 776),     # ragged M, K % 32 == 8
    (2048, 2048, 512, 2048),   # 256 tiles: more than one per CTA
])
def test_f32x3_bits_pinned(M, N, K, ldc, mode, lower):
    A, B, C0 = pinned_inputs(M, N, K, ldc, mode, lower)
    ops = Operands(torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda())
    c = torch.from_numpy(C0).cuda()
    ops.gemm(c, ldc, 0, M, 0, N, mode, lower)
    got = c.cpu().numpy()
    assert not np.array_equal(got, C0)
    assert hashlib.sha256(got.tobytes()).hexdigest() == PINNED[(M, N, K, ldc, mode, lower)]
