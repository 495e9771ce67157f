"""GPU: the 3xTF32 tensor-core GEMM block and the blocked Cholesky-inverse built on it.
Floating point, tolerances stated: fp32-level for the GEMM (3xTF32 drops ~2^-22), 1e-3
relative on Hinv_U (north_star) — measured far tighter."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def _split(x):
    from llmc_b200._lib import call, ptr, stream_ptr
    hi, lo = torch.empty_like(x), torch.empty_like(x)
    call('llmc_split_tf32', ptr(x), x.shape[0], x.shape[1], x.shape[1], ptr(hi), ptr(lo),
         stream_ptr(x.device))
    return hi, lo


def _gemm(a, a_mn, b, b_mn, c, M, N, K, mode, lower=0):
    from llmc_b200._lib import call, ptr, stream_ptr
    ah, al = _split(a)
    bh, bl = _split(b)
    call('llmc_gemm_f32x3', ptr(ah), ptr(al), a_mn, a.shape[1], ptr(bh), ptr(bl), b_mn, b.shape[1],
         ptr(c), c.shape[1], M, N, K, mode, lower, stream_ptr(c.device))


@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize('M,N,K', [(128, 256, 32), (384, 512, 128), (1000, 776, 128), (4096, 2048, 64)])
def test_f32x3_all_layouts(a_mn, b_mn, M, N, K):
    torch.manual_seed(M + N + K + a_mn * 2 + b_mn)
    A = torch.randn(M, K, device='cuda')
    B = torch.randn(N, K, device='cuda')
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    C0 = torch.randn(M, N, device='cuda')
    ref = A.double() @ B.double().t()
    c = C0.clone()
    _gemm(a, a_mn, b, b_mn, c, M, N, K, mode=1)
    err = (c.double() - ref).abs().max().item()
    assert err <= 2e-6 * K ** 0.5 * ref.abs().max().item() + 1e-6, err
    c = C0.clone()
    _gemm(a, a_mn, b, b_mn, c, M, N, K, mode=0)
    err = (c.double() - (C0.double() - ref)).abs().max().item()
    assert err <= 2e-6 * K ** 0.5 * ref.abs().max().item() + 1e-6, err


def test_f32x3_exact_on_integers_and_lower_only():
    M = N = 512
    K = 128
    A = torch.randint(-8, 9, (M, K), device='cuda').float()
    C0 = torch.zeros(M, N, device='cuda')
    c = C0.clone()
    _gemm(A, 0, A, 0, c, M, N, K, mode=0, lower=1)
    ref = -(A @ A.t())
    low = torch.tril(torch.ones(M, N, device='cuda', dtype=torch.bool))
    assert torch.equal(c[low], ref[low]), 'lower triangle must be exact on small integers'


@pytest.mark.parametrize('C', [128, 256, 512, 1024, 4096, 1096])
def test_chol_inv_upper_matches_cusolver_and_definition(C):
    from llmc_b200 import gptq_ops as ops
    torch.manual_seed(C)
    T = 4 * C
    X = (torch.randn(T, C, device='cuda') * torch.exp(torch.randn(C, device='cuda') * 0.7))
    H = (2.0 / T) * (X.t() @ X)
    H += 0.01 * torch.diag(H).mean() * torch.eye(C, device='cuda')     # percdamp like gptq.py:169
    U, info = ops.chol_inv_upper(H, return_info=True)
    assert int(info.item()) == 0
    assert torch.equal(U, torch.triu(U)) and (torch.diagonal(U) > 0).all()
    Uref = ops.chol_inv_upper(H, backend='cusolver')
    rel = ((U - Uref).abs().max() / Uref.abs().max()).item()
    assert rel < 1e-3, rel
    # definition: U^T U == H^-1  <=>  U H U^T == I, checked in fp64
    Ud, Hd = U.double(), H.double()
    I = Ud @ Hd @ Ud.t()
    resid = (I - torch.eye(C, device='cuda', dtype=torch.float64)).abs().max().item()
    Ir = Uref.double() @ Hd @ Uref.double().t()
    resid_ref = (Ir - torch.eye(C, device='cuda', dtype=torch.float64)).abs().max().item()
    assert resid < max(5 * resid_ref, 1e-3), (resid, resid_ref)


def test_chol_reports_non_spd():
    from llmc_b200 import gptq_ops as ops
    H = torch.eye(256, device='cuda')
    H[100, 100] = -1.0
    _, info = ops.chol_inv_upper(H, return_info=True)
    # the factorisation runs on the index-reversed matrix (DESIGN.md K4): minor 256 - 100 fails first
    assert int(info.item()) == 156


def test_gptq_raises_on_non_spd_hessian():
    """ADVICE r1: the reference raises from torch.linalg.cholesky (gptq.py:172); the GPU path must
    not sweep NaNs into layer.weight silently."""
    import pytest as _pt
    from llmc_b200.blockwise import AttrDict
    from llmc_b200.gptq import GPTQ
    from llmc_b200.synth import SynthModel
    cfg = AttrDict.wrap({'quant': {'method': 'GPTQ', 'quant_out': True,
                                   'weight': {'bit': 4, 'symmetric': False, 'granularity': 'per_group',
                                              'group_size': 128},
                                   'special': {'actorder': True, 'static_groups': False, 'percdamp': 0.01,
                                               'blocksize': 128, 'true_sequential': True}}})
    model = SynthModel('tiny-llama', n_layers=1, device='cuda')
    inp = model.first_block_input(4, 64, bs=1, device='cuda')
    algo = GPTQ(model, cfg.quant, inp, None, cfg)
    algo.percdamp = -10.0                    # H - 10*mean(diag)*I is indefinite
    with _pt.raises(torch.linalg.LinAlgError):
        algo.run_block_loop()
