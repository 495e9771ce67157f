"""GPU: the blocked Cholesky inverse, built on the 3xTF32 update (tested in test_gpu_tf32x3.py).
Floating point, tolerance stated: 1e-3 relative on Hinv_U (north_star) — measured far tighter."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


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
