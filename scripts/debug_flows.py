"""Debug: per-layer comparison of the hook schedule vs the progressive schedule on tiny-llama
(LLMC_B200_SIMT_TRAILING=1 forces the fp32 CUDA-core trailing update), then the blocked Cholesky
against chol_inv_upper(backend='cusolver')."""
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from test_gpu_framework import GPTQ_CFG, _run_gptq  # noqa: E402
from llmc_b200 import gptq_ops as ops  # noqa: E402

print('SIMT', os.environ.get('LLMC_B200_SIMT_TRAILING'))
m1, a1 = _run_gptq(False)
m2, a2 = _run_gptq(True)
for bi, (b1, b2) in enumerate(zip(m1.get_blocks(), m2.get_blocks())):
    l1, l2 = m1.get_block_linears(b1), m2.get_block_linears(b2)
    for n in l1:
        w1 = l1[n].w_qdq(l1[n]).float()
        w2 = l2[n].w_qdq(l2[n]).float()
        frac = (w1 != w2).float().mean().item()
        k = f'{bi}.{n}'
        print(f'{k:24s} frac_diff={frac:.4f} loss_hook={a1.layer_loss(k):.6g} loss_prog={a2.layer_loss(k):.6g} '
              f'scale_rel={((l1[n].buf_scales - l2[n].buf_scales).abs().max() / l1[n].buf_scales.abs().max()).item():.3g}')

# conditioning / determinism probe on a down_proj-like Hessian
torch.manual_seed(0)
C = 512
X = torch.randn(1024, C, device='cuda') * torch.exp(torch.randn(C, device='cuda') * 1.5)
H = (2.0 / 1024) * X.t() @ X
H += 0.01 * torch.diag(H).mean() * torch.eye(C, device='cuda')
U1 = ops.chol_inv_upper(H, backend='b200')
U2 = ops.chol_inv_upper(H, backend='b200')
Uc = ops.chol_inv_upper(H, backend='cusolver')
Hp = H * (1 + 1e-7 * torch.randn_like(H))
Hp = (Hp + Hp.t()) / 2
Ucp = ops.chol_inv_upper(Hp, backend='cusolver')
U1p = ops.chol_inv_upper(Hp, backend='b200')
print('b200 deterministic:', torch.equal(U1, U2))
print('b200 vs cusolver rel:', ((U1 - Uc).abs().max() / Uc.abs().max()).item())
print('cusolver sensitivity to 1e-7 perturbation:', ((Ucp - Uc).abs().max() / Uc.abs().max()).item())
print('b200 sensitivity to 1e-7 perturbation:', ((U1p - U1).abs().max() / U1.abs().max()).item())
print('cond(H) ~', (torch.linalg.eigvalsh(H.double()).max() / torch.linalg.eigvalsh(H.double()).min()).item())
