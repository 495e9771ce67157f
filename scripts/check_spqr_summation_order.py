"""How far the SpQR end-to-end run (tests/test_gpu_e2e.py::test_spqr_pipeline_matches_reference)
lands from the reference when only floating-point summation orders change.

The same inputs (tests/golden/e2e_spqr_llama.pt) go through the pipeline four ways:
  wgmma          the library as shipped (wgmma GEMM / SYRK, wgmma 3xTF32 trailing update)
  wgmma+simt     the same, trailing update on the fp32 CUDA-core kernel (LLMC_B200_SIMT_TRAILING=1)
  cublas         forwards through torch F.linear (cuBLAS), Hessians as torch fp32 X^T X
  cublas+simt    both substitutions
and each layer's Losses.sum() deviation from the reference is printed next to the reference's own
eager-vs-sdpa self-divergence.  If the cuBLAS runs land as far away as the shipped one, the spread
comes from summation order, not from the library's kernels.

    python scripts/check_spqr_summation_order.py      (one GPU; JSON on stdout)
"""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from llmc_b200 import gptq_ops, module_utils, synth  # noqa: E402
from llmc_b200.spqr import SpQR  # noqa: E402
from test_gpu_e2e import _load, _run  # noqa: E402


def torch_linear(x, weight, bias=None):
    return F.linear(x, weight, bias)


@torch.no_grad()
def torch_hessian_add_batch(H, nsamples, inp):
    """gptq.py:283-290 as the reference writes it (fp32 GEMM on X.float())."""
    if inp.dim() == 2:
        inp = inp.unsqueeze(0)
    b = inp.shape[0]
    x = inp.reshape(-1, inp.shape[-1]).t().float()
    H *= nsamples / (nsamples + b)
    x = (2.0 / (nsamples + b)) ** 0.5 * x
    H += x.matmul(x.t())
    return nsamples + b


def run(variant):
    """One variant in this process (the trailing-update switch is read once per process)."""
    d, init = _load(os.path.join(ROOT, 'tests', 'golden'), 'spqr_llama')
    if variant.startswith('cublas'):
        module_utils.linear_forward = synth.linear_forward = torch_linear
        gptq_ops.hessian_add_batch = torch_hessian_add_batch
    _, algo = _run(d, init, SpQR)
    return {k: abs(algo.layer_loss(k) - v) / v for k, v in d['losses'].items()}


def main():
    if len(sys.argv) > 1:                       # worker: one variant, JSON on stdout
        print(json.dumps(run(sys.argv[1])))
        return
    d, _ = _load(os.path.join(ROOT, 'tests', 'golden'), 'spqr_llama')
    self_dev = d['self_divergence']['loss_rel_dev']
    out = {'gpu': torch.cuda.get_device_name(), 'reference_self_divergence': self_dev,
           'reference_self_divergence_max': max(self_dev.values())}
    for v in ('wgmma', 'wgmma+simt', 'cublas', 'cublas+simt'):
        env = dict(os.environ)
        env.pop('LLMC_B200_SIMT_TRAILING', None)
        if v.endswith('simt'):
            env['LLMC_B200_SIMT_TRAILING'] = '1'
        res = subprocess.run([sys.executable, os.path.abspath(__file__), v], env=env, check=True,
                             stdout=subprocess.PIPE, text=True)
        dev = json.loads(res.stdout.strip().splitlines()[-1])
        worst = max(dev, key=dev.get)
        out[v] = {'loss_rel_dev': dev, 'max': dev[worst], 'max_layer': worst}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
