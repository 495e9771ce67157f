"""Generate tests/golden/e2e_gptq_block1.npz by running the REFERENCE's GPTQ pipeline on CPU (the
gptq_llama case of gen_e2e_golden.py, same initial weights and calibration ids) and recording what
block 1 of the tiny Llama received and produced:

  * x1     — block 0's quant_out output, i.e. the calibration input of block 1 ([16, 128, 256]
             bf16, stored as its uint16 bit pattern, compressed);
  * losses — Losses.sum() of block 1's seven linears in the same run.

Block 1's input is computed by bf16 CPU kernels whose results depend on the CPU and its thread
count, and GPTQ amplifies such roundings; pinning block 1 to the reference's own input keeps the
comparison of tests/test_oracle_golden.py at its 2e-3 bar on any host.  Build container only
(needs the reference checkout):

    python oracle/gen_block1_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..'))
from oracle import gen_e2e_golden as ge  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(HERE, '..', 'tests', 'golden', 'e2e_gptq_block1.npz')


def main():
    rh.setup()
    from llmc.compression.quantization.gptq import GPTQ
    gold = torch.load(os.path.join(ge.OUT, 'e2e_gptq_llama.pt'), weights_only=False)
    rec = {}
    orig_bo, orig_lt, orig_wt = GPTQ.block_opt, GPTQ.layer_transform, GPTQ.weight_transform

    def bo(self, block, *a, **k):
        if self.block_idx == 1:
            rec['x1'] = torch.cat([t.detach().clone() for t in self.input['data']], dim=0)
        return orig_bo(self, block, *a, **k)

    def lt(self, layer, name):
        rec['cur'] = f'{self.block_idx}.{name}'
        return orig_lt(self, layer, name)

    def wt(self, W, Hinv, Losses, tmp):
        r = orig_wt(self, W, Hinv, Losses, tmp)
        rec.setdefault('losses', {})[rec['cur']] = float(Losses.sum().item())
        return r
    GPTQ.block_opt, GPTQ.layer_transform, GPTQ.weight_transform = bo, lt, wt
    try:
        from transformers import LlamaConfig
        model = rh.shape_llama(LlamaConfig(**ge.TINY), torch.bfloat16, seed=0)
        sd0 = torch.load(os.path.join(ge.OUT, 'e2e_init_llama.pt'), weights_only=False)['sd0']
        assert all(torch.equal(sd0[k], v) for k, v in model.model.state_dict().items() if k in sd0)
        rh.run_algo(model, ge.GPTQ_QUANT, gold['calib_ids'], bs=gold['bs'], seq_len=gold['calib_ids'].shape[1])
    finally:
        GPTQ.block_opt, GPTQ.layer_transform, GPTQ.weight_transform = orig_bo, orig_lt, orig_wt
    x1 = rec['x1']
    assert x1.dtype == torch.bfloat16 and x1.shape == (16, 128, 256), (x1.dtype, x1.shape)
    names = sorted(k for k in rec['losses'] if k.startswith('1.'))
    np.savez_compressed(OUT, x1=x1.view(torch.int16).numpy().view(np.uint16),
                        loss_names=np.array(names), losses=np.array([rec['losses'][k] for k in names]))
    print('block 0 losses vs e2e_gptq_llama.pt:',
          {k: round(abs(v - gold['losses'][k]) / gold['losses'][k], 7) for k, v in rec['losses'].items()
           if k.startswith('0.')})
    print(f'{OUT}: {os.path.getsize(OUT)} bytes')


if __name__ == '__main__':
    main()
