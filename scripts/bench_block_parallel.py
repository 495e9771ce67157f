"""Block-parallel GPTQ calibration benchmark — BASELINE.json north_star's multi-GPU split and
configs[3] ("GPTQ W4A16 on Llama-3-70B-shaped weights, layer-parallel across 8 GPUs with NCCL
activation broadcast").

    python -m torch.distributed.run --nproc-per-node N scripts/bench_block_parallel.py \
        --model llama-3-70b --layers 16 --samples 128 --seq-len 2048

Runs llmc_b200.block_parallel.BlockParallelRunner over `--layers` decoder blocks of the shape model
(every block has the same cost; a prefix keeps weights + activations inside one GPU's HBM and the
run inside the GPU budget) with the GPTQ YAML of configs/gptq_w_only.yml except `quant_out: False`,
`true_sequential: False` — the setting in which blocks are independent given their fp inputs
(SURVEY.md 8(e)).  Timing: barrier + synchronize around the whole run, CUDA events, max over
ranks; prints ONE JSON line on rank 0 with layers/s and the per-phase breakdown.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from llmc_b200.block_parallel import BlockParallelRunner  # noqa: E402
from llmc_b200.blockwise import AttrDict  # noqa: E402
from llmc_b200.gptq import GPTQ  # noqa: E402
from llmc_b200.prof import TIMER  # noqa: E402
from llmc_b200.synth import SynthModel  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--model', default='llama-3-70b')
    ap.add_argument('--layers', type=int, default=16)
    ap.add_argument('--samples', type=int, default=128)
    ap.add_argument('--seq-len', dest='seq_len', type=int, default=2048)
    ap.add_argument('--sync', default='rank0', choices=['all', 'rank0', 'none'])
    args = ap.parse_args()
    rank, world = int(os.environ.get('RANK', '0')), int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    cfg = AttrDict.wrap({
        'base': {'seed': 0}, 'calib': {'n_samples': args.samples, 'bs': 1, 'seq_len': args.seq_len},
        'quant': {'method': 'GPTQ', 'quant_out': False,
                  'weight': {'bit': 4, 'symmetric': False, 'granularity': 'per_group', 'group_size': 128},
                  'special': {'actorder': True, 'static_groups': False, 'percdamp': 0.01, 'blocksize': 128,
                              'true_sequential': False}}})
    model = SynthModel(args.model, n_layers=args.layers, seed=0, device='cuda', with_head=False, init='device')
    # every rank builds only ITS contiguous chunk of the calibration inputs (same token ids)
    assert args.samples % world == 0
    nl = args.samples // world
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, model.shape['vocab'], (args.samples, args.seq_len), generator=g)
    inp = model.first_block_input(0, 0, bs=1, device='cuda', ids=ids[rank * nl:(rank + 1) * nl])

    class BenchGPTQ(GPTQ):
        def collect_model_qparams(self):          # seeds collected per block inside block_opt
            self._qparams_pending = set(range(len(self.blocks)))
    # warm-up on a throw-away prefix of the same shape (one round: `world` blocks, the rank's first
    # samples): kernel module loads, function attributes, the NCCL rings and the caching allocator's
    # first cudaMallocs stay out of the timed run
    wm = SynthModel(args.model, n_layers=world, seed=1, device='cuda', with_head=False, init='device')
    winp = {'data': [d.clone() for d in inp['data'][:max(1, min(2, nl))]],
            'kwargs': inp['kwargs'][:max(1, min(2, nl))]}
    walgo = BenchGPTQ(wm, cfg.quant, winp, None, cfg)
    BlockParallelRunner(walgo, sync=None if args.sync == 'none' else args.sync, input_is_local=True).run()
    del wm, walgo, winp
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    algo = BenchGPTQ(model, cfg.quant, inp, None, cfg)
    runner = BlockParallelRunner(algo, sync=None if args.sync == 'none' else args.sync, input_is_local=True)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    TIMER.enabled = True
    TIMER.reset()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    runner.run()
    e.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ms = torch.tensor([s.elapsed_time(e)], device='cuda', dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    kern = TIMER.summary()
    if rank == 0:
        ms = float(ms.item())
        layers = 7 * args.layers
        spans = {k: {'calls': v['calls'], 'ms': round(v['ms'], 1)} for k, v in
                 sorted(kern.items(), key=lambda kv: -kv[1]['ms'])}
        print(json.dumps({
            'metric': 'GPTQ-W4 layers/sec, block-parallel (quant_out False)', 'value': round(layers / (ms / 1e3), 3),
            'unit': 'layers/s', 'n_gpus': world, 'ms_total': round(ms, 1), 'ms_per_block': round(ms / args.layers, 2),
            'config': {'model': args.model, 'blocks': args.layers, 'samples': args.samples, 'seq_len': args.seq_len,
                       'parallelism': f'block-parallel x{world}: dp fp forward, NCCL all-gather of block inputs to their owners, '
                                      f'owner-local calibration, results -> {args.sync}'},
            'rank0_spans': spans,
            'peak_mem_gb': round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
