"""Block-parallel calibration across the GPUs of one box — BASELINE.json north_star's multi-GPU
split ("calibration partitions layer-parallel across the 8 GPUs with NCCL broadcast of
calibration activations over NVLink"), SURVEY.md 8(e) axis "Blocks".

Valid when block i+1 is calibrated on the FLOATING-POINT output of block i, i.e. `quant_out:
False` (base_blockwise_quantization.py:436-444), and for data-free algorithms (RTN, export): then
blocks are independent given their fp input activations.  (`quant_out: True` — the shipped GPTQ /
AWQ YAMLs — makes blocks sequentially dependent; that mode stays on data-parallel calibration,
llmc_b200/gptq.py + dist_utils.)

Schedule, one process per GPU (N ranks, block i owned by rank i mod N):
  1. fp forward, data-parallel: rank r pushes ITS contiguous chunk of the calibration samples
     through all blocks in floating point and keeps every block's input chunk
     (L x n/N x S x hidden, e.g. 8.6 GB for Llama-3-8B at N = 8);
  2. per round of N blocks, one NCCL all-gather per block hands its owner the full [n, S, hidden]
     input of the block in the original sample order — the "activation broadcast" of the
     north_star, 2-4 GiB per block over NVLink / NVSwitch (ring collective);
  3. every owner runs the unchanged `block_opt` on its block: no collective inside;
  4. the calibrated block (weights + buf_* qparams) is broadcast from its owner (or only sent to
     rank 0, which saves) — metadata first, because GPTQ changes dtypes and adds buffers.
Results are bit-identical to the single-GPU run of the same YAML: the fp forward is per-sample,
and each block's calibration sees the same tensors in the same order.
"""
import torch
import torch.distributed as dist

from .dist_utils import global_rank, global_world, no_data_parallel
from .prof import TIMER


def _chunk_bounds(n, r, w):
    assert n % w == 0, f'{n} calibration samples do not split over {w} ranks'
    c = n // w
    return r * c, (r + 1) * c


class BlockParallelRunner:
    def __init__(self, algo, sync='all', fwd_chunk=16, input_is_local=False):
        """algo: a constructed algorithm object whose `input` holds ALL n calibration samples'
        first-block inputs (each rank builds them from the same token ids; only its chunk is used).
        sync: 'all' broadcast calibrated blocks to every rank | 'rank0' | None (leave them on
        their owners)."""
        if getattr(algo, 'quant_out', False) and not algo.data_free:
            raise ValueError('block-parallel calibration needs quant_out: False (blocks must be '
                             'independent given their fp inputs); use data-parallel calibration for '
                             'quant_out: True')
        self.algo, self.sync, self.fwd_chunk = algo, sync, fwd_chunk
        # input_is_local: algo.input already holds only THIS rank's contiguous chunk of the samples
        self.input_is_local = input_is_local
        self.r, self.w = global_rank(), global_world()

    # ---- stage 1 ----------------------------------------------------------------------------------
    @torch.no_grad()
    def _fp_forward_all(self, x_local, kwargs):
        """Returns the list of every block's input chunk [n_local, S, hidden] (fp forward)."""
        blocks = self.algo.blocks
        inputs = []
        x = x_local
        for b in blocks:
            inputs.append(x)
            y = torch.empty_like(x)
            for i in range(0, x.shape[0], self.fwd_chunk):
                out = b(x[i:i + self.fwd_chunk], **kwargs)
                y[i:i + self.fwd_chunk] = out[0] if isinstance(out, tuple) else out
            x = y
        return inputs

    # ---- stage 4 ----------------------------------------------------------------------------------
    @staticmethod
    def _named_tensors(block):
        out = [(n, p.data) for n, p in block.named_parameters()]
        out += [(n, b) for n, b in block.named_buffers() if torch.is_tensor(b)]
        return out

    def _sync_block(self, idx, owner):
        blk = self.algo.blocks[idx]
        dev = next(blk.parameters()).device
        meta = [None]
        if self.r == owner:
            meta[0] = [(n, tuple(t.shape), t.dtype, t.is_cuda) for n, t in self._named_tensors(blk)]
        dist.broadcast_object_list(meta, src=owner)
        for n, shape, dtype, on_dev in meta[0]:
            mod_name, _, leaf = n.rpartition('.')
            mod = blk.get_submodule(mod_name) if mod_name else blk
            if self.r == owner:
                t = (mod._parameters[leaf].data if leaf in mod._parameters else mod._buffers[leaf])
                t = t.to(dev).contiguous()
            else:
                t = torch.empty(shape, dtype=dtype, device=dev)
            if self.sync == 'all':
                dist.broadcast(t, src=owner)
            elif self.sync == 'rank0' and owner != 0:
                if self.r == owner:
                    dist.send(t, dst=0)
                elif self.r == 0:
                    dist.recv(t, src=owner)
            if self.r != owner and (self.sync == 'all' or (self.sync == 'rank0' and self.r == 0)):
                t = t if on_dev else t.cpu()
                if leaf in mod._parameters:
                    mod._parameters[leaf].data = t
                else:
                    mod._buffers[leaf] = t

    # ---- the loop ---------------------------------------------------------------------------------
    @torch.no_grad()
    def run(self):
        algo, r, w = self.algo, self.r, self.w
        blocks = algo.blocks
        L = len(blocks)
        if algo.data_free:
            for i in range(r, L, w):
                algo.block_idx = i
                with no_data_parallel():
                    algo.block_opt(blocks[i])
        else:
            data, kwargs = algo.input['data'], algo.input['kwargs']
            bs_list = [d.shape[0] for d in data]
            X = data[0] if len(data) == 1 else torch.cat(data, dim=0)
            if self.input_is_local:
                lo, hi = 0, X.shape[0]
                bs_list = bs_list * w
            else:
                lo, hi = _chunk_bounds(X.shape[0], r, w)
            kw = kwargs[0]
            with TIMER.span('bp_fp_forward'):
                inputs = self._fp_forward_all(X[lo:hi].contiguous(), kw)
            del X, data
            algo.input = None
            nl = hi - lo
            for k in range(0, L, w):
                mine = k + r
                full = None
                # The activation "broadcast": one NCCL all-gather per block of the round; the owner
                # keeps the result, the other ranks reuse one scratch buffer.  (A single all-to-all
                # would move 1/N of the bytes, but ncclSend/Recv-based all_to_all_single was measured
                # two orders of magnitude slower per rank than the ring collectives.)
                scratch = None
                for j in range(w):
                    b = k + j
                    if b >= L:
                        break
                    src = inputs[b]
                    with TIMER.span('bp_all_gather', nbytes=float(src.numel() * src.element_size() * w)):
                        if w > 1:
                            if j == r:
                                dst = torch.empty((w * nl,) + tuple(src.shape[1:]), dtype=src.dtype,
                                                  device=src.device)
                            else:
                                if scratch is None:
                                    scratch = torch.empty((w * nl,) + tuple(src.shape[1:]), dtype=src.dtype,
                                                          device=src.device)
                                dst = scratch
                            dist.all_gather_into_tensor(dst, src.contiguous())
                        else:
                            dst = src
                    if j == r:
                        full = dst
                    inputs[b] = None
                del scratch
                if mine < L:
                    algo.input = {'data': list(torch.split(full, bs_list, dim=0)),
                                  'kwargs': [kw] * len(bs_list), 'stacked': full}
                    algo.block_idx = mine
                    with no_data_parallel():         # a different block on every rank: no DP collectives
                        algo.block_opt(blocks[mine])
                    algo.input = None
                del full
        if hasattr(algo, 'check_factorizations'):
            algo.check_factorizations(wait=True)
        if self.sync and w > 1:
            with TIMER.span('bp_sync_blocks'):
                for i in range(L):
                    self._sync_block(i, i % w)
        return algo
