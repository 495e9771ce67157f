"""Block-wise quantisation framework — thin Python mirror of
llmc/compression/blockwise_optimization.py (BlockwiseOpt :8-114) and
llmc/compression/quantization/base_blockwise_quantization.py (BaseBlockwiseQuantization
:41-1038), reduced to what RTN / GPTQ / AWQ need (SURVEY.md §8(b): "boundary, not a kernel").

Same override points (`block_opt`, `block_transform`, `subset_transform`, `cache_input_hook`,
`block_init`, `subset_init`, `w_qdq`, `w_q`, `a_qdq`), same `buf_*` buffers, same
`deploy(quant_format)` formats.  Everything stays resident on the GPU (180 GB of HBM3e holds a
70B model + activations), so the reference's block.cuda()/block.cpu() shuttling
(base_blockwise_quantization.py:397,418) disappears.
"""
import functools
from collections import defaultdict

import torch

from .module_utils import (_REALQUANT_LINEAR_MAP_, EffcientFakeQuantLinear, FakeQuantLinear,
                           OriginFloatLinear)
from .quant import IntegerQuantizer
from .registry import ALGO_REGISTRY  # noqa: F401  (re-exported for algorithm modules)


def _same_act_scale(a, b):
    """Whether linears a and b hold one static activation scale (buf_act_scales_0).  Read once per
    pair of buffer versions and cached on a, as synth._same_input_scale does, so that later forwards
    do not synchronise."""
    sa, sb = a.buf_act_scales_0, b.buf_act_scales_0
    if sa is sb:
        return True
    key = (sa.data_ptr(), sa._version, sb.data_ptr(), sb._version)
    cached = getattr(a, '_same_act_scale', None)
    if cached is None or cached[0] != key:
        cached = (key, sa.numel() == sb.numel() and torch.equal(sa.reshape(-1).float(), sb.reshape(-1).float()))
        a._same_act_scale = cached
    return cached[1]


class AttrDict(dict):
    """The 10-line stand-in for easydict (not installed): cfg.quant.weight.bit style access."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError:
            raise AttributeError(k) from None
        return v

    def __setattr__(self, k, v):
        self[k] = v

    @classmethod
    def wrap(cls, obj):
        if isinstance(obj, dict):
            return cls({k: cls.wrap(v) for k, v in obj.items()})
        if isinstance(obj, list):
            return [cls.wrap(v) for v in obj]
        return obj


class BlockStreamer:
    """Host-resident model, device-resident working set: the double-buffered form of the
    reference's `block = block.cuda(); block_opt(block); block = block.cpu()`
    (blockwise_optimization.py:36-47).

    Block i+1's weights travel host->device on one copy stream while block i is calibrated, and
    block i's results (calibrated weights + qparam buffers) travel device->host on another while
    block i+1 runs, so neither copy is on the critical path.  Host tensors are pinned.  After
    `release(i)` every parameter / buffer of block i is a pinned host tensor again, like after
    the reference's `block.cpu()`.
    """

    def __init__(self, blocks, device, writeback=True):
        """writeback=False (data-parallel ranks other than the saving one — the reference saves
        from rank 0 only): results are not copied back; the block's parameters return to their
        original pinned host tensors and the device copies are dropped."""
        self.blocks = list(blocks)
        self.device = torch.device(device)
        self.writeback = writeback
        self.h2d = torch.cuda.Stream(self.device)
        self.d2h = torch.cuda.Stream(self.device)
        self.host_in = [None] * len(self.blocks)      # {name: pinned tensor}
        self.host_out = [None] * len(self.blocks)     # {name: pinned tensor}, allocated ahead or lazily
        self.staged = {}                              # block idx -> ({name: device tensor}, event)
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    @staticmethod
    def _named_tensors(block):
        for n, p in block.named_parameters():
            yield n, p, True
        for n, b in block.named_buffers():
            yield n, b, False

    def offload(self):
        """Move every block's parameters to pinned host memory and release the device copies."""
        for i, blk in enumerate(self.blocks):
            d = {}
            for n, p in blk.named_parameters():
                h = torch.empty(p.shape, dtype=p.dtype, pin_memory=True)
                h.copy_(p.data)
                d[n] = h
                p.data = h
            self.host_in[i] = d
        torch.cuda.synchronize(self.device)
        torch.cuda.empty_cache()

    def preallocate_results(self, template_idx, targets):
        """Pinned result buffers for blocks `targets`, shaped like block `template_idx`'s current
        (already calibrated) tensors — pinning memory is slow, so do it outside the block loop."""
        if not self.writeback:
            return
        shapes = {n: (t.shape, t.dtype) for n, t, _ in self._named_tensors(self.blocks[template_idx])}
        for i in targets:
            self.host_out[i] = {n: torch.empty(s, dtype=dt, pin_memory=True) for n, (s, dt) in shapes.items()}

    def prefetch(self, i):
        if i in self.staged or self.host_in[i] is None:
            return
        cur = torch.cuda.current_stream(self.device)
        dev = {n: torch.empty(h.shape, dtype=h.dtype, device=self.device) for n, h in self.host_in[i].items()}
        self.h2d.wait_stream(cur)            # the buffers were carved out of memory `cur` may still use
        with torch.cuda.stream(self.h2d):
            for n, h in self.host_in[i].items():
                dev[n].copy_(h, non_blocking=True)
                self.h2d_bytes += h.numel() * h.element_size()
        ev = torch.cuda.Event()
        ev.record(self.h2d)
        for t in dev.values():
            t.record_stream(self.h2d)
        self.staged[i] = (dev, ev)

    def acquire(self, i):
        self.prefetch(i)
        dev, ev = self.staged.pop(i)
        torch.cuda.current_stream(self.device).wait_event(ev)
        for n, p in self.blocks[i].named_parameters():
            p.data = dev[n]

    def release(self, i):
        cur = torch.cuda.current_stream(self.device)
        done = torch.cuda.Event()
        done.record(cur)
        blk = self.blocks[i]
        if not self.writeback:
            for n, p in blk.named_parameters():
                if p.is_cuda and n in (self.host_in[i] or {}):
                    p.data = self.host_in[i][n]
            return
        out = self.host_out[i] or {}
        self.d2h.wait_event(done)
        with torch.cuda.stream(self.d2h):
            for n, t, is_param in list(self._named_tensors(blk)):
                if not t.is_cuda:
                    continue
                h = out.get(n)
                if h is None or h.shape != t.shape or h.dtype != t.dtype:
                    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                    out[n] = h
                src = t.data if is_param else t
                h.copy_(src, non_blocking=True)
                src.record_stream(self.d2h)
                self.d2h_bytes += h.numel() * h.element_size()
                if is_param:
                    t.data = h
                else:
                    mod, _, leaf = n.rpartition('.')
                    owner = blk.get_submodule(mod) if mod else blk
                    owner._buffers[leaf] = h
        self.host_out[i] = out

    def finish(self):
        self.h2d.synchronize()
        self.d2h.synchronize()


class BlockwiseOpt:
    """blockwise_optimization.py:8-51."""

    def __init__(self, model, compress_config, input, padding_mask, config):
        self.model = model
        self.blocks = model.get_blocks()
        self.quant_config = compress_config
        self.input = input
        self.padding_mask = padding_mask
        self.data_free = False if self.input else True
        self.config = config
        self.block_idx = None
        self.num_blocks = len(self.blocks)
        if self.input:
            for kw in input['kwargs']:
                kw.pop('use_cache', None)
                if 'past_key_value' in kw:
                    kw['past_key_value'] = None
            self.n_samples = sum(d.shape[0] for d in input['data'])

    def run_block_loop(self, first=0, last=None, streamer=None, on_block_done=None):
        """blockwise_optimization.py:30-51.  With a `BlockStreamer` the model lives in pinned host
        memory and each block is brought in / written back around `block_opt` (the reference's
        block.cuda() / block.cpu()), copies overlapped with the neighbouring blocks' work;
        without one, everything is already resident on the GPU.  `on_block_done(i)` runs after
        block i has been queued (e.g. to read a loss back)."""
        last = len(self.blocks) if last is None else last
        if streamer is not None and first < last:
            streamer.prefetch(first)
        for i in range(first, last):
            if streamer is not None:
                streamer.acquire(i)
                if i + 1 < last:
                    streamer.prefetch(i + 1)
            self.block_idx = i
            self.block_opt(self.blocks[i])
            if streamer is not None:
                streamer.release(i)
            if on_block_done is not None:
                on_block_done(i)
        if streamer is not None:
            streamer.finish()

    def cache_input_hook(self, m, x, y, name, feat_dict):
        """blockwise_optimization.py:53-61 — kept on the device (the reference moves every
        hooked input to the CPU)."""
        inputs = [i.detach() for i in x]
        if len(inputs) == 1:
            inp = inputs[0]
            if inp.dim() == 2:
                inp = inp.unsqueeze(0)
            feat_dict[name].append(inp)
        else:
            feat_dict[name].append(tuple(inputs))

    def block_opt(self, block):
        raise NotImplementedError

    def layer_init(self, layer):
        pass

    def subset_init(self, subset):
        pass

    def block_init(self, block):
        pass


class BaseBlockwiseQuantization(BlockwiseOpt):
    def __init__(self, model, quant_config, input, padding_mask, config):
        super().__init__(model, quant_config, input, padding_mask, config)
        self.set_quant_config()

    # ---- quantizer selection (base_blockwise_quantization.py:133-268) --------------------------
    def set_quant_config(self):
        qc = self.quant_config
        self.mixed_precision = 'ignored_layers' in (self.config or {})
        if self.mixed_precision:
            ig = self.config['ignored_layers']
            self.ignored_block_ids = ig.get('block_ids', [])
            self.ignored_layer_names = ig.get('layer_names', [])
            self.ignored_speical_names = ig.get('speical_names', [])
        self.quant_out = qc.get('quant_out', False)
        self.tp = qc.get('tp', 1)
        wkw = dict(qc['weight'])
        quant_type = wkw.pop('quant_type', 'int-quant')
        if quant_type == 'int-quant':
            if wkw['bit'] == 48:
                raise NotImplementedError('Weight48IntegerQuantizer (quant.py:1232-1369)')
            self.weight_quant_module = IntegerQuantizer
        elif quant_type == 'float-quant':
            from .quant_float import FloatQuantizer
            self.weight_quant_module = FloatQuantizer
        else:
            raise ValueError(quant_type)
        wkw['tp'] = self.tp
        self.wquantizer = self.weight_quant_module(**wkw)
        if 'act' in qc:
            akw = dict(qc['act'])
            self.w_only = False
            aquant_type = akw.pop('quant_type', 'int-quant')
            if aquant_type == 'float-quant':
                from .quant_float import FloatQuantizer
                self.act_quant_module = FloatQuantizer
            else:
                self.act_quant_module = IntegerQuantizer
            akw['tp'] = self.tp
            self.aquantizer = self.act_quant_module(**akw)
            self.act_static = akw.get('static', False)
            if self.act_static:
                assert akw['granularity'] == 'per_tensor', 'Only support per_tensor static quant'
        else:
            self.w_only = True
            self.aquantizer = None
            self.act_static = False
        if 'kvcache' in qc:
            raise NotImplementedError('KV-cache quantisation is out of scope (SURVEY §2 #11)')
        self.quant_kvcache = False
        self.quant_attn = self.quant_softmax = self.quant_act_fn = False
        special = qc.get('special', {}) or {}
        self.true_sequential = special.get('true_sequential', False)
        self.online_rotate = False
        self.modality = qc.get('modality', 'language')

    # ---- replacement callbacks (base_blockwise_quantization.py:46-131) ---------------------------
    def w_qdq(self, module, wquantizer):
        args = {'lowbound_factor': None, 'upbound_factor': None}
        if hasattr(module, 'buf_lowbound_factor'):
            args['lowbound_factor'] = module.buf_lowbound_factor
        if hasattr(module, 'buf_upbound_factor'):
            args['upbound_factor'] = module.buf_upbound_factor
        return wquantizer.fake_quant_weight_dynamic(module.weight, args)

    def w_q(self, module, wquantizer):
        return wquantizer.real_quant_weight_dynamic(module.weight.data)

    def a_qdq(self, act, module, aquantizer, input_index=0):
        if self.act_static:
            args = {k: getattr(module, f'buf_act_{k}_{input_index}', None)
                    for k in ('scales', 'zeros', 'qmax', 'qmin')}
            return aquantizer.fake_quant_act_static(act, args)
        return aquantizer.fake_quant_act_dynamic(act)

    def a_qdq_routed(self, linears, aquantizer):
        """The routed twin of a_qdq, for a grouped MoE layer (module_utils.moe_forward): linears[e] are
        the linears of expert e that take the same rows (w1 and w3, or w2).  Returns f(act,
        expert_of_row) that gives, in one pass over the routed rows act [M, K] (expert_of_row [M] on
        the device), what a_qdq(rows of e, m) gives every m in linears[e], bit for bit; or None when
        one pass cannot:
          dynamic, per_token / per_channel / per_group: every row's qparams come from that row alone,
            so fake_quant_act_dynamic over all rows;
          static, per_tensor, symmetric: the quantiser's static pass with one scale per row, the
            buf_act_scales_0 of the row's expert gathered on the device (0-dim scales only, whose
            arithmetic that pass restates).  qmin / qmax are the quantiser's own, the values
            register_act_qparams stores.  The linears of one expert must hold one scale (read once
            per buffer version, then cached), since each quantises the same rows.
        Refused: per_tensor dynamic activations (the scale depends on the expert's whole segment),
        asymmetric static ones and every other form."""
        from .quant_float import FloatQuantizer
        q = aquantizer
        if type(q) not in (IntegerQuantizer, FloatQuantizer):
            return None
        if not self.act_static:
            if q.granularity not in ('per_token', 'per_channel', 'per_group'):
                return None
            if type(q) is IntegerQuantizer and (q.calib_algo not in ('minmax', 'learnable') or not q.round_zp):
                return None
            return lambda act, expert_of_row: q.fake_quant_act_dynamic(act)
        if q.granularity != 'per_tensor' or not q.sym:
            return None
        for ms in linears:
            for m in ms:
                sc = getattr(m, 'buf_act_scales_0', None)
                if sc is None or sc.dim() != 0 or not sc.is_cuda or not sc.is_floating_point():
                    return None
            if not all(_same_act_scale(ms[0], m) for m in ms[1:]):
                return None
        first = [ms[0] for ms in linears]

        def qdq(act, expert_of_row):
            table = torch.stack([m.buf_act_scales_0.float() for m in first])
            return q.fake_quant_act_static_rows(act, table.index_select(0, expert_of_row))
        return qdq

    def w_packed(self, module, wquantizer):
        """K6 hand-off for EffcientFakeQuantLinear: the packed form of exactly what `w_qdq` would
        materialise, or None when this layer / quantizer is not a plain INT2 / INT3 / INT4 / INT8 group or
        channel weight quantizer (then the wrapper materialises as before)."""
        from .module_utils import pack_unsigned_codes
        from .quant_float import FloatQuantizer
        q, w = wquantizer, module.weight
        if isinstance(q, FloatQuantizer):
            return self._fp8_packed(module, q)
        if not (isinstance(q, IntegerQuantizer) and q.bit in (2, 3, 4, 8) and q.calib_algo == 'minmax'
                and q.granularity in ('per_group', 'per_channel') and q.round_zp
                and w.dim() == 2 and w.is_cuda and w.dtype in (torch.float16, torch.bfloat16)):
            return None
        if hasattr(module, 'buf_lowbound_factor') or hasattr(module, 'buf_upbound_factor'):
            return None
        K = w.shape[1]
        group = q.group_size if q.granularity == 'per_group' else K
        if K % 64 or group % 64 or K % group:
            return None
        codes, scales, zeros = q.real_quant_weight_dynamic(w.data)
        return dict(qweight=pack_unsigned_codes(codes, q.bit, signed=q.sym), scales=scales.contiguous(),
                    zeros=None if zeros is None else zeros.to(scales.dtype).contiguous(),
                    bits=q.bit, group=group, dtype=w.dtype)

    @staticmethod
    def _fp8_packed(module, q):
        """w_packed on an e4m3 / e5m2 grid (FloatQuantizer, minmax): the bytes and scales of the very
        pass fake_quant_weight_dynamic runs (`_dynamic`: byte mode instead of QDQ mode).  per_tensor's
        fp32 scalar is expanded to one fp32 scale per row; per_channel / per_group keep their scales in
        the weight dtype.  None for per_block, clipped layers, and K or groups not a multiple of 64."""
        w = module.weight
        if not (q.calib_algo == 'minmax' and q.granularity in ('per_tensor', 'per_channel', 'per_group')
                and w.dim() == 2 and w.is_cuda and w.dtype in (torch.float16, torch.bfloat16)):
            return None
        if hasattr(module, 'buf_lowbound_factor') or hasattr(module, 'buf_upbound_factor'):
            return None
        N, K = w.shape
        # FloatQuantizer._layout: a row shorter than the group is one group
        group = q.group_size if q.granularity == 'per_group' and K >= q.group_size else K
        if K % 64 or group % 64 or K % group:
            return None
        wq, scales = q._dynamic(w.data, 2)
        if q.granularity == 'per_tensor':
            scales = scales.reshape(1).float().expand(N, 1)
        return dict(qweight=wq.reshape(N, K), scales=scales.reshape(N, K // group).contiguous(), zeros=None,
                    bits=8, group=group, dtype=w.dtype)

    def get_replacement_params(self, mode='fake_quant', w_only=False, name=None):
        params = {}
        if mode in ('fake_quant', 'fake_quant_wo_kv'):
            params['a_qdq'] = (functools.partial(self.a_qdq, aquantizer=self.aquantizer)
                               if not w_only else None)
            params['w_qdq'] = functools.partial(self.w_qdq, wquantizer=self.wquantizer)
            # the packed twin of w_qdq: only a class that defines w_qdq knows what it materialises,
            # so the packer is the `w_packed` that same class defines (the base one for RTN / AWQ,
            # GPTQ's own, act-order included; HQQ's and SpQR's real-valued zero-points, SpQR's
            # outliers included).  A subclass that overrides w_qdq without a w_packed of its own
            # keeps the materialised path.
            owner = next(c for c in type(self).__mro__ if 'w_qdq' in c.__dict__)
            if 'w_packed' in owner.__dict__:
                params['w_qdq'].packed = functools.partial(self.w_packed, wquantizer=self.wquantizer)
            # the routed twin of a_qdq (a grouped MoE layer's activations in one pass), by the same
            # rule: only the class that defines a_qdq knows what it computes
            owner = next(c for c in type(self).__mro__ if 'a_qdq' in c.__dict__)
            if params['a_qdq'] is not None and 'a_qdq_routed' in owner.__dict__:
                params['a_qdq'].routed = functools.partial(self.a_qdq_routed, aquantizer=self.aquantizer)
        elif mode in _REALQUANT_LINEAR_MAP_:
            params['w_q'] = functools.partial(self.w_q, wquantizer=self.wquantizer)
            params['quant_config'] = self.quant_config
        return params

    # ---- RTN qparams of a block (base_blockwise_quantization.py:337-365) -------------------------
    @torch.no_grad()
    def collect_block_qparams(self, block):
        for n, m in self.model.get_block_linears(block).items():
            args = {}
            if hasattr(m, 'buf_lowbound_factor'):
                args['lowbound_factor'] = m.buf_lowbound_factor
            if hasattr(m, 'buf_upbound_factor'):
                args['upbound_factor'] = m.buf_upbound_factor
            _, scales, zeros, max_int, min_int = self.wquantizer.get_tensor_qparams(
                m.weight.data, args=args)
            m.register_buffer('buf_scales', scales.detach())
            m.register_buffer('buf_zeros', zeros.detach())
            # 0-dim integer bounds stay on the host: they are kernel *arguments*, and reading a
            # device scalar back (`.item()`) would drain the stream once per use
            # (get_qparams returns the quantizer's own qmax/qmin moved to the device)
            del max_int, min_int
            m.register_buffer('buf_qmax', self.wquantizer.qmax.clone().cpu())
            m.register_buffer('buf_qmin', self.wquantizer.qmin.clone().cpu())

    # ---- block loop (base_blockwise_quantization.py:367-526) ---------------------------------------
    def block_forward(self, block, input_data=None):
        if input_data is None:
            input_data = self.input['data']
        dev = next(block.parameters()).device if any(True for _ in block.parameters()) else \
            next(block.buffers()).device
        output = []
        for i in range(len(input_data)):
            with torch.no_grad():
                out = block(input_data[i].to(dev), **self.input['kwargs'][i])
            output.append(out[0] if isinstance(out, tuple) else out)
        return output

    def block_opt(self, block):
        named_linears = self.model.get_block_linears(block)
        extra_modules = self.model.get_extra_modules(block)       # base_bq.py:398-408
        input_feat = defaultdict(list)
        handles = self.register_hooks({**named_linears, **extra_modules}, input_feat)
        self.block_init(block)
        self.run(block, input_feat, handles)

    def register_hooks(self, modules, input_feat):
        handles = []
        if not self.data_free:
            for name, m in modules.items():
                handles.append(m.register_forward_hook(
                    functools.partial(self.cache_input_hook, name=name, feat_dict=input_feat)))
        return handles

    def run(self, block, input_feat, handles):
        if not self.data_free:
            if self.quant_out:
                self.block_forward(block)
            else:
                self.input['data'] = self.block_forward(block)
            for h in handles:
                h.remove()
            self.block_transform(block, input_feat, self.input['kwargs'])
        else:
            self.block_transform(block)
        if not self.data_free and self.quant_out:
            self.model.replace_module_block(
                FakeQuantLinear, block, self.block_idx,
                self.get_replacement_params(mode='fake_quant', w_only=self.w_only, name=None))
            self.input['data'] = self.block_forward(block)

    def block_transform(self, block, input_feat=None, block_kwargs=None):
        subsets = self.model.get_subsets_in_block(block)
        for index, subset in enumerate(subsets):
            subset_kwargs = block_kwargs if subset['has_kwargs'] else {}
            self.subset_transform(subset, input_feat, subset_kwargs)
            if self.act_static:
                self.register_act_qparams(subset['layers'], input_feat[subset['input'][0]])
            if self.true_sequential and index != len(subsets) - 1:
                input_feat.update(self.rehook_next_subset(block, subset, subsets[index + 1]))

    def rehook_next_subset(self, block, subset, next_subset):
        self.subset_init(next_subset)
        self.model.replace_module_subset(
            FakeQuantLinear, block, subset, self.block_idx,
            self.get_replacement_params(mode='fake_quant', w_only=self.w_only, name=None))
        input_feat_subset = defaultdict(list)
        handles = self.register_hooks(next_subset['layers'], input_feat_subset)
        self.block_forward(block)
        for h in handles:
            h.remove()
        return input_feat_subset

    def subset_transform(self, subset, input_feat, subset_kwargs):
        pass

    # ---- static activation qparams (base_blockwise_quantization.py:566-588) ------------------------
    @torch.no_grad()
    def register_act_qparams(self, layers_dict, act_tensors):
        scales_list, zeros_list, qmin_list, qmax_list = \
            self.aquantizer.get_batch_tensors_qparams(list(act_tensors))
        from .dist_utils import world as _dp_world
        world = _dp_world()
        for i in range(len(scales_list)):
            scales, zeros = scales_list[i].cuda(), zeros_list[i].cuda()
            if world > 1:
                torch.distributed.all_reduce(scales)
                scales = scales / world
            for name, layer in layers_dict.items():
                layer.register_buffer(f'buf_act_scales_{i}', scales)
                layer.register_buffer(f'buf_act_zeros_{i}', zeros)
                layer.register_buffer(f'buf_act_qmin_{i}', qmin_list[i].cuda())
                layer.register_buffer(f'buf_act_qmax_{i}', qmax_list[i].cuda())

    # ---- deploy (base_blockwise_quantization.py:932-986) ---------------------------------------------
    @torch.no_grad()
    def deploy(self, quant_format, keep_device=False):
        mapping = {'origin_float': OriginFloatLinear, 'fake_quant': EffcientFakeQuantLinear,
                   'fake_quant_wo_kv': EffcientFakeQuantLinear}
        mapping.update(_REALQUANT_LINEAR_MAP_)
        if quant_format not in mapping:
            raise NotImplementedError(f"Quant format '{quant_format}' is not implemented.")
        self.model.replace_language_module_all(
            mapping[quant_format],
            self.get_replacement_params(mode=quant_format, w_only=self.w_only),
            keep_device=keep_device)
