"""GPTQ — mirror of llmc/compression/quantization/gptq.py (class GPTQ :21-478) on the CUDA
kernels.  Same YAML knobs (`special: actorder, static_groups, percdamp, blocksize,
true_sequential, chunk_num`), same hook / subset flow, same `buf_*` hand-off to
FakeQuantLinear / the real-quant packers.

What differs from the reference is only HOW the numbers are produced:
  * add_batch        -> one wgmma SYRK per hooked batch (gptq_ops.hessian_add_batch); the
                        per-batch all_reduce of H (gptq.py:292-295) becomes ONE all_reduce per
                        layer before it is used (same mean, linear in H);
  * layer_transform  -> prepare gather kernel, Cholesky triple, one fused column-block sweep
                        (gptq_ops.weight_transform) that also writes tmp[:, invperm];
  * linears that share an input (q/k/v, gate/up) share perm + Hinv (the reference recomputes
    the identical H, perm and Cholesky for each; gptq.py:113-117).
"""
import math
import os

import torch
import torch.distributed as dist
import torch.nn as nn

from . import dist_utils
from . import gptq_ops as ops
from .blockwise import ALGO_REGISTRY, BaseBlockwiseQuantization
from .module_utils import (_LLMC_LINEAR_TYPES_, _TRANSFORMERS_LINEAR_TYPES_, FakeQuantLinear,
                           linear_residual)


def norm_into(ln, src, dst):
    """dst <- ln(src): the fused RMSNorm kernel when `ln` is an RMSNorm it can run (8-wide rows,
    weight in the activations' dtype), else the module itself."""
    if hasattr(ln, 'variance_epsilon') and src.shape[-1] % 8 == 0 and ln.weight.dtype == src.dtype:
        from . import block_ops
        block_ops.rmsnorm(src, ln.weight.data, ln.variance_epsilon, out=dst)
    else:
        dst.copy_(ln(src))


@ALGO_REGISTRY
class GPTQ(BaseBlockwiseQuantization):
    def __init__(self, model, quant_config, input, padding_mask, config, modality='language'):
        super().__init__(model, quant_config, input, padding_mask, config)
        self.dev = torch.device('cuda')
        self.model_dtype = next(self.model.model.parameters()).dtype
        self.add_quant_config()
        self.layers_cache = {}
        self.losses = {}           # name -> Losses.sum() (the reference logs it, gptq.py:184)
        self._chol_infos = []      # (name, device int32[1]) of the current block's factorisations
        self._chol_pending = []    # (names, pinned flags, event) travelling to the host
        self.collect_model_qparams()

    @torch.no_grad()
    def add_quant_config(self):
        """gptq.py:33-56."""
        self.prefix = self.model.block_name_prefix
        sp = self.quant_config['special']
        self.true_sequential = sp['true_sequential']
        self.static_groups = sp['static_groups']
        self.actorder = sp['actorder']
        self.percdamp = sp['percdamp']
        self.blocksize = sp['blocksize']
        if self.blocksize != 128:
            raise NotImplementedError('the fused column-block kernel is built for blocksize 128 '
                                      '(every shipped GPTQ YAML uses 128)')
        if sp.get('owq', False):
            raise NotImplementedError('OWQ mixed precision (gptq.py:47-50) is not on the hot path')
        self.owq = False
        if self.float_grid:
            # FloatQuantizer itself refuses use_qtorch False (quant.py:1005-1027) and grids other
            # than e4m3 / e5m2 (:982-988); the sweep covers the granularities of gptq.py:212-227
            wq = self.wquantizer
            if wq.granularity not in ('per_channel', 'per_tensor', 'per_group'):
                raise NotImplementedError(f'GPTQ on an FP8 grid with granularity {wq.granularity} '
                                          '(gptq.py:212-227 sweeps per_channel / per_tensor / per_group)')
            if wq.calib_algo != 'minmax':
                raise NotImplementedError(f'GPTQ on an FP8 grid with calib_algo {wq.calib_algo} '
                                          '(the sweep searches minmax scales, quant.py:1043-1059)')
        self.chunk_num = sp.get('chunk_num', 1)
        self.need_perm = (self.wquantizer.granularity == 'per_group'
                          and not self.static_groups and self.actorder)

    @property
    def float_grid(self):
        """The weights go onto an FP8 grid (FloatQuantizer, llmc_gptq_colblock_fp8)."""
        from .quant_float import FloatQuantizer
        return isinstance(self.wquantizer, FloatQuantizer)

    # ---- Hessian collection ---------------------------------------------------------------------
    @torch.no_grad()
    def cache_input_hook(self, m, inp, out, name, feat_dict):
        """gptq.py:246-251."""
        if isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
            self.add_batch(self.named_layers[name], name, inp[0].data, out.data)
        if self.act_static:
            super().cache_input_hook(m, inp, out, name, feat_dict)

    @staticmethod
    def _input_key(inp):
        return (inp.data_ptr(), tuple(inp.shape), tuple(inp.stride()), inp.dtype)

    @torch.no_grad()
    def add_batch(self, layer, name, inp, out):
        """gptq.py:253-295 (nn.Linear / FakeQuantLinear inputs)."""
        cache = self.layers_cache[name]
        share = cache.get('share')
        if share is None:
            return    # a later subset whose first-pass Hessian would be discarded (subset_init)
        if share != name:
            # H is accumulated once per distinct input, by the subset's first linear.  That is only
            # valid while this linear is fed the very tensor the leader was fed in this forward
            # (q/k/v, gate/up); anything else (e.g. MoE experts, which see routed tokens) must keep
            # its own H like the reference (gptq.py:310-322) — _init_layers arranges that, this is
            # the guard that it did.
            if self.layers_cache[share].get('last_input') != self._input_key(inp):
                raise RuntimeError(
                    f'GPTQ: {name} shares the Hessian of {share} but was called with a different '
                    'input tensor; the subset does not have a common input')
            return
        cache['last_input'] = self._input_key(inp)
        cache['nsamples'] = ops.hessian_add_batch(cache['H'], cache['nsamples'], inp)

    @torch.no_grad()
    def layer_init(self, layer, name):
        """gptq.py:297-308."""
        C = layer.weight.shape[1]
        self.layers_cache[name]['H'] = torch.zeros((C, C), device=self.dev)
        self.layers_cache[name]['nsamples'] = 0
        self.layers_cache[name]['columns'] = C

    def _init_layers(self, named_layers, subsets):
        """One H per distinct input.  A subset's linears hang off one leader only when the model
        wrapper declares that they consume the same tensor: `subset['input']` names one of the
        subset's own linears (llama.py:52-91: q/k/v -> 'self_attn.q_proj', gate/up ->
        'mlp.gate_proj').  Mixtral's expert subset names the MoE module instead
        (mixtral.py:62-75): every expert sees its own routed tokens and the router all tokens, so
        each linear keeps its own H exactly like the reference (gptq.py:310-322)."""
        self.named_layers = named_layers
        leader = {}
        for sub in subsets:
            names = [n for n in sub['layers'] if n in named_layers]
            src = (sub.get('input') or [None])[0]
            if src in names:
                for n in names:
                    leader[n] = src
        for name, layer in named_layers.items():
            if not isinstance(layer, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                continue        # a non-linear subset member (DeepseekV2Gate): no Hessian (gptq.py:246-251)
            self.layers_cache[name] = {}
            lead = leader.get(name, name)
            if lead == name or lead not in self.layers_cache:
                self.layer_init(layer, name)
                self.layers_cache[name]['share'] = name
            else:
                self.layers_cache[name] = {'share': lead, 'columns': layer.weight.shape[1]}

    @torch.no_grad()
    def subset_init(self, subset):
        """gptq.py:310-315."""
        self._init_layers(subset['layers'], [subset])

    @torch.no_grad()
    def block_init(self, block):
        """gptq.py:317-322.  Under true_sequential the Hessians of later subsets collected in the
        first pass are thrown away by subset_init (rehook_next_subset), so they are not computed."""
        subsets = self.model.get_subsets_in_block(block)
        linears = self.model.get_block_linears(block)
        if self.true_sequential and subsets:
            first = {n: linears[n] for n in subsets[0]['layers'] if n in linears}
            self._init_layers(first, subsets[:1])
            for n in linears:
                if n not in first:
                    self.layers_cache[n] = {'share': None, 'columns': linears[n].weight.shape[1]}
            self.named_layers = linears
        else:
            self._init_layers(linears, subsets)

    # ---- GPU-first block execution: ONE progressive pass instead of five forwards ------------------
    def progressive_ok(self, block):
        """The staged whole-batch pass reproduces the reference's schedule in two cases:
          true_sequential + quant_out       : every linear sees the output of the already-quantised
                                              prefix (Appendix E-9) — quantise between stages;
          not true_sequential, not quant_out: every Hessian comes from the ONE fp forward of run()
                                              (base_blockwise_quantization.py:436-444) and the block
                                              hands its fp output on — quantise after the pass.
        (The two mixed settings re-run the block on self.input, which run() has already replaced;
        they stay on the generic hook schedule.)"""
        staged = (self.true_sequential and self.quant_out) or \
                 (not self.true_sequential and not self.quant_out)
        return (staged and not self.data_free
                and not self.act_static and hasattr(block, 'mlp') and hasattr(block, 'self_attn')
                and hasattr(block.self_attn, 'qkv_rope') and hasattr(block.mlp, 'gate_up_act'))

    @torch.no_grad()
    def block_opt(self, block):
        if self.block_idx in self._qparams_pending:      # host-resident at __init__ (BlockStreamer)
            self._qparams_pending.discard(self.block_idx)
            self.collect_block_qparams(block)
        if self.progressive_ok(block) and getattr(self, 'progressive', True):
            self.block_opt_progressive(block)
        else:
            super().block_opt(block)
        self.check_factorizations(wait=False)

    @torch.no_grad()
    def block_opt_progressive(self, block, chunk=16):
        """SURVEY.md Appendix E-9: with true_sequential + quant_out the reference runs the block
        five times over every calibration sample (run + 3x rehook_next_subset + the quant_out
        pass, base_blockwise_quantization.py:436-526).  Every linear sees exactly one distinct
        input in that schedule — the output of the already-quantised prefix — so one staged pass
        produces the same Hessians and the same block output:
            ln1 -> [H_qkv] -> quantise q,k,v -> attention -> [H_o] -> quantise o -> residual
            -> ln2 -> [H_gate/up] -> quantise -> act -> [H_down] -> quantise -> residual.
        Samples are streamed in chunks of `chunk` to bound activation memory."""
        a, m = block.self_attn, block.mlp
        subsets = self.model.get_subsets_in_block(block)
        data, kwargs = self.input['data'], self.input['kwargs']
        params = self.get_replacement_params(mode='fake_quant', w_only=self.w_only, name=None)
        # all samples as ONE [N, S, hidden] tensor: whole-batch SYRK / GEMM launches
        X = self.input.get('stacked')            # the previous block's output, already one tensor
        if X is None or X.shape[0] != sum(d.shape[0] for d in data):
            X = data[0] if len(data) == 1 else torch.cat(data, dim=0)
        N = X.shape[0]
        pos = kwargs[0].get('position_embeddings')
        bs_list = [d.shape[0] for d in data]

        between = self.quant_out          # see progressive_ok: quantise between stages, or after
        deferred = []

        def stage(subset, x_all):
            """H of the subset's shared input over all samples (one SYRK, b = N samples: the same
            running mean as N add_batch calls), quantise its linears, swap in FakeQuantLinear."""
            self.subset_init(subset)
            lead = next(iter(subset['layers']))
            cache = self.layers_cache[lead]
            cache['nsamples'] = ops.hessian_add_batch(cache['H'], cache['nsamples'], x_all)
            if not between:
                deferred.append(subset)
                return
            self.subset_transform(subset, None, None)
            self.model.replace_module_subset(FakeQuantLinear, block, subset, self.block_idx, params)

        def chunks():
            for i in range(0, N, chunk):
                yield slice(i, min(i + chunk, N))

        x1 = torch.empty_like(X)
        for s in chunks():
            norm_into(block.input_layernorm, X[s], x1[s])
        stage(subsets[0], x1)
        att = torch.empty((N, X.shape[1], a.heads * a.head_dim), dtype=X.dtype, device=X.device)
        w_fused = a.fused_qkv_weight(X.dtype)       # the stage's weights, once for every chunk
        for s in chunks():
            att[s] = a.sdpa(*a.qkv_rope(x1[s], pos, w_fused))
        del x1, w_fused
        stage(subsets[1], att)
        h = torch.empty_like(X)
        for s in chunks():
            linear_residual(a.o_proj, att[s], X[s], out=h[s])
        del att
        x3 = torch.empty_like(X)
        for s in chunks():
            norm_into(block.post_attention_layernorm, h[s], x3[s])
        stage(subsets[2], x3)
        act = torch.empty((N, X.shape[1], m.gate_proj.out_features), dtype=X.dtype, device=X.device)
        w_fused = m.fused_gate_up_weight(X.dtype)
        for s in chunks():
            m.gate_up_act(x3[s], out=act[s], w_gate_up=w_fused)
        del x3, w_fused
        stage(subsets[3], act)
        for s in chunks():
            linear_residual(m.down_proj, act[s], h[s], out=h[s])
        del act
        self.input['stacked'] = h
        self.input['data'] = list(torch.split(h, bs_list, dim=0))
        for subset in deferred:            # fp pass done: transform every subset on its fp Hessian
            self.subset_transform(subset, None, None)

    @torch.no_grad()
    def collect_model_qparams(self):
        """gptq.py:324-330 (the reference moves every block to the GPU and back for this).  Blocks
        whose weights are in host memory (BlockStreamer) are collected when they arrive in
        block_opt instead — their weights are untouched until then, so the seeds are the same."""
        self._qparams_pending = set()
        for i, block in enumerate(self.blocks):
            if all(p.is_cuda for p in block.parameters()):
                self.collect_block_qparams(block)
            else:
                self._qparams_pending.add(i)

    # ---- per-layer transform ------------------------------------------------------------------------
    @torch.no_grad()
    def subset_transform(self, subset, input_feat, subset_kwargs):
        """gptq.py:96-111.  Linears that share one Hessian (q/k/v, gate/up) are swept together:
        rows of a linear are independent given Hinv (SURVEY 8(e)), so their permuted weights are
        stacked row-wise and ONE column sweep serves them all — bit-identical per row, a third /
        half of the sequential 128-column chains."""
        groups = {}
        for name, layer in subset['layers'].items():
            if not isinstance(layer, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                continue
            groups.setdefault(self.layers_cache[name]['share'], []).append((name, layer))
        for members in groups.values():
            self._transform_group(members)
        for name in list(subset['layers']):
            self.free(name)

    def _hessian_of(self, name):
        lead = self.layers_cache[name]['share']
        cache = self.layers_cache[lead]
        if not cache.get('reduced', False):
            dist_utils.allreduce_mean_symmetric_(cache['H'])           # gptq.py:292-295, once
            cache['reduced'] = True
        return lead, cache['H']

    @torch.no_grad()
    def layer_transform(self, layer, name, shared=None):
        """gptq.py:113-196 for one linear."""
        self._transform_group([(name, layer)])

    @torch.no_grad()
    def _transform_group(self, members):
        """gptq.py:113-196 for the linears `members` = [(name, layer)] that share one Hessian."""
        name0, layer0 = members[0]
        lead, H = self._hessian_of(name0)
        wq = self.wquantizer
        Ws = []
        for _, layer in members:
            W = layer.weight.data
            Ws.append(W.flatten(1) if isinstance(layer, nn.Conv2d) else W)
        C = Ws[0].shape[1]
        assert all(W.shape[1] == C for W in Ws)
        Rs = [W.shape[0] for W in Ws]
        R = sum(Rs)
        offs = [0]
        for r in Rs:
            offs.append(offs[-1] + r)
        gran = wq.granularity
        group = wq.group_size if gran == 'per_group' else C
        ng = C // group
        # hessian_sorting (:58-64), dead columns, damping, Cholesky triple: depend on H only
        perm = torch.argsort(torch.diag(H), descending=True) if self.actorder else None
        invperm = torch.argsort(perm) if perm is not None else None
        Wp = torch.empty((R, C), dtype=torch.float32, device=H.device)
        Hp = None
        for i, W in enumerate(Ws):
            _, hp = ops.prepare(W, H, perm, self.percdamp, want_h=(i == 0), wp_out=Wp[offs[i]:offs[i + 1]])
            Hp = hp if i == 0 else Hp
        Hinv, info = ops.chol_inv_upper(Hp, return_info=True, inplace=True)
        self._chol_infos.append((f'{self.block_idx}.{lead}', info))
        del Hp
        static, gmap = None, None
        if gran != 'per_group' or self.static_groups:
            parts = [self._static_qparams(layer, r, ng) for (_, layer), r in zip(members, Rs)]
            zs = [p[1] for p in parts]
            static = (torch.cat([p[0] for p in parts]) if len(parts) > 1 else parts[0][0],
                      None if zs[0] is None else (torch.cat(zs) if len(zs) > 1 else zs[0]))
            if gran == 'per_group' and perm is not None:
                gmap = (perm // group).to(torch.int32)
        # N > 1: rows are independent given Hinv, so each rank sweeps R/world rows and the results
        # are all-gathered (bit-identical to sweeping all rows on every rank)
        bounds = dist_utils.row_shard(R) if getattr(self, 'row_sharded_sweep', True) else None
        if bounds is None:
            tmp, losses, scales, zeros = ops.weight_transform(
                Wp, Hinv, wq.bit, wq.sym, group, static_qparams=static, gmap=gmap, out_perm=perm)
        else:
            lo, hi = bounds
            st_l = None
            if static is not None:
                st_l = (static[0].reshape(R, -1)[lo:hi].reshape(-1).contiguous(),
                        None if static[1] is None else
                        static[1].reshape(R, -1)[lo:hi].reshape(-1).contiguous())
            tmp_l, losses_l, scales_l, zeros_l = ops.weight_transform(
                Wp[lo:hi], Hinv, wq.bit, wq.sym, group, static_qparams=st_l, gmap=gmap,
                out_perm=perm)
            with dist_utils.comm_span('allgather_rows', tmp_l, world_factor=True):
                tmp = dist_utils.all_gather_rows(tmp_l, R)
                losses = dist_utils.all_gather_rows(losses_l, R)
                scales, zeros = (static if static is not None else (None, None))
                if static is None:
                    scales = dist_utils.all_gather_rows(scales_l.reshape(hi - lo, ng), R)
                    zeros = None if zeros_l is None else \
                        dist_utils.all_gather_rows(zeros_l.reshape(hi - lo, ng), R)
        del Wp, Hinv
        for i, (name, layer) in enumerate(members):
            r0, r1 = offs[i], offs[i + 1]
            if self.actorder:
                layer.register_buffer('buf_perm', perm)
                layer.register_buffer('buf_invperm', invperm)
            self.losses[f'{self.block_idx}.{name}'] = losses[r0:r1]   # summed lazily: no host sync
            layer.weight.data = tmp[r0:r1].reshape(layer.weight.shape)  # fp32 until convert_dtype (:193)
            if gran == 'per_group' and not self.static_groups:        # update_model_qparams (:397-409)
                layer.buf_scales = scales.reshape(R, ng)[r0:r1].reshape(-1, 1)
                if not wq.sym:
                    layer.buf_zeros = zeros.reshape(R, ng)[r0:r1].reshape(-1, 1)
            elif self.float_grid:
                # FloatQuantizer.quant sets zero scales to 1 IN PLACE (quant.py:1062), and the sweep
                # hands it the layer's own buf_scales (search_layer_qparams / search_group_qparams,
                # gptq.py:368-395): a 16-bit scale that underflowed to 0 stays 1 for deploy / export
                layer.buf_scales.masked_fill_(layer.buf_scales == 0, 1)

    def _static_qparams(self, layer, R, ng):
        """The kernel indexes static qparams as [row * ng + group]; expand what
        collect_block_qparams stored for the coarser granularities the way broadcasting does in
        the reference's quant_dequant (merge_qparams, gptq.py:338-352)."""
        def expand(t):
            t = t.to(layer.weight.device)
            if t.numel() == R * ng:
                return t.reshape(-1)
            if t.numel() == 1:                                     # per_tensor
                return t.reshape(1).expand(R * ng).contiguous()
            if self.wquantizer.granularity == 'per_head' and ng == 1 and R % t.numel() == 0:
                # [head_num, 1] over weight.reshape(head_num, -1): R/head_num consecutive rows
                return t.reshape(-1).repeat_interleave(R // t.numel())
            raise NotImplementedError(
                f'GPTQ static qparams of {t.numel()} elements for a [{R} x {ng} groups] sweep '
                f'(granularity {self.wquantizer.granularity})')
        scales = expand(layer.buf_scales)
        z = getattr(layer, 'buf_zeros', None)
        zeros = None
        if torch.is_tensor(z) and not self.wquantizer.sym:
            zeros = expand(z)
        assert scales.numel() == R * ng
        return scales, zeros

    def check_factorizations(self, wait=True):
        """The reference's torch.linalg.cholesky raises on a non-SPD damped Hessian
        (gptq.py:172).  llmc_chol_inv_upper reports the failing leading minor in a device flag;
        the flags of a block are copied to pinned memory asynchronously at the end of block_opt
        and read one block late (or here, with wait=True), so the sweep never stalls on them."""
        if self._chol_infos:
            names = [n for n, _ in self._chol_infos]
            dev_flags = torch.cat([t for _, t in self._chol_infos])
            host = torch.empty(dev_flags.shape, dtype=dev_flags.dtype, pin_memory=True)
            host.copy_(dev_flags, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev_flags.device))
            self._chol_pending.append((names, host, ev))
            self._chol_infos = []
        keep = 0 if wait else 1
        while len(self._chol_pending) > keep:
            names, host, ev = self._chol_pending.pop(0)
            ev.synchronize()
            bad = [(n, int(v)) for n, v in zip(names, host.tolist()) if v != 0]
            if bad:
                n, k = bad[0]
                raise torch.linalg.LinAlgError(
                    f'GPTQ: the damped Hessian of {n} is not positive-definite (leading minor of '
                    f'order {k}); {len(bad)} factorisation(s) failed')

    def run_block_loop(self, *a, **kw):
        super().run_block_loop(*a, **kw)
        self.check_factorizations(wait=True)

    def layer_loss(self, key):
        self.check_factorizations(wait=True)
        return float(self.losses[key].double().sum().item())

    # ---- deploy-time callbacks --------------------------------------------------------------------------
    @torch.no_grad()
    def w_q(self, module, wquantizer):
        """gptq.py:411-422."""
        args = {'scales': module.buf_scales.to(self.model_dtype), 'zeros': module.buf_zeros,
                'qmax': module.buf_qmax, 'qmin': module.buf_qmin}
        return wquantizer.real_quant_weight_static(module.weight.data, args)

    @torch.no_grad()
    def w_qdq(self, module, wquantizer):
        """gptq.py:424-452: W[:, perm] -> static qdq -> model dtype -> [:, invperm], one pass."""
        if self.float_grid:
            # the FP8 static kernel has no group map: the column gathers of gptq.py:427-450 as written
            w = module.weight.data
            if self.need_perm:
                w = w[:, module.buf_perm]
            w = wquantizer.fake_quant_weight_static(w, {'scales': module.buf_scales}).to(self.model_dtype)
            return w[:, module.buf_invperm] if self.need_perm else w
        args = {'scales': module.buf_scales,
                'zeros': module.buf_zeros if hasattr(module, 'buf_zeros') else None,
                'qmax': module.buf_qmax, 'qmin': module.buf_qmin, 'out_dtype': self.model_dtype}
        if self.need_perm:
            args['gmap'] = (module.buf_invperm // wquantizer.group_size).to(torch.int32)
        return wquantizer.fake_quant_weight_static(module.weight.data, args)

    @torch.no_grad()
    def w_packed(self, module, wquantizer):
        """The packed form of exactly what `w_qdq` materialises, for EffcientFakeQuantLinear: codes of
        the calibrated fp32 weight (original column order) from the same static quantisation pass
        w_qdq runs, packed for llmc_gemm_w2a16 / w3a16 / w4a16 / w8a16; qparams as GPTQ stores them
        (dynamic groups: fp32 in the permuted group order; static groups and per-channel: the model
        dtype, original order); `g_idx` = invperm // group_size when act-order reorders the groups.  None when the
        layer does not fit the packed GEMM; it is then materialised as before."""
        from .module_utils import pack_unsigned_codes
        from .quant import OUT_CODES_I32, IntegerQuantizer
        q, w = wquantizer, module.weight.data
        if self.float_grid:
            return self._fp8_packed_static(module, q)
        if not (isinstance(q, IntegerQuantizer) and q.bit in (2, 3, 4, 8) and q.calib_algo == 'minmax'
                and q.granularity in ('per_group', 'per_channel') and q.round_zp
                and w.dim() == 2 and w.is_cuda and w.is_floating_point()
                and self.model_dtype in (torch.float16, torch.bfloat16)):
            return None
        R, K = w.shape
        group = q.group_size if q.granularity == 'per_group' else K
        if K % 64 or K % group or (not self.need_perm and group % 64):
            return None
        scales = module.buf_scales.to(w.device).reshape(R, -1)
        ng = scales.shape[1]
        zeros = getattr(module, 'buf_zeros', None) if not q.sym else None
        if ng != K // group or scales.dtype not in (torch.float32, self.model_dtype):
            return None
        if zeros is not None:
            zeros = zeros.to(device=w.device, dtype=scales.dtype).reshape(R, ng)
        g_idx = (module.buf_invperm // group).to(torch.int32) if self.need_perm else None
        codes = torch.empty((R, K), dtype=torch.int32, device=w.device)
        q._static(w, scales.reshape(-1), zeros, module.buf_qmax, module.buf_qmin, OUT_CODES_I32, codes,
                  self.model_dtype, ng, group, gmap=g_idx)
        return dict(qweight=pack_unsigned_codes(codes, q.bit, signed=q.sym), scales=scales.contiguous(),
                    zeros=None if zeros is None else zeros.contiguous(), bits=q.bit, group=group,
                    dtype=self.model_dtype, g_idx=g_idx)

    def _fp8_packed_static(self, module, q):
        """w_packed on an e4m3 / e5m2 grid: the bytes of w_qdq's static pass on W[:, perm] (byte mode
        instead of QDQ mode), gathered back with [:, invperm]; the scales as that pass reads them —
        buf_scales in the weight's dtype (fp32 until convert_dtype), a per-tensor scale as fp32, one per
        row — so that fp32(byte) * s rounds once to the model dtype exactly as w_qdq's
        `.to(model_dtype)` does.  g_idx = invperm // group_size under act-order."""
        w = module.weight.data
        if not (q.granularity in ('per_tensor', 'per_channel', 'per_group') and w.dim() == 2 and w.is_cuda
                and w.dtype in (torch.float32, self.model_dtype)
                and self.model_dtype in (torch.float16, torch.bfloat16)):
            return None
        R, K = w.shape
        group = q.group_size if q.granularity == 'per_group' else K
        if K % 64 or K % group or (not self.need_perm and group % 64):
            return None
        s = module.buf_scales.to(w.device)
        if s.numel() == 1:
            scales = s.reshape(1).float().expand(R, 1).contiguous()
        else:
            scales = s.reshape(R, -1).to(w.dtype).contiguous()
        if scales.shape[1] != K // group:
            return None
        src = w[:, module.buf_perm] if self.need_perm else w
        wq = q._static(src, module.buf_scales, 2).reshape(R, K)
        g_idx = None
        if self.need_perm:
            wq = wq.view(torch.uint8)[:, module.buf_invperm].view(wq.dtype)
            g_idx = (module.buf_invperm // group).to(torch.int32)
        return dict(qweight=wq.contiguous(), scales=scales, zeros=None, bits=8, group=group,
                    dtype=self.model_dtype, g_idx=g_idx)

    @torch.no_grad()
    def deploy(self, quant_format):
        """gptq.py:454-459."""
        self.check_factorizations(wait=True)
        if quant_format not in ['fake_quant', 'origin_float']:
            assert not self.need_perm
        super().deploy(quant_format)
        self.model.convert_dtype(self.model_dtype)

    @torch.no_grad()
    def free(self, name):
        """gptq.py:466-472."""
        self.layers_cache.pop(name, None)
