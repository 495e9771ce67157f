"""AWQ — mirror of llmc/compression/quantization/awq.py (class Awq :28-372) and
auto_clip.py (class AutoClipper :22-281) on the CUDA kernels, plus the scale-migration helpers of
base_blockwise_quantization.py (:596-778, :876-897).

Same YAML knobs (`special: trans, trans_version, weight_clip, clip_sym, clip_version, save_scale,
awq_bs`), same 20-point grid, same selection rule (running weighted loss, strict `<`, updated
inside the batch loop, awq.py:245-248).  What changes is how the numbers are produced:
  * `W*s -> group fake-quant` is ONE pass (llmc_quant_dynamic col_scale) that never modifies the
    module weights, so the reference's per-step `load_state_dict` from a CPU copy (awq.py:199,244)
    disappears while each grid step still starts from the original weights;
  * x / s, |x| column means and the MSE are single kernels; losses and the running best stay on
    the device (the reference synchronises with `.item()` every grid step);
  * the per-input |x| mean is computed once per subset (the reference recomputes it 20 times);
  * module forwards run on the wgmma GEMM through the swapped weights;
  * auto-clip evaluates its 10 shrink levels in one kernel without the [256, 512, ng, g]
    broadcast temporaries (auto_clip.py:127-179).
"""
import torch
import torch.distributed as dist
import torch.nn as nn

from . import dist_utils
from ._lib import call, dtype_enum, ptr, require_cuda, stream_ptr
from .blockwise import ALGO_REGISTRY, BaseBlockwiseQuantization
from .gptq_ops import _workspace
from .module_utils import _LLMC_LINEAR_TYPES_, _TRANSFORMERS_LINEAR_TYPES_, FakeQuantLinear
from .prof import TIMER
from .quant import OUT_QDQ

_LN_TYPES = (nn.LayerNorm,)


def _is_norm(m):
    return isinstance(m, _LN_TYPES) or type(m).__name__.endswith('RMSNorm') or \
        type(m).__name__.endswith('LayerNorm')


# ---- tensor ops -----------------------------------------------------------------------------------
def absmean_cols(x):
    """awq.py:74-85: x.abs().view(-1, C).mean(0), dtype of x."""
    require_cuda(x)
    x2 = x.reshape(-1, x.shape[-1])
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    T, C = x2.shape
    out = torch.empty(C, dtype=x.dtype, device=x.device)
    nfl = 256 * C
    ws = _workspace(nfl * 4, x.device, 'awq_f32')
    with TIMER.span('awq_absmean', nbytes=float(x2.element_size()) * T * C):
        call('llmc_absmean_cols', ptr(x2), T, C, dtype_enum(x.dtype), ptr(out), ptr(ws), nfl,
             stream_ptr(x.device))
    return out


def div_cols(x, s):
    """base_blockwise_quantization.py:876-889: x / s.view(1, -1)."""
    require_cuda(x, s)
    x2 = x.reshape(-1, x.shape[-1])
    x2 = x2 if x2.is_contiguous() else x2.contiguous()
    s = s.to(x.dtype).contiguous()
    out = torch.empty_like(x2)
    with TIMER.span('awq_div_cols', nbytes=2.0 * x2.element_size() * x2.numel()):
        call('llmc_div_cols', ptr(x2), ptr(s), x2.shape[0], x2.shape[1], dtype_enum(x.dtype),
             ptr(out), stream_ptr(x.device))
    return out.reshape(x.shape)


def mse(a, b):
    """awq.py:134-145 for one batch: (a - b).float().pow(2).mean() as a DEVICE fp32 scalar."""
    require_cuda(a, b)
    assert a.shape == b.shape and a.dtype == b.dtype
    a = a if a.is_contiguous() else a.contiguous()
    b = b if b.is_contiguous() else b.contiguous()
    out = torch.empty(1, dtype=torch.float32, device=a.device)
    ws = _workspace(1024 * 4, a.device, 'awq_mse')
    with TIMER.span('awq_mse', nbytes=2.0 * a.element_size() * a.numel()):
        call('llmc_mse', ptr(a), ptr(b), a.numel(), dtype_enum(a.dtype), ptr(out), ptr(ws),
             stream_ptr(a.device))
    return out[0]


def scaled_fake_quant(wquantizer, weight, scales):
    """awq.py:147-164: fake_quant_weight_dynamic(W.mul_(s.view(1, -1))) without touching W."""
    src = weight if weight.is_contiguous() else weight.contiguous()
    out = torch.empty_like(src)
    cs = scales.to(src.dtype).contiguous()
    wquantizer._dynamic(src, OUT_QDQ, out=out, out_dtype=src.dtype, col_scale=cs)
    return out


# ---- AutoClipper (auto_clip.py) -----------------------------------------------------------------------
class AutoClipper:
    def __init__(self, w_only, wquantizer, aquantizer, clip_version, clip_sym, save_clip,
                 padding_mask):
        self.wquantizer, self.aquantizer = wquantizer, aquantizer
        self.clip_version, self.clip_sym = clip_version, clip_sym
        self.save_clip, self.padding_mask, self.w_only = save_clip, padding_mask, w_only
        self.weight_clips = {}
        if clip_version != 'v1':
            raise NotImplementedError('clip_version v2 (learnable bound factors, auto_clip.py:212-256)')
        if not w_only:
            raise NotImplementedError('auto-clip with activation fake-quant (auto_clip.py:276-281)')

    @torch.no_grad()
    def run(self, block, block_idx, input_feat, n_sample_token):
        """auto_clip.py:43-81."""
        for n, m in block.named_modules():
            if not isinstance(m, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
                continue
            if any(k in n for k in ['q_', 'k_', 'query', 'key', 'Wqkv']):
                continue
            inputs = [torch.cat(input_feat[n])] if len(input_feat[n]) != 1 else input_feat[n]
            max_val, min_val = self.auto_clip_layer(block_idx, n, m.weight, inputs,
                                                    n_sample_token=n_sample_token)
            if dist_utils.world() > 1:
                for t in (max_val, min_val):
                    dist.all_reduce(t, op=dist.ReduceOp.SUM)
                    t /= dist_utils.world()
            self.apply_clip(block_idx, m, min_val, max_val, n)

    @torch.no_grad()
    def auto_clip_layer(self, block_idx, layer_name, w, inputs, n_grid=20, max_shrink=0.5,
                        n_sample_token=512, eps=0.0):
        """auto_clip.py:83-191 -> (best_max [R, ng, 1], best_min [R, ng, 1])."""
        assert w.dim() == 2 and n_grid == 20 and max_shrink == 0.5
        require_cuda(w)
        q = self.wquantizer
        group = q.group_size if q.granularity == 'per_group' else w.shape[1]
        R, C = w.shape
        assert len(inputs) == 1, 'inputs are concatenated by run() (auto_clip.py:60-64)'
        x = inputs[0].reshape(-1, C)
        if self.padding_mask and self.padding_mask[0].numel() == x.shape[0]:
            # auto_clip.py:136-138 — as in the reference this only matches a single (bs: -1) batch:
            # run() has already concatenated multi-batch inputs
            x = x[self.padding_mask[0].flatten().bool().to(x.device)]
        if n_sample_token is None:
            n_sample_token = min(x.shape[0], 512)
        step = max(1, x.shape[0] // n_sample_token)
        xs = x[0::step].contiguous()                      # auto_clip.py:144-147
        ns = xs.shape[0]
        ng = C // group
        wc = w.data if w.data.is_contiguous() else w.data.contiguous()
        best_max = torch.empty((R, ng, 1), dtype=w.dtype, device=w.device)
        best_min = torch.empty_like(best_max)
        nfl = R * ng * 10
        ws = _workspace(nfl * 4, w.device, 'awq_clip')
        with TIMER.span('awq_clip', flops=2.0 * 11 * ns * R * C):
            call('llmc_awq_clip', ptr(wc), R, C, ptr(xs), ns, dtype_enum(w.dtype), int(group),
                 int(q.bit), int(bool(q.sym)), int(bool(self.clip_sym)), ptr(best_max),
                 ptr(best_min), ptr(ws), nfl, stream_ptr(w.device))
        return best_max, best_min

    @torch.no_grad()
    def apply_clip(self, block_idx, layer, min_val, max_val, layer_name):
        """auto_clip.py:193-211 (v1): one elementwise clamp per layer."""
        org_shape = layer.weight.shape
        w = layer.weight.data.reshape(*max_val.shape[:2], -1)
        if self.clip_sym:
            min_val = -max_val
        layer.weight.data = torch.clamp(w, min_val, max_val).reshape(org_shape)


# ---- Awq ---------------------------------------------------------------------------------------------------
@ALGO_REGISTRY
class Awq(BaseBlockwiseQuantization):
    def __init__(self, model, quant_config, input, padding_mask, config):
        super().__init__(model, quant_config, input, padding_mask, config)
        sp = self.quant_config.get('special', {}) or {}
        self.trans = sp.get('trans', True)
        self.trans_version = sp.get('trans_version', 'v2')
        self.save_scale = sp.get('save_scale', False)
        self.awq_bs = sp.get('awq_bs', None)
        self.save_mem = sp.get('save_mem', True)
        self.weight_clip = sp.get('weight_clip', True)          # base_bq.py:223-240
        self.clip_version = sp.get('clip_version', 'v1')
        self.clip_sym = sp.get('clip_sym', self.wquantizer.sym)
        self.act_scales = {}
        # base_bq.py:267-284: GQA v_proj -> o_proj migration with the kv scales repeated per group
        self.do_gqa_trans = bool(sp.get('do_gqa_trans', False))
        shape = getattr(self.model, 'shape', None) or {}
        self.num_heads = int(shape.get('heads', 0) or 0)
        self.num_key_value_heads = int(shape.get('kv_heads', self.num_heads) or 0)
        self.head_dim = (int(shape.get('hidden', 0)) // self.num_heads) if self.num_heads else 0
        self.num_key_value_groups = (self.num_heads // self.num_key_value_heads) if self.num_key_value_heads else 1
        self.has_gqa = self.num_key_value_groups > 1
        if self.weight_clip:
            self.auto_clipper = AutoClipper(self.w_only, self.wquantizer, self.aquantizer,
                                            self.clip_version, self.clip_sym,
                                            sp.get('save_clip', False), padding_mask)
        self.search_log = {}      # '<block>.<input_name>' -> device tensor of the 20 losses

    # -- pieces of search_scale_subset -------------------------------------------------------------------
    def get_weight_scale(self, layers_dict):
        """awq.py:48-72; only trans_version v1 consumes it — a handful of elementwise torch ops on
        the device (not worth a kernel: v2, the shipped default, never reads the result)."""
        total = None
        for m in layers_dict.values():
            w = m.weight.data.clone()
            shape = w.shape
            r = self.wquantizer.reshape_tensor(w)
            a = r.abs()
            ls = a.div_(a.amax(dim=1, keepdim=True)).view(shape)
            total = ls.mean(0) if total is None else total.add_(ls.mean(0))
        return total.div_(len(layers_dict))

    def get_act_scale(self, x):
        """awq.py:74-85 (batch loop included: mean of per-_bs-chunk means)."""
        if x.shape[0] == self._bs:
            return absmean_cols(x)
        b_num = x.shape[0] // self._bs
        means = [absmean_cols(x[i * self._bs:(i + 1) * self._bs]) for i in range(b_num)]
        return sum(means) / len(means)

    @torch.no_grad()
    def repeat_gqa_scales(self, scales):
        """base_bq.py:591-594: [kv_heads * head_dim] -> [1, heads, head_dim], every kv head's
        scales repeated for the query heads of its group."""
        scales = scales.view(1, self.num_key_value_heads, self.head_dim)
        return torch.repeat_interleave(scales, dim=1, repeats=self.num_key_value_groups)

    @torch.no_grad()
    def get_scales(self, prev_op, x, w_max, is_gqa, ratio, x_mean=None):
        """awq.py:87-108; `x_mean` lets the caller reuse get_act_scale(x) — for is_gqa
        get_act_scale(prev_op(x)), the statistics of v_proj's OUTPUT — across the grid."""
        if x_mean is None:
            x_mean = self.get_act_scale(prev_op(x) if is_gqa else x)
        x_tmp = x_mean
        if self.trans_version == 'v1' and not is_gqa:
            scales = (x_tmp.pow(ratio) / w_max.pow(1 - ratio)).clamp(min=1e-4).view(-1)
        else:
            scales = x_tmp.pow(ratio).clamp(min=1e-4).view(-1)
        return scales / (scales.max() * scales.min()).sqrt()

    def inspect_module_forward(self, x, inspect_module, kwargs):
        """awq.py:110-126."""
        def run(t):
            out = inspect_module(t, **kwargs)
            return out[0] if isinstance(out, tuple) else out
        if self._bs == x.shape[0]:
            return run(x)
        b_num = x.shape[0] // self._bs
        return torch.cat([run(x[i * self._bs:(i + 1) * self._bs]) for i in range(b_num)], dim=0)

    def calculate_loss(self, org_out, out):
        """awq.py:134-145 -> device scalar."""
        if out.shape[0] == self._bs:
            return mse(org_out, out)
        b_num = org_out.shape[0] // self._bs
        tot = sum(mse(org_out[i * self._bs:(i + 1) * self._bs], out[i * self._bs:(i + 1) * self._bs])
                  for i in range(b_num))
        return tot / b_num

    def scaling_input(self, x, scales, is_gqa=False):
        """base_bq.py:876-889."""
        if is_gqa:
            scales = self.repeat_gqa_scales(scales).reshape(-1)
        return div_cols(x, scales)

    @torch.no_grad()
    def search_scale_subset(self, prev_op, layers_dict, input, inspect_module, is_gqa, subset_kwargs):
        """awq.py:178-278."""
        self._bs = input[0].shape[0] if self.awq_bs is None else self.awq_bs
        w_max = self.get_weight_scale(layers_dict) if self.trans_version == 'v1' else None
        dev = input[0].device
        n_grid = 20
        best_error = torch.full((), float('inf'), device=dev)
        best_scales = None
        org_w = {name: fc.weight.data for name, fc in layers_dict.items()}
        org_out, x_means = {}, {}
        losses_log = []
        try:
            for n in range(n_grid):
                loss_mean = torch.zeros((), device=dev)
                scales_mean = 0
                for i in range(len(input)):
                    x = input[i]
                    kwargs = subset_kwargs[i] if isinstance(subset_kwargs, list) else subset_kwargs
                    if i not in org_out:
                        for name, fc in layers_dict.items():
                            fc.weight.data = org_w[name]
                        org_out[i] = self.inspect_module_forward(x, inspect_module, kwargs)
                        x_means[i] = self.get_act_scale(prev_op(x) if is_gqa else x)   # awq.py:89-96
                    ratio = n * 1 / n_grid
                    scales = self.get_scales(prev_op, x, w_max, is_gqa, ratio, x_mean=x_means[i])
                    # awq.py:40-46: the weight columns see the kv scales repeated per query group
                    w_scales = self.repeat_gqa_scales(scales).reshape(-1) if is_gqa else scales
                    for name, fc in layers_dict.items():
                        fc.weight.data = scaled_fake_quant(self.wquantizer, org_w[name], w_scales)
                    x_tmp = self.scaling_input(x, scales, is_gqa)
                    if not self.w_only:
                        x_tmp = self.aquantizer.fake_quant_act_dynamic(x_tmp)
                    out = self.inspect_module_forward(x_tmp, inspect_module, kwargs)
                    oo = org_out[i]
                    if self.padding_mask and oo.shape[1] == self.padding_mask[i].shape[-1]:
                        pm = self.padding_mask[i].unsqueeze(dim=-1).to(oo.device)   # awq.py:231-233
                        oo, out = oo * pm, out * pm
                    loss = self.calculate_loss(oo, out)
                    n_samples = x.shape[0] if len(input) == 1 else self.n_samples
                    wgt = x.shape[0] * 1.0 / n_samples
                    loss_mean = loss_mean + wgt * loss
                    scales_mean = scales_mean + wgt * scales
                    is_best = loss_mean < best_error                  # awq.py:245-248, on device
                    best_error = torch.where(is_best, loss_mean, best_error)
                    best_scales = scales_mean if best_scales is None else \
                        torch.where(is_best, scales_mean, best_scales)
                losses_log.append(loss_mean)
        finally:
            for name, fc in layers_dict.items():
                fc.weight.data = org_w[name]                           # "load_state_dict(org_sd)"
        self._last_losses = torch.stack(losses_log)
        if dist_utils.world() > 1:
            # awq.py:255-273: global MIN of the best error, broadcast of the winner's scales
            err = best_error.reshape(1).clone()
            dist.all_reduce(err, op=dist.ReduceOp.MIN)
            mine = (best_error.reshape(1) - err).abs() < 1e-5
            r = torch.where(mine, torch.tensor([dist_utils.rank()], device=dev),
                            torch.tensor([-1], device=dev))
            dist.all_reduce(r, op=dist.ReduceOp.MAX)
            src = int(r.item())
            if src < 0 or best_scales is None:
                raise RuntimeError('AWQ scale search: no finite loss on any rank (NaN outputs?)')
            dist.broadcast(best_scales, src=src)
        return best_scales

    # -- scale migration (base_blockwise_quantization.py:596-778) -----------------------------------------
    @torch.no_grad()
    def apply_scale(self, scales, prev_op, layers):
        assert len(prev_op) == 1
        p = prev_op[0]
        if isinstance(p, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_)):
            assert len(layers) == 1
            self.scale_fc_fc(p, layers[0], scales)
        elif _is_norm(p):
            self.scale_ln_fcs(p, layers, scales)
        else:
            raise NotImplementedError(f'prev_op {type(p)} not supported yet!')

    @torch.no_grad()
    def scale_fc_fc(self, fc1, fc2, scales):
        """base_bq.py:631-700 (out_features == in_features * {1, 2, 3}, or the GQA-repeat branch
        :678-685 under `do_gqa_trans`)."""
        scales = scales.to(fc1.weight.device)
        if fc1.out_features == fc2.in_features * 3:
            # fused qkv -> out_proj (:633-653): only the V third of every head is divided
            num_heads = self.model.get_num_attention_heads()
            W = fc1.weight.data.t()                                  # [in, 3 * hidden]
            org_shape = W.shape
            W3 = W.reshape(org_shape[0] * num_heads, 3, -1).clone()
            value = W3[:, 2, :].reshape(org_shape[0], -1)
            W3[:, 2, :] = value.div(scales.view(-1)).reshape(W3[:, 2, :].shape)
            fc1.weight.data = W3.reshape(org_shape).t().contiguous()
            if getattr(fc1, 'bias', None) is not None:
                b3 = fc1.bias.data.reshape(num_heads, 3, -1).clone()
                b3[:, 2, :] = b3[:, 2, :].reshape(-1).div(scales.view(-1)).reshape(b3[:, 2, :].shape)
                fc1.bias.data = b3.reshape(-1)
        elif fc1.out_features == fc2.in_features * 2:
            fc1.weight.data[fc1.weight.data.shape[0] // 2:].div_(scales.view(-1, 1))
            if getattr(fc1, 'bias', None) is not None:
                fc1.bias.data[fc1.bias.data.shape[0] // 2:].div_(scales.view(-1))
        elif fc1.out_features == fc2.in_features:
            if getattr(fc1, 'bias', None) is not None:
                fc1.bias.div_(scales.view(-1))
            fc1.weight.div_(scales.view(-1, 1))
        elif self.has_gqa and self.do_gqa_trans:
            if getattr(fc1, 'bias', None) is not None:
                fc1.bias.div_(scales.view(-1))
            fc1.weight.div_(scales.view(-1, 1))
            if fc1.out_features != fc2.in_features:
                scales = self.repeat_gqa_scales(scales)
        else:
            raise Exception('Can not scale this fc-fc.')
        fc2.weight.mul_(scales.view(1, -1))

    @torch.no_grad()
    def scale_ln_fcs(self, ln, fcs, scales):
        """base_bq.py:749-778."""
        if not isinstance(fcs, list):
            fcs = [fcs]
        scales = scales.to(ln.weight.device).to(ln.weight.dtype)
        ln.weight.div_(scales)
        if getattr(ln, 'bias', None) is not None:
            ln.bias.div_(scales)
        for fc in fcs:
            fc.weight.mul_(scales.view(1, -1))

    @torch.no_grad()
    def update_input_feat(self, scale, input_feat, layers_dict, is_gqa=False):
        """base_bq.py:891-897."""
        for name in layers_dict:
            for i in range(len(input_feat[name])):
                input_feat[name][i] = self.scaling_input(input_feat[name][i], scale, is_gqa)

    # -- framework hooks ---------------------------------------------------------------------------------
    @torch.no_grad()
    def block_transform(self, block, input_feat, block_kwargs):
        """awq.py:280-296."""
        if self.trans:
            super().block_transform(block, input_feat, block_kwargs)
        if self.weight_clip:
            self.auto_clipper.run(block, self.block_idx, input_feat,
                                  n_sample_token=(self.config.get('calib', {}) or {}).get('seq_len', None))

    @torch.no_grad()
    def subset_transform(self, subset, input_feat, subset_kwargs):
        """awq.py:298-372."""
        layers_dict, prev_op = subset['layers'], subset['prev_op']
        input_name, inspect_module = subset['input'][0], subset['inspect']
        if not subset.get('do_trans', True):
            return
        assert len(prev_op) in (0, 1), 'Only support single prev_op.'
        if len(prev_op) == 0 or prev_op[0] is None:
            return
        p = prev_op[0]
        is_linear = isinstance(p, tuple(_LLMC_LINEAR_TYPES_ + _TRANSFORMERS_LINEAR_TYPES_))
        if not (is_linear or _is_norm(p)):
            return
        layers = list(layers_dict.values())
        is_gqa = False
        if is_linear and p.out_features not in (layers[0].in_features * 3, layers[0].in_features * 2,
                                                layers[0].in_features):
            if not (self.has_gqa and self.do_gqa_trans):
                return    # GQA v_proj -> o_proj: "Cannot apply scale" (awq.py:349-352)
            # awq.py:345-348: the search then runs on the PREVIOUS entry of input_feat (the
            # q/k/v input) — the reference's behaviour, reproduced as is
            is_gqa = True
            keys = list(input_feat.keys())
            input_name = keys[keys.index(input_name) - 1]
        scale = self.search_scale_subset(p, layers_dict, input_feat[input_name], inspect_module,
                                         is_gqa, subset_kwargs)
        self.search_log[f'{self.block_idx}.{next(iter(layers_dict))}'] = self._last_losses
        self.apply_scale(scale, prev_op, layers)
        self.update_input_feat(scale, input_feat, layers_dict, is_gqa)
        if self.save_scale:
            for n in layers_dict:
                self.act_scales[f'{self.model.block_name_prefix}.{self.block_idx}.{n}'] = scale
