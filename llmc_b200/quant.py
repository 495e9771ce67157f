"""Quantizers — host-side mirror of llmc/compression/quantization/quant.py.

Same constructor kwargs, method names, argument meaning, return shapes/dtypes and error
behaviour as the reference's `BaseQuantizer` / `IntegerQuantizer` (quant.py:46-960) and
`FloatQuantizer` (:963-1229), so `quant.weight` / `quant.act` YAML dicts construct them
unchanged (base_blockwise_quantization.py:150-179).  The arithmetic runs in the sm_90a
kernels of libllmc_b200.so (csrc/quant.cu) through the C ABI; tensors must live on a CUDA
device — there is no CPU path here (the CPU restatement is oracle/, test-only).
"""
import ctypes

import torch

from . import _lib
from .prof import TIMER
from ._lib import (OUT_CODES_I8, OUT_CODES_I32, OUT_CODES_U8, OUT_NONE, OUT_PACK_VLLM,
                   OUT_QDQ, call, dtype_enum, ptr, require_cuda, stream_ptr)


def ceil_div(a, b):
    return (a + b - 1) // b


def _as_int(v):
    return int(v.item()) if torch.is_tensor(v) else int(v)


class BaseQuantizer(object):
    """quant.py:46-101 — parses the YAML kwargs; range-search knobs are kept for API parity."""

    def __init__(self, bit, symmetric, granularity, **kwargs):
        self.bit = bit
        self.sym = symmetric
        self.granularity = granularity
        self.kwargs = kwargs
        self.calib_algo = kwargs.get('calib_algo', 'minmax')
        if granularity == 'per_group':
            self.group_size = kwargs['group_size']
        elif granularity == 'per_head':
            self.head_num = kwargs['head_num']
        elif granularity == 'per_block':
            assert self.calib_algo == 'minmax' and self.sym
            self.block_size = kwargs['block_size']
        if kwargs.get('ste', False) or kwargs.get('ste_all', False):
            raise NotImplementedError(
                'straight-through rounding is a training-time feature (quant.py:63-71); the '
                'the CUDA kernels implement inference-time round-half-even only')
        self.round_func = torch.round
        self.ste_all = False
        self.round_zp = kwargs.get('round_zp', True)
        self.mse_b_num = kwargs.get('mse_b_num', 1)
        self.maxshrink = kwargs.get('maxshrink', 0.8)
        self.mse_grid = kwargs.get('mse_grid', 100)
        self.bins = kwargs.get('bins', 2048)
        self.sigmoid = torch.nn.Sigmoid()

    # ---- layout helpers (quant.py:612-658); pure views, no arithmetic -----------------------
    def reshape_tensor(self, tensor, allow_padding=False):
        if self.granularity == 'per_group':
            if tensor.shape[-1] >= self.group_size:
                if tensor.shape[-1] % self.group_size == 0:
                    return tensor.reshape(-1, self.group_size)
                if allow_padding:
                    deficiency = self.group_size - tensor.shape[1] % self.group_size
                    pad = torch.zeros((*tensor.shape[:-1], deficiency), device=tensor.device,
                                      dtype=tensor.dtype)
                    return torch.cat((tensor, pad), dim=-1).reshape(-1, self.group_size)
                raise ValueError(f'Dimension {tensor.shape[-1]} '
                                 f'not divisible by group size {self.group_size}')
            return tensor
        if self.granularity == 'per_head':
            return tensor.reshape(self.head_num, -1)
        if self.granularity == 'per_block':
            m, n = tensor.shape
            bs = self.block_size
            padded = torch.zeros((ceil_div(m, bs) * bs, ceil_div(n, bs) * bs),
                                 dtype=tensor.dtype, device=tensor.device)
            padded[:m, :n] = tensor
            return padded.view(-1, bs, padded.size(1) // bs, bs)
        return tensor

    def restore_tensor(self, tensor, shape):
        if tensor.shape == shape:
            return tensor
        if self.granularity == 'per_block':
            try:
                return tensor.reshape(-1, shape[-1])[:shape[0], :]
            except RuntimeError:
                return tensor.reshape(shape[0], -1)[:, :shape[1]]
        try:
            return tensor.reshape(shape)
        except RuntimeError:
            deficiency = self.group_size - shape[1] % self.group_size
            return tensor.reshape(*shape[:-1], -1)[..., :-deficiency]

    # ---- small range helpers: a handful of torch ops on [groups,1] tensors (not the hot path) --
    def get_minmax_range(self, tensor):
        """quant.py:132-143."""
        if self.granularity == 'per_tensor':
            require_cuda(tensor)
            t = tensor.contiguous()
            mm = torch.empty(2, dtype=t.dtype, device=t.device)
            ws = torch.empty(2048, dtype=torch.float32, device=t.device)
            call('llmc_minmax_tensor', ptr(t), t.numel(), dtype_enum(t.dtype), ptr(mm), ptr(ws),
                 stream_ptr(t.device))
            return (mm[0], mm[1])
        if self.granularity == 'per_block':
            min_val = tensor.abs().float().amin(dim=(1, 3), keepdim=True)
            max_val = tensor.abs().float().amax(dim=(1, 3), keepdim=True)
            return (min_val, max_val)
        return (tensor.amin(dim=-1, keepdim=True), tensor.amax(dim=-1, keepdim=True))

    def get_learnable_range(self, tensor, lowbound_factor=None, upbound_factor=None):
        """quant.py:205-219 (AWQ clip v2 / OmniQuant bound factors)."""
        min_val, max_val = self.get_minmax_range(tensor)
        if self.sym:
            if upbound_factor is not None:
                abs_max = torch.max(max_val.abs(), min_val.abs()).clamp(min=1e-5)
                abs_max = self.sigmoid(upbound_factor) * abs_max
                min_val, max_val = -abs_max, abs_max
        elif upbound_factor is not None and lowbound_factor is not None:
            min_val = self.sigmoid(lowbound_factor) * min_val
            max_val = self.sigmoid(upbound_factor) * max_val
        return (min_val, max_val)

    def get_tensor_range(self, tensor, args={}):
        """quant.py:122-130."""
        if self.calib_algo == 'learnable':
            return self.get_learnable_range(tensor, **args)
        if self.calib_algo == 'mse':
            return self.get_mse_range(tensor)
        return self.get_minmax_range(tensor)

    def get_mse_range(self, tensor, norm=2.4, bs=256):
        """quant.py:145-203 on the reshaped [groups, g] tensor: ONE launch of llmc_mse_range
        (csrc/range.cu) instead of int(maxshrink*mse_grid) = 80 eager quantise-dequantise passes.
        Returns fp32 (min, max) [groups, 1] like the reference (`tensor.float()`, :151)."""
        assert self.mse_b_num >= 1 and tensor.shape[0] % self.mse_b_num == 0, \
            'Batch number must be divisible by tensor.shape[0],'
        if getattr(self, 'quant_type', 'int-quant') == 'float-quant':
            raise NotImplementedError('mse range for float quantizers (quant.py:173-181)')
        if self.granularity in ('per_tensor', 'per_block') or tensor.dim() != 2:
            raise NotImplementedError('mse range is built for row-wise ranges (per_channel / per_group '
                                      '/ per_head / per_token), the granularities the shipped YAMLs use')
        require_cuda(tensor)
        t = tensor if tensor.is_contiguous() else tensor.contiguous()
        rows, cols = t.shape
        mn = torch.empty((rows, 1), dtype=torch.float32, device=t.device)
        mx = torch.empty_like(mn)
        steps = int(self.maxshrink * self.mse_grid)
        with TIMER.span('mse_range', nbytes=float(t.element_size()) * rows * cols):
            call('llmc_mse_range', ptr(t), rows, cols, dtype_enum(t.dtype), int(bool(self.sym)),
                 _as_int(self.qmin), _as_int(self.qmax), steps, float(self.mse_grid), float(norm),
                 ptr(mn), ptr(mx), stream_ptr(t.device))
        return (mn, mx)

    def get_qparams(self, tensor_range, device):
        """quant.py:545-559 — elementwise on the (tiny) range tensors."""
        min_val, max_val = tensor_range[0], tensor_range[1]
        qmin = self.qmin.to(device)
        qmax = self.qmax.to(device)
        if self.sym:
            abs_max = torch.max(max_val.abs(), min_val.abs()).clamp(min=1e-5)
            scales = abs_max / qmax
            zeros = torch.tensor(0.0)
        else:
            scales = (max_val - min_val).clamp(min=1e-5) / (qmax - qmin)
            zeros = (qmin - torch.round(min_val / scales)).clamp(qmin, qmax)
            if not self.round_zp:
                zeros = qmin - (min_val / scales)
        return scales, zeros, qmax, qmin

    # ---- static activation calibration (quant.py:103-120, 221-263, 561-586) -------------------
    def reshape_batch_tensors(self, act_tensors):
        assert len(act_tensors) > 0, (
            'Calibration data is insufficient. Please provide more data to ensure '
            'all experts in the MOE receive an adequate number of tokens.')
        if isinstance(act_tensors[0], tuple):
            return [torch.stack(tl) for tl in zip(*act_tensors)]
        if len(act_tensors) == 1:
            act_tensors[0] = [act_tensors[0][i] for i in range(act_tensors[0].size(0))]
            return act_tensors
        return [act_tensors]

    def get_static_minmax_range(self, act_tensors):
        act_tensors = self.reshape_batch_tensors(act_tensors)
        min_vals, max_vals = [], []
        for tensors in act_tensors:
            mins, maxs = [], []
            for tensor in tensors:
                mn, mx = self.get_minmax_range(self.reshape_tensor(tensor))
                mins.append(mn.float().reshape(1))
                maxs.append(mx.float().reshape(1))
            min_vals.append(torch.cat(mins).mean())
            max_vals.append(torch.cat(maxs).mean())
        return min_vals, max_vals

    def get_static_moving_minmax_range(self, act_tensors, alpha):
        act_tensors = self.reshape_batch_tensors(act_tensors)
        mins, maxs = [], []
        for tensors in act_tensors:
            mv_min = mv_max = None
            for tensor in tensors:
                mn, mx = self.get_minmax_range(self.reshape_tensor(tensor))
                if mv_min is None:
                    mv_min, mv_max = mn, mx
                else:
                    mv_min = mv_min + alpha * (mn - mv_min)
                    mv_max = mv_max + alpha * (mx - mv_max)
            mins.append(mv_min)
            maxs.append(mv_max)
        return mins, maxs

    # ---- static histogram observer (quant.py:265-522; the PyTorch HistogramObserver scheme) -----
    # Per calibration tensor ONE histogram kernel (llmc_histc) runs on the device; the 2048-bin
    # bookkeeping (re-binning when the range grows, the quantile walk that minimises the expected
    # L2 quantisation error) is O(bins) host arithmetic, kept on the CPU like in the reference.
    upsample_rate = 16

    def _histc(self, tensor, lo, hi):
        require_cuda(tensor)
        t = tensor if tensor.is_contiguous() else tensor.contiguous()
        hist = torch.empty(self.bins, dtype=torch.float32, device=t.device)
        call('llmc_histc', ptr(t), t.numel(), dtype_enum(t.dtype), int(self.bins), float(lo), float(hi),
             ptr(hist), stream_ptr(t.device))
        return hist.cpu()

    def _rebin(self, hist, o_min, o_max, n_min, n_max):
        """_upscale_histogram (:332-366): the old histogram expressed in the new, wider range."""
        up = self.upsample_rate
        fine = hist.repeat_interleave(up) / up
        bin_size = (o_max - o_min) / (self.bins * up)
        mids = torch.linspace(o_min, o_max, self.bins * up + 1)[:-1] + 0.5 * bin_size
        edges = torch.linspace(n_min, n_max, self.bins + 1)
        idx = (torch.bucketize(mids, edges, right=True) - 1).clamp_(0, self.bins - 1)
        return torch.bincount(idx, weights=fine, minlength=self.bins)

    def _merge_hist(self, hist, o_min, o_max, upd, n_min, n_max):
        """_combine_histograms (:368-401)."""
        if n_min == o_min and n_max == o_max:
            return hist + upd
        if o_min == o_max:
            return torch.histc(o_min, bins=self.bins, min=n_min, max=n_max) * torch.sum(upd) + upd
        assert n_min <= o_min and n_max >= o_max
        return upd + self._rebin(hist, o_min, o_max, n_min, n_max)

    def _expected_l2(self, hist, min_val, max_val, first, last):
        """get_quantization_error (:279-330): expected squared error of mapping the source bins
        [first, last] onto dst_nbins uniform levels, each source bin taken as uniformly filled."""
        bw = (max_val.item() - min_val.item()) / self.bins
        dw = bw * (last - first + 1) / self.dst_nbins
        if dw == 0.0:
            return 0.0
        src = torch.arange(self.bins)
        beg = (src - first) * bw
        end = beg + bw
        d_beg = torch.clamp(torch.div(beg, dw, rounding_mode='floor'), 0, self.dst_nbins - 1)
        d_end = torch.clamp(torch.div(end, dw, rounding_mode='floor'), 0, self.dst_nbins - 1)
        dens = hist / bw

        def cube(lo, hi):                       # density * integral_lo^hi x^2 dx   (get_norm :265-277)
            return dens * ((hi * hi * hi - lo * lo * lo) / 3)
        half = dw / 2
        norm = torch.zeros(self.bins)
        norm += cube(beg - (d_beg + 0.5) * dw, torch.ones(self.bins) * half)
        norm += (d_end - d_beg - 1) * cube(torch.tensor(-half), torch.tensor(half))
        norm += cube(torch.tensor(-half), end - (d_end * dw + half))
        return norm.sum().item()

    def get_hist_threshold(self, histogram, min_val, max_val):
        """:403-460 — walk the two quantile bounds inwards, 1e-8 of the mass at a time, while the
        expected L2 error keeps falling."""
        assert histogram.size()[0] == self.bins, 'bins mismatch'
        bin_width = (max_val - min_val) / self.bins
        total = torch.sum(histogram).item()
        csum = torch.cumsum(histogram, dim=0).tolist()
        step, alpha, beta = 1e-8, 0.0, 1.0
        first, last = 0, self.bins - 1
        best = float('inf')
        while alpha < beta:
            na, nb = alpha + step, beta - step
            lo, hi = first, last
            while lo < last and csum[lo] < na * total:
                lo += 1
            while hi > first and csum[hi] > nb * total:
                hi -= 1
            nf, nl = first, last
            if (lo - first) > (last - hi):
                nf, alpha = lo, na
            else:
                nl, beta = hi, nb
            if nf == first and nl == last:
                continue
            err = self._expected_l2(histogram, min_val, max_val, nf, nl)
            if err > best:
                break
            best, first, last = err, nf, nl
        return min_val + bin_width * first, min_val + bin_width * (last + 1)

    def get_static_hist_range(self, act_tensors):
        """:462-522."""
        act_tensors = self.reshape_batch_tensors(act_tensors)
        mins, maxs = [], []
        for tensors in act_tensors:
            lo = hi = None
            hist = torch.zeros(self.bins)
            for tensor in tensors:
                mn, mx = self.get_minmax_range(self.reshape_tensor(tensor))
                x_min, x_max = mn.float().cpu().reshape(()), mx.float().cpu().reshape(())
                if lo is None:
                    hist = self._histc(tensor, x_min.item(), x_max.item())
                    lo, hi = x_min, x_max
                    continue
                n_min, n_max = torch.min(lo, x_min), torch.max(hi, x_max)
                upd = self._histc(tensor, n_min.item(), n_max.item())
                hist = self._merge_hist(hist, lo, hi, upd, n_min, n_max)
                lo, hi = n_min, n_max
            new_min, new_max = self.get_hist_threshold(hist, lo, hi)
            mins.append(new_min)
            maxs.append(new_max)
        return mins, maxs

    def get_batch_tensors_qparams(self, act_tensors, alpha=0.01, args={}):
        if self.calib_algo == 'static_minmax':
            min_vals, max_vals = self.get_static_minmax_range(act_tensors)
        elif self.calib_algo == 'static_moving_minmax':
            min_vals, max_vals = self.get_static_moving_minmax_range(act_tensors, alpha)
        elif self.calib_algo == 'static_hist':
            assert self.sym is True and self.granularity == 'per_tensor', \
                'Only support per tensor static symmetric int quantize.'
            min_vals, max_vals = self.get_static_hist_range(act_tensors)
        else:
            raise ValueError(f'Unsupported calibration algorithm: {self.calib_algo}')
        scales_list, zeros_list, qmin_list, qmax_list = [], [], [], []
        for min_val, max_val in zip(min_vals, max_vals):
            scales, zeros, qmax, qmin = self.get_qparams((min_val, max_val), min_val.device)
            scales_list.append(scales)
            zeros_list.append(zeros)
            qmin_list.append(qmin)
            qmax_list.append(qmax)
        return scales_list, zeros_list, qmin_list, qmax_list


class IntegerQuantizer(BaseQuantizer):
    """quant.py:661-960.  `quant.weight: {bit, symmetric, granularity, group_size, ...}`."""

    def __init__(self, bit, symmetric, granularity, **kwargs):
        super().__init__(bit, symmetric, granularity, **kwargs)
        self.quant_type = 'int-quant'
        if 'int_range' in self.kwargs:
            qmin, qmax = self.kwargs['int_range'][0], self.kwargs['int_range'][1]
        elif self.sym:
            qmin, qmax = -(2 ** (self.bit - 1)), 2 ** (self.bit - 1) - 1
        else:
            qmin, qmax = 0.0, 2 ** self.bit - 1
        self.qmin = torch.tensor(qmin)
        self.qmax = torch.tensor(qmax)
        self.dst_nbins = 2 ** bit

    # ---- kernel launch helpers ----------------------------------------------------------------
    def _group_of(self, t2d):
        """Elements per quantisation group along the last dim of the 2-D view."""
        cols = t2d.shape[-1]
        if self.granularity == 'per_group':
            if cols >= self.group_size:
                if cols % self.group_size != 0:
                    raise ValueError(f'Dimension {cols} '
                                     f'not divisible by group size {self.group_size}')
                return self.group_size
            return cols
        return cols  # per_channel / per_token / per_head (caller reshapes rows)

    def _view2d(self, tensor):
        if self.granularity == 'per_head':
            return tensor.reshape(self.head_num, -1)
        return tensor.reshape(-1, tensor.shape[-1])

    def _dynamic(self, tensor, out_mode, out=None, out_dtype=None, col_scale=None):
        """One fused launch: group min/max -> qparams -> codes / qdq / packed words."""
        require_cuda(tensor)
        if self.calib_algo not in ('minmax', 'learnable') or not self.round_zp:
            raise NotImplementedError(f'calib_algo={self.calib_algo} round_zp={self.round_zp}')
        t2d = self._view2d(tensor)
        if not t2d.is_contiguous():
            t2d = t2d.contiguous()
        rows, cols = t2d.shape
        group = self._group_of(t2d)
        ng = cols // group
        dt = dtype_enum(t2d.dtype)
        scales = torch.empty((rows * ng, 1), dtype=t2d.dtype, device=t2d.device)
        zeros = None if self.sym else torch.empty_like(scales)
        qmin, qmax = _as_int(self.qmin), _as_int(self.qmax)
        with TIMER.span('quant_dynamic', nbytes=float(t2d.element_size()) * rows * cols):
            call('llmc_quant_dynamic', ptr(t2d), rows, cols, cols, dt, group, int(self.bit),
                 int(bool(self.sym)), 1, qmin, qmax, ptr(col_scale), ptr(scales), ptr(zeros),
                 out_mode, ptr(out),
                 0, dtype_enum(out_dtype) if out_dtype is not None else dt,
                 stream_ptr(t2d.device))
        return scales, zeros

    def _static(self, tensor2d, scales, zeros, qmax, qmin, out_mode, out, out_dtype,
                q_row_stride, group, gmap=None, round_dtype=-1):
        require_cuda(tensor2d, scales)
        w = tensor2d if tensor2d.is_contiguous() else tensor2d.contiguous()
        rows, cols = w.shape
        s = scales.contiguous()
        z = None
        if torch.is_tensor(zeros) and zeros.numel() > 1:
            # per-row / per-group zero-points; after BlockStreamer.release they may sit in pinned
            # host memory — move them, never drop them (an asymmetric tensor quantised without
            # its zero-points is silently wrong)
            if zeros.numel() != s.numel():
                raise ValueError(f'zeros has {zeros.numel()} elements, scales {s.numel()}')
            z = zeros.to(device=s.device, dtype=s.dtype).reshape(s.shape).contiguous()
        elif torch.is_tensor(zeros) and zeros.numel() == 1 and (zeros.is_cuda or float(zeros) != 0.0):
            z = zeros.to(device=s.device, dtype=s.dtype).reshape(1).expand(s.numel()).reshape(s.shape).contiguous()
        if not self.round_zp:
            out_mode |= 0x100          # LLMC_OUT_FLAG_ZP_INSIDE: round(x / s + z), quant.py:702-707
        with TIMER.span('quant_static', nbytes=float(w.element_size()) * rows * cols):
            call('llmc_quant_static', ptr(w), rows, cols, cols, dtype_enum(w.dtype), ptr(s),
                 ptr(z), dtype_enum(s.dtype), round_dtype, q_row_stride, group, ptr(gmap),
                 int(self.bit), _as_int(qmin), _as_int(qmax), out_mode, ptr(out), 0,
                 dtype_enum(out_dtype), stream_ptr(w.device))

    # ---- reference API ------------------------------------------------------------------------
    def get_tensor_qparams(self, tensor, args={}):
        """quant.py:690-697 -> (reshaped tensor, scales, zeros, qmax, qmin)."""
        if self.calib_algo == 'hqq':
            raise NotImplementedError('HQQ (quant.py:680-688) is a SURVEY §8(f) "next" row')
        reshaped = self.reshape_tensor(tensor)
        dev = tensor.device
        if self.granularity in ('per_tensor', 'per_block') or self.calib_algo == 'mse' or \
                not self.round_zp or (
                self.calib_algo == 'learnable' and any(v is not None for v in args.values())):
            tensor_range = self.get_tensor_range(reshaped, args)
            scales, zeros, qmax, qmin = self.get_qparams(tensor_range, dev)
            return reshaped, scales, zeros, qmax, qmin
        scales, zeros = self._dynamic(tensor, OUT_NONE)
        if self.sym:
            zeros = torch.tensor(0.0)
        # qmax / qmin stay 0-dim HOST tensors (the reference moves them to the device): they are
        # kernel arguments here, and a pageable H2D copy of a scalar is a synchronous cudaMemcpy
        # that makes the host lose its lead over the GPU (the GPU idles for every such call)
        return reshaped, scales, zeros, self.qmax, self.qmin

    def quant(self, tensor, scales, zeros, qmax, qmin):
        """quant.py:699-708: clamp(round(x / s) + z, qmin, qmax), integer-valued, dtype of x."""
        return self._elementwise(tensor, scales, zeros, qmax, qmin, dequant=False)

    def dequant(self, tensor, scales, zeros):
        """quant.py:710-712 — two elementwise torch ops on codes (not a hot path by itself)."""
        return (tensor - zeros) * scales

    def quant_dequant(self, tensor, scales, zeros, qmax, qmin, output_scale_factor=1):
        """quant.py:714-717."""
        if output_scale_factor != 1:
            q = self.quant(tensor, scales, zeros, qmax, qmin)
            return self.dequant(q, scales * output_scale_factor, zeros)
        return self._elementwise(tensor, scales, zeros, qmax, qmin, dequant=True)

    def _elementwise(self, tensor, scales, zeros, qmax, qmin, dequant):
        """Broadcast `scales`/`zeros` ([N,1], [N] or scalar) against a [N, g] tensor."""
        require_cuda(tensor)
        t2d = tensor.reshape(-1, tensor.shape[-1]) if tensor.dim() != 2 else tensor
        rows, cols = t2d.shape
        scales = scales if torch.is_tensor(scales) else torch.tensor(scales)
        rd = -1
        if scales.dim() == 0:
            # 0-dim scale (per_tensor): torch's CPU kernels keep a scalar operand in fp32 and
            # round each result to the tensor dtype (ATen BinaryOpsKernel.cpp div/mul scalar
            # branch) — the reference CPU path, hence the parity target.
            ct = t2d.dtype
            s = scales.reshape(1).to(device=t2d.device, dtype=torch.float32)
            stride = 0
            if ct != torch.float32:
                rd = dtype_enum(ct)
        elif scales.numel() == 1:
            ct = torch.promote_types(t2d.dtype, scales.dtype)
            s = scales.reshape(1).to(device=t2d.device, dtype=ct)
            stride = 0
        else:
            ct = torch.promote_types(t2d.dtype, scales.dtype)
            if scales.numel() != rows and scales.dim() == tensor.dim():
                # per_block: [M/bs, 1, N/bs, 1] qparams against a [M/bs, bs, N/bs, bs] tensor — one
                # value per row of the 2-D view after broadcasting over the tile's rows
                lead = tensor.shape[:-1]
                scales = scales.expand(*lead, 1).reshape(-1)
                if torch.is_tensor(zeros) and zeros.numel() > 1:
                    zeros = zeros.expand(*lead, 1).reshape(-1)
            assert scales.numel() == rows, (scales.shape, t2d.shape)
            s = scales.reshape(rows).to(ct)
            stride = 1
        out = torch.empty(t2d.shape, dtype=ct, device=t2d.device)
        if dequant:
            self._static(t2d, s, zeros, qmax, qmin, OUT_QDQ, out, ct, stride, cols, round_dtype=rd)
        else:
            codes = torch.empty(t2d.shape, dtype=torch.int32, device=t2d.device)
            self._static(t2d, s, zeros, qmax, qmin, OUT_CODES_I32, codes, ct, stride, cols,
                         round_dtype=rd)
            out = codes.to(ct)
        return out.reshape(tensor.shape)

    # -- fake quant ----------------------------------------------------------------------------
    def fake_quant_weight_dynamic(self, weight, args={}):
        """quant.py:833-869."""
        if 'int_indices' in args:
            raise NotImplementedError('mixed-precision column subsets (quant.py:834-838)')
        transpose = 'dim' in args and 'ic' in args['dim']
        q_weight = weight.T if transpose else weight
        org_bit = self.bit
        if 'current_bit' in args:
            self.bit = args['current_bit']
        try:
            fast = (self.granularity in ('per_group', 'per_channel', 'per_head', 'per_token')
                    and self.calib_algo == 'minmax')
            if fast:
                src = q_weight.contiguous()
                out = torch.empty_like(src)
                self._dynamic(src, OUT_QDQ, out=out, out_dtype=src.dtype)
                q_weight = out
            else:
                org_shape, org_dtype = q_weight.shape, q_weight.dtype
                t, scales, zeros, qmax, qmin = self.get_tensor_qparams(q_weight, args)
                t = self.quant_dequant(t, scales, zeros, qmax, qmin)
                q_weight = self.restore_tensor(t, org_shape).to(org_dtype)
        finally:
            self.bit = org_bit
        return q_weight.T if transpose else q_weight

    def fake_quant_weight_static(self, weight, args):
        """quant.py:785-831; `args['gmap']` (int32 [C]) is an extension of this library that fuses
        GPTQ's act-order gather (gptq.py:427-450) into the same pass."""
        if 'int_indices' in args or 'rounding' in args:
            raise NotImplementedError('int_indices / TesseraQ rounding (quant.py:786-799)')
        transpose = 'dim' in args and 'ic' in args['dim']
        q_weight = weight.T if transpose else weight
        scales, zeros, qmax, qmin = args['scales'], args['zeros'], args['qmax'], args['qmin']
        osf = args.get('output_scale_factor', 1)
        org_shape, org_dtype = q_weight.shape, q_weight.dtype
        out_dtype = args.get('out_dtype', org_dtype)
        if osf != 1 or self.granularity in ('per_block',) or scales.numel() == 1:
            t = self.reshape_tensor(q_weight)
            t = self.quant_dequant(t, scales, zeros, qmax, qmin, osf)
            q_weight = self.restore_tensor(t, org_shape).to(org_dtype)
        else:
            w2d = q_weight.reshape(-1, q_weight.shape[-1])
            rows, cols = w2d.shape
            group = self._group_of(w2d)
            stride = cols // group
            s = scales.reshape(-1)
            assert s.numel() == rows * stride, (scales.shape, w2d.shape, group)
            out = torch.empty(w2d.shape, dtype=out_dtype, device=w2d.device)
            self._static(w2d, s, zeros, qmax, qmin, OUT_QDQ, out, out_dtype, stride, group,
                         gmap=args.get('gmap'))
            q_weight = out.reshape(org_shape)
        return q_weight.T if transpose else q_weight

    def fake_quant_act_dynamic(self, act, args={}):
        """quant.py:754-783 (per_token / per_tensor / per_group activations)."""
        if 'int_indices' in args:
            raise NotImplementedError('mixed-precision activation subsets (quant.py:755-757)')
        org_bit = self.bit
        if 'current_bit' in args:
            self.bit = args['current_bit']
        try:
            if self.granularity in ('per_token', 'per_group', 'per_channel'):
                src = act.contiguous()
                out = torch.empty_like(src)
                self._dynamic(src, OUT_QDQ, out=out, out_dtype=src.dtype)
                return out
            org_shape, org_dtype = act.shape, act.dtype
            t, scales, zeros, qmax, qmin = self.get_tensor_qparams(act, args)
            t = self.quant_dequant(t, scales, zeros, qmax, qmin)
            return self.restore_tensor(t, org_shape).to(org_dtype)
        finally:
            self.bit = org_bit

    def fake_quant_act_static(self, act, args={}):
        """quant.py:719-752."""
        if 'int_indices' in args:
            raise NotImplementedError('mixed-precision activation subsets (quant.py:720-722)')
        org_shape, org_dtype = act.shape, act.dtype
        t = self.reshape_tensor(act)
        t = self.quant_dequant(t, args['scales'], args['zeros'], args['qmax'], args['qmin'])
        return self.restore_tensor(t, org_shape).to(org_dtype)

    # -- real quant -------------------------------------------------------------------------------
    def _code_dtype(self):
        if self.bit == 8:
            return (torch.int8, OUT_CODES_I8) if self.qmin != 0 else (torch.uint8, OUT_CODES_U8)
        return torch.int32, OUT_CODES_I32

    def _finish_real(self, weight, scales, zeros, osf):
        """Common tail of quant.py:888-914 / :927-953."""
        dtype, _ = self._code_dtype()
        scales = scales * osf
        if not self.sym and self.round_zp:
            zeros = zeros.to(dtype)
        elif self.sym:
            zeros = None
        if self.granularity == 'per_tensor':
            qshape = 1
        elif self.granularity == 'per_block':
            qshape = (scales.shape[0], scales.shape[2])
        else:
            qshape = (weight.shape[0], -1)
        if zeros is not None:
            zeros = zeros.view(qshape)
        return weight, scales.view(qshape), zeros

    def real_quant_weight_dynamic(self, weight, args={}):
        """quant.py:916-953 -> (codes, scales [R, ng], zeros or None)."""
        osf = args.pop('output_scale_factor', 1) if 'output_scale_factor' in args else 1
        dtype, mode = self._code_dtype()
        if self.granularity in ('per_group', 'per_channel', 'per_head') and \
                self.calib_algo == 'minmax':
            src = weight.contiguous()
            codes = torch.empty(src.shape, dtype=dtype, device=src.device)
            scales, zeros = self._dynamic(src, mode, out=codes)
            return self._finish_real(codes, scales, zeros, osf)
        org_shape = weight.shape
        t, scales, zeros, qmax, qmin = self.get_tensor_qparams(weight, args)
        t = self.restore_tensor(self.quant(t, scales, zeros, qmax, qmin), org_shape).to(dtype)
        return self._finish_real(t, scales, zeros, osf)

    def real_quant_weight_static(self, weight, args):
        """quant.py:871-914."""
        osf = args.pop('output_scale_factor', 1) if 'output_scale_factor' in args else 1
        scales, zeros, qmax, qmin = args['scales'], args['zeros'], args['qmax'], args['qmin']
        dtype, mode = self._code_dtype()
        if self.granularity in ('per_group', 'per_channel') and scales.numel() > 1:
            w2d = weight.reshape(-1, weight.shape[-1])
            rows, cols = w2d.shape
            group = self._group_of(w2d)
            s = scales.reshape(-1)
            codes = torch.empty(w2d.shape, dtype=dtype, device=w2d.device)
            self._static(w2d, s, zeros, qmax, qmin, mode, codes, w2d.dtype, cols // group, group)
            return self._finish_real(codes.reshape(weight.shape), scales, zeros, osf)
        org_shape = weight.shape
        t = self.reshape_tensor(weight)
        t = self.restore_tensor(self.quant(t, scales, zeros, qmax, qmin), org_shape).to(dtype)
        return self._finish_real(t, scales, zeros, osf)

    def real_quant_pack_vllm_dynamic(self, weight):
        """Fast path for VllmRealQuantLinear.quant_pack (module_utils.py:821-862):
        quantise + pack in ONE pass (the reference round-trips int32 codes through numpy)."""
        assert self.granularity in ('per_group', 'per_channel') and self.bit in (4, 8)
        src = weight.contiguous()
        rows, cols = src.shape
        pf = 32 // self.bit
        packed = torch.empty((rows, ceil_div(cols, pf)), dtype=torch.int32, device=src.device)
        scales, zeros = self._dynamic(src, OUT_PACK_VLLM, out=packed)
        return packed, scales.view(rows, -1), zeros

    def __repr__(self):
        return (f'IntegerQuantizer(bit={self.bit}, sym={self.sym},'
                f'granularity={self.granularity},'
                f'kwargs={self.kwargs}, qmin={self.qmin}, qmax={self.qmax})')
