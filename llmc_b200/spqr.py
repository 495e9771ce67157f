"""SpQR — mirror of llmc/compression/quantization/spqr.py (class SpQR :19-398), the remaining
SURVEY §8(f)-3 sibling of GPTQ: the same Hessian / act-order / Cholesky pipeline, a column sweep
that (a) searches every group's statistics with a leave-one-out outlier test, (b) quantises the
group scales and zeros themselves ("bilevel"), (c) keeps weights whose compensated error exceeds
a threshold unquantised (an unstructured outlier mask).

Same YAML knobs (`special: actorder, percdamp, blocksize, true_sequential, relative_threshold,
simplified_outliers, scale: {...}, zero: {...}`), same `buf_*` hand-off to FakeQuantLinear.
What runs where:
  * Hessians              -> the wgmma SYRK of GPTQ (spqr.py:270-299 is gptq.py:253-295);
  * Cholesky triple       -> llmc_chol_inv_upper;
  * weight_transform      -> llmc_spqr_colblock (csrc/gptq.cu: one thread per weight row through
                             csrc/spqr_row.cuh, super-panel trailing updates on 3xTF32 tensor cores);
  * damping / threshold   -> a few O(C^2) / O(R*C) torch reductions on the device per layer.
Deviations, all stated: `buf_mask` is a dense uint8 buffer (the reference stores a sparse COO float
tensor, :169); linears that share an input share ONE Hessian, permutation and Cholesky factor (the
reference recomputes identical ones per linear).
"""
import math

import torch
import torch.nn as nn

from . import gptq_ops as ops
from .blockwise import ALGO_REGISTRY
from .gptq import GPTQ


def _level2(cfg, what):
    """special.scale / special.zero -> (bit, symmetric, round_zp).  The reference builds an
    IntegerQuantizer from the dict (spqr.py:54-55) and feeds it the [R, 1] scale / zero tensor;
    per_group / per_channel / per_token statistics of a one-column tensor are per-row statistics,
    which is what the kernel evaluates.  per_tensor would couple all rows — not built."""
    gran = cfg.get('granularity', 'per_group')
    if gran not in ('per_group', 'per_channel', 'per_token'):
        raise NotImplementedError(f'SpQR special.{what}.granularity {gran} (statistics across rows)')
    if gran == 'per_group' and int(cfg.get('group_size', 0)) <= 1:
        raise NotImplementedError(f'SpQR special.{what}.group_size must be > 1')
    if cfg.get('calib_algo', 'minmax') != 'minmax' or 'int_range' in cfg:
        raise NotImplementedError(f'SpQR special.{what}: only minmax calibration of the full integer range')
    return int(cfg['bit']), bool(cfg['symmetric']), bool(cfg.get('round_zp', True))


@ALGO_REGISTRY
class SpQR(GPTQ):
    @torch.no_grad()
    def add_quant_config(self):
        """spqr.py:33-58."""
        if self.wquantizer.granularity != 'per_group':
            raise AssertionError('SpQR only supports per_group quantization')      # spqr.py:22-24
        sp = self.quant_config['special']
        self.prefix = self.model.block_name_prefix
        self.true_sequential = sp['true_sequential']
        self.actorder = sp['actorder']
        self.percdamp = sp['percdamp']
        self.blocksize = sp['blocksize']
        if self.blocksize != 128:
            raise NotImplementedError('the fused column-block kernel is built for blocksize 128 '
                                      '(the shipped SpQR YAML uses 128)')
        rt = sp['relative_threshold']
        self.relative_threshold = math.inf if rt == 'inf' else float(rt)
        self.simplified_outliers = bool(sp['simplified_outliers'])
        if self.quant_config.get('quant_type', 'int-quant') == 'float-quant':
            raise AssertionError('SPQR do not support Float quant now.')           # spqr.py:52-53
        wq = self.wquantizer
        if self.float_grid:
            raise NotImplementedError('SpQR on an FP8 weight grid: the reference refuses float quant '
                                      '(spqr.py:53) and the SpQR kernel is integer only')
        if wq.sym:
            # the reference fails here too: zeros is a 0-dim tensor that zero_quantizer's
            # reshape_tensor cannot index (spqr.py:334, quant.py:614)
            raise ValueError('SpQR needs an asymmetric weight quantizer')
        if wq.group_size not in (16, 32, 64, 128):
            raise NotImplementedError(f'SpQR group_size {wq.group_size}: the kernel serves 16 / 32 / 64 / 128')
        if getattr(wq, 'calib_algo', 'minmax') != 'minmax':
            raise NotImplementedError('SpQR with a non-minmax weight calibration')
        self.scale_cfg = _level2(sp['scale'], 'scale')
        self.zero_cfg = _level2(sp['zero'], 'zero')
        self.static_groups = False
        self.owq = False
        self.chunk_num = 1
        self.need_perm = bool(self.actorder)                                      # spqr.py:44-45

    @torch.no_grad()
    def _damped_permuted_hessian(self, H, perm):
        """spqr.py:134-151.  Not gptq.py:139-171: the damping mean is taken over |diag(H)| with dead
        columns still at zero, and a dead diagonal ends up exactly 1 (not 1 + damp)."""
        d = torch.diag(H)
        dead = d == 0
        Hp = H[perm][:, perm] if perm is not None else H.clone()
        if perm is not None:
            d, dead = d[perm], dead[perm]
        dp = torch.diagonal(Hp)
        if self.percdamp > 0:
            dp.add_(self.percdamp * d.abs().mean())
        dp.copy_(torch.where(dead, torch.ones_like(dp), dp))
        return Hp

    @torch.no_grad()
    def _transform_group(self, members):
        """spqr.py:116-170 for the linears `members` that share one Hessian: one permutation and
        one Cholesky triple for all of them, one sweep each (the outlier threshold is a statistic of
        the individual weight, :194-195)."""
        name0, _ = members[0]
        lead, H = self._hessian_of(name0)
        wq = self.wquantizer
        group = wq.group_size
        perm = torch.argsort(torch.diag(H), descending=True) if self.actorder else None
        invperm = torch.argsort(perm) if perm is not None else None
        Hp = self._damped_permuted_hessian(H, perm)
        Hinv, info = ops.chol_inv_upper(Hp, return_info=True, inplace=True)
        self._chol_infos.append((f'{self.block_idx}.{lead}', info))
        del Hp
        wcfg = (wq.bit, wq.sym, bool(getattr(wq, 'round_zp', True)), group)
        for name, layer in members:
            W = layer.weight.data
            W = W.flatten(1) if isinstance(layer, nn.Conv2d) else W
            R, C = W.shape
            if C % group:
                raise ValueError(f'Dimension {C} not divisible by group size {group}')
            Wp, _ = ops.prepare(W, H, perm, self.percdamp, want_h=False)   # W.float()[:, perm], dead -> 0
            thr = ops.spqr_threshold(Wp, Hinv, self.relative_threshold)
            tmp, mask, losses, scales, zeros = ops.spqr_transform(
                Wp, Hinv, wcfg, self.scale_cfg, self.zero_cfg, thr, self.simplified_outliers,
                out_perm=perm)
            if self.actorder:
                layer.register_buffer('buf_perm', perm)
                layer.register_buffer('buf_invperm', invperm)
            self.losses[f'{self.block_idx}.{name}'] = losses
            layer.weight.data = tmp.reshape(layer.weight.shape)            # fp32 until save_model (:394-396)
            layer.buf_scales = scales.reshape(-1, 1)                       # set_model_qparams (:353-361)
            layer.buf_zeros = zeros.reshape(-1, 1)
            layer.register_buffer('buf_mask', mask)
        del Hinv

    @torch.no_grad()
    def w_q(self, module, wquantizer):
        """spqr.py:359-361 (`pass`)."""
        raise AssertionError('SpQR does not support real quantization')

    @torch.no_grad()
    def w_qdq(self, module, wquantizer):
        """spqr.py:363-386: W[:, perm] -> static qdq -> model dtype -> [:, invperm], outliers keep
        their (compensated) weight."""
        mask = module.buf_mask.bool()
        weight = module.weight.data
        args = {'scales': module.buf_scales, 'zeros': module.buf_zeros,
                'qmax': module.buf_qmax, 'qmin': module.buf_qmin, 'out_dtype': self.model_dtype}
        if self.need_perm:
            args['gmap'] = (module.buf_invperm // wquantizer.group_size).to(torch.int32)
        y = wquantizer.fake_quant_weight_static(weight, args)
        return torch.where(mask, weight.to(self.model_dtype), y)

    @torch.no_grad()
    def w_packed(self, module, wquantizer):
        """The packed form of exactly what `w_qdq` materialises, for EffcientFakeQuantLinear: codes of
        the static pass w_qdq runs (act-order gmap included), in the original column order; the fp32
        statistics as [ng, R] with g_idx = invperm // group (k // group without act-order); the
        outliers of buf_mask as a CSR with their weights in the model dtype.  None when
        llmc_gemm_w*a16_rz does not serve the layer; it is then materialised as before."""
        from .module_utils import outliers_to_csr, pack_unsigned_codes
        from .quant import OUT_CODES_I32, IntegerQuantizer
        q, w = wquantizer, module.weight.data
        if not (isinstance(q, IntegerQuantizer) and q.bit in (2, 3, 4, 8) and q.granularity == 'per_group'
                and w.dim() == 2 and w.is_cuda and w.is_floating_point()
                and self.model_dtype in (torch.float16, torch.bfloat16)):
            return None
        R, K = w.shape
        group = q.group_size
        if K % 64 or K % group:
            return None
        ng = K // group
        scales = module.buf_scales.to(w.device)
        zeros = module.buf_zeros.to(w.device)
        if scales.dtype != torch.float32 or zeros.dtype != torch.float32 or scales.numel() != R * ng:
            return None
        scales, zeros = scales.reshape(R, ng), zeros.reshape(R, ng)
        gmap = (module.buf_invperm // group).to(torch.int32) if self.need_perm else None
        codes = torch.empty((R, K), dtype=torch.int32, device=w.device)
        q._static(w, scales.reshape(-1), zeros, module.buf_qmax, module.buf_qmin, OUT_CODES_I32, codes,
                  self.model_dtype, ng, group, gmap=gmap)
        g_idx = gmap if gmap is not None else (torch.arange(K, device=w.device) // group).to(torch.int32)
        mask = module.buf_mask.to(w.device)
        outliers = outliers_to_csr(mask, w.to(self.model_dtype)) if bool(mask.any()) else None
        return dict(qweight=pack_unsigned_codes(codes, q.bit, signed=q.sym), scales=scales.t().contiguous(),
                    zeros=zeros.t().contiguous(), bits=q.bit, group=group, dtype=self.model_dtype, g_idx=g_idx,
                    rz=True, sym=q.sym, group_axis=0, outliers=outliers)

    @torch.no_grad()
    def deploy(self, quant_format):
        """spqr.py:388-392."""
        if quant_format == 'real_quant':
            assert False, 'SpQR does not support real quantization'
        super().deploy(quant_format)
