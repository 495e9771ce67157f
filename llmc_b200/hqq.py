"""HQQ — mirror of llmc/compression/quantization/hqq.py (class HQQ :12-103), a SURVEY §8(f)-3
sibling: data-free half-quadratic optimisation of the zero-points.  Per linear the RTN qparams come
from the hot path's kernel (`get_tensor_qparams` on the fp32, optionally transposed, weight); the
proximal iterations (:36-61) are a handful of elementwise passes over the weight per iteration with
one global mean deciding the early exit — evaluated on the device with eager tensor ops (≤ 20
iterations per layer, once per model; not worth a dedicated kernel), the result handed to the
static fake-quant kernel through `buf_scales / buf_zeros` exactly like the reference's `w_qdq`.
"""
import torch

from .blockwise import ALGO_REGISTRY, BaseBlockwiseQuantization
from .quant import IntegerQuantizer


@ALGO_REGISTRY
class HQQ(BaseBlockwiseQuantization):
    def __init__(self, model, quant_config, input, padding_mask, config):
        super().__init__(model, quant_config, input, padding_mask, config)
        sp = self.quant_config['special']
        self.lp_norm, self.beta, self.kappa = sp['lp_norm'], sp['beta'], sp['kappa']
        self.iters, self.axis = sp['iters'], sp['axis']
        self.data_free = True

    def shrink_op(self, x, beta):
        """hqq.py:24-33: generalised soft-thresholding of the l_p proximal step."""
        if self.lp_norm == 1:
            return torch.sign(x) * torch.nn.functional.relu(torch.abs(x) - 1.0 / self.beta)
        return torch.sign(x) * torch.nn.functional.relu(
            torch.abs(x) - (1.0 / self.beta) * torch.pow(torch.abs(x), self.lp_norm - 1))

    @torch.no_grad()
    def optimize_weights_proximal(self, W_f, scales, zeros, qmax, qmin):
        """hqq.py:36-61.  The early exit compares a global mean; it is read back once per iteration
        (the reference does the same with `float(...)`)."""
        best_error = 1e4
        current_beta, current_kappa = self.beta, self.kappa
        scales = 1 / scales
        qmin_f, qmax_f = float(qmin), float(qmax)
        for _ in range(self.iters):
            W_q = torch.round(W_f * scales + zeros).clamp(qmin_f, qmax_f)
            W_r = (W_q - zeros) / scales
            W_e = self.shrink_op(W_f - W_r, current_beta)
            zeros = torch.mean(W_q - (W_f - W_e) * scales, axis=-1, keepdim=True)
            current_beta *= current_kappa
            current_error = float(torch.abs(W_f - W_r).mean())
            if current_error < best_error:
                best_error = current_error
            else:
                break
        return 1 / scales, zeros

    @torch.no_grad()
    def block_opt(self, block):
        """hqq.py:63-92."""
        for name, layer in self.model.get_block_linears(block).items():
            tensor = layer.weight.data.float()
            if self.axis == 0:
                tensor = tensor.T
            tensor, org_scales, org_zeros, qmax, qmin = self.wquantizer.get_tensor_qparams(tensor)
            org_zeros = org_zeros.to(tensor.device) if torch.is_tensor(org_zeros) else org_zeros
            best_scales, best_zeros = self.optimize_weights_proximal(tensor, org_scales, org_zeros, qmax, qmin)
            layer.register_buffer('buf_scales', best_scales)
            layer.register_buffer('buf_zeros', best_zeros)
            layer.register_buffer('buf_qmax', torch.as_tensor(qmax).clone().cpu())
            layer.register_buffer('buf_qmin', torch.as_tensor(qmin).clone().cpu())

    def w_qdq(self, module, wquantizer):
        """hqq.py:94-103."""
        args = {'scales': module.buf_scales, 'zeros': module.buf_zeros, 'qmax': module.buf_qmax,
                'qmin': module.buf_qmin}
        if self.axis == 0:
            args['dim'] = 'ic'
        return wquantizer.fake_quant_weight_static(module.weight, args)

    def w_packed(self, module, wquantizer):
        """The packed form of exactly what `w_qdq` materialises, for EffcientFakeQuantLinear: codes from
        the same static pass (round_zp False puts the real-valued zero-point inside the rounding), on
        weight.T for axis 0 and transposed back to [R, C]; the fp32 buf_scales / buf_zeros as stored —
        [C, R/group], groups along N, for axis 0; [R, C/group] for axis 1, handed over as [C/group, R]
        with g_idx = k // group.  None (materialise) for what llmc_gemm_w*a16_rz does not serve."""
        from .module_utils import pack_unsigned_codes
        from .quant import OUT_CODES_I32
        q, w = wquantizer, module.weight
        if not (isinstance(q, IntegerQuantizer) and q.bit in (2, 3, 4, 8) and q.granularity == 'per_group'
                and w.dim() == 2 and w.is_cuda and w.dtype in (torch.float16, torch.bfloat16)):
            return None
        R, C = w.shape
        src = w.data.T if self.axis == 0 else w.data          # the tensor w_qdq quantises
        rows, cols = src.shape
        group = q.group_size if cols >= q.group_size else cols  # IntegerQuantizer._group_of
        if C % 64 or cols % group:
            return None
        s = module.buf_scales.to(w.device)
        if s.dtype != torch.float32 or s.numel() != rows * (cols // group):
            return None
        s = s.reshape(rows, cols // group)
        zeros = module.buf_zeros
        z = None                                             # what _static reads: zero-points, or 0
        if torch.is_tensor(zeros) and zeros.numel() > 1:
            z = zeros.to(device=w.device, dtype=torch.float32).reshape(s.shape)
        elif torch.is_tensor(zeros) and zeros.numel() == 1 and (zeros.is_cuda or float(zeros) != 0.0):
            z = zeros.to(device=w.device, dtype=torch.float32).reshape(1, 1).expand(s.shape)
        codes = torch.empty((rows, cols), dtype=torch.int32, device=w.device)
        q._static(src, s.reshape(-1), zeros, module.buf_qmax, module.buf_qmin, OUT_CODES_I32, codes, w.dtype,
                  cols // group, group)
        packed = dict(bits=q.bit, group=group, dtype=w.dtype, rz=True, sym=q.sym, outliers=None)
        if self.axis == 0:
            packed.update(qweight=pack_unsigned_codes(codes.t(), q.bit, signed=q.sym), scales=s.contiguous(),
                          zeros=z.contiguous() if z is not None else None, group_axis=1, g_idx=None)
        else:
            g_idx = (torch.arange(C, device=w.device) // group).to(torch.int32)
            packed.update(qweight=pack_unsigned_codes(codes, q.bit, signed=q.sym), scales=s.t().contiguous(),
                          zeros=z.t().contiguous() if z is not None else None, group_axis=0, g_idx=g_idx)
        return packed
