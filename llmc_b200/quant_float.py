"""FloatQuantizer — mirror of llmc/compression/quantization/quant.py:963-1229 for the
`use_qtorch: True` configuration every shipped FP8 YAML uses (configs/quantization/backend/*/fp8).

PARITY UNPINNED: the rounding step is `qtorch.quant.float_quantize`, an unpinned third-party
dependency absent from /root/reference and from this image (SURVEY.md §8c).  It is restated as
IEEE round-to-nearest-even onto the e4m3fn / e5m2 grid with saturation (csrc/fp8.cu); the dtype
flow around it (x/s rounded to the tensor dtype, fp32 grid value, fp32 * scale, cast back)
follows the reference line by line.  The non-qtorch log2 emulation (quant.py:1005-1027) is not
provided.
"""
import torch

from ._lib import call, dtype_enum, ptr, require_cuda, stream_ptr
from .prof import TIMER
from .quant import BaseQuantizer

_FP8 = {'e4m3': (torch.float8_e4m3fn, 0), 'e5m2': (torch.float8_e5m2, 1)}


class FloatQuantizer(BaseQuantizer):
    def __init__(self, bit, symmetric, granularity, **kwargs):
        super().__init__(bit, symmetric, granularity, **kwargs)
        self.sym = True                                    # quant.py:966
        self.quant_type = 'float-quant'
        self.e_bits, self.m_bits = int(self.bit[1]), int(self.bit[-1])
        self.num_bits = self.e_bits + self.m_bits + 1
        self.use_qtorch = self.kwargs.get('use_qtorch')
        if not self.use_qtorch:
            raise NotImplementedError('FloatQuantizer without use_qtorch (quant.py:1005-1027 log2 '
                                      'emulation) has no CUDA kernel here; every shipped fp8 YAML sets it')
        if self.bit not in _FP8:
            raise NotImplementedError(f'{self.bit}: only e4m3 / e5m2 have hardware conversions '
                                      '(e2m1/e3m2/e4m7 of quant.py:982-988 are not built)')
        if 'float_range' in self.kwargs:
            qmin, qmax = self.kwargs['float_range']
        else:
            fi = torch.finfo(_FP8[self.bit][0])
            qmin, qmax = fi.min, fi.max
        self.qmax, self.qmin = torch.tensor(qmax), torch.tensor(qmin)
        self.dst_nbins = 2 ** self.num_bits

    # ---- kernel launcher ----------------------------------------------------------------------
    def _run(self, t2d, group, dynamic, scales, out_mode, q_row_stride=0, scale_f32=0):
        require_cuda(t2d)
        rows, cols = t2d.shape
        fp8_dtype, e5m2 = _FP8[self.bit]
        out = None
        if out_mode == 1:
            out = torch.empty_like(t2d)
        elif out_mode == 2:
            out = torch.empty(t2d.shape, dtype=torch.uint8, device=t2d.device)
        with TIMER.span('fp8_quant', nbytes=float(t2d.element_size() + 1) * rows * cols):
            call('llmc_fp8_quant', ptr(t2d), rows, cols, dtype_enum(t2d.dtype), int(group), e5m2,
                 int(dynamic), ptr(scales), int(q_row_stride), int(scale_f32), out_mode, ptr(out),
                 stream_ptr(t2d.device))
        if out_mode == 2:
            out = out.view(fp8_dtype)
        return out

    def _layout(self, tensor):
        t2d = tensor.reshape(-1, tensor.shape[-1])
        t2d = t2d if t2d.is_contiguous() else t2d.contiguous()
        cols = t2d.shape[1]
        if self.granularity == 'per_group' and cols >= self.group_size:
            if cols % self.group_size:
                raise ValueError(f'Dimension {cols} not divisible by group size {self.group_size}')
            return t2d, self.group_size
        return t2d, cols

    def _dynamic(self, tensor, out_mode):
        """-> (out, scales [rows*ng, 1] or 0-dim)."""
        if self.calib_algo != 'minmax':
            raise NotImplementedError(f'FloatQuantizer calib_algo={self.calib_algo}')
        if self.granularity == 'per_block':
            return self._block(tensor, out_mode)
        t2d, group = self._layout(tensor)
        if self.granularity == 'per_tensor':
            mn, mx = self.get_minmax_range(t2d)
            scales, _, _, _ = self.get_qparams((mn, mx), t2d.device)     # 0-dim (fp32 for T != fp32)
            s32 = scales.reshape(1).float().contiguous()
            out = self._run(t2d, t2d.shape[1], 0, s32, out_mode, 0, 1) if out_mode else None
            return out, scales
        rows, cols = t2d.shape
        scales = torch.empty((rows * (cols // group), 1), dtype=t2d.dtype, device=t2d.device)
        out = self._run(t2d, group, 1, scales, out_mode)
        return out, scales

    def _block(self, tensor, out_mode):
        """128 x 128 block scales (quant.py:137-139, 545-553 in fp32) -> (out, scales [Mb, 1, Nb, 1])."""
        require_cuda(tensor)
        assert tensor.dim() == 2
        w = tensor if tensor.is_contiguous() else tensor.contiguous()
        M, N = w.shape
        bs = self.block_size
        mb, nb = -(-M // bs), -(-N // bs)
        fp8_dtype, e5m2 = _FP8[self.bit]
        scales = torch.empty((mb, nb), dtype=torch.float32, device=w.device)
        out = None
        if out_mode == 1:
            out = torch.empty_like(w)
        elif out_mode == 2:
            out = torch.empty(w.shape, dtype=torch.uint8, device=w.device)
        with TIMER.span('fp8_block_quant', nbytes=float(w.element_size() + 1) * M * N):
            call('llmc_fp8_block_quant', ptr(w), M, N, dtype_enum(w.dtype), int(bs), e5m2, ptr(scales),
                 out_mode, ptr(out), stream_ptr(w.device))
        if out_mode == 2:
            out = out.view(fp8_dtype)
        return out, scales.view(mb, 1, nb, 1)

    def _static(self, tensor, scales, out_mode):
        t2d, group = self._layout(tensor)
        s = scales
        if s.dim() == 0 or s.numel() == 1:
            s32 = s.reshape(1).to(device=t2d.device, dtype=torch.float32).contiguous()
            return self._run(t2d, t2d.shape[1], 0, s32, out_mode, 0, 1)
        s = s.reshape(-1).to(t2d.dtype).contiguous()
        return self._run(t2d, group, 0, s, out_mode, t2d.shape[1] // group, 0)

    # ---- reference API -----------------------------------------------------------------------------
    def get_tensor_qparams(self, tensor, args={}):
        """quant.py:1043-1059."""
        reshaped = self.reshape_tensor(tensor)
        if self.granularity == 'per_tensor':
            scales, zeros, qmax, qmin = self.get_qparams(self.get_minmax_range(reshaped), tensor.device)
            return reshaped, scales, zeros, qmax, qmin
        _, scales = self._dynamic(tensor, 0)
        return reshaped, scales, torch.tensor(0.0), self.qmax, self.qmin

    def quant(self, tensor, scales, zeros, qmax, qmin):
        """quant.py:1061-1072 -> fp32 tensor of grid values."""
        return self._static(tensor, scales, 2).float().reshape(tensor.shape)

    def dequant(self, tensor, scales, zeros):
        return (tensor - zeros) * scales

    def quant_dequant(self, tensor, scales, zeros, qmax, qmin):
        """quant.py:1078-1081 (result dtype: fp32 * T -> fp32, callers cast back)."""
        return self._static(tensor, scales, 1).reshape(tensor.shape)

    def fake_quant_weight_dynamic(self, weight, args={}):
        """quant.py:1142-1159."""
        tr = 'dim' in args and 'ic' in args['dim']
        w = weight.T if tr else weight
        out, _ = self._dynamic(w, 1)
        out = out.reshape(w.shape).to(w.dtype)
        return out.T if tr else out

    def fake_quant_weight_static(self, weight, args):
        """quant.py:1111-1140."""
        tr = 'dim' in args and 'ic' in args['dim']
        w = weight.T if tr else weight
        out = self._static(w, args['scales'], 1).reshape(w.shape).to(w.dtype)
        return out.T if tr else out

    def fake_quant_act_dynamic(self, act, args={}):
        """quant.py:1100-1109."""
        out, _ = self._dynamic(act, 1)
        return out.reshape(act.shape).to(act.dtype)

    def fake_quant_act_static(self, act, args={}):
        """quant.py:1083-1098."""
        return self._static(act, args['scales'], 1).reshape(act.shape).to(act.dtype)

    def _qshape(self, weight, scales):
        if self.granularity == 'per_tensor':
            return scales.view(1)
        if self.granularity == 'per_block':
            return scales.view(scales.shape[0], scales.shape[2])        # quant.py:1213-1214
        return scales.view(weight.shape[0], -1)

    def real_quant_weight_dynamic(self, weight, args={}):
        """quant.py:1195-1221 -> (fp8 weight, scales, None)."""
        osf = args.pop('output_scale_factor', 1) if 'output_scale_factor' in args else 1
        out, scales = self._dynamic(weight, 2)
        return out.reshape(weight.shape), self._qshape(weight, scales * osf), None

    def real_quant_weight_static(self, weight, args):
        """quant.py:1161-1193."""
        osf = args.pop('output_scale_factor', 1) if 'output_scale_factor' in args else 1
        out = self._static(weight, args['scales'], 2)
        return out.reshape(weight.shape), self._qshape(weight, args['scales'] * osf), None

    def __repr__(self):
        return (f'FloatQuantizer(bit={self.bit},e_bits={self.e_bits}, m_bits={self.m_bits},'
                f'granularity={self.granularity},kwargs={self.kwargs}, qmin={self.qmin}, qmax={self.qmax})')


def weight_cast_to_fp8(weight, block_size):
    """quant.py:32-43 -> (fp8 weight [M, N], scale_inv [ceil(M/bs), ceil(N/bs)] fp32)."""
    q = FloatQuantizer(bit='e4m3', symmetric=True, granularity='per_block', block_size=block_size,
                       use_qtorch=True)
    fp8_weight, fp8_scale, _ = q.real_quant_weight_dynamic(weight)
    return fp8_weight, fp8_scale


def weight_cast_to_bf16(weight, scale, block_size):
    """quant.py:18-29: block-FP8 checkpoint weight -> bf16."""
    require_cuda(weight, scale)
    assert weight.dtype in (torch.float8_e4m3fn, torch.float8_e5m2) and weight.dim() == 2
    w = weight.contiguous()
    M, N = w.shape
    s = scale.to(torch.float32).contiguous()
    assert s.shape == (-(-M // block_size), -(-N // block_size)), (s.shape, w.shape, block_size)
    out = torch.empty((M, N), dtype=torch.bfloat16, device=w.device)
    with TIMER.span('fp8_block_dequant', nbytes=3.0 * M * N):
        call('llmc_fp8_block_dequant', ptr(w.view(torch.uint8)), M, N, int(block_size),
             int(weight.dtype == torch.float8_e5m2), ptr(s), ptr(out), stream_ptr(w.device))
    return out
