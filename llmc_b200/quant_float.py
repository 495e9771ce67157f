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


def _zeros_to_one(scales):
    """quant.py:1062 `scales[scales == 0] = 1`, in place on the caller's tensor as in the reference:
    its quant() changes the scales it is handed, and dequant / real_quant_* go on with those.  A 16-bit
    scale underflows to 0 for small groups (fp16: absmax / 57344 below ~1.7e-3 on e5m2); such a group
    is quantised with scale 1, so 1 is the scale its bytes must be exported with."""
    if torch.is_tensor(scales):
        scales.masked_fill_(scales == 0, 1)
    return scales


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
            # quant.py:979-980 would take qmin / qmax from it, but the kernels here (the quantiser, the
            # FP8 GPTQ sweep, the fp8 dequant GEMM) all scale to finfo.max and saturate there
            raise NotImplementedError('FloatQuantizer float_range: only the finfo range of e4m3 / e5m2 '
                                      'is built (no shipped fp8 YAML sets float_range)')
        fi = torch.finfo(_FP8[self.bit][0])
        self.qmax, self.qmin = torch.tensor(fi.max), torch.tensor(fi.min)
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
        if self.granularity == 'per_head':                   # quant.py:633-634: one group per head
            t2d = tensor.reshape(self.head_num, -1)
        else:
            t2d = tensor.reshape(-1, tensor.shape[-1])
        t2d = t2d if t2d.is_contiguous() else t2d.contiguous()
        cols = t2d.shape[1]
        if self.granularity == 'per_group' and cols >= self.group_size:
            if cols % self.group_size:
                raise ValueError(f'Dimension {cols} not divisible by group size {self.group_size}')
            return t2d, self.group_size
        return t2d, cols

    def _dynamic(self, tensor, out_mode):
        """-> (out, scales [rows*ng, 1] or 0-dim).  out_mode 0 returns get_qparams' scales as they
        are; the byte mode (2) returns the scales the bytes were quantised with, zeros set to 1
        (quant.py:1062), which is what real_quant_weight_dynamic exports and the fp8 GEMM reads."""
        if self.calib_algo != 'minmax':
            raise NotImplementedError(f'FloatQuantizer calib_algo={self.calib_algo}')
        if self.granularity == 'per_block':
            out, scales = self._block(tensor, out_mode)
        else:
            t2d, group = self._layout(tensor)
            if self.granularity == 'per_tensor':
                mn, mx = self.get_minmax_range(t2d)
                scales, _, _, _ = self.get_qparams((mn, mx), t2d.device)     # 0-dim (fp32 for T != fp32)
                s32 = scales.reshape(1).float().contiguous()
                out = self._run(t2d, t2d.shape[1], 0, s32, out_mode, 0, 1) if out_mode else None
            else:
                rows, cols = t2d.shape
                scales = torch.empty((rows * (cols // group), 1), dtype=t2d.dtype, device=t2d.device)
                out = self._run(t2d, group, 1, scales, out_mode)
        if out_mode == 2:
            _zeros_to_one(scales)
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
        """quant.py:1063 `tensor / scales + zeros` with torch's type promotion.  A 0-dim scale, or one of
        the tensor's dtype T, gives a T quotient (a one-element scale divides in fp32, torch's CPU
        scalar-operand path).  Scales with dimensions of another dtype promote the quotient, and the
        QDQ product, to fp32: the tensor is widened to fp32 first, so nothing is rounded to T (out_mode
        1 then returns fp32, which the callers cast back as the reference's `.to(org_dtype)` does)."""
        t2d, group = self._layout(tensor)
        s = scales.to(t2d.device)
        if s.dim() and s.dtype != t2d.dtype:
            if torch.promote_types(t2d.dtype, s.dtype) != torch.float32:
                raise TypeError(f'FloatQuantizer static scales of {s.dtype} for a {t2d.dtype} tensor')
            t2d = t2d.float()
        if s.numel() == 1:
            s32 = s.reshape(1).float().contiguous()
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
        """quant.py:1061-1072 -> fp32 tensor of grid values (zero scales set to 1 in place)."""
        _zeros_to_one(scales)
        return self._static(tensor, scales, 2).float().reshape(tensor.shape)

    def dequant(self, tensor, scales, zeros):
        return (tensor - zeros) * scales

    def quant_dequant(self, tensor, scales, zeros, qmax, qmin):
        """quant.py:1078-1081: the fp32 grid values times the scales -> fp32 (callers cast back)."""
        return self.dequant(self.quant(tensor, scales, zeros, qmax, qmin), scales, zeros)

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
        out = self._static(w, _zeros_to_one(args['scales']), 1).reshape(w.shape).to(w.dtype)
        return out.T if tr else out

    def fake_quant_act_dynamic(self, act, args={}):
        """quant.py:1100-1109."""
        out, _ = self._dynamic(act, 1)
        return out.reshape(act.shape).to(act.dtype)

    def fake_quant_act_static(self, act, args={}):
        """quant.py:1083-1098."""
        return self._static(act, _zeros_to_one(args['scales']), 1).reshape(act.shape).to(act.dtype)

    def fake_quant_act_static_rows(self, act, scales):
        """fake_quant_act_static on a 0-dim scale, with one scale per row of act instead (a grouped MoE
        layer's rows each under their expert's scale): the same llmc_fp8_quant pass in QDQ mode with
        fp32 scales and row stride 1, as real_quant_act runs it for bytes, so row r is bit for bit what
        the 0-dim scales[r] gives it.  Zero scales read as 1 (quant.py:1062) on a copy: the caller's
        tensor is not modified."""
        t2d = act.reshape(-1, act.shape[-1])
        t2d = t2d if t2d.is_contiguous() else t2d.contiguous()
        s = scales.reshape(-1).to(device=t2d.device, dtype=torch.float32, copy=True)
        _zeros_to_one(s)
        return self._run(t2d, t2d.shape[1], 0, s, 1, 1, 1).reshape(act.shape)

    def real_quant_act(self, act, input_scale=None):
        """The e4m3 bytes and fp32 scales of the W8A8 real-quant forward (llmc_gemm_w8a8_fp8): the bytes
        the fake-quant forward of the same config rounds to, from the same llmc_fp8_quant pass, so
        rT(fp32(byte) * scale) is its QDQ activation bit for bit.  A zero scale is returned as 1, the
        scale the bytes were quantised with (quant.py:1062).  -> (e4m3 [rows, K], fp32 [rows] or [1]).
          input_scale None: per-token dynamic (fake_quant_act_dynamic).
          input_scale given: per-tensor static (fake_quant_act_static on its 0-dim scale); the caller's
            tensor is not modified.  One value, or one per row (a grouped MoE layer's rows each under
            their expert's input_scale): the same pass and arithmetic, row r under scale r; -> scales
            fp32 [1] or [rows]."""
        if self.bit != 'e4m3':
            raise NotImplementedError(f'W8A8 real-quant FP8 activations are e4m3, not {self.bit}')
        t2d = act.reshape(-1, act.shape[-1])
        t2d = t2d if t2d.is_contiguous() else t2d.contiguous()
        if input_scale is None:
            if self.granularity != 'per_token':
                raise NotImplementedError(f'dynamic FP8 activations are per_token, not {self.granularity}')
            out, scales = self._dynamic(t2d, 2)
            return out, scales.reshape(-1).float()
        if self.granularity != 'per_tensor' or input_scale.numel() not in (1, t2d.shape[0]):
            raise NotImplementedError('static FP8 activations take one per_tensor input_scale (or one per row)')
        s = input_scale.reshape(-1).to(device=t2d.device, dtype=torch.float32, copy=True)
        _zeros_to_one(s)
        return self._run(t2d, t2d.shape[1], 0, s, 2, int(s.numel() != 1), 1), s

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
        out = self._static(weight, _zeros_to_one(args['scales']), 2)
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


_FP8_BLOCK_ONLY_128 = ('block_size={}: the block-FP8 forward is built for 128 only — the reference '
                       "hard-wires fp8_gemm's K step and scale index to 128 (kernel.py:143, 196)")


def act_quant(x, block_size=128):
    """kernel.py:31-53 -> (e4m3 tensor of x's shape, fp32 scales [*x.shape[:-1], K/128]).

    Per contiguous group of 128 elements s = max|x| / 448 and y = e4m3(x / s), with the approximate
    division the reference's kernel compiles to (csrc/fp8.cu).  An all-zero group gives s = 0 and NaN
    codes, as in the reference.  x: bf16, fp16 or fp32, any leading dims."""
    if block_size != 128:
        raise NotImplementedError(_FP8_BLOCK_ONLY_128.format(block_size))
    require_cuda(x)
    K = x.shape[-1]
    if K % block_size:
        raise ValueError(f'Last dimension size must be divisible by block_size (block_size={block_size})')
    xc = x if x.is_contiguous() else x.contiguous()
    y = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    s = torch.empty((*x.shape[:-1], K // block_size), dtype=torch.float32, device=x.device)
    rows = x.numel() // K if K else 0
    if rows:
        with TIMER.span('fp8_act_quant', nbytes=(x.element_size() + 1 + 4.0 / block_size) * rows * K):
            call('llmc_fp8_act_quant', ptr(xc), rows, K, dtype_enum(x.dtype), ptr(y), ptr(s),
                 stream_ptr(x.device))
    return y.view(torch.float8_e4m3fn), s


def gemm_fp8_block(a, a_s, b, b_s, out_dtype, bias=None):
    """llmc_gemm_fp8_block: a [..., K] e4m3 with a_s [..., K/128], b [N, K] e4m3 with
    b_s [ceil(N/128), K/128] -> [..., N] of out_dtype (fp32, or bf16 with an optional bias added
    after the rounding)."""
    require_cuda(a, a_s, b, b_s, bias)
    if a.dtype != torch.float8_e4m3fn or b.dtype != torch.float8_e4m3fn:
        raise TypeError(f'fp8 GEMM operands must be float8_e4m3fn (got {a.dtype}, {b.dtype})')
    K = a.shape[-1]
    N = b.shape[0]
    if b.dim() != 2 or b.shape[1] != K:
        raise ValueError(f'weight shape {tuple(b.shape)} does not match K={K}')
    if K % 128:
        raise ValueError(f'K={K} must be a multiple of 128')
    a2 = a.reshape(-1, K)
    a2 = a2 if a2.is_contiguous() else a2.contiguous()
    M = a2.shape[0]
    sa = a_s.reshape(M, K // 128).to(torch.float32).contiguous()
    sb = b_s.to(torch.float32).contiguous()
    if tuple(sb.shape) != (-(-N // 128), K // 128):
        raise ValueError(f'weight scales {tuple(sb.shape)} != [ceil(N/128), K/128] = '
                         f'[{-(-N // 128)}, {K // 128}]')
    bc = b if b.is_contiguous() else b.contiguous()
    bt = None
    if bias is not None:
        bt = bias.contiguous()
        if bt.dtype not in (torch.float32, torch.float16, torch.bfloat16) or bt.numel() != N:
            raise ValueError(f'bias must be [N={N}] fp32 / fp16 / bf16 (got {bt.dtype} {tuple(bt.shape)})')
    y = torch.empty((M, N), dtype=out_dtype, device=a.device)
    with TIMER.span('gemm_fp8_block', flops=2.0 * M * N * K,
                    nbytes=float(M * K + N * K) + 4.0 * (M + N / 128) * K / 128 + y.element_size() * M * N):
        call('llmc_gemm_fp8_block', ptr(a2.view(torch.uint8)), ptr(sa), ptr(bc.view(torch.uint8)), ptr(sb),
             ptr(bt), dtype_enum(bt.dtype) if bt is not None else 0, ptr(y), dtype_enum(out_dtype),
             M, N, K, stream_ptr(a.device))
    return y.reshape(*a.shape[:-1], N)


def fp8_gemm(a, a_s, b, b_s):
    """kernel.py:217-242: block-scaled e4m3 GEMM on the FP8 tensor cores -> [..., N] of
    torch.get_default_dtype() (fp32 unless changed; bf16 is also built)."""
    dt = torch.get_default_dtype()
    if dt not in (torch.float32, torch.bfloat16):
        raise NotImplementedError(f'fp8_gemm output dtype {dt}: only fp32 and bf16 are built')
    return gemm_fp8_block(a, a_s, b, b_s, dt)


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
