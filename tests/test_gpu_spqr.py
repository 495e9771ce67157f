"""GPU parity: SpQR's column sweep (llmc_spqr_colblock through the C ABI) and the SpQR algorithm class
against layers the reference's own SpQR produced (tests/golden/spqr_kat.pt, oracle/gen_spqr_golden.py)
and against the CPU oracle.

Bars: a 128-column problem involves no GEMM between blocks -> tmp / mask / scales / zeros bit-exact;
multi-block layers see the 3xTF32 trailing update instead of the reference's fp32 GEMM -> 1e-4 on tmp,
>= 99.5 % equal mask bits; from (W, H) through the GPU Hessian-free path (the golden H) and
llmc_chol_inv_upper -> 1e-3 on the loss."""
import math
import os

import pytest
import torch

from oracle import spqr_oracle as so

pytestmark = pytest.mark.gpu


def _kat(golden_dir):
    return torch.load(os.path.join(golden_dir, 'spqr_kat.pt'), weights_only=False)


def _cfgs(c):
    wk, l2 = c['weight_kwargs'], c['level2']
    wcfg = (wk['bit'], wk['symmetric'], wk.get('round_zp', True), wk['group_size'])
    l2c = (l2['bit'], l2['symmetric'], l2.get('round_zp', True))
    return wcfg, l2c


def _sweep(c, Wp, Hinv):
    from llmc_b200 import gptq_ops as ops
    wcfg, l2c = _cfgs(c)
    Wp, Hinv = Wp.cuda().contiguous(), Hinv.cuda().contiguous()
    thr = ops.spqr_threshold(Wp, Hinv, c['special']['relative_threshold'])
    out = ops.spqr_transform(Wp.clone(), Hinv, wcfg, l2c, l2c, thr, c['special']['simplified_outliers'])
    return thr, [t.cpu() for t in out]


def test_threshold_matches_reference_formula(golden_dir):
    for c in _kat(golden_dir):
        from llmc_b200 import gptq_ops as ops
        thr = ops.spqr_threshold(c['Wp'].cuda(), c['Hinv'].cuda(), c['special']['relative_threshold'])
        ref = so.threshold_of(c['Wp'], c['Hinv'], c['special']['relative_threshold'])
        if math.isinf(ref):
            assert math.isinf(float(thr))
        else:
            assert abs(float(thr) - ref) <= 1e-5 * ref


def test_single_block_bit_exact(golden_dir):
    """First 128 columns of every golden layer as a problem of its own, with the ORACLE's threshold
    handed to the kernel (the device reduction of var / mean may differ in the last bit)."""
    from llmc_b200 import gptq_ops as ops
    for c in _kat(golden_dir):
        wcfg, l2c = _cfgs(c)
        cnt = 128
        Wb, Hb = c['Wp'][:, :cnt].contiguous(), c['Hinv'][:cnt, :cnt].contiguous()
        thr = so.threshold_of(c['Wp'], c['Hinv'], c['special']['relative_threshold'])
        cfg = so.make_cfg(c['weight_kwargs'], c['special'], c['level2'], c['level2'], thr)
        ref = so.row_block(Wb, Hb, cfg)
        thr_t = torch.tensor([thr], dtype=torch.float32, device='cuda')
        tmp, mask, losses, S, Z = ops.spqr_transform(Wb.cuda(), Hb.cuda(), wcfg, l2c, l2c, thr_t,
                                                      c['special']['simplified_outliers'])
        assert torch.equal(tmp.cpu(), ref[0]), c['name']
        assert torch.equal(mask.cpu(), ref[2]), c['name']
        assert torch.equal(S.cpu(), ref[3]) and torch.equal(Z.cpu(), ref[4]), c['name']
        assert torch.equal(losses.cpu(), ref[5]), c['name']
        # and therefore equal to what the reference itself produced for those columns
        assert torch.equal(tmp.cpu(), c['tmp_perm'][:, :cnt])
        assert torch.equal(mask.cpu().bool(), c['mask_perm'][:, :cnt])


def test_layers_match_reference(golden_dir):
    for c in _kat(golden_dir):
        thr, (tmp, mask, losses, S, Z) = _sweep(c, c['Wp'], c['Hinv'])
        ref_max = float(c['tmp_perm'].abs().max())
        assert float((tmp - c['tmp_perm']).abs().max()) <= 1e-4 * ref_max, c['name']
        assert float((mask.bool() == c['mask_perm']).float().mean()) >= 0.995, c['name']
        assert abs(float(losses.double().sum()) - c['losses_sum']) <= 1e-4 * c['losses_sum'], c['name']
        assert float((S.reshape(-1, 1) - c['buf_scales']).abs().max()) <= 1e-4 * float(c['buf_scales'].abs().max())
        assert float((Z.reshape(-1, 1) - c['buf_zeros']).abs().max()) <= 1e-3 * float(c['buf_zeros'].abs().max())


def _fake_layer_algo(c):
    """A SpQR object around ONE linear, fed the golden Hessian (the SYRK has its own tests)."""
    from llmc_b200.quant import IntegerQuantizer
    from llmc_b200.spqr import SpQR, _level2
    a = SpQR.__new__(SpQR)
    wk = dict(c['weight_kwargs'])
    a.wquantizer = IntegerQuantizer(**wk)
    sp = c['special']
    a.actorder, a.percdamp = sp['actorder'], sp['percdamp']
    a.relative_threshold = math.inf if sp['relative_threshold'] == 'inf' else float(sp['relative_threshold'])
    a.simplified_outliers = sp['simplified_outliers']
    a.scale_cfg, a.zero_cfg = _level2(c['level2'], 'scale'), _level2(c['level2'], 'zero')
    a.need_perm = bool(a.actorder)
    a.model_dtype = torch.bfloat16
    a.block_idx, a.losses, a._chol_infos, a._chol_pending = 0, {}, [], []
    layer = torch.nn.Linear(c['W'].shape[1], c['W'].shape[0], bias=False).cuda()
    layer.weight.data = c['W'].cuda()
    _, s, z, qmax, qmin = a.wquantizer.get_tensor_qparams(layer.weight.data)
    for k, v in (('buf_scales', s), ('buf_zeros', z), ('buf_qmax', qmax), ('buf_qmin', qmin)):
        layer.register_buffer(k, v.clone() if torch.is_tensor(v) else torch.tensor(v))
    a.layers_cache = {'l': {'share': 'l', 'H': c['H'].cuda().clone(), 'reduced': True}}
    return a, layer


def test_layer_transform_and_wqdq_match_reference(golden_dir):
    """SpQR._transform_group (damping rule of spqr.py:143-151, llmc_chol_inv_upper, sweep) and
    w_qdq on its result, against the reference's layer_transform / w_qdq of the same (W, H)."""
    for c in _kat(golden_dir):
        a, layer = _fake_layer_algo(c)
        a._transform_group([('l', layer)])
        a.check_factorizations(wait=True)
        loss = float(a.losses['0.l'].double().sum())
        assert abs(loss - c['losses_sum']) <= 1e-3 * c['losses_sum'], (c['name'], loss, c['losses_sum'])
        if c['perm'] is not None:
            assert float((layer.buf_perm.cpu() == c['perm']).float().mean()) >= 0.95
        same_mask = float((layer.buf_mask.cpu().float() == c['buf_mask']).float().mean())
        assert same_mask >= 0.99, (c['name'], same_mask)
        rel = float((layer.weight.data.cpu() - c['new_weight']).abs().max() / c['new_weight'].abs().max())
        assert rel <= 2e-2, (c['name'], rel)          # a flipped outlier moves one weight by up to a step
        q = a.w_qdq(layer, a.wquantizer).cpu()
        assert q.dtype == torch.bfloat16
        same = float((q == c['qdq']).float().mean())
        assert same >= 0.97, (c['name'], same)
        # w_qdq alone, on the reference's own buffers: exact
        layer.weight.data = c['new_weight'].cuda()
        layer.buf_scales, layer.buf_zeros = c['buf_scales'].cuda(), c['buf_zeros'].cuda()
        layer.register_buffer('buf_mask', c['buf_mask'].to(torch.uint8).cuda())
        if c['perm'] is not None:
            layer.register_buffer('buf_perm', c['perm'].cuda())
            layer.register_buffer('buf_invperm', torch.argsort(c['perm']).cuda())
        assert torch.equal(a.w_qdq(layer, a.wquantizer).cpu(), c['qdq']), c['name']


def test_model_width_properties():
    """4096 x 4096, group 16 (the shipped spqr_w_only.yml): deterministic, finite, a plausible
    outlier rate, outliers keep their compensated weight, everything else lies on its group's grid."""
    from llmc_b200 import gptq_ops as ops
    torch.manual_seed(3)
    R = C = 4096
    W = (torch.randn(R, C, device='cuda') * 0.02)
    W[torch.rand(R, C, device='cuda') < 0.002] *= 10
    chan = torch.exp(torch.randn(C, device='cuda') * 0.7)
    H = torch.zeros(C, C, device='cuda')
    n = 0
    for _ in range(4):
        n = ops.hessian_add_batch(H, n, (torch.randn(1, 2048, C, device='cuda') * chan).bfloat16())
    perm = torch.argsort(torch.diag(H), descending=True)
    Wp, Hp = ops.prepare(W.bfloat16(), H, perm, 1.0)
    Hinv = ops.chol_inv_upper(Hp)
    thr = ops.spqr_threshold(Wp, Hinv, 0.2)
    cfg = ((4, False, False, 16), (3, False, False), (3, False, False))
    outs = [ops.spqr_transform(Wp.clone(), Hinv, *cfg, thr, False, out_perm=perm) for _ in range(2)]
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    tmp, mask, losses, S, Z = outs[0]
    assert torch.isfinite(tmp).all() and torch.isfinite(losses).all() and torch.isfinite(S).all()
    frac = float(mask.float().mean())
    assert frac < 0.2, frac
    # permuted view: quantise the non-outliers with the returned qparams -> error below half a step
    tp = tmp[:, perm].reshape(R, C // 16, 16)
    s, z = S.unsqueeze(-1), Z.unsqueeze(-1)
    q = torch.clamp(torch.round(tp / s.clamp_min(1e-9) + z), 0, 15)
    dq = (q - z) * s
    inside = (q > 0) & (q < 15)
    assert float(((dq - tp).abs() / s)[inside].max()) <= 0.5 + 1e-3


def test_lane_kernel_bit_identical_to_row_kernel(golden_dir, monkeypatch):
    """The 16-lanes-per-row in-block kernel (the default) against the thread-per-row kernel
    (LLMC_B200_SPQR_KERNEL=row): same per-element operation sequences (spqr_row.cuh: lanes_* vs row_block, equal on the
    host by tests/test_oracle_golden.py), so every output must be bit-identical — on the reference
    layers and on a 1000 x 1024 layer with act-order scatter; timings of both go to gpurun_out/."""
    import json
    import time
    from llmc_b200 import gptq_ops as ops
    cases = []
    for c in _kat(golden_dir):
        wcfg, l2c = _cfgs(c)
        cases.append((c['name'], c['Wp'].cuda(), c['Hinv'].cuda(), wcfg, l2c, c['special']['relative_threshold'],
                      c['special']['simplified_outliers'], None))
    torch.manual_seed(9)
    R, C = 1000, 1024
    W = torch.randn(R, C, device='cuda') * 0.02
    W[torch.rand(R, C, device='cuda') < 0.01] *= 8
    H = torch.zeros(C, C, device='cuda')
    ops.hessian_add_batch(H, 0, (torch.randn(1, 4096, C, device='cuda') * torch.exp(torch.randn(C, device='cuda') * 0.7)).bfloat16())
    perm = torch.argsort(torch.diag(H), descending=True)
    Wp, Hp = ops.prepare(W.bfloat16(), H, perm, 1.0)
    cases.append(('rand_1000x1024', Wp, ops.chol_inv_upper(Hp), (4, False, False, 16), (3, False, False), 0.2, False, perm))
    times = {}
    for name, Wp, Hinv, wcfg, l2c, rel, simp, op in cases:
        thr = ops.spqr_threshold(Wp, Hinv, rel)
        outs = {}
        for kern in ('row', 'lanes'):
            monkeypatch.setenv('LLMC_B200_SPQR_KERNEL', kern)
            ops.spqr_transform(Wp.clone(), Hinv, wcfg, l2c, l2c, thr, simp, out_perm=op)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs[kern] = ops.spqr_transform(Wp.clone(), Hinv, wcfg, l2c, l2c, thr, simp, out_perm=op)
            torch.cuda.synchronize()
            times[f'{name}_{kern}_ms'] = (time.perf_counter() - t0) * 1e3
        monkeypatch.delenv('LLMC_B200_SPQR_KERNEL')
        for a, b in zip(outs['row'], outs['lanes']):
            assert torch.equal(a, b), name
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, 'spqr_kernels.json'), 'w') as fh:
            json.dump(times, fh, indent=1)
    except OSError:
        pass
