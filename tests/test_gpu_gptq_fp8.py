"""GPU: GPTQ on FP8 weight grids — llmc_gptq_colblock_fp8 (csrc/gptq.cu) against the oracle, and the
shipped vLLM / SGLang FP8 GPTQ recipes end to end.

The sweep is checked bit for bit on the structured Hinv of test_gpu_sweep_trailing.py (real 128 x 128
diagonal blocks, one exact power-of-two entry per later column), where every trailing-update
schedule gives the oracle's bits: tmp and the dynamic group scales must be identical, per-row losses
agree to 1e-5 (the kernel sums a row in another order).  On the reference's own layers
(gptq_fp8_kat.pt, a real Hinv) the first 128-column block is bit-exact and the rest differs from the
CPU BLAS only by the summation order of the trailing dot products.
PARITY UNPINNED at the rounding step itself (qtorch; oracle/fp8_oracle.py)."""
import functools
import math
import os

import pytest
import torch

import test_gpu_sweep_trailing as tst
from oracle import fp8_oracle as fo
from oracle import gptq_fp8_oracle as gfo

pytestmark = pytest.mark.gpu

DT = {'fp16': torch.float16, 'bf16': torch.bfloat16}
# bit, model dtype, R, C, granularity (group size or 'channel'), static groups, act-order, saturating
CASES = {
    'e4m3-channel-fp16-333x1152-actorder': dict(bit='e4m3', dt='fp16', R=333, C=1152, group=None, perm=True),
    'e5m2-channel-bf16-200x2560': dict(bit='e5m2', dt='bf16', R=200, C=2560, group=None),
    'e4m3-channel-bf16-333x1152-saturating': dict(bit='e4m3', dt='bf16', R=333, C=1152, group=None, sat=True),
    'e5m2-channel-fp16-96x1000-saturating-simt': dict(bit='e5m2', dt='fp16', R=96, C=1000, group=None,
                                                       sat=True),
    'e4m3-g128-dynamic-333x1152-actorder': dict(bit='e4m3', dt='bf16', R=333, C=1152, group=128, perm=True),
    'e5m2-g128-dynamic-200x2560': dict(bit='e5m2', dt='fp16', R=200, C=2560, group=128),
    'e4m3-g64-dynamic-333x1664': dict(bit='e4m3', dt='fp16', R=333, C=1664, group=64),
    'e4m3-g128-static-fp16-520x2560-actorder-gmap': dict(bit='e4m3', dt='fp16', R=520, C=2560, group=128,
                                                         static=True, perm=True),
    'e5m2-g128-static-bf16-333x1152': dict(bit='e5m2', dt='bf16', R=333, C=1152, group=128, static=True),
}


@functools.lru_cache(maxsize=None)
def _problem(name):
    c = CASES[name]
    R, C, dt = c['R'], c['C'], DT[c['dt']]
    g = tst._seed(name)
    W = (torch.randn(R, C, generator=g) * 0.02 * torch.exp(0.3 * torch.randn(R, 1, generator=g))).to(dt).float()
    Hinv = tst._structured_hinv(tst._diag_blocks(C, g), g)
    perm = torch.randperm(C, generator=g) if c.get('perm') else None
    group = c['group'] or C
    gran = 'per_group' if c['group'] else 'per_channel'
    static = None
    if gran == 'per_channel' or c.get('static'):
        # collect_block_qparams on the model-dtype weight in its original column order; a saturating
        # case takes the scales of half the weight, so |w / s| reaches twice finfo.max
        W_orig = (W[:, torch.argsort(perm)] if perm is not None else W).to(dt)
        if c.get('sat'):
            W_orig = W_orig * 0.5
        t = W_orig.reshape(-1, group) if gran == 'per_group' else W_orig
        static = fo.qparams(t, c['bit'], gran).reshape(R, -1)
        assert static.dtype == dt
    return dict(c, W=W, Hinv=Hinv, perm=perm, group=group, gran=gran, static=static,
                tensor_path=C % 8 == 0)


@functools.lru_cache(maxsize=None)
def _oracle(name):
    p = _problem(name)
    sq = s = p['static']
    if s is not None and p['gran'] == 'per_group':
        sq = [s[:, i:i + 1] for i in range(s.shape[1])]
    return gfo.weight_transform(p['W'], p['Hinv'], p['bit'], p['gran'], p['group'], static_qparams=sq,
                                perm=p['perm'], trailing_split=p['tensor_path'])


def _sweep(p, W=None, rows=None):
    """ops.weight_transform on the device as GPTQ._transform_group calls it (rows: a row range)."""
    from llmc_b200 import gptq_ops as ops
    W = p['W'] if W is None else W
    lo, hi = rows or (0, W.shape[0])
    kw = {}
    if p['static'] is not None:
        kw['static_qparams'] = (p['static'][lo:hi].reshape(-1).cuda(), None)
        if p['perm'] is not None and p['gran'] == 'per_group':
            kw['gmap'] = (p['perm'] // p['group']).to(torch.int32).cuda()
    if p['perm'] is not None:
        kw['out_perm'] = p['perm'].cuda()
    out = ops.weight_transform(W[lo:hi].cuda().contiguous(), p['Hinv'].cuda(), p['bit'], True, p['group'], **kw)
    tmp, losses, scales, zeros = (t.cpu() if t is not None else None for t in out)
    assert zeros is None
    if p['perm'] is not None:
        tmp = tmp[:, p['perm']]
    return tmp, losses, scales


@pytest.mark.parametrize('name', list(CASES))
def test_fp8_sweep_bit_exact(name, monkeypatch):
    p = _problem(name)
    tmp_o, L_o, groups = _oracle(name)
    if p.get('sat'):
        fmax = torch.finfo(fo.FP8[p['bit']]).max
        assert (tmp_o.abs() > fmax * p['static'].float()).any(), 'the case must saturate'
    bad = {}
    for sched in tst._schedules(monkeypatch):
        tmp, losses, scales = _sweep(p)
        msgs = [tst._diff('tmp', tmp, tmp_o)]
        if p['static'] is None:
            msgs.append(tst._diff('scales', scales, torch.cat(groups, 1)))
        if not torch.allclose(losses, L_o.sum(1), rtol=1e-5, atol=0):
            msgs.append('losses: max rel %.3g' % float(((losses - L_o.sum(1)).abs() / L_o.sum(1)).max()))
        msgs = [m for m in msgs if m]
        if msgs:
            bad[sched] = msgs
    assert not bad, bad


@pytest.mark.parametrize('name', ['e4m3-g128-dynamic-333x1152-actorder', 'e5m2-channel-bf16-200x2560'])
def test_stacked_and_row_sharded_sweeps_equal_per_linear(name):
    """Rows are independent given Hinv: stacking two linears row-wise (q/k/v, gate/up) and sweeping a
    row range (the data-parallel shard) give each row the bits of its own sweep."""
    p = _problem(name)
    R = p['W'].shape[0]
    full = _sweep(p)
    cut = R // 3
    parts = [_sweep(p, rows=(0, cut)), _sweep(p, rows=(cut, R))]
    for i in range(3):
        assert torch.equal(torch.cat([parts[0][i], parts[1][i]]), full[i])


def test_kat_layers_first_block_bit_exact(golden_dir):
    """The reference's own layers (real Hinv): block 0 bit-exact, the rest within summation order."""
    from llmc_b200 import gptq_ops as ops
    kat = torch.load(os.path.join(golden_dir, 'gptq_fp8_kat.pt'), weights_only=False)
    for c in kat:
        wkw, sp = c['weight_kwargs'], c['special']
        R, C = c['Wp'].shape
        gran = wkw['granularity']
        gs = wkw.get('group_size') if gran == 'per_group' else C
        kw = {}
        if gran != 'per_group' or sp['static_groups']:
            s = c['rtn_scales']
            s = s.reshape(1).expand(R) if s.dim() == 0 else s
            kw['static_qparams'] = (s.reshape(-1).contiguous().cuda(), None)
            if gran == 'per_group' and c['perm'] is not None:
                kw['gmap'] = (c['perm'] // gs).to(torch.int32).cuda()
        Hinv = gfo.unpack_upper(c['Hinv_upper'], C).cuda()
        tmp, losses, scales, _ = ops.weight_transform(c['Wp'].cuda().clone(), Hinv, wkw['bit'], True, gs, **kw)
        tmp = tmp.cpu()
        assert torch.equal(tmp[:, :128], c['tmp_perm'][:, :128]), c['name']
        ls = losses.double().sum().item()
        assert abs(ls - c['losses_sum']) <= 2e-3 * abs(c['losses_sum']), (c['name'], ls, c['losses_sum'])
        assert (tmp - c['tmp_perm']).abs().max().item() <= 2e-2 * c['tmp_perm'].abs().max().item()
        if 'static_qparams' not in kw:
            ng = C // gs
            ref = c['buf_scales'].reshape(-1, ng)
            assert torch.equal(scales.cpu()[:, :1], ref[:, :1]), c['name']


def test_fp8_entry_point_validates_arguments():
    from llmc_b200._lib import load
    lib = load()
    W = torch.zeros(128, 256, device='cuda')
    H = torch.eye(256, device='cuda')
    s = torch.ones(128, 2, device='cuda')
    out = torch.empty_like(W)
    loss = torch.empty(128, device='cuda')
    nb = lib.llmc_gptq_workspace_bytes(128, 256)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    p = lambda t: t.data_ptr()   # noqa: E731

    def run(e5m2=0, group=128, static=0, q_dtype=0, wsb=nb):
        return lib.llmc_gptq_colblock_fp8(p(W), p(H), 128, 256, group, e5m2, static, None, p(s), q_dtype,
                                          p(out), None, p(loss), p(ws), wsb, None)
    assert run(e5m2=2) == -1
    assert run(group=96) == -1
    assert run(q_dtype=1) == -1                 # dynamic groups write fp32 scales
    assert run(wsb=16) == -1
    assert run() == 0
    torch.cuda.synchronize()
    assert torch.equal(out, W) and float(loss.abs().max()) == 0.0


YAMLS = ['backend/vllm/fp8/gptq_fp8.yml', 'backend/sglang/fp8/gptq_fp8.yml']


def _linear_weights(model):
    return {n + '.weight': m.weight.detach().clone() for n, m in model.get_model().named_modules()
            if hasattr(m, 'weight') and isinstance(getattr(m, 'weight', None), torch.Tensor)
            and m.weight.dim() == 2 and 'layers.' in n}


@pytest.mark.parametrize('rel', YAMLS)
def test_shipped_fp8_gptq_yaml_runs_end_to_end(rel, tmp_path):
    """`python -m llmc_b200` main on the tiny Llama, the YAML used as shipped (model / data / sizes /
    save path overridden): finite fake-quant PPL, and the saved checkpoint holds weights on the
    e4m3 grid whose product with weight_scale is the deployed fake-quant weight.  The reference's
    config.json patch then fails on these YAMLs: with float-quant activations it reads
    weight.block_size (export_vllm.py:33-39), which a per-channel weight does not have; export.py
    does the same."""
    from safetensors.torch import load_file
    from llmc_b200.__main__ import adapt_reference_config, main
    from llmc_b200.synth import perplexity
    from test_ref_yamls import _docs
    doc = _docs()[rel]
    kw = dict(n_samples=8, seq_len=128, eval_seq_len=128)
    cfg = adapt_reference_config(doc, 'tiny-llama', save_path=str(tmp_path), **kw)
    assert cfg['quant'] == doc['quant']
    # 1. calibration + fake-quant evaluation, without the save step
    cfg_eval = dict(cfg)
    cfg_eval.pop('save')
    algo, model, report = main(cfg_eval, quiet=True)
    assert type(algo.wquantizer).__name__ == 'FloatQuantizer' and algo.wquantizer.bit == 'e4m3'
    if 'ppl_fake_quant' not in report:          # eval_pos 'fake-quant' (sic) is not an eval position
        algo.deploy('fake_quant')
        g = torch.Generator().manual_seed(4)
        tokens = torch.randint(0, model.shape['vocab'], (1, 128 * 8), generator=g)
        report['ppl_fake_quant'] = perplexity(model, tokens, 128, 1)
    ppl = report['ppl_fake_quant']
    assert math.isfinite(ppl) and ppl < 1e4, ppl
    fake = _linear_weights(model)
    assert fake
    # 2. the same run with the save step: the checkpoint is written, then config.json patching fails
    with pytest.raises(AttributeError, match='block_size'):
        main(cfg, quiet=True)
    sd = load_file(os.path.join(str(tmp_path), 'sgl_quant_model', 'model.safetensors'))
    n = 0
    for name, w in fake.items():
        # GPTQ.deploy ends in convert_dtype (gptq.py:459; `blocks[i].to(dtype)` in the reference), which
        # casts the e4m3 codes to the model dtype as well: the saved weight holds e4m3 grid values
        q = sd[name].float()
        assert torch.equal(q.to(torch.float8_e4m3fn).float(), q), name
        s = sd[name[:-len('weight')] + 'weight_scale'].reshape(-1, 1)
        assert s.shape[0] == q.shape[0]
        deq = (q.float() * s.float()).to(w.dtype)
        assert torch.equal(deq, w.cpu()), name
        n += 1
    assert n == len(fake)


@pytest.mark.parametrize('weight,special', [
    (dict(bit='e5m2', granularity='per_group', group_size=128), dict(actorder=True, static_groups=False)),
    (dict(bit='e4m3', granularity='per_group', group_size=128), dict(actorder=True, static_groups=True)),
    (dict(bit='e4m3', granularity='per_group', group_size=64), dict(actorder=False, static_groups=False)),
    (dict(bit='e4m3', granularity='per_tensor'), dict(actorder=False, static_groups=False)),
])
def test_gptq_fp8_granularities_through_main(weight, special):
    """The GPTQ host path on the other FP8 configurations (dynamic groups with act-order deploy through
    the W[:, perm] / [:, invperm] gathers of gptq.py:427-450): weight-only, the shipped FP8 recipe's
    other settings, finite fake-quant PPL close to the unquantised model's."""
    from llmc_b200.__main__ import adapt_reference_config, main
    from test_ref_yamls import _docs
    doc = _docs()['backend/sglang/fp8/gptq_fp8.yml']
    cfg = adapt_reference_config(doc, 'tiny-llama', n_samples=8, seq_len=128, eval_seq_len=128)
    cfg.pop('save')
    cfg['quant'] = dict(cfg['quant'], weight=dict(cfg['quant']['weight'], **weight),
                        special=dict(cfg['quant']['special'], **special))
    cfg['quant'].pop('act')
    cfg['eval']['eval_pos'] = ['pretrain', 'fake_quant']
    algo, model, report = main(cfg, quiet=True)
    assert algo.need_perm == (weight['granularity'] == 'per_group' and special['actorder']
                              and not special['static_groups'])
    ppl, ppl0 = report['ppl_fake_quant'], report['ppl_pretrain']
    assert math.isfinite(ppl) and abs(ppl - ppl0) <= 0.05 * ppl0, (ppl, ppl0)
