"""CPU: the GPTQ oracle on FP8 weight grids (oracle/gptq_fp8_oracle.py) against the reference's own
GPTQ run on the same layers (tests/golden/gptq_fp8_kat.pt, written by oracle/gen_gptq_fp8_golden.py
with fp8_oracle.float_quantize standing in for qtorch's rounding).

Both sides start from the reference's permuted weights and Hinv and run on one thread, so every op,
the trailing GEMMs included, has the same summation order: tmp, Losses, the scales and the deployed
fake-quant weight must agree bit for bit."""
import os

import pytest
import torch

from oracle import gptq_fp8_oracle as gfo

KAT = os.path.join(os.path.dirname(__file__), 'golden', 'gptq_fp8_kat.pt')
NAMES = [c['name'] for c in torch.load(KAT, weights_only=False)]


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _case(name):
    return next(c for c in torch.load(KAT, weights_only=False) if c['name'] == name)


def static_qparams(c):
    """What GPTQ hands the sweep for per_channel / per_tensor (search_layer_qparams, gptq.py:368-377)
    and static groups (search_group_qparams / split_qparams, :333-341, 379-395)."""
    wkw, sp = c['weight_kwargs'], c['special']
    s = c['rtn_scales'].clone()
    if wkw['granularity'] != 'per_group':
        return s
    if not sp['static_groups']:
        return None
    ng = c['Wp'].shape[1] // wkw['group_size']
    cols = s.reshape(-1, ng).t()
    return [cols[i].reshape(-1, 1) for i in range(ng)]


def test_kat_covers_the_issue_matrix():
    cases = torch.load(KAT, weights_only=False)
    bits = {c['weight_kwargs']['bit'] for c in cases}
    grans = {(c['weight_kwargs']['granularity'], c['special']['static_groups'], c['special']['actorder'])
             for c in cases}
    assert bits == {'e4m3', 'e5m2'}
    assert {('per_channel', False, True), ('per_group', False, True), ('per_group', True, True)} <= grans
    assert {c['dtype'] for c in cases} == {torch.float16, torch.bfloat16}
    assert any(c['saturated'] > 0 and c['Wp'].shape[1] > 128 for c in cases), 'a multi-block saturating layer'
    # the all-zero row of an fp16 per-channel layer: its scale underflows to 0 and the reference's
    # quant() sets it to 1 in place (quant.py:1062), which the stored buf_scales show
    c = _case('e4m3_channel_actorder_fp16')
    assert float(c['rtn_scales'][1]) == 0.0 and float(c['buf_scales'][1]) == 1.0


@pytest.mark.parametrize('name', NAMES)
def test_oracle_reproduces_reference_sweep(name, one_thread):
    c = _case(name)
    wkw, sp = c['weight_kwargs'], c['special']
    C = c['Wp'].shape[1]
    gran, gs = wkw['granularity'], wkw.get('group_size')
    Hinv = gfo.unpack_upper(c['Hinv_upper'], C)
    tmp, Losses, groups = gfo.weight_transform(c['Wp'], Hinv, wkw['bit'], gran, gs,
                                               static_qparams=static_qparams(c), perm=c['perm'])
    assert torch.equal(tmp, c['tmp_perm'])
    assert torch.equal(Losses, c['Losses'])
    assert Losses.sum().item() == c['losses_sum']
    if gran == 'per_group' and not sp['static_groups']:
        scales = torch.stack(groups, dim=1).reshape(-1, 1)                 # update_model_qparams
        assert scales.dtype == torch.float32
        assert torch.equal(scales, c['buf_scales'])
    else:
        s = c['rtn_scales'].clone()
        s[s == 0] = 1
        assert torch.equal(s, c['buf_scales'])
    invperm = torch.argsort(c['perm']) if c['perm'] is not None else None
    new_weight = tmp[:, invperm] if invperm is not None else tmp             # gptq.py:186-193
    need_perm = gran == 'per_group' and not sp['static_groups'] and sp['actorder']
    qdq = gfo.w_qdq(new_weight, c['buf_scales'], wkw['bit'], gran, gs, c['perm'] if need_perm else None,
                    invperm, c['dtype'])
    assert qdq.dtype == c['dtype'] and torch.equal(qdq, c['qdq'])
