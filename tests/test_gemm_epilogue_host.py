"""CPU: the host side of the fused GEMM epilogues — the interleaved gate / up weight, which linears
count as having a dense forward weight, which block shapes take the fused path, and the argument
checks of the C entry points (made before any CUDA call)."""
import ctypes

import pytest
import torch
import torch.nn as nn

from llmc_b200 import module_utils as mu
from llmc_b200 import synth


def test_interleave_gate_up_layout():
    K = 3
    wg = torch.arange(256 * K, dtype=torch.float32).reshape(256, K)
    wu = -wg - 1
    w = mu.interleave_gate_up(wg, wu)
    assert w.shape == (512, K)
    assert torch.equal(w[0:128], wg[0:128]) and torch.equal(w[128:256], wu[0:128])
    assert torch.equal(w[256:384], wg[128:256]) and torch.equal(w[384:512], wu[128:256])


def _fake_quant(lin, a_qdq=None):
    calls = []

    def w_qdq(m):
        calls.append(1)
        return m.weight.data * 2
    return mu.FakeQuantLinear.new(lin, w_qdq, a_qdq), calls


def test_dense_forward_weight_rules():
    dt = torch.bfloat16
    lin = synth.B200Linear(16, 8, bias=False).to(dt)
    assert mu.dense_forward_weight(lin, dt) is lin.weight
    assert mu.dense_forward_weight(lin, torch.float16) is None                  # dtype mismatch
    assert mu.dense_forward_weight(synth.B200Linear(16, 8).to(dt), dt) is None  # bias
    assert mu.dense_forward_weight(nn.Linear(16, 8, bias=False).to(dt), dt) is None
    h = lin.register_forward_hook(lambda *a: None)
    assert mu.dense_forward_weight(lin, dt) is None                             # hooks see the call
    h.remove()
    fq, calls = _fake_quant(lin)
    w = mu.dense_forward_weight(fq, dt)
    assert calls == [1] and w is fq.tmp_weight and torch.equal(w, lin.weight * 2)
    assert mu.dense_forward_weight(fq, dt) is w and calls == [1]                # cached, as forward
    fq.dynamic_quant_tmp_weight = True
    assert mu.dense_forward_weight(fq, dt) is None
    fq_a, _ = _fake_quant(lin, a_qdq=lambda x, m: x)
    assert mu.dense_forward_weight(fq_a, dt) is None                            # activation qdq


@pytest.mark.parametrize('hidden,heads,kv_heads,fused', [
    (512, 4, 2, True),       # head_dim 128, q 512, k / v 256
    (256, 4, 2, False),      # tiny-llama: head_dim 64
    (256, 2, 1, False),      # k width 128: not a multiple of 256
    (1024, 8, 2, True),
])
def test_fused_qkv_weight_eligibility(hidden, heads, kv_heads, fused):
    a = synth.LlamaAttention(hidden, heads, kv_heads).to(torch.bfloat16)
    w = a.fused_qkv_weight(torch.bfloat16)
    if not fused:
        assert w is None
        return
    assert torch.equal(w, torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]))
    assert a.fused_qkv_weight(torch.float16) is None
    a.v_proj = synth.B200Linear(hidden, kv_heads * 128).to(torch.bfloat16)   # with a bias
    assert a.fused_qkv_weight(torch.bfloat16) is None


@pytest.mark.parametrize('inter,fused', [(1024, True), (512, True), (520, False), (200, False)])
def test_fused_gate_up_weight_eligibility(inter, fused):
    m = synth.LlamaMLP(256, inter).to(torch.bfloat16)
    w = m.fused_gate_up_weight(torch.bfloat16)
    if not fused:
        assert w is None
        return
    assert torch.equal(w, mu.interleave_gate_up(m.gate_proj.weight, m.up_proj.weight))
    m.up_proj, _ = _fake_quant(m.up_proj, a_qdq=lambda x, mod: x)
    assert m.fused_gate_up_weight(torch.bfloat16) is None


def test_cpu_forward_keeps_the_unfused_path():
    """On CPU tensors the methods run the projections and the eager glue, as forward did."""
    torch.manual_seed(0)
    a = synth.LlamaAttention(512, 4, 2)
    x = torch.randn(2, 8, 512)
    cos, sin = synth.rope_cos_sin(8, 128, 'cpu', torch.float32)
    q, k, v = a.qkv_rope(x, (cos, sin))
    ref = a.attend(a.q_proj(x), a.k_proj(x), a.v_proj(x), (cos, sin))
    assert torch.equal(a.sdpa(q, k, v), ref)
    m = synth.LlamaMLP(512, 256)
    assert torch.equal(m.gate_up_act(x), m.act(m.gate_proj(x), m.up_proj(x)))


def test_fused_entry_points_check_arguments_without_gpu():
    from llmc_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(256)

    def last():
        return lib.llmc_b200_last_error().decode()
    assert lib.llmc_gemm_rope_qkv(p, p, p, p, p, p, p, 256, 128, 256, 256, 512, 128, 2, None) == -1
    assert 'n_q=128 and n_k=256 must be multiples of 256' in last()
    assert lib.llmc_gemm_rope_qkv(p, p, p, p, p, p, p, 200, 256, 256, 256, 512, 128, 2, None) == -1
    assert 'M a multiple of seq' in last()
    assert lib.llmc_gemm_swiglu(p, p, p, 128, 200, 512, 2, None) == -1
    assert 'inter=200 must be a positive multiple of 128' in last()
    assert lib.llmc_gemm_residual(p, p, p, p, 128, 12, 512, 2, None) == -1
    assert 'N=12 must be a multiple of 8' in last()
    assert lib.llmc_gemm_residual(p, p, None, p, 128, 16, 512, 2, None) == -1
    assert 'null pointer' in last()
