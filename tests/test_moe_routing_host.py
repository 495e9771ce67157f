"""CPU: the routing metadata of the grouped MoE forward (module_utils.moe_routing) against a Python
loop, and what the grouped MoE entry points refuse before any CUDA call."""
import ctypes
import os
import re

import pytest
import torch

from llmc_b200.module_utils import moe_routing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _routing_loop(sel, E):
    """perm / offsets / rows as the eager loop sees them: expert by expert, torch.where order."""
    T, k = sel.shape
    perm, offsets, where = [], [0], {}
    for e in range(E):
        tok, slot = torch.where(sel == e)
        for t, s in zip(tok.tolist(), slot.tolist()):
            where[(t, s)] = len(perm)
            perm.append(t * k + s)
        offsets.append(len(perm))
    rows = [[where[(t, s)] for s in sorted(range(k), key=lambda s: int(sel[t, s]))] for t in range(T)]
    return (torch.tensor(perm, dtype=torch.int64), torch.tensor(offsets, dtype=torch.int32),
            torch.tensor(rows, dtype=torch.int64).view(T, k))


def _random_sel(T, E, k, g):
    return torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int64)


def _check(sel, E):
    perm, offsets, rows = moe_routing(sel, E)
    p_o, off_o, rows_o = _routing_loop(sel, E)
    assert perm.dtype == torch.int64 and offsets.dtype == torch.int32 and rows.dtype == torch.int64
    assert torch.equal(perm, p_o)
    assert torch.equal(offsets, off_o)
    assert torch.equal(rows, rows_o)
    # every token's k rows hold its k (token, slot) pairs, experts ascending
    T, k = sel.shape
    flat = sel.reshape(-1)
    for t in range(T):
        pairs = perm[rows[t]]
        assert sorted((pairs // k).tolist()) == [t] * k
        assert flat[pairs].tolist() == sorted(sel[t].tolist())


@pytest.mark.parametrize('k', [1, 2])
@pytest.mark.parametrize('T,E', [(1, 8), (7, 4), (300, 8), (129, 3)])
def test_random_routings(T, E, k):
    g = torch.Generator().manual_seed(T * 31 + E * 7 + k)
    _check(_random_sel(T, E, k, g), E)


@pytest.mark.parametrize('k', [1, 2])
def test_empty_experts(k):
    g = torch.Generator().manual_seed(5)
    sel = _random_sel(50, 3, k, g)
    sel = torch.where(sel == 2, torch.full_like(sel, 7), sel)       # experts 2..6 get nothing
    sel = torch.where(sel == 1, torch.full_like(sel, 4), sel)
    _check(sel, 8)
    off = moe_routing(sel, 8)[1].tolist()
    assert [off[e + 1] - off[e] for e in (1, 2, 3, 5, 6)] == [0] * 5


def test_all_tokens_on_one_expert():
    sel = torch.full((200, 1), 5, dtype=torch.int64)
    _check(sel, 8)
    assert moe_routing(sel, 8)[1].tolist() == [0] * 6 + [200] * 3
    sel2 = torch.stack([torch.full((200,), 6), torch.full((200,), 2)], dim=1).to(torch.int64)
    _check(sel2, 8)
    assert moe_routing(sel2, 8)[1].tolist() == [0, 0, 0, 200, 200, 200, 200, 400, 400]


def test_moe_cap_matches_header():
    from llmc_b200 import _lib
    src = open(os.path.join(ROOT, 'include', 'llmc_b200.h')).read()
    assert int(re.search(r'#define LLMC_MOE_MAX_EXPERTS (\d+)', src).group(1)) == _lib.MOE_MAX_EXPERTS
    assert _lib.MOE_MAX_EXPERTS >= 8            # Mixtral-8x7B


def test_moe_argument_validation_without_gpu():
    """The grouped MoE entry points reject bad arguments before any CUDA call."""
    from llmc_b200 import _lib
    lib = _lib.load()
    p, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    cap = _lib.MOE_MAX_EXPERTS

    def ptrs(n, addr=256):
        return (ctypes.c_void_p * n)(*([addr] * n))

    def last():
        return lib.llmc_b200_last_error().decode()

    swiglu, down, combine = lib.llmc_moe_gemm_swiglu, lib.llmc_moe_gemm_down, lib.llmc_moe_combine
    w = ptrs(cap + 1)
    # more experts than the kernel-parameter space holds, and none
    assert swiglu(p, w, w, p, p, 256, 512, 256, cap + 1, _lib.BF16, null) == -1
    assert 'experts outside 1..%d' % cap in last()
    assert down(p, w, p, p, p, 256, 256, 512, 0, _lib.BF16, null) == -1
    assert 'experts outside' in last()
    # inter not a multiple of 128, N not a multiple of 8
    assert swiglu(p, w, w, p, p, 256, 500, 256, 4, _lib.BF16, null) == -1
    assert 'inter=500' in last()
    assert down(p, w, p, p, p, 256, 100, 512, 4, _lib.BF16, null) == -1
    assert 'N=100' in last()
    # K not a multiple of 8 / a misaligned pointer
    assert swiglu(p, w, w, p, p, 256, 512, 100, 4, _lib.BF16, null) == -4
    assert 'K=100' in last()
    assert swiglu(ctypes.c_void_p(258), w, w, p, p, 256, 512, 256, 4, _lib.BF16, null) == -4
    assert swiglu(p, ptrs(4, 264), w, p, p, 256, 512, 256, 4, _lib.BF16, null) == -4
    assert 'expert 0 not 16-byte aligned' in last()
    # null pointers: the offsets, the routing weights, one expert's weight
    assert swiglu(p, w, w, null, p, 256, 512, 256, 4, _lib.BF16, null) == -1
    assert 'null pointer' in last()
    assert down(p, w, p, null, p, 256, 256, 512, 4, _lib.BF16, null) == -1
    assert 'null pointer' in last()
    w3 = ptrs(4)
    w3[2] = None
    assert swiglu(p, w, w3, p, p, 256, 512, 256, 4, _lib.BF16, null) == -1
    assert 'null weight of expert 2' in last()
    # fp32 is not a GEMM dtype, refused before the rows == 0 return like every scalar argument
    assert swiglu(p, w, w, p, p, 256, 512, 256, 4, _lib.F32, null) == -1
    assert swiglu(null, w, w, null, null, 0, 512, 256, 4, _lib.F32, null) == -1
    assert 'dtype must be bf16 or fp16' in last()
    # combine: N not a multiple of 8, top_k 0, dtype
    assert combine(p, p, p, 16, 2, 100, _lib.BF16, null) == -4
    assert combine(p, p, p, 16, 0, 128, _lib.BF16, null) == -1
    assert combine(p, p, p, 16, 2, 128, _lib.F32, null) == -1
    # no rows / tokens: a no-op that touches no pointer
    assert swiglu(null, w, w, null, null, 0, 512, 256, 4, _lib.BF16, null) == 0
    assert down(null, w, null, null, null, 0, 256, 512, 4, _lib.BF16, null) == 0
    assert combine(null, null, null, 0, 2, 128, _lib.BF16, null) == 0
