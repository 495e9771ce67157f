"""GPU parity for the wgmma kernels: GEMM (fake-quant forward) and SYRK (GPTQ Hessian).
Floating point: compared with an fp32/fp64 torch reference of the same op; tolerance stated
per test (north_star: 1e-3 relative on the Hessian)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lin(x, w, b=None):
    from llmc_b200.module_utils import linear_forward
    return linear_forward(x, w, b)


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('M,N,K', [(128, 256, 64), (256, 512, 128), (2048, 4096, 4096),
                                   (1000, 768, 3072), (77, 264, 200), (4096, 1024, 4096)])
def test_gemm_matches_fp32_reference(dtype, M, N, K):
    torch.manual_seed(M + N + K)
    x = torch.randn(M, K, device='cuda').to(dtype)
    w = (torch.randn(N, K, device='cuda') * 0.05).to(dtype)
    b = torch.randn(N, device='cuda').to(dtype)
    y = _lin(x, w, b)
    ref = (x.double() @ w.double().t() + b.double())
    # single rounding of an fp32 accumulation: error <= 1 ulp of the output dtype plus
    # accumulation noise; bound it by 2^-8 (bf16) / 2^-10 (fp16) relative to max|ref|
    tol = (2 ** -7 if dtype == torch.bfloat16 else 2 ** -9)
    err = (y.double() - ref).abs().max().item()
    assert err <= tol * ref.abs().max().item() + 1e-6, (err, ref.abs().max().item())
    # and tighter in the mean: rounding-level
    rel = ((y.double() - ref).abs().mean() / ref.abs().mean()).item()
    assert rel < (4e-3 if dtype == torch.bfloat16 else 6e-4), rel


def test_gemm_exact_on_integer_grid():
    """Small integers are exactly representable: the tensor-core result must be exact,
    which pins the operand layouts (any swizzle / descriptor slip scrambles it)."""
    torch.manual_seed(0)
    M, N, K = 384, 768, 320
    x = torch.randint(-4, 5, (M, K), device='cuda').to(torch.bfloat16)
    w = torch.randint(-4, 5, (N, K), device='cuda').to(torch.bfloat16)
    y = _lin(x, w)
    ref = (x.float() @ w.float().t())
    assert ref.abs().max() < 2 ** 8 * 40
    assert torch.equal(y.float(), ref.to(torch.bfloat16).float())


def test_gemm_3d_input_and_no_bias():
    x = torch.randn(2, 130, 256, device='cuda', dtype=torch.float16)
    w = torch.randn(512, 256, device='cuda', dtype=torch.float16) * 0.1
    y = _lin(x, w)
    assert y.shape == (2, 130, 512)
    ref = x.float() @ w.float().t()
    assert (y.float() - ref).abs().max() < 0.05


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('T,C', [(64, 128), (512, 256), (4096, 1024), (1000, 768), (8192, 4096),
                                 (2048, 14336 // 4)])
def test_syrk_matches_reference_formula(dtype, T, C):
    """gptq.py:283-290 in fp64 vs the kernel: <= 1e-3 relative (north_star); measured ~1e-6."""
    from llmc_b200.gptq_ops import hessian_add_batch
    torch.manual_seed(T + C)
    chan = torch.exp(torch.randn(C, device='cuda'))
    H = torch.zeros(C, C, device='cuda')
    Href = torch.zeros(C, C, device='cuda', dtype=torch.float64)
    n = 0
    for bs in (1, 2):
        x = (torch.randn(bs, T, C, device='cuda') * chan).to(dtype)
        Href *= n / (n + bs)
        xf = x.reshape(-1, C).double()
        Href += (2.0 / (n + bs)) * (xf.t() @ xf)
        n = hessian_add_batch(H, n, x)
    assert n == 3
    assert torch.equal(H, H.t()), 'H must come back exactly symmetric'
    scale = Href.abs().max().item()
    err = (H.double() - Href).abs().max().item()
    assert err <= 1e-4 * scale, (err, scale)   # fp32 accumulation over 3*T terms
    d = torch.diagonal(H).double()
    dref = torch.diagonal(Href)
    assert ((d - dref).abs() / dref).max().item() < 1e-4


def test_syrk_exact_on_integer_grid():
    from llmc_b200.gptq_ops import hessian_add_batch
    torch.manual_seed(1)
    T, C = 2048, 640
    x = torch.randint(-3, 4, (1, T, C), device='cuda').to(torch.bfloat16)
    H = torch.zeros(C, C, device='cuda')
    hessian_add_batch(H, 0, x)
    xf = x.reshape(-1, C).float()
    ref = 2.0 * (xf.t() @ xf)       # n=0, b=1: H = 2 * X^T X, all integers < 2^24
    assert torch.equal(H, ref)
