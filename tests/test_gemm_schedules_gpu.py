"""The encoder GEMM's three schedules (cooperative 128x128 for small problems; ping-pong 128x128 for large problems with short K;
cooperative 128x256 for large problems with long K) and its bf16-output epilogues, which store 16 bytes per lane after
exchanging accumulators inside each quad of lanes.

A bf16 output must be the bf16 rounding of the fp32 value the same launch shape computes, bit for bit: any misplaced column of
the exchange shows up as a mismatch. Rows past M are never written.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(300, 384, 192, 0),        # small problem, tail tile of 44 rows: cooperative 128x128 (variant 0)
          (9500, 768, 768, 1),       # ping-pong (variant 1)
          (9259, 3072, 768, 1),      # ping-pong, N = 3072, tail tile of 43 rows
          (9500, 768, 3072, 1)]      # long K: cooperative 128x256 (variant 1)


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _gemm(L, a, b, M, N, K, bias=None, gelu_in=None, act=0, out_f32=None, out_bf16=None, out_pre=None):
    p = lambda t: None if t is None else t.data_ptr()
    L.check(L.lib().aph_gemm_epi_test(p(a), p(b), M, N, K, p(bias), None, p(gelu_in), act, p(out_f32), p(out_bf16), p(out_pre),
                                      0, 0, L.stream_ptr()), 'gemm')


def _qg(x):
    return x * torch.sigmoid(1.702 * x)


@pytest.mark.parametrize('M,N,K,variant', SHAPES)
def test_bf16_epilogues_round_the_fp32_result(L, M, N, K, variant):
    lib = L.lib()
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device='cuda') * 0.5).bfloat16()
    b = (torch.randn(N, K, device='cuda') * K ** -0.5).bfloat16()
    bias = torch.randn(N, device='cuda')
    hpre = torch.randn(M, N, device='cuda').bfloat16()
    pad = 64                                                    # rows past M: must stay untouched
    new = lambda: torch.full((M + pad, N), -7., device='cuda', dtype=torch.bfloat16)
    before = lib.aph_gemm_variant_launches(variant, -1)
    f32 = torch.empty(M, N, device='cuda')
    _gemm(L, a, b, M, N, K, out_f32=f32)
    o_bf16, o_bias, o_act, o_pre, o_grad = new(), new(), new(), new(), new()
    _gemm(L, a, b, M, N, K, out_bf16=o_bf16)
    _gemm(L, a, b, M, N, K, bias=bias, out_bf16=o_bias)
    _gemm(L, a, b, M, N, K, bias=bias, act=1, out_bf16=o_act, out_pre=o_pre)
    _gemm(L, a, b, M, N, K, gelu_in=hpre, out_bf16=o_grad)
    torch.cuda.synchronize()
    assert lib.aph_gemm_variant_launches(variant, -1) == before + 5, 'the shape did not run the expected schedule'
    assert torch.equal(o_bf16[:M], f32.bfloat16())
    assert torch.equal(o_bias[:M], (f32 + bias).bfloat16())
    assert torch.equal(o_pre[:M], (f32 + bias).bfloat16())
    # QuickGELU and its derivative use tanh.approx in the kernel: within a few bf16 ulps of the exact functions
    h = f32 + bias
    assert torch.allclose(o_act[:M].float(), _qg(h), rtol=2e-2, atol=2e-2)
    x = hpre.float()
    s = torch.sigmoid(1.702 * x)
    assert torch.allclose(o_grad[:M].float(), f32 * (s * (1. + 1.702 * x * (1. - s))), rtol=2e-2, atol=2e-2)
    for o in (o_bf16, o_bias, o_act, o_pre, o_grad):
        assert bool((o[M:] == -7.).all()), 'a row past M was written'


def test_misaligned_bf16_output_is_refused(L):
    """The bf16 epilogues store 16 bytes per lane, so their operands must be 16-byte aligned: an unaligned pointer is an
    error returned by the call, and nothing is launched."""
    from aphantasia_b200 import _lib
    M, N, K = 256, 256, 64
    a = torch.randn(M, K, device='cuda').bfloat16(); b = torch.randn(N, K, device='cuda').bfloat16()
    out = torch.zeros(M * N + 8, device='cuda', dtype=torch.bfloat16)
    n0 = L.lib().aph_launch_count()
    rc = L.lib().aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, None, None, None, 0, None, out.data_ptr() + 2, None, 0, 0,
                                   L.stream_ptr())
    assert L.lib().aph_launch_count() == n0
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        _lib.check(rc, 'gemm')
