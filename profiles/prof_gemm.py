"""Stand-alone launcher of the wgmma GEMM on the step's shapes: prints time and TFLOP/s per shape (and is a small target for profilers)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from aphantasia_b200 import _lib
lib, ck = _lib.lib(), _lib.check
shapes = [(9500, 768, 768), (9500, 3072, 768), (9500, 768, 3072), (9500, 2304, 768)]
for (M, N, K) in shapes:
    a = torch.randn(M, K, device='cuda').bfloat16(); b = torch.randn(N, K, device='cuda').bfloat16(); c = torch.empty(M, N, device='cuda')
    for _ in range(3):
        ck(lib.aph_gemm_bf16_tn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, _lib.stream_ptr()), 'gemm')
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ck(lib.aph_gemm_bf16_tn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, _lib.stream_ptr()), 'gemm')
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print('%dx%dx%d: %.1f us  %.0f TFLOP/s' % (M, N, K, ms * 1e3, 2.0 * M * N * K / ms / 1e9))
