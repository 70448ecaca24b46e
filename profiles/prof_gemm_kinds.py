"""Per-shape / per-epilogue timing of the wgmma GEMM against cuBLASLt (torch) on the same shapes, isolated launches.

    python profiles/prof_gemm_kinds.py > gemm_kinds.json

Every GEMM launch of one C2 step (ViT-B/32, S=190: M=9500 token rows) with its real fused epilogue, through the test entry
aph_gemm_epi_test, 20 timed repetitions after 3 warm-ups (CUDA events on the launching stream). Between repetitions a 256 MB
buffer is written so the operands do not sit in the 50 MB L2 (flush=1) -- and once more without the flush (what back-to-back
kernels of the step see). The cuBLASLt column is torch's bf16 matmul (+ the UNFUSED epilogue as separate torch ops, which is
what the reference's PyTorch path launches).
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aphantasia_b200 import _lib  # noqa: E402

lib, ck = _lib.lib(), _lib.check
M = 9500
SHAPES = [('bias_bf16', M, 2304, 768, 'qkv'), ('bias_resid', M, 768, 768, 'out_proj + residual'), ('bias_gelu', M, 3072, 768, 'fc1 + QuickGELU'),
          ('bias_resid', M, 768, 3072, 'fc2 + residual'), ('gelugrad', M, 3072, 768, 'd fc2 x gelu\''), ('bf16', M, 768, 3072, 'd fc1'),
          ('bf16', M, 768, 768, 'd out_proj'), ('bf16', M, 768, 2304, 'd qkv')]
PER_STEP = {'qkv': 12, 'out_proj + residual': 12, 'fc1 + QuickGELU': 12, 'fc2 + residual': 12, 'd fc2 x gelu\'': 12, 'd fc1': 12, 'd out_proj': 12, 'd qkv': 12}
flushbuf = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')


def timeit(fn, flush, reps=20):
    for _ in range(3):
        fn()
    tot = 0.
    for _ in range(reps):
        if flush:
            flushbuf.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps * 1e3      # us


def qg(x):
    return x * torch.sigmoid(1.702 * x)


def main():
    st = _lib.stream_ptr()
    rows = []
    for kind, m, n, k, what in SHAPES:
        a = (torch.randn(m, k, device='cuda') * 0.5).bfloat16(); b = (torch.randn(n, k, device='cuda') * k ** -0.5).bfloat16()
        bias = torch.randn(n, device='cuda'); resid = torch.randn(m, n, device='cuda'); hpre = torch.randn(m, n, device='cuda').bfloat16()
        of = torch.empty(m, n, device='cuda'); ob = torch.empty(m, n, device='cuda', dtype=torch.bfloat16); op = torch.empty_like(ob)
        N = None
        args = {'f32': (N, N, N, 0, of.data_ptr(), N, N), 'bf16': (N, N, N, 0, N, ob.data_ptr(), N),
                'bias_bf16': (bias.data_ptr(), N, N, 0, N, ob.data_ptr(), N), 'bias_gelu': (bias.data_ptr(), N, N, 1, N, ob.data_ptr(), op.data_ptr()),
                'bias_resid': (bias.data_ptr(), resid.data_ptr(), N, 0, of.data_ptr(), N, N), 'gelugrad': (N, N, hpre.data_ptr(), 0, N, ob.data_ptr(), N)}[kind]

        def ours():
            ck(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), m, n, k, *args, 0, 0, st), kind)
        bias_b = bias.bfloat16()

        def cublas():
            if kind == 'f32':
                return torch.matmul(a, b.T).float()
            if kind == 'bf16':
                return torch.matmul(a, b.T)
            if kind == 'bias_bf16':
                return torch.nn.functional.linear(a, b, bias_b)
            if kind == 'bias_gelu':
                h = torch.nn.functional.linear(a, b, bias_b)
                return h, qg(h)
            if kind == 'bias_resid':
                return resid + torch.nn.functional.linear(a, b, bias_b).float()
            return torch.matmul(a, b.T) * (torch.sigmoid(1.702 * hpre) * (1 + 1.702 * hpre * (1 - torch.sigmoid(1.702 * hpre))))

        def cublas_mm_only():
            return torch.matmul(a, b.T)
        fl = 2.0 * m * n * k
        r = {'kind': kind, 'what': what, 'M': m, 'N': n, 'K': k}
        for flush in (1, 0):
            t_o, t_c, t_m = timeit(ours, flush), timeit(cublas, flush), timeit(cublas_mm_only, flush)
            r['flush%d' % flush] = {'ours_us': round(t_o, 2), 'ours_tflops': round(fl / t_o / 1e6, 1), 'cublaslt_unfused_us': round(t_c, 2),
                                   'cublaslt_matmul_only_us': round(t_m, 2), 'cublaslt_matmul_only_tflops': round(fl / t_m / 1e6, 1)}
        rows.append(r)
    step = {f: {'ours_ms': sum(r[f]['ours_us'] * PER_STEP[r['what']] for r in rows) / 1e3,
                'cublaslt_unfused_ms': sum(r[f]['cublaslt_unfused_us'] * PER_STEP[r['what']] for r in rows) / 1e3,
                'cublaslt_matmul_only_ms': sum(r[f]['cublaslt_matmul_only_us'] * PER_STEP[r['what']] for r in rows) / 1e3} for f in ('flush1', 'flush0')}
    print(json.dumps({'device': torch.cuda.get_device_name(0), 'rows': rows, 'sum_over_the_96_layer_gemms_of_a_step': step}, indent=1))


if __name__ == '__main__':
    main()
