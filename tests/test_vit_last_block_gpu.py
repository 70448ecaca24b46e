"""The encoder's last residual block runs on the class-token rows only after its attention (out_proj, ln_2, fc1, fc2 and their
data-gradients at M = S), because the caller only receives what ln_post reads: rows s*T of the last block's output.

- Forward and data-gradient against the fp32 oracle at small batches (tail tiles at small M) and at the benchmark batches,
  eager / graph capture / graph replay.
- One handle driven through different batch sizes gives what a fresh handle gives (the last block's attention gradient buffer
  is zero between the cls rows and is never cleared again).
- One forward + backward at the benchmark batch launches 92 large-problem and 8 small-problem GEMMs.
- The strided GEMM operands the last block uses (A rows, residual rows and output rows at a stride) against dense launches.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restate as R  # noqa: E402


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _run(L, vis, x, cot):
    """one forward + backward through the C ABI: (embeddings, image gradient)"""
    lib = L.lib()
    S = x.shape[0]
    emb = torch.full((S, 512), float('nan'), device='cuda'); gx = torch.full(tuple(x.shape), float('nan'), device='cuda')
    L.check(lib.aph_vit_fwd(vis.handle, x.data_ptr(), S, emb.data_ptr(), 1, L.stream_ptr()), 'vit_fwd')
    L.check(lib.aph_vit_bwd(vis.handle, cot.data_ptr(), S, gx.data_ptr(), L.stream_ptr()), 'vit_bwd')
    torch.cuda.synchronize()
    return emb, gx


def _inputs(S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(S, 3, 224, 224, generator=g), torch.randn(S, 512, generator=g) * 0.1


@pytest.mark.parametrize('patch,S', [(32, 1), (32, 3), (32, 190), (16, 47)])
def test_last_block_vs_oracle_eager_capture_replay(L, patch, S):
    from aphantasia_b200.clip import VisionTransformer
    lib = L.lib()
    sd = R.synthetic_visual_state_dict(patch, 0)
    vis = VisionTransformer(sd, max_batch=S)
    x, cot = _inputs(S, 100 + S)
    xo = x.clone().requires_grad_(True)
    eo = R.build_visual(sd)(xo)
    (eo * cot).sum().backward()
    xc, cc = x.cuda(), cot.cuda()
    small, large = lambda: lib.aph_gemm_variant_launches(0, -1), lambda: lib.aph_gemm_variant_launches(1, -1)
    s0, l0 = small(), large()
    runs = [_run(L, vis, xc, cc)]                             # eager: the GEMM variant counters see each launch once
    n_small, n_large = small() - s0, large() - l0
    runs += [_run(L, vis, xc, cc) for _ in range(2)]         # capture, replay
    assert n_small + n_large == 100, (n_small, n_large)
    if S * (224 // patch) ** 2 > 9000:
        assert (n_large, n_small) == (92, 8), (n_large, n_small)
    for emb, gx in runs:
        e_emb, e_grad = _rel(emb, eo), _rel(gx, xo.grad)
        assert e_emb < 2e-2 and e_grad < 2e-2, (patch, S, e_emb, e_grad)
    for emb, gx in runs[1:]:
        assert torch.equal(emb, runs[0][0]) and torch.equal(gx, runs[0][1]), 'graph capture / replay differ from the eager call'


def test_one_handle_through_batch_sizes_matches_fresh_handles(L):
    """S = 190, 47, 190, 47, 190 on one handle (eager, eager, capture, capture, replay) against a fresh handle per batch size.
    The last block writes its attention-output gradient only on rows s*T of a buffer zeroed at creation; rows a larger batch
    wrote are either rewritten or outside what a smaller batch reads, so nothing stale can leak into a result."""
    from aphantasia_b200.clip import VisionTransformer
    sd = R.synthetic_visual_state_dict(32, 0)
    inputs = {S: tuple(t.cuda() for t in _inputs(S, 7 + S)) for S in (190, 47)}
    want = {}
    for S in (190, 47):
        fresh = VisionTransformer(sd, max_batch=S)
        want[S] = _run(L, fresh, *inputs[S])
        fresh.close()
    vis = VisionTransformer(sd, max_batch=190)
    for S in (190, 47, 190, 47, 190):
        emb, gx = _run(L, vis, *inputs[S])
        assert torch.equal(emb, want[S][0]) and torch.equal(gx, want[S][1]), 'S=%d differs from a fresh handle' % S


# ---------------------------------------------------------------------------------------------- strided GEMM operands
STRIDED = [(190, 768, 768, 50),      # the last block's out_proj / d out_proj (ViT-B/32, T = 50): small schedule
           (190, 3072, 768, 50),     # fc1, d fc2
           (190, 768, 3072, 50),     # fc2, d fc1
           (47, 768, 768, 197),      # ViT-B/16, T = 197
           (9500, 768, 768, 2),      # a row stride on the ping-pong schedule
           (9500, 768, 3072, 2)]     # ... and on the cooperative 128x256 schedule
KINDS = ['f32', 'bf16', 'bias_bf16', 'bias_gelu', 'bias_resid', 'gelugrad']


@pytest.mark.parametrize('M,N,K,T', STRIDED)
def test_strided_gemm_matches_dense_for_every_epilogue(L, M, N, K, T):
    """Rows m*T of A, of the residual and of the outputs (gelu_in at the outputs' stride), against the dense GEMM on compact
    copies (bit for bit: same schedule, same arithmetic) and against torch. Rows between the strided output rows stay untouched."""
    lib = L.lib()
    torch.manual_seed(M + N + K + T)
    p = lambda t: None if t is None else t.data_ptr()
    st = L.stream_ptr()
    a_full = (torch.randn(M * T, K, device='cuda') * 0.5).bfloat16()
    b = (torch.randn(N, K, device='cuda') * K ** -0.5).bfloat16()
    bias = torch.randn(N, device='cuda')
    resid_full = torch.randn(M * T, N, device='cuda')
    hpre_full = torch.randn(M * T, N, device='cuda').bfloat16()
    a, resid, hpre = a_full[::T].contiguous(), resid_full[::T].contiguous(), hpre_full[::T].contiguous()
    acc = a.float() @ b.float().T
    for kind in KINDS:
        f32 = kind in ('f32', 'bias_resid')
        use_bias = kind in ('bias_bf16', 'bias_gelu', 'bias_resid')
        args = lambda A, lda, R, ldr, G, of, ob, op, ldo: (p(A), lda, p(b), M, N, K, p(bias) if use_bias else None, p(R), ldr, p(G),
                                                            int(kind == 'bias_gelu'), p(of), p(ob), p(op), ldo, st)
        mk = lambda rows: (torch.full((rows, N), -7., device='cuda', dtype=torch.float32 if f32 else torch.bfloat16))
        d_out, s_out = mk(M), mk(M * T)
        d_pre, s_pre = (mk(M), mk(M * T)) if kind == 'bias_gelu' else (None, None)
        R_d, R_s = (resid, resid_full) if kind == 'bias_resid' else (None, None)
        G_d, G_s = (hpre, hpre_full) if kind == 'gelugrad' else (None, None)
        L.check(lib.aph_gemm_epi_strided_test(*args(a, 0, R_d, 0, G_d, d_out if f32 else None, None if f32 else d_out, d_pre, 0)), kind)
        L.check(lib.aph_gemm_epi_strided_test(*args(a_full, T * K, R_s, T * N, G_s, s_out if f32 else None, None if f32 else s_out,
                                                     s_pre, T * N)), kind)
        torch.cuda.synchronize()
        for d, s in ((d_out, s_out), (d_pre, s_pre)):
            if d is None:
                continue
            assert torch.equal(s[::T], d), (kind, 'strided rows differ from the dense launch')
            between = s.reshape(M, T, N)[:, 1:]
            assert bool((between == -7.).all()), (kind, 'a row between the strided output rows was written')
        want = {'f32': acc, 'bf16': acc, 'bias_bf16': acc + bias, 'bias_gelu': acc + bias, 'bias_resid': acc + bias + resid,
                'gelugrad': acc * (lambda x, s: s * (1. + 1.702 * x * (1. - s)))(hpre.float(), torch.sigmoid(1.702 * hpre.float()))}[kind]
        got = d_pre if kind == 'bias_gelu' else d_out
        assert _rel(got.float(), want) < (1e-5 if f32 else 5e-3), (kind, _rel(got.float(), want))


def test_misaligned_row_strides_are_refused(L):
    """Row strides are part of the 16-byte alignment the TMA map and the 16-byte bf16 stores need: nothing is launched."""
    lib = L.lib()
    M, N, K = 256, 256, 64
    a = torch.zeros(M * 2, K + 8, device='cuda').bfloat16(); b = torch.zeros(N, K, device='cuda').bfloat16()
    out = torch.zeros(M * 2, N + 8, device='cuda').bfloat16()
    n0 = lib.aph_launch_count()
    for lda, ldo in ((K + 4, 0), (0, N + 4)):
        rc = lib.aph_gemm_epi_strided_test(a.data_ptr(), lda, b.data_ptr(), M, N, K, None, None, 0, None, 0, None, out.data_ptr(), None,
                                           ldo, L.stream_ptr())
        with pytest.raises(RuntimeError, match='16-byte aligned'):
            L.check(rc, 'gemm')
    assert lib.aph_launch_count() == n0
