"""GPU parity at the BENCHMARK configuration: the kernels bench.py actually times (VERDICT r1 items 2a-2e).

At S=190 ViT-B/32 (M = 9500 token rows) and S=47 ViT-B/16 (M = 9259) launch_gemm selects the 128 x 256 tiles with fused
epilogues and the forward / backward launch chains are replayed from the CUDA-graph cache; the small-shape tests of
test_gpu_parity.py never reach those code paths. Reference call sites: clip_fft.py:254 (encode_image at S=190), :240
(slice_imgs), :235-295 (whole step). Tolerances: north_star (1e-3 fp32, 2e-2 bf16), norm-wise.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restate as R  # noqa: E402


def _rel(a, b):
    a = torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a)).double()
    b = torch.as_tensor(np.asarray(b.detach().cpu() if torch.is_tensor(b) else b)).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _seed(s):
    torch.manual_seed(int(s)); np.random.seed(int(s))


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


EPI = dict(f32=0, bf16=1, bias_bf16=2, bias_gelu=3, bias_resid=4, gelugrad=5, unpatch=6)


def _quickgelu(x):
    return x * torch.sigmoid(1.702 * x)


def _quickgelu_grad(x):
    s = torch.sigmoid(1.702 * x)
    return s * (1. + 1.702 * x * (1. - s))


# ---------------------------------------------------------------------------------------------- (b) every epilogue kind, wide tiles
@pytest.mark.parametrize('kind,M,N,K', [
    ('f32', 9500, 768, 3072),            # d fc1 (ViT-B/32 data-gradient)
    ('bf16', 9500, 768, 768),            # d out_proj
    ('bf16', 9500, 768, 3072),           # d fc1 (bf16 gradient into the LayerNorm backward)
    ('bf16', 9500, 768, 2304),           # d qkv
    ('bf16', 9259, 768, 768),            # ViT-B/16 batch: tail tile of 43 rows
    ('bias_bf16', 9500, 2304, 768),      # qkv
    ('bias_gelu', 9500, 3072, 768),      # fc1 + QuickGELU (saves the pre-activation)
    ('bias_resid', 9500, 768, 3072),     # fc2 + residual
    ('bias_resid', 9500, 768, 768),      # out_proj + residual
    ('gelugrad', 9500, 3072, 768),       # d fc2 x gelu'(h)
    ('unpatch', 9310, 3072, 768),        # conv1 data-gradient scattered to NCHW (ViT-B/32: 190 x 49 patches, p=32)
    ('bias_resid', 9259, 768, 3072),     # ViT-B/16, S=47: M = 47*197 (tail tile of 43 rows)
    ('gelugrad', 9259, 3072, 768),
    ('unpatch', 9212, 768, 768),         # ViT-B/16: 47 x 196 patches, p=16
])
# test id kept stable across the port: the large-tile variant it checks is now the 128x256 wgmma tile
def test_pair_gemm_epilogue_kinds_at_bench_size(L, kind, M, N, K):
    lib = L.lib()
    _seed(M + N + K + EPI[kind])
    dev = 'cuda'
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=dev) * (K ** -0.5)).bfloat16()
    acc = a.float() @ b.float().T
    bias = torch.randn(N, device=dev)
    resid = torch.randn(M, N, device=dev)
    hpre = torch.randn(M, N, device=dev).bfloat16()
    nul = None
    wide_launches = lambda: lib.aph_gemm_variant_launches(1, EPI[kind])     # 128x256 tiles
    before = wide_launches()
    st = L.stream_ptr()
    if kind == 'f32':
        out = torch.full((M, N), float('nan'), device=dev)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, nul, nul, nul, 0, out.data_ptr(), nul, nul, 0, 0, st), kind)
        checks = [(out, acc, 1e-5)]
    elif kind == 'bf16':
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, nul, nul, nul, 0, nul, out.data_ptr(), nul, 0, 0, st), kind)
        checks = [(out.float(), acc, 3e-3)]
    elif kind == 'bias_bf16':
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, bias.data_ptr(), nul, nul, 0, nul, out.data_ptr(), nul, 0, 0, st), kind)
        checks = [(out.float(), acc + bias, 3e-3)]
    elif kind == 'bias_gelu':
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16); pre = torch.zeros_like(out)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, bias.data_ptr(), nul, nul, 1, nul, out.data_ptr(), pre.data_ptr(), 0, 0, st), kind)
        checks = [(pre.float(), acc + bias, 3e-3), (out.float(), _quickgelu(acc + bias), 4e-3)]
    elif kind == 'bias_resid':
        out = torch.full((M, N), float('nan'), device=dev)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, bias.data_ptr(), resid.data_ptr(), nul, 0, out.data_ptr(), nul, nul, 0, 0, st), kind)
        checks = [(out, acc + bias + resid, 1e-5)]
    elif kind == 'gelugrad':
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, nul, nul, hpre.data_ptr(), 0, nul, out.data_ptr(), nul, 0, 0, st), kind)
        checks = [(out.float(), acc * _quickgelu_grad(hpre.float()), 4e-3)]
    else:
        p = int(round((N // 3) ** 0.5)); g = 224 // p; S = M // (g * g)
        assert S * g * g == M and 3 * p * p == N
        out = torch.full((S, 3, 224, 224), float('nan'), device=dev)
        L.check(lib.aph_gemm_epi_test(a.data_ptr(), b.data_ptr(), M, N, K, nul, nul, nul, 0, out.data_ptr(), nul, nul, p, g, st), kind)
        ref = acc.reshape(S, g, g, 3, p, p).permute(0, 3, 1, 4, 2, 5).reshape(S, 3, 224, 224)
        checks = [(out, ref, 1e-5)]
    torch.cuda.synchronize()
    assert wide_launches() == before + 1, 'this shape did not run the 128x256-tile kernel'
    for got, want, tol in checks:
        assert torch.isfinite(got).all()
        assert _rel(got, want) < tol, (kind, M, N, K, _rel(got, want))
    # rows past M must not have been touched by the tail tile: outputs are exactly M rows here, so check the last valid row instead
    assert _rel(checks[0][0][-1:], checks[0][1][-1:]) < 10 * checks[0][2]


# ---------------------------------------------------------------------------------------------- (a) ViT at the benchmark batch
@pytest.mark.parametrize('patch,S', [(32, 190), (16, 47)])
def test_vit_at_bench_batch_vs_oracle_incl_graph_replay(L, patch, S):
    """Forward + data-gradient of the full ViT-B at the benchmark batch through the C ABI with FIXED buffers, three times:
    call 1 runs eagerly, call 2 captures the CUDA graph, call 3 replays it. All three must match the fp32 oracle."""
    from aphantasia_b200.clip import VisionTransformer
    lib = L.lib()
    sd = R.synthetic_visual_state_dict(patch, 0)
    vis = VisionTransformer(sd, max_batch=S)
    ref = R.build_visual(sd)
    _seed(40 + patch)
    x = torch.randn(S, 3, 224, 224)
    cot = torch.randn(S, 512) * 0.1
    xo = x.clone().requires_grad_(True)
    eo = ref(xo)
    (eo * cot).sum().backward()
    xc, gc = x.cuda(), cot.cuda()
    emb = torch.empty(S, 512, device='cuda'); gx = torch.empty(S, 3, 224, 224, device='cuda')
    wides = lambda: lib.aph_gemm_variant_launches(1, -1)
    wide_before = wides()
    errs = []
    for it in range(3):
        emb.fill_(float('nan')); gx.fill_(float('nan'))
        L.check(lib.aph_vit_fwd(vis.handle, xc.data_ptr(), S, emb.data_ptr(), 1, L.stream_ptr()), 'vit_fwd')
        L.check(lib.aph_vit_bwd(vis.handle, gc.data_ptr(), S, gx.data_ptr(), L.stream_ptr()), 'vit_bwd')
        torch.cuda.synchronize()
        if it == 0:
            assert wides() - wide_before >= 90, 'the 128x256-tile kernels were not selected at this batch'
        errs.append((_rel(emb, eo), _rel(gx, xo.grad)))
    print('vit B/%d S=%d: rel err (emb, grad) eager %s capture %s replay %s' % (patch, S, errs[0], errs[1], errs[2]))
    for e_emb, e_grad in errs:
        assert e_emb < 2e-2 and e_grad < 2e-2
    assert abs(errs[2][0] - errs[0][0]) < 1e-3 and abs(errs[2][1] - errs[0][1]) < 1e-3       # the replay computes the same thing


# ---------------------------------------------------------------------------------------------- (c) sampler at C2
def test_sampler_c2_values_and_canvas_gradient(L):
    """720x1280 canvas, S=190, transforms_fast (BASELINE configs[1]) vs the oracle's per-crop loop (utils.py:243-253)."""
    from aphantasia_b200 import _rng, transforms
    from aphantasia_b200.utils import slice_imgs
    H, W, S = 720, 1280, 190
    _seed(21)
    canvas = torch.rand(1, 3, H, W)
    cc = canvas.cuda().requires_grad_(True)
    _seed(22)
    out = slice_imgs([cc], S, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
    _seed(22)
    tabs, _ = _rng.draw_crop_table(S, (H, W), 224, 2, 'uniform', 0.4)
    co = canvas.clone().requires_grad_(True)
    ref = R.sample_crops(co, tabs[0], 224, 2)
    _seed(23)
    cot = torch.randn(ref.shape)
    (out * cot.cuda()).sum().backward()
    (ref * cot).sum().backward()
    assert tuple(out.shape) == (S, 3, 224, 224)
    assert _rel(out, ref) < 1e-5
    assert _rel(cc.grad, co.grad) < 1e-4


# ---------------------------------------------------------------------------------------------- (d) the whole C2 step
def test_full_step_config2_vs_oracle(L):
    """BASELINE configs[1] (1280x720 FFT, S=190, ViT-B/32, mix loss): loss, embeddings and d loss / d spectrum vs the oracle,
    through the reference-facing entry points (what clip_fft.py's train(i) executes)."""
    from aphantasia_b200 import _rng, transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.image import fft_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    h, w, S = 720, 1280, 190
    sd = synthetic_visual_state_dict(patch=32, seed=0)
    model = CLIP('ViT-B/32', sd, True)
    _seed(0)
    params, image_f, _ = fft_image([1, 3, h, w], 0.07, 1.5, None)
    rgb_f = to_valid_rgb(image_f, colors=1.8)
    g = torch.Generator().manual_seed(1234)
    txt = torch.randn(1, 512, generator=g); txt = (10. * txt / txt.norm()).cuda()
    _seed(1)
    crops = slice_imgs([rgb_f()], S, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
    emb = model.encode_image(crops)
    loss = -1. * sim_func(txt, emb, 'mix')
    loss.backward()
    _seed(1)
    tabs, _ = _rng.draw_crop_table(S, (h, w), 224, 2, 'uniform', 0.4)
    o_loss, o_grad, o_emb = R.reference_step(params[0].detach().cpu(), R.fft_scale(h, w, 1.5), (h, w), R.color_matrix(1.8), tabs[0],
                                             R.build_visual(sd), txt.cpu(), 'mix')
    e_emb, e_grad = _rel(emb, o_emb), _rel(params[0].grad, o_grad)
    print('config2: loss ours %.6f oracle %.6f; rel emb %.3e grad %.3e' % (loss.item(), o_loss.item(), e_emb, e_grad))
    assert e_emb < 2e-2 and e_grad < 2e-2
    assert abs(loss.item() - o_loss.item()) < 2e-3


# ---------------------------------------------------------------------------------------------- (e) C3 at S=47
def test_full_step_config3_vs_oracle_unpinned_dwt(L):
    """BASELINE configs[2]: --dwt --wave db3 1920x1080, S=47, ViT-B/16. The DWT restatement is PARITY UNPINNED
    (pytorch_wavelets / PyWavelets absent); everything downstream of it is pinned as in the other tests."""
    from aphantasia_b200 import _rng, transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.image import dwt_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    h, w, S = 1080, 1920, 47
    sd = synthetic_visual_state_dict(patch=16, seed=0)
    model = CLIP('ViT-B/16', sd, True)
    _seed(5)
    Ys, gen, _ = dwt_image([1, 3, h, w], 'db3', 0.3, 1.8, None)
    rgb_f = to_valid_rgb(gen, colors=1.8)
    g = torch.Generator().manual_seed(1234)
    txt = torch.randn(1, 512, generator=g); txt = (10. * txt / txt.norm()).cuda()
    _seed(6)
    crops = slice_imgs([rgb_f()], S, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
    emb = model.encode_image(crops)
    loss = -1. * sim_func(txt, emb, 'mix')
    loss.backward()
    # oracle
    _seed(6)
    tabs, _ = _rng.draw_crop_table(S, (h, w), 224, 2, 'uniform', 0.4)
    rec_lo, rec_hi = R.wavelet_filters('db3')
    Yo = [y.detach().cpu().clone().requires_grad_(True) for y in Ys]
    o_rgb = R.valid_rgb(R.synth_dwt(Yo, rec_lo, rec_hi, 0.3, 1.0), R.color_matrix(1.8))
    o_emb = R.build_visual(sd)(R.sample_crops(o_rgb, tabs[0], 224, 2))
    o_loss = -1. * R.sim_func(txt.cpu(), o_emb, 'mix')
    o_loss.backward()
    ga = torch.cat([y.grad.reshape(-1) for y in Ys]); gb = torch.cat([y.grad.reshape(-1) for y in Yo])
    e_emb, e_grad = _rel(emb, o_emb), _rel(ga, gb)
    print('config3: loss ours %.6f oracle %.6f; rel emb %.3e grad %.3e' % (loss.item(), o_loss.item(), e_emb, e_grad))
    assert e_emb < 2e-2 and e_grad < 2.5e-2
    assert abs(loss.item() - o_loss.item()) < 2e-3


# ---------------------------------------------------------------------------------------------- --enforce: two forwards, one backward
def test_two_grad_tracked_forwards_before_backward(L):
    """clip_fft.py --enforce (:254, :276) runs encode_image twice on the same model before loss.backward(); the handle owns one
    activation arena, so the first call's backward must recompute its forward (ADVICE r1, high). Checked against the oracle."""
    from aphantasia_b200.clip import CLIP
    from aphantasia_b200.utils import sim_func
    S = 4
    sd = R.synthetic_visual_state_dict(32, 0)
    model = CLIP('ViT-B/32', sd, True)
    ref = R.build_visual(sd)
    _seed(9)
    x1, x2 = torch.randn(S, 3, 224, 224), torch.randn(S, 3, 224, 224)
    txt = torch.randn(1, 512)
    a1, a2 = x1.cuda().requires_grad_(True), x2.cuda().requires_grad_(True)
    e1 = model.encode_image(a1)
    e2 = model.encode_image(a2)
    loss = -sim_func(txt.cuda(), e1, 'mix') - 0.5 * sim_func(e1, e2, 'mix')          # clip_fft.py:259,277
    loss.backward()
    b1, b2 = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
    o1, o2 = ref(b1), ref(b2)
    (-R.sim_func(txt, o1, 'mix') - 0.5 * R.sim_func(o1, o2, 'mix')).backward()
    assert model.visual.recomputes == 1
    assert _rel(a1.grad, b1.grad) < 2e-2 and _rel(a2.grad, b2.grad) < 2e-2


# ---------------------------------------------------------------------------------------------- sampler -> encoder patch operand
@pytest.mark.parametrize('patch', [32, 16])
def test_sampler_emits_patch_operand_for_the_encoder(L, patch):
    """SURVEY 2.4 k10-k12: slice_imgs' last stage writes the bf16 patch-major conv1 operand into the encoder handle and
    encode_image on that very tensor skips k_patchify. Same embeddings and canvas gradient, bit for bit, as the plain route
    (the operand is the same rounding of the same fp32 values); a derived tensor, an in-place edit, a second forward on the stale
    buffer or two live encoders must take the plain route."""
    import gc
    from aphantasia_b200 import _patchlink, transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.utils import sim_func, slice_imgs
    gc.collect()
    lib = L.lib()
    model = CLIP('ViT-B/%d' % patch, synthetic_visual_state_dict(patch=patch, seed=0), True)
    vis = model.visual
    _patchlink._consumers.clear()                 # encoders other tests left alive would (correctly) switch the hand-over off
    _patchlink.register(vis)
    _seed(3)
    canvas = torch.rand(1, 3, 360, 640, device='cuda')
    txt = torch.randn(1, 512).cuda()

    def run(fuse, kind=transforms.transforms_fast, mutate=None):
        os.environ['APH_PATCH_FUSE'] = '1' if fuse else '0'
        c = canvas.clone().requires_grad_(True)
        _seed(5)
        n0, f0 = lib.aph_launch_count(), vis.prepatched_forwards
        crops = slice_imgs([c], 12, 224, kind, 'uniform', 0.4)[0]
        if mutate:
            crops = mutate(crops)
        emb = model.encode_image(crops)
        n1 = lib.aph_launch_count()
        (-sim_func(txt, emb, 'mix')).backward()
        return emb.detach().clone(), c.grad.clone(), n1 - n0, vis.prepatched_forwards - f0
    try:
        for _ in range(3):
            run(False)                                                     # past the encoder's eager / capture steps: launch counts settle
        e0, g0, n_plain, f_plain = run(False)
        e1, g1, n_fused, f_fused = run(True)
        assert f_plain == 0 and f_fused == 1
        assert torch.equal(e0, e1), 'embeddings differ between the plain and the prepatched route: %g' % _rel(e1, e0)
        assert _rel(g1, g0) < 1e-5                                         # (the canvas gradient accumulates with atomics: not bit-stable)
        assert n_fused == n_plain - 1, (n_plain, n_fused)                  # k_patchify is gone, nothing else changed
        e2, g2, _, f2 = run(True, kind=transforms.normalize())             # the resize kernel emits the operand for kinds without a warp stage
        e3, g3, _, f3 = run(False, kind=transforms.normalize())
        assert f2 == 1 and f3 == 0 and torch.equal(e2, e3) and _rel(g2, g3) < 1e-5
        e4, g4, _, f4 = run(True, mutate=lambda t: t * 1.0)                # a derived tensor carries no stamp
        assert f4 == 0 and torch.equal(e4, e0)
        # a second forward of the same batch after another batch went through the encoder: the buffer is stale -> plain route
        c = canvas.clone()
        _seed(5)
        crops = slice_imgs([c], 12, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
        other = model.encode_image(torch.randn(12, 3, 224, 224, device='cuda'))
        f0 = vis.prepatched_forwards
        again = model.encode_image(crops)
        assert vis.prepatched_forwards == f0 and torch.equal(again, e0) and not torch.equal(other, e0)
        # in-place edit of the stamped tensor -> version mismatch -> plain route on the edited values
        _seed(5)
        crops = slice_imgs([c], 12, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
        crops.mul_(0.5)
        f0 = vis.prepatched_forwards
        half = model.encode_image(crops)
        assert vis.prepatched_forwards == f0 and not torch.equal(half, e0)
        # two live encoders (--dualmod): no target
        model2 = CLIP('ViT-B/16' if patch == 32 else 'ViT-B/32', synthetic_visual_state_dict(patch=48 - patch, seed=0), True)
        assert _patchlink.target(224) is None
        del model2
    finally:
        os.environ.pop('APH_PATCH_FUSE', None)
        del model, vis
        gc.collect()


# ---------------------------------------------------------------------------------------------- loss heads, fused Adam (rows f2 / f4)
def test_derivat_and_aesthetic_head_vs_torch(L):
    from aphantasia_b200.utils import aesthetic_model, derivat
    _seed(3)
    img = torch.rand(1, 3, 90, 130)
    ic = img.cuda().requires_grad_(True)
    v = derivat(ic, mode='naiv')
    (v * 3.).backward()
    io = img.clone().requires_grad_(True)
    dx = torch.mean(torch.abs(io[:, :, :, 1:] - io[:, :, :, :-1])); dy = torch.mean(torch.abs(io[:, :, 1:, :] - io[:, :, :-1, :]))
    ((0.5 * (dx + dy)) * 3.).backward()                                   # utils.py:265-268
    assert _rel(v, 0.5 * (dx + dy)) < 1e-6 and _rel(ic.grad, io.grad) < 1e-5
    head = aesthetic_model('ViT-B/32').cuda()
    e = torch.randn(19, 512)
    ec = e.cuda().requires_grad_(True)
    out = head(ec)
    assert tuple(out.shape) == (19, 1)
    (-0.001 * 0.5 * out.mean()).backward()                                # clip_fft.py:256
    eo = e.clone().requires_grad_(True)
    ro = torch.nn.functional.linear(eo, head.weight.cpu().reshape(1, -1), head.bias.cpu())
    (-0.001 * 0.5 * ro.mean()).backward()
    assert _rel(out, ro) < 1e-6 and _rel(ec.grad, eo.grad) < 1e-6


def test_fused_adam_shim_matches_torch_adam(L):
    """aphantasia_b200.optim.Adam over an fft_image spectrum (update fused into the synthesis backward) vs torch.optim.Adam on
    the same gradients, 3 steps incl. an lr change between steps (the script's --prog writes param_groups[...]['lr'])."""
    from aphantasia_b200 import optim
    from aphantasia_b200.image import fft_image, to_valid_rgb
    h, w = 96, 160
    _seed(5)
    pa, fa, _ = fft_image([1, 3, h, w], 0.07, 1.5, None)
    pb, fb, _ = fft_image([1, 3, h, w], 0.07, 1.5, pa[0].detach().clone())
    ra, rb = to_valid_rgb(fa, colors=1.8), to_valid_rgb(fb, colors=1.8)
    oa = optim.Adam(pa, 0.05, betas=(.0, .999))
    ob = torch.optim.Adam(pb, 0.05, betas=(.0, .999))
    for i in range(3):
        for grp in list(oa.param_groups) + list(ob.param_groups):
            grp['lr'] = 0.05 * (1 + i)
        cot = torch.randn(1, 3, h, w, device='cuda')
        oa.zero_grad(); (ra() * cot).sum().backward(); oa.step()
        ob.zero_grad(); (rb() * cot).sum().backward(); ob.step()
        with torch.no_grad():
            ra(contrast=1.1)                                               # the script's preview synthesis between steps (no grad)
    assert oa.fused_steps == 3 and pa[0].grad is None
    assert _rel(pa[0], pb[0]) < 1e-5
