"""CLIP ViT-L/14 on the GPU: the streaming attention kernels (T > 256) against float64, the patch-14 embedding (operand rows
padded from 3 p^2 = 588 to 640 columns), the encoder against the fp32 oracle at small and full geometry, the 768-wide text
tower, a whole optimisation step, and the public clip.load('ViT-L/14') path.

Attention bars: the rounding budget of tests/test_encoder_kernels_gpu.py (module docstring): 2u = 7.8e-3 per (sample, head)
block for every output and 1e-2 per output row of the forward, against a float64 reference computed from the same bf16
operands, with dS / 8 rounded to bf16 where the kernels round it. The streaming kernels round at the same places as the
resident ones: P (the A operand of P V, and of dV = P^T dO), dS / 8, and each output.
"""
import ctypes as C
import gc
import os

import numpy as np
import pytest
import torch

from oracle import restate as R
from test_encoder_kernels_gpu import BLOCK_BAR, REGIMES, ROW_BAR, make_qkv, ref_attention, rel_err, split_heads

pytestmark = pytest.mark.gpu
VITL14 = dict(patch=14, width=1024, layers=24, heads=16, out_dim=768, res=224)
LONG_SEQ = [257, 258, 271, 272, 273, 320, 577]
SHORT_SEQ = [1, 197, 256]


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _seed(s):
    torch.manual_seed(int(s)); np.random.seed(int(s))


def _rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def per_sample_err(a, b):
    a, b = a.detach().cpu().double().flatten(1), b.detach().cpu().double().flatten(1)
    return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item(), float((a - b).norm() / b.norm())


# ---------------------------------------------------------------------------------------------------------- streaming attention
def run_long(L, fwd, qkv, dout, S, T, heads):
    D = 64 * heads
    out = torch.full((S * T, D if fwd else 3 * D), float('nan'), device='cuda', dtype=torch.bfloat16)
    L.check(L.lib().aph_attn_long_test(int(fwd), qkv.data_ptr(), None if dout is None else dout.data_ptr(), out.data_ptr(), S, T, D, heads,
                                       L.stream_ptr()), 'aph_attn_long_test')
    torch.cuda.synchronize()
    return out


def long_errors(L, S, T, heads, regime, seed):
    qkv = make_qkv(S, T, heads, regime, seed)
    g = torch.Generator().manual_seed(seed + 1)
    dout = (torch.randn(S * T, 64 * heads, generator=g) * 0.5).bfloat16().cuda()
    out = run_long(L, True, qkv, None, S, T, heads)
    dqkv = run_long(L, False, qkv, dout, S, T, heads)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(dqkv).all()), 'non-finite (unwritten or overflowed) outputs'
    o_ref, dq, dk, dv = ref_attention(qkv, dout, S, T, heads)
    o = split_heads(out, S, T, heads, 1)[0]
    errs = {'out_block': rel_err(o, o_ref, 2), 'out_row': rel_err(o, o_ref, 1)}
    for name, gt, rf in zip(('dq', 'dk', 'dv'), split_heads(dqkv, S, T, heads, 3), (dq, dk, dv)):
        if T == 1 and name != 'dv':          # one key: dQ = dK = 0 exactly (the reference is exactly 0 too)
            assert bool((gt == 0).all()), name
            continue
        errs[name + '_block'] = rel_err(gt, rf, 2)
    return errs


def _check(errs, what):
    bad = {k: v for k, v in errs.items() if v > (ROW_BAR if k.endswith('_row') else BLOCK_BAR)}
    assert not bad, (what, bad)


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('heads', [1, 16])
@pytest.mark.parametrize('T', SHORT_SEQ + LONG_SEQ)
def test_stream_attention_vs_float64(L, T, heads, regime):
    """The streaming kernels at T = 257 .. 577 (one key past a tile edge, mid-tile, at and around the 16-key sub-tile edges,
    several tiles) and, through the same hook, at T = 1, 197 and 256, where the encoder runs the resident kernels."""
    _check(long_errors(L, 3, T, heads, regime, seed=T * 100 + heads), (T, heads, regime))


@pytest.mark.parametrize('T', [257, 577])
def test_stream_attention_is_deterministic(L, T):
    """No atomics: two runs give bit-identical outputs and dqkv."""
    S, heads = 8, 16
    qkv = make_qkv(S, T, heads, 'sharp', T)
    dout = (torch.randn(S * T, 64 * heads, device='cuda') * 0.5).bfloat16()
    runs = [(run_long(L, True, qkv, None, S, T, heads), run_long(L, False, qkv, dout, S, T, heads)) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_stream_attention_refuses_bad_shapes(L):
    """A head dim other than 64 and an empty sequence return an error and launch nothing."""
    lib = L.lib()
    buf = torch.zeros(4 * 3 * 128, device='cuda', dtype=torch.bfloat16)
    n0 = lib.aph_launch_count()
    for T, D, heads in ((0, 128, 2), (5, 96, 2)):
        rc = lib.aph_attn_long_test(1, buf.data_ptr(), None, buf.data_ptr(), 1, T, D, heads, L.stream_ptr())
        with pytest.raises(RuntimeError, match='aph_attn_long_test'):
            L.check(rc, 'aph_attn_long_test')
    assert lib.aph_launch_count() == n0


# ---------------------------------------------------------------------------------------------------------- the encoder
def perturb(sd, seed=0, qk_scale=2.0):
    """tests/test_encoder_kernels_gpu.py perturbed_visual_state_dict's perturbation, applied to a state dict of any geometry"""
    g = torch.Generator().manual_seed(7919 + seed)
    uni = lambda shape, b: (torch.rand(shape, generator=g) * 2 - 1) * b
    sd = dict(sd)
    for k in list(sd):
        v = sd[k]
        if k.endswith(('ln_pre.weight', 'ln_post.weight', 'ln_1.weight', 'ln_2.weight')):
            sd[k] = 1 + uni(v.shape, 0.5)
        elif k.endswith(('ln_pre.bias', 'ln_post.bias', 'ln_1.bias', 'ln_2.bias')):
            sd[k] = uni(v.shape, 0.5)
        elif k.endswith(('attn.in_proj_bias', 'attn.out_proj.bias')):
            sd[k] = uni(v.shape, 0.2)
        elif k.endswith('attn.in_proj_weight'):
            w = v.clone()
            w[:2 * w.shape[1]] *= qk_scale
            sd[k] = w
    return sd


def encode(L, vis, x, cot):
    """aph_vit_fwd(_sized) + aph_vit_bwd(_sized) on x [S,3,side,side] -> (emb, grad_x)"""
    lib, S, side = L.lib(), x.shape[0], x.shape[-1]
    emb = torch.full((S, vis.output_dim), float('nan'), device='cuda')
    gx = torch.full(tuple(x.shape), float('nan'), device='cuda')
    if side == vis.input_resolution:
        L.check(lib.aph_vit_fwd(vis.handle, x.data_ptr(), S, emb.data_ptr(), 1, L.stream_ptr()), 'vit_fwd')
        L.check(lib.aph_vit_bwd(vis.handle, cot.data_ptr(), S, gx.data_ptr(), L.stream_ptr()), 'vit_bwd')
    else:
        L.check(lib.aph_vit_fwd_sized(vis.handle, x.data_ptr(), S, side, emb.data_ptr(), 1, L.stream_ptr()), 'vit_fwd_sized')
        L.check(lib.aph_vit_bwd_sized(vis.handle, cot.data_ptr(), S, side, gx.data_ptr(), L.stream_ptr()), 'vit_bwd_sized')
    torch.cuda.synchronize()
    return emb, gx


def oracle(sd, x, cot):
    xo = x.detach().cpu().clone().requires_grad_(True)
    eo = R.build_visual(sd)(xo)
    (eo * cot.cpu()).sum().backward()
    return eo.detach(), xo.grad


def check_vs_oracle(L, sd, S, res, seed, runs=3):
    """forward and data-gradient against the oracle (2e-2 per sample and globally); eager, capture and replay bit-identical"""
    from aphantasia_b200.clip import VisionTransformer
    vis = VisionTransformer(sd, max_batch=S)
    g = torch.Generator().manual_seed(seed)
    x, cot = torch.randn(S, 3, res, res, generator=g), torch.randn(S, vis.output_dim, generator=g) * 0.1
    eo, go = oracle(sd, x, cot)
    xc, cc = x.cuda(), cot.cuda()
    outs = [encode(L, vis, xc, cc) for _ in range(runs)]
    for emb, gx in outs:
        errs = per_sample_err(emb, eo) + per_sample_err(gx, go)
        assert max(errs) < 2e-2, errs
    for emb, gx in outs[1:]:
        assert torch.equal(emb, outs[0][0]) and torch.equal(gx, outs[0][1]), 'graph capture / replay differ from the eager call'
    vis.close()
    return outs[0]


@pytest.mark.parametrize('perturbed', [False, True])
def test_patch14_small_vs_oracle(L, perturbed):
    """patch 14, width 128, res 56: T = 17, the resident attention; the operand rows carry 52 pad columns"""
    sd = R.synthetic_visual_state_dict(14, 3, width=128, layers=2, heads=2, out_dim=128, res=56)
    check_vs_oracle(L, perturb(sd, 3) if perturbed else sd, 3, 56, seed=31)


@pytest.mark.parametrize('perturbed', [False, True])
def test_width256_t257_vs_oracle(L, perturbed):
    """patch 14 at res 224, width 256: T = 257 runs the streaming attention inside the encoder"""
    sd = R.synthetic_visual_state_dict(14, 4, width=256, layers=2, heads=4, out_dim=128, res=224)
    check_vs_oracle(L, perturb(sd, 4) if perturbed else sd, 3, 224, seed=41)


def test_vitl14_vs_oracle(L):
    from aphantasia_b200.clip import synthetic_visual_state_dict
    check_vs_oracle(L, synthetic_visual_state_dict(seed=0, **VITL14), 2, 224, seed=51)


def test_vitl14_perturbed_vs_oracle(L):
    from aphantasia_b200.clip import synthetic_visual_state_dict
    check_vs_oracle(L, perturb(synthetic_visual_state_dict(seed=1, **VITL14), 1), 3, 224, seed=52, runs=2)


def test_vitl14_handle_reuse_across_batch_sizes(L):
    """One handle (max_batch 8) taken through S = 2, 8, 3 gives, bit for bit, what a fresh handle of each size gives."""
    from aphantasia_b200.clip import VisionTransformer, synthetic_visual_state_dict
    sd = synthetic_visual_state_dict(seed=2, **VITL14)
    g = torch.Generator().manual_seed(61)
    x, cot = torch.randn(8, 3, 224, 224, generator=g).cuda(), (torch.randn(8, 768, generator=g) * 0.1).cuda()
    vis = VisionTransformer(sd, max_batch=8)
    shared = {S: encode(L, vis, x[:S].contiguous(), cot[:S].contiguous()) for S in (2, 8, 3)}
    vis.close()
    for S in (2, 8, 3):
        fresh = VisionTransformer(sd, max_batch=S)
        e, gx = encode(L, fresh, x[:S].contiguous(), cot[:S].contiguous())
        fresh.close()
        assert torch.equal(e, shared[S][0]) and torch.equal(gx, shared[S][1]), S


# ---------------------------------------------------------------------------------------------------------- patch operand
class _DevInt16:
    """a CUDA array interface over device memory the library owns (read back for inspection; torch does not own it)"""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': '<i2', 'data': (ptr, False), 'version': 3}


def patch_operand(L, vis, S):
    """the handle's bf16 patch operand [S*g*g, 640] as an int16 view (a bf16 zero is an int16 zero)"""
    p, patch, grid = C.c_void_p(), C.c_int(), C.c_int()
    L.check(L.lib().aph_vit_patch_operand(vis.handle, S, C.byref(p), C.byref(patch), C.byref(grid)), 'aph_vit_patch_operand')
    assert patch.value == 14
    return torch.as_tensor(_DevInt16(p.value, (S * grid.value ** 2, 640)), device='cuda')


def im2col14(x, res=224):
    """[S,3,side,side] -> bf16 [S*16*16, 588] of the top-left res x res window, col = c*196 + py*14 + px"""
    S, g = x.shape[0], res // 14
    w = x[:, :, :res, :res].reshape(S, 3, g, 14, g, 14).permute(0, 2, 4, 1, 3, 5).reshape(S * g * g, 588)
    return w.bfloat16()


@pytest.mark.parametrize('side', [224, 232])
def test_patch14_window_and_operand(L, side):
    """images of side 224 and 232 (the size + 8 batches of transforms_custom / _elastic) at patch 14: the window gradient
    matches the oracle, the margin of the image gradient is exactly zero, and the operand k_patchify wrote is the bf16 im2col
    of the window with its 52 pad columns zero."""
    from aphantasia_b200.clip import VisionTransformer
    sd = perturb(R.synthetic_visual_state_dict(14, 5, width=256, layers=2, heads=4, out_dim=128, res=224), 5)
    S = 3
    vis = VisionTransformer(sd, max_batch=S)
    g = torch.Generator().manual_seed(71 + side)
    x, cot = torch.randn(S, 3, side, side, generator=g), torch.randn(S, 128, generator=g) * 0.1
    emb, gx = encode(L, vis, x.cuda(), cot.cuda())
    op = patch_operand(L, vis, S)
    assert bool((op[:, 588:] == 0).all()), 'a pad column of the patch operand is not zero'
    assert torch.equal(op[:, :588].view(torch.bfloat16), im2col14(x.cuda()))
    eo, go = oracle(sd, x[:, :, :224, :224].contiguous(), cot)
    assert max(per_sample_err(emb, eo) + per_sample_err(gx[:, :, :224, :224], go)) < 2e-2
    if side > 224:
        assert bool((gx[:, :, 224:, :] == 0).all()) and bool((gx[:, :, :, 224:] == 0).all()), 'the margin gradient is not exactly zero'
    vis.close()


def test_patch14_fused_operand_matches_plain_route(L):
    """slice_imgs -> encode_image with the sampler writing the patch-14 operand is bit-identical to APH_PATCH_FUSE=0, for
    kinds none, fast, custom and elastic (the last two at side 232); after the fused write the pad columns are still zero."""
    from aphantasia_b200 import _patchlink, transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.utils import slice_imgs
    gc.collect()
    sd = perturb(R.synthetic_visual_state_dict(14, 6, width=256, layers=2, heads=4, out_dim=128, res=224), 6)
    model = CLIP('ViT-L/14', sd, True)
    vis = model.visual
    _patchlink._consumers.clear()
    _patchlink.register(vis)
    canvas = torch.rand(1, 3, 360, 640, device='cuda')
    S = 6

    def run(fuse, kind):
        os.environ['APH_PATCH_FUSE'] = '1' if fuse else '0'
        _seed(5)
        f0 = vis.prepatched_forwards
        crops = slice_imgs([canvas], S, 224, kind, 'uniform', 0.4)[0]
        if fuse:
            op = patch_operand(L, vis, S)
            assert bool((op[:, 588:] == 0).all()), 'the sampler wrote into the pad columns'
            assert torch.equal(op[:, :588].view(torch.bfloat16), im2col14(crops)), 'fused operand != im2col of the batch'
        emb = model.encode_image(crops)
        torch.cuda.synchronize()
        return emb.detach().clone(), vis.prepatched_forwards - f0
    try:
        run(False, transforms.transforms_fast)
        for kind in (None, transforms.transforms_fast, transforms.transforms_custom, transforms.transforms_elastic):
            e0, f_plain = run(False, kind)
            e1, f_fused = run(True, kind)
            assert f_plain == 0 and f_fused == 1, (kind, f_plain, f_fused)
            assert torch.equal(e0, e1), (kind, _rel(e1, e0))
    finally:
        os.environ.pop('APH_PATCH_FUSE', None)
        del model, vis
        gc.collect()


# ---------------------------------------------------------------------------------------------------------- text, step, load
def test_text_tower_vitl14_geometry():
    """the ViT-L/14 text tower (width 768, 12 heads, 12 layers, out 768) against the restatement at the text tests' bar"""
    import text_oracle as TO
    from aphantasia_b200 import clip
    from test_text_tower_gpu import _tokens
    cfg = dict(width=768, layers=12, heads=12, out_dim=768, context=77, vocab=49408)
    sd = clip.synthetic_text_state_dict(seed=5, **cfg)
    ref = TO.build_text(sd)
    tower = clip.TextTransformer(sd)
    toks = _tokens(3, 77, cfg['vocab'], [1, 38, 76], seed=3)
    got = tower(toks.cuda())
    with torch.no_grad():
        want = ref(toks)
    assert got.shape == (3, 768) and _rel(got, want) < 2e-2, _rel(got, want)
    tower.close()


def test_full_step_vitl14_vs_oracle(L):
    """224 x 224 canvas, S = 3, transforms_fast, ViT-L/14, sim 'mix': loss and d loss / d spectrum vs the CPU oracle"""
    from aphantasia_b200 import _rng, transforms
    from aphantasia_b200.clip import CLIP, synthetic_visual_state_dict
    from aphantasia_b200.image import fft_image, to_valid_rgb
    from aphantasia_b200.utils import sim_func, slice_imgs
    h = w = 224; S = 3
    sd = synthetic_visual_state_dict(seed=0, **VITL14)
    model = CLIP('ViT-L/14', sd, True)
    _seed(0)
    params, image_f, _ = fft_image([1, 3, h, w], 0.07, 1.5, None)
    rgb_f = to_valid_rgb(image_f, colors=1.8)
    txt = model.encode_text(torch.zeros(1, 77, dtype=torch.long)).cuda()
    _seed(1)
    crops = slice_imgs([rgb_f()], S, 224, transforms.transforms_fast, 'uniform', 0.4)[0]
    emb = model.encode_image(crops)
    loss = -1. * sim_func(txt, emb, 'mix')
    loss.backward()
    _seed(1)
    tabs, _ = _rng.draw_crop_table(S, (h, w), 224, 2, 'uniform', 0.4)
    o_loss, o_grad, o_emb = R.reference_step(params[0].detach().cpu(), R.fft_scale(h, w, 1.5), (h, w), R.color_matrix(1.8), tabs[0],
                                             R.build_visual(sd), txt.cpu(), 'mix')
    assert _rel(emb, o_emb) < 2e-2
    assert abs(loss.item() - o_loss.item()) < 2e-3
    assert _rel(params[0].grad, o_grad) < 3e-2
    model.visual.close()


def test_clip_load_vitl14(L):
    from aphantasia_b200 import clip
    from aphantasia_b200.utils import aesthetic_model
    for k in [k for k in os.environ if k.startswith('APH_CLIP_WEIGHTS')]:
        assert not os.path.isfile(os.environ[k]), 'this test wants the synthetic weights'
    model, _ = clip.load('ViT-L/14', jit=False)
    assert model.visual.input_resolution == 224 and model.embed_dim == 768 and model.visual.patch_size == 14
    x = torch.rand(2, 3, 224, 224, device='cuda', requires_grad=True)
    emb = model.encode_image(x)
    assert emb.shape == (2, 768)
    head = aesthetic_model('ViT-L/14').cuda()
    out = head(emb)
    assert tuple(out.shape) == (2, 1)
    out.mean().backward()
    assert x.grad is not None and bool(torch.isfinite(x.grad).all()) and float(x.grad.abs().sum()) > 0
    with pytest.raises(RuntimeError, match='not available'):
        clip.load('ViT-L/14@336px')
    model.visual.close()


def test_vitl14_handle_at_200_samples(L):
    """a ViT-L/14 handle sized for 200 samples creates, and reports what it holds (about 32 GB estimated from the layout)"""
    from aphantasia_b200.clip import VisionTransformer, synthetic_visual_state_dict
    gc.collect()
    vis = VisionTransformer(synthetic_visual_state_dict(seed=0, **VITL14), max_batch=200)
    nbytes = L.lib().aph_vit_bytes(vis.handle)
    print('ViT-L/14 handle at S = 200: %.2f GB' % (nbytes / 1e9))
    assert 20e9 < nbytes < 45e9, nbytes
    x = torch.rand(200, 3, 224, 224, device='cuda')
    emb = torch.empty(200, 768, device='cuda')
    L.check(L.lib().aph_vit_fwd(vis.handle, x.data_ptr(), 200, emb.data_ptr(), 0, L.stream_ptr()), 'vit_fwd')
    torch.cuda.synchronize()
    assert bool(torch.isfinite(emb).all())
    vis.close()
