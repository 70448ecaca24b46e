"""Every handle and plan gives back, when it is destroyed, exactly the device memory it held, and a stream-ordered temporary is
gone when its call returns. Each object is created and run forward and backward (and through its analysis, for the plans), so
that every scratch it owns has grown before it is destroyed. aph_device_bytes() counts what the library holds: on a shared GPU,
cudaMemGetInfo also counts other processes' memory. The sampler, whose scratch lives as long as the process, is not run here."""
import contextlib
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from aphantasia_b200 import _lib, clip, cppn, lpips
from aphantasia_b200._wavelets import reconstruction_filters

pytestmark = pytest.mark.gpu


def _held():
    torch.cuda.synchronize()
    return _lib.lib().aph_device_bytes()


@contextlib.contextmanager
def _quiet_gc():
    """no other test's handle is collected, and so destroyed, while a measurement runs"""
    gc.collect()
    gc.disable()
    try:
        yield
    finally:
        gc.enable()


def _ok(rc, what):
    _lib.check(rc, what)


def _vit():
    sd = clip.synthetic_visual_state_dict(patch=32, width=128, layers=2, heads=2, out_dim=128, res=64, seed=0)
    h = _lib.Handle('aph_vit', C.byref(_lib.VitConfig(32, 128, 2, 2, 128, 64, 2, 0)))
    h.load(sd)
    img = torch.rand(2, 3, 64, 64, device='cuda')
    emb, g = torch.empty(2, 128, device='cuda'), torch.randn(2, 128, device='cuda')
    gimg = torch.empty_like(img)
    for _ in range(3):              # eager, captured, replayed: the handle's graph cache holds entries when it is destroyed
        _ok(_lib.lib().aph_vit_fwd(h, img.data_ptr(), 2, emb.data_ptr(), 1, _lib.stream_ptr()), 'aph_vit_fwd')
        _ok(_lib.lib().aph_vit_bwd(h, g.data_ptr(), 2, gimg.data_ptr(), _lib.stream_ptr()), 'aph_vit_bwd')
    return h.close


def _text():
    sd = clip.synthetic_text_state_dict(width=128, layers=2, heads=2, out_dim=128, context=16, vocab=500, seed=0)
    h = _lib.Handle('aph_text', C.byref(_lib.TextConfig(128, 2, 2, 128, 16, 500, 2, 0)))
    h.load(sd)
    tokens = torch.randint(0, 500, (2, 16), device='cuda')
    emb = torch.empty(2, 128, device='cuda')
    _ok(_lib.lib().aph_text_fwd(h, tokens.data_ptr(), 2, emb.data_ptr(), _lib.stream_ptr()), 'aph_text_fwd')   # no backward
    return h.close


def _lpips():
    model = lpips.LPIPS(net='vgg', verbose=False, vgg_state_dict=lpips.synthetic_vgg_state_dict(),
                        lin_state_dict=lpips.synthetic_lin_state_dict())
    x = torch.rand(2, 3, 64, 64, device='cuda', requires_grad=True)
    model(x, torch.rand(2, 3, 64, 64, device='cuda')).sum().backward()
    return model.close


def _cppn():
    net = cppn.CPPN(nf_hid=64, num_layers=10).cuda()      # too large for shared memory: the backward's z_l go to handle scratch
    net(torch.rand(1, 2, 32, 32, device='cuda') * 2 - 1).sum().backward()
    return net._handle.close


def _fft():
    H, W = 64, 96
    Wh = W // 2 + 1
    plan = _lib.Handle('aph_fft_plan', H, W)
    P, scale = torch.randn(3, H, Wh, 2, device='cuda'), 0.5 + torch.rand(H, Wh, device='cuda')
    x, out = torch.empty(3, H, W, device='cuda'), torch.empty(3, H, W, device='cuda')
    stats = torch.empty(4, device='cuda', dtype=torch.float64)
    st = _lib.stream_ptr()
    _ok(_lib.lib().aph_synth_fft_fwd(plan, P.data_ptr(), scale.data_ptr(), None, 0, 1.0, None, 1, x.data_ptr(), stats.data_ptr(),
                                     out.data_ptr(), st), 'aph_synth_fft_fwd')
    gp, cot = torch.empty_like(P), torch.randn_like(out)
    _ok(_lib.lib().aph_synth_fft_bwd(plan, cot.data_ptr(), out.data_ptr(), x.data_ptr(), stats.data_ptr(), scale.data_ptr(), 1.0, None, 1,
                                     gp.data_ptr(), st), 'aph_synth_fft_bwd')
    _ok(_lib.lib().aph_fft_analyze(plan, out.data_ptr(), scale.data_ptr(), gp.data_ptr(), st), 'aph_fft_analyze')
    return plan.close


def _dwt_filters(wave='coif2'):
    lo, hi = reconstruction_filters(wave)
    return (C.c_float * len(lo))(*np.asarray(lo, dtype=np.float32)), (C.c_float * len(hi))(*np.asarray(hi, dtype=np.float32)), len(lo)


def _dwt_run(plan, H, W):
    """synthesis forward and backward, then the analysis of the synthesised image (stream-ordered temporaries per level)"""
    J, dims, ohw = C.c_int(), (C.c_int * 32)(), (C.c_int * 2)()
    _ok(_lib.lib().aph_dwt_plan_levels(plan, C.byref(J), dims, ohw), 'aph_dwt_plan_levels')
    shapes = [(dims[2 * i], dims[2 * i + 1]) for i in range(J.value)]
    Ys = [torch.randn(3, *shapes[-1], device='cuda')] + [torch.randn(3, 3, *hw, device='cuda') for hw in shapes]
    ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
    scales = (C.c_float * J.value)(*([0.5] * J.value))
    x, out = torch.empty(3, ohw[0], ohw[1], device='cuda'), torch.empty(3, ohw[0], ohw[1], device='cuda')
    stats = torch.empty(4, device='cuda', dtype=torch.float64)
    st = _lib.stream_ptr()
    _ok(_lib.lib().aph_synth_dwt_fwd(plan, ptrs, scales, 1.0, None, 1, x.data_ptr(), stats.data_ptr(), out.data_ptr(), st), 'aph_synth_dwt_fwd')
    grads = [torch.empty_like(y) for y in Ys]
    gptrs = (C.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
    cot = torch.randn_like(out)
    _ok(_lib.lib().aph_synth_dwt_bwd(plan, cot.data_ptr(), out.data_ptr(), x.data_ptr(), stats.data_ptr(), scales, 1.0, None, 1, gptrs, st),
        'aph_synth_dwt_bwd')
    img = torch.rand(3, H, W, device='cuda')
    _ok(_lib.lib().aph_dwt_analyze(plan, img.data_ptr(), scales, gptrs, st), 'aph_dwt_analyze')
    torch.cuda.synchronize()


def _dwt():
    H, W = 64, 96
    lo, hi, L = _dwt_filters()
    plan = _lib.Handle('aph_dwt_plan', H, W, lo, hi, L)
    _dwt_run(plan, H, W)
    return plan.close


OBJECTS = {'vit': _vit, 'text': _text, 'lpips': _lpips, 'cppn': _cppn, 'fft_plan': _fft, 'dwt_plan': _dwt}


@pytest.mark.parametrize('kind', list(OBJECTS))
def test_destroy_gives_back_every_device_byte(kind):
    with _quiet_gc():
        start = _held()
        close = OBJECTS[kind]()
        alive = _held()
        close()
        assert alive > start, (kind, start, alive)
        assert _held() == start, (kind, start, alive, _held())


def test_refused_creates_hold_nothing():
    lo, hi, L = _dwt_filters()
    with _quiet_gc():
        start = _held()
        plan = C.c_void_p()
        rc = _lib.lib().aph_dwt_plan_create(C.byref(plan), 1 << 17, 1 << 17, lo, hi, L)       # 17 levels: one more than a plan holds
        assert rc != 0 and plan.value is None and '17 levels' in _lib.lib().aph_last_error().decode()
        rc = _lib.lib().aph_fft_plan_create(C.byref(plan), 64, 17 * 4)                       # a prime factor > 13
        assert rc != 0 and plan.value is None and 'prime factor' in _lib.lib().aph_last_error().decode()
        assert _held() == start


def test_temporaries_are_gone_when_the_call_returns():
    """aph_dwt_analyze's per-level row buffers, aph_attn_long_test's backward statistics and aph_lpips_conv_test's packed weights
    are freed on their stream before the call returns; the plan's own memory stays until it is destroyed."""
    H, W = 64, 96
    lo, hi, L = _dwt_filters()
    with _quiet_gc():
        plan = _lib.Handle('aph_dwt_plan', H, W, lo, hi, L)
        try:
            start = _held()
            _dwt_run(plan, H, W)
            assert _held() == start
        finally:
            plan.close()
        S, T, heads = 2, 257, 2
        D = 64 * heads
        qkv = (torch.randn(S * T, 3 * D, device='cuda') * 0.5).to(torch.bfloat16)
        dout = torch.randn(S * T, D, device='cuda').to(torch.bfloat16)
        dqkv = torch.empty(S * T, 3 * D, device='cuda', dtype=torch.bfloat16)
        x = torch.randn(1, 8, 8, 64, device='cuda').to(torch.bfloat16)
        w, b = torch.randn(64, 64, 3, 3, device='cuda') * 0.05, torch.zeros(64, device='cuda')
        y = torch.empty(1, 8, 8, 64, device='cuda', dtype=torch.bfloat16)
        start = _held()
        _ok(_lib.lib().aph_attn_long_test(0, qkv.data_ptr(), dout.data_ptr(), dqkv.data_ptr(), S, T, D, heads, _lib.stream_ptr()),
            'aph_attn_long_test')
        for fwd in (1, 0):
            _ok(_lib.lib().aph_lpips_conv_test(fwd, x.data_ptr(), w.data_ptr(), b.data_ptr(), None, y.data_ptr(), 1, 8, 8, 64, 64,
                                               _lib.stream_ptr()), 'aph_lpips_conv_test')
        assert _held() == start
        assert bool(torch.isfinite(dqkv.float()).all()) and bool(torch.isfinite(y.float()).all())
