"""GPU: the DWT kernels at the filter lengths the built-in symlets and coiflets bring (coif3 18, coif4 24, coif6 36 taps; sym4
8, sym8 16, sym20 40), which no other test runs at 18, 24 or 36 taps. The kernels get the package's fp32 taps; the float64
references use the 60-digit tables of tests/wavelet_tables.py rounded to float64, not the package's literals.

Bars follow tests/test_synth_kernels_gpu.py and tests/test_image_resume_gpu.py: 5e-6 per level against that level's own norm,
widened by sqrt(L / 12) for filters longer than coif2's 12 taps, for the synthesis forward, its adjoint and the analysis;
perfect reconstruction (analysis, then synthesis) 1e-5 norm-wise, widened the same way; one fused-Adam step against the stock
step 1e-6 per tensor, as tests/test_fused_optim_gpu.py. Measured on an H100 80GB HBM3 at a 700 W power limit: forward
<= 1.7e-7, level gradients <= 7.1e-7, Yl <= 1.0e-6, analysis <= 1.0e-6, picture bands <= 1.1e-6, round trip <= 5.2e-7, Adam
<= 1.2e-7. Sizes include 33x47 and 5x7, where every filter here is longer than
the coarse levels and the symmetric extension wraps around a line several times.
"""
import ctypes as C
import functools
import math
import os

import numpy as np
import pytest
import torch

import resume_oracle as RO
import test_fused_optim_gpu as FO
import test_synth_kernels_gpu as G
import wavelet_tables as T
from oracle import restate as R
from test_image_resume_gpu import PR_BAR, dwt_analyze, dwt_plan, per_channel, picture_file, rel, report, smooth_picture
from test_real_script import SCRIPT, _run

pytestmark = pytest.mark.gpu
WAVES = ['coif3', 'coif4', 'coif6', 'sym4', 'sym8', 'sym20']
SIZES = [(64, 96), (33, 47), (5, 7)]


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


@functools.lru_cache(maxsize=None)
def filters(wave):
    """(lo32, hi32, lo64, hi64): the fp32 reconstruction taps the kernels get, and the generator's float64 taps"""
    from aphantasia_b200._wavelets import reconstruction_filters
    lo, hi = reconstruction_filters(wave)
    n = int(wave.lstrip('cofisym'))
    dec = [float(v) for v in (T.coiflet_dec_lo(n) if wave.startswith('coif') else T.symlet_dec_lo(n))]
    lo64, hi64 = dec[::-1], [(-1) ** k * dec[k] for k in range(len(dec))]
    assert np.abs(np.array(lo) - lo64).max() <= 1e-15 and np.abs(np.array(hi) - hi64).max() <= 1e-15
    return np.asarray(lo, dtype=np.float32), np.asarray(hi, dtype=np.float32), lo64, hi64


def widen(bar, wave):
    return bar * math.sqrt(max(1., len(filters(wave)[0]) / 12.))


CASES = [(h, w, wave) for wave in WAVES for h, w in SIZES]
IDS = ['%dx%d-%s' % c for c in CASES]


@pytest.mark.parametrize('H,W,wave', CASES, ids=IDS)
def test_dwt_synthesis_and_adjoint_vs_float64(L, monkeypatch, H, W, wave):
    """aph_synth_dwt_fwd / _bwd: x_raw, the RGB output, the statistics, and the gradient of Yl and of every level."""
    monkeypatch.setattr(G, 'dwt_filters32', filters)
    errs, nt = G.dwt_case(L, H, W, wave, seed=H * 3 + W + len(wave))
    bar = G.dwt_bar(nt)
    G.check(errs, (H, W, wave), {k: bar for k in errs if k in ('x_raw', 'out') or k.startswith('grad')})


@pytest.mark.parametrize('H,W,wave', CASES, ids=IDS)
def test_dwt_analysis_vs_float64(L, H, W, wave):
    lo32, hi32, lo64, hi64 = filters(wave)
    plan, shapes, _ = dwt_plan(L, H, W, lo32, hi32)
    try:
        assert shapes == [tuple(t) for t in R.dwt_level_shapes(H, W, len(lo32))]
        inv = [float(np.float32(1. / s)) for s in R.dwt_scales(shapes, 0.3)]
        x = torch.randn(3, H, W, generator=torch.Generator().manual_seed(H * 5 + W + len(wave)))
        Ys = dwt_analyze(L, plan, x.cuda(), shapes, inv)
        torch.cuda.synchronize()
    finally:
        L.lib().aph_dwt_plan_destroy(plan)
    ref = RO.dwt_analysis(x.double()[None], lo64, hi64)
    ref = [ref[0][0]] + [y[0] * s for y, s in zip(ref[1:], inv)]
    assert all(bool(torch.isfinite(y).all()) for y in Ys)
    report(('dwt analysis', H, W, wave), [rel(y.cpu(), r) for y, r in zip(Ys, ref)], widen(G.DWT_BAR, wave))


@pytest.mark.parametrize('h,w,wave', [(h, w, wave) for wave in WAVES for h, w in ((45, 64), (33, 47), (5, 7))],
                         ids=['%dx%d-%s' % (h, w, wave) for wave in WAVES for h, w in ((45, 64), (33, 47), (5, 7))])
def test_picture_round_trip_through_dwt_image(L, tmp_path, h, w, wave):
    """dwt_image(shape, wave, 0.3, 1.8, path): the bands against the float64 analysis of un_rgb(picture) divided by the
    scales, img2dwt gives the same bits, and the synthesis of those bands (contrast 1, no colour matrix) gives the picture back
    on its first h x w."""
    from aphantasia_b200.image import dwt_image, img2dwt
    lo32, hi32, lo64, hi64 = filters(wave)
    img = smooth_picture(h, w, len(wave) + w)
    Ys, gen, size = dwt_image([1, 3, 64, 64], wave, 0.3, 1.8, picture_file(tmp_path, img))
    assert tuple(size) == (h, w) and [tuple(y.shape) for y in Ys] == gen.param_shapes()
    x64 = RO.un_rgb(img, 1.8, torch.float64)
    ref = RO.dwt_analysis(x64, lo64, hi64)
    scales = R.dwt_scales([tuple(y.shape[3:5]) for y in ref[1:]], 0.3)
    ref = [ref[0]] + [y / s for y, s in zip(ref[1:], scales)]
    report(('dwt_image picture bands', h, w, wave), [rel(y.detach().cpu(), r) for y, r in zip(Ys, ref)], widen(G.DWT_BAR, wave))
    assert all(torch.equal(a, b.detach()) for a, b in zip(img2dwt(img, wave, 0.3, 1.8), Ys))
    oh, ow = gen.out_hw
    x_raw = torch.empty(3, oh, ow, device='cuda'); out = torch.empty_like(x_raw)
    stats = torch.empty(4, device='cuda', dtype=torch.float64)
    ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
    L.check(L.lib().aph_synth_dwt_fwd(gen.plan, ptrs, gen.scales_c, 1.0, None, 0, x_raw.data_ptr(), stats.data_ptr(), out.data_ptr(),
                                      L.stream_ptr()), 'aph_synth_dwt_fwd')
    torch.cuda.synchronize()
    assert (oh, ow) == (h + h % 2, w + w % 2)
    report(('dwt picture round trip', h, w, wave), [per_channel(x_raw[:, :h, :w].cpu(), x64[0])], widen(PR_BAR, wave))


@pytest.mark.parametrize('H,W', [(360, 640), (33, 47)])
@pytest.mark.parametrize('wave', WAVES)
def test_fused_adam_step_matches_backward_then_step(H, W, wave):
    """aphantasia_b200.optim.Adam (the update inside aph_synth_dwt_bwd) against the plain backward and the stock Adam step."""
    from aphantasia_b200 import image, optim

    def make():
        torch.manual_seed(3)
        params, gen, _ = image.dwt_image([1, 3, H, W], wave, 0.3, 1.)
        return params, image.to_valid_rgb(gen, colors=1.5)
    (pa, fa), (pb, fb) = make(), make()
    assert all(torch.equal(a, b) for a, b in zip(pa, pb))
    kw = FO._f32_betas({})
    a, b = (pa, fa, optim.Adam(pa, 0.05, **kw)), (pb, fb, optim._stock_adam(pb, 0.05, **kw))
    grad_out = torch.randn(1, 3, *fa().shape[2:], device='cuda', generator=torch.Generator(device='cuda').manual_seed(7))
    for side in (a, b):
        side[2].zero_grad()
        (side[1]() * grad_out).sum().backward()
        side[2].step()
    err = FO._compare(a, b)
    print('errors fused adam', wave, H, W, '%.2e' % err)
    assert err <= FO.BAR


needs_script = pytest.mark.skipif(not os.path.isfile(SCRIPT), reason='no copy of the original clip_fft.py: build() stages one into oracle/_ref/')


@needs_script
@pytest.mark.parametrize('wave', ['coif3', 'coif4', 'sym8'])
def test_unmodified_clip_fft_dwt_wave(tmp_path, wave):
    """The unmodified clip_fft.py --dwt --wave <wave>, without PyWavelets: a few steps with finite similarities."""
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--dwt', '--wave', wave, '--size', '320-256', '--samples', '8', '--steps', '3'])
    assert tr['encode_image_calls'] == 3 and len(tr['sims']) == 3 and all(math.isfinite(s) for s in tr['sims'])
