"""Starting from an image file on the GPU: the analysis kernels against float64 references computed from the same fp32 inputs
(aph_un_rgb, aph_fft_analyze in csrc/synth_fft.cu, aph_dwt_analyze in csrc/synth_dwt.cu), round trips through the existing
synthesis kernels, the drop-in entry points against the reference's own outputs (tests/golden/reference_golden_resume.npz),
and the unmodified clip_fft.py with --resume.

Rounding budget (u = 2^-24), following tests/test_synth_kernels_gpu.py:
Measured values are from an H100 80GB HBM3 at a 700 W power limit.
  un_rgb   x / 255, - mean, / std and a 3-term mix in fp32: a few u of the terms' magnitudes, which the result shares
           (|(x/255 - mean) / std| <= 2.1 against a result of order 1). Bar 1e-6 per channel, norm-wise, against float64
           from the same uint8 input and the same fp32 inverse matrix (measured <= 7.7e-8).
  FFT      The analysis is the synthesis backward's forward DFTs: a length-W complex DFT of two real rows, a split with the
           factor 1/2 norm, a length-H DFT times the fp32 analysis scale. Same stage count as the synthesis, so the same
           bar: 2e-6 per channel and radial frequency band (f < 0.05, 0.05 - 0.25, >= 0.25) against float64
           ascale * rfftn(img, 'ortho'), each band against its own norm or, if larger, the norm a white spectrum puts in
           it (measured <= 2.1e-7; a band of one bin, the DC bin at 11 x 13, can be small by chance, and the FFT's error
           is relative to the whole transform). The round trip (analysis, then aph_synth_fft_fwd with scale = 1 / ascale)
           adds the synthesis's error and two roundings of the scales: 2e-6 norm-wise per channel on x_raw (measured
           <= 3.1e-7).
  DWT      Each coefficient is an L-tap sum along W followed by an L-tap sum along H in fp32; levels chain through LL. Bar as
           the synthesis: 5e-6 per level against that level's own norm, widened by sqrt(L / 12) for filters longer than
           coif2's 12 taps (measured <= 5.6e-7). The float64 reference is oracle/restate.py's afb1d_sym (pytorch_wavelets'
           symmetric-mode afb1d restated), so parity with pytorch_wavelets itself is unpinned. Perfect reconstruction
           through aph_synth_dwt_fwd: 1e-5 norm-wise on the first H x W (measured <= 1.5e-7).
  Entry    The drop-in functions against the reference's fp32 outputs: both sides round, 1e-5 per band (spectra) or
           norm-wise (pixels) (measured <= 4.0e-6, in the sparse high band of the grey picture's spectrum).
"""
import ctypes as C
import glob
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import resume_oracle as RO
from oracle import restate as R
from test_real_script import SCRIPT, _run
from test_synth_kernels_gpu import DWT_BAR, FFT_SIZES, FWD_BAR, WAVES, dwt_filters32, fft_plan, per_channel, rel

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNRGB_BAR = 1e-6
ENTRY_BAR = 1e-5
PR_BAR = 1e-5
MEAN = [float(np.float32(v)) for v in R.CLIP_MEAN]
STD = [float(np.float32(v)) for v in R.CLIP_STD]


@pytest.fixture(scope='module')
def L():
    from aphantasia_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


@pytest.fixture(scope='module')
def fx():
    with np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_golden_resume.npz')) as z:
        return {k: z[k] for k in z.files}


def report(what, errs, bar):
    print('errors', what, ' '.join('%.2e' % e for e in errs))
    assert max(errs) <= bar, (what, errs)


def picture_file(tmp_path, img, name='pic.png'):
    path = str(tmp_path / name)
    Image.fromarray(img).save(path)
    return path


def smooth_picture(h, w, seed):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 90 * np.sin(2 * np.pi * (xx / w * (k + 1) + yy / h * (2 - k)) + k) for k in range(3)], -1)
    return np.clip(np.rint(img + rng.normal(0, 20, (h, w, 3))), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------- un_rgb
@pytest.mark.parametrize('h,w,colors,gain', [(37, 53, 1.0, 1.0), (240, 320, 1.6, 1.0), (720, 1280, 2.0, 3.3)])
def test_un_rgb_vs_float64(L, h, w, colors, gain):
    from aphantasia_b200 import image
    img = np.random.RandomState(h + w).randint(0, 256, (h, w, 3)).astype(np.uint8)
    got = image._un_rgb(img, colors, gain)[0].cpu()
    inv = torch.linalg.inv(image._color_correlation(colors).T).double()              # the fp32 inverse the kernel gets
    x = torch.tensor(img, dtype=torch.float64).permute(2, 0, 1) / 255.
    x = (x - torch.tensor(MEAN, dtype=torch.float64).view(3, 1, 1)) / torch.tensor(STD, dtype=torch.float64).view(3, 1, 1)
    ref = gain * torch.einsum('chw,cd->dhw', x, inv)
    report(('un_rgb', h, w, colors, gain), [per_channel(got, ref)], UNRGB_BAR)
    report(('un_rgb vs fp32 reference order', h, w), [per_channel(got, gain * RO.un_rgb(img, colors)[0])], UNRGB_BAR)


# ---------------------------------------------------------------------------------------------------------------- FFT analysis
def fft_analyze(L, plan, x, ascale):
    H, W = x.shape[1], x.shape[2]
    spec = torch.full((3, H, W // 2 + 1, 2), float('nan'), device='cuda')
    L.check(L.lib().aph_fft_analyze(plan, x.data_ptr(), ascale.data_ptr(), spec.data_ptr(), L.stream_ptr()), 'aph_fft_analyze')
    return spec


def white_band_errors(got, ref, H, W):
    """Per channel and radial band, ||error|| over the larger of the band's norm and the norm a white spectrum puts there,
    ||ref|| sqrt(bins in band / bins): the FFT's error is relative to the whole transform, and a band of one or two bins (the
    DC bin alone below f = 0.05 at 11 x 13) can be near zero by chance."""
    errs = []
    for m in RO.radial_bands(H, W):
        if bool(m.any()):
            frac = math.sqrt(float(m.sum()) / m.numel())
            errs.append(max(float((got[c][m] - ref[c][m]).norm() / max(ref[c][m].norm(), ref[c].norm() * frac)) for c in range(3)))
    return errs


@pytest.mark.parametrize('H,W', FFT_SIZES, ids=['%dx%d' % hw for hw in FFT_SIZES])
def test_fft_analysis_vs_float64_and_round_trip(L, H, W):
    """White image and white analysis scale U(0.5, 1.5): every bin counts. Then aph_synth_fft_fwd with scale = 1 / ascale
    (no shift, colour matrix or sigmoid) must return the image in x_raw."""
    Wh = W // 2 + 1
    g = torch.Generator().manual_seed(H * 7 + W)
    x = torch.randn(3, H, W, generator=g)
    ascale = (0.5 + torch.rand(H, Wh, generator=g)).float()
    ref = torch.view_as_real(torch.fft.rfftn(x.double(), dim=(1, 2), norm='ortho')) * ascale.double()[..., None]
    plan = fft_plan(L, H, W)
    try:
        xc, ac = x.cuda(), ascale.cuda()
        spec = fft_analyze(L, plan, xc, ac)
        x_raw = torch.full((3, H, W), float('nan'), device='cuda')
        out = torch.empty_like(x_raw)
        stats = torch.empty(4, device='cuda', dtype=torch.float64)
        inv = (1. / ascale.double()).float().cuda()
        L.check(L.lib().aph_synth_fft_fwd(plan, spec.data_ptr(), inv.data_ptr(), None, 0, 1.0, None, 0, x_raw.data_ptr(), stats.data_ptr(),
                                          out.data_ptr(), L.stream_ptr()), 'aph_synth_fft_fwd')
        torch.cuda.synchronize()
    finally:
        L.lib().aph_fft_plan_destroy(plan)
    assert bool(torch.isfinite(spec).all())
    report(('fft analysis', H, W), white_band_errors(spec.cpu().double(), ref, H, W), FWD_BAR)
    report(('fft round trip', H, W), [per_channel(x_raw.cpu(), x.double())], FWD_BAR)


# ---------------------------------------------------------------------------------------------------------------- DWT analysis
def dwt_plan(L, H, W, lo32, hi32):
    plan = C.c_void_p()
    L.check(L.lib().aph_dwt_plan_create(C.byref(plan), H, W, lo32.ctypes.data_as(C.c_void_p), hi32.ctypes.data_as(C.c_void_p), len(lo32)),
            'aph_dwt_plan_create')
    J = C.c_int(); dims = (C.c_int * 32)(); ohw = (C.c_int * 2)()
    L.check(L.lib().aph_dwt_plan_levels(plan, C.byref(J), dims, ohw), 'aph_dwt_plan_levels')
    return plan, [(dims[2 * i], dims[2 * i + 1]) for i in range(J.value)], (ohw[0], ohw[1])


def dwt_analyze(L, plan, x, shapes, inv_scales):
    Ys = [torch.full((3, *shapes[-1]), float('nan'), device='cuda')] + [torch.full((3, 3, *hw), float('nan'), device='cuda') for hw in shapes]
    ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
    L.check(L.lib().aph_dwt_analyze(plan, x.data_ptr(), (C.c_float * len(inv_scales))(*inv_scales), ptrs, L.stream_ptr()), 'aph_dwt_analyze')
    return Ys


DWT_CASES = ([(64, 96, w) for w in WAVES] + [(33, 47, w) for w in WAVES] + [(135, 240, w) for w in ('db3', 'coif2', 'db8')]
             + [(5, 7, 'db20'), (20, 20, 'db20'), (8, 8, 'db8'), (3, 130, 'db8'), (2, 2, 'coif2'), (130, 3, 'db4')])


@pytest.mark.parametrize('H,W,wave', DWT_CASES, ids=['%dx%d-%s' % c for c in DWT_CASES])
def test_dwt_analysis_vs_float64(L, H, W, wave):
    """Every built-in wavelet at even (64x96) and odd sizes; at 33x47 the coarse lines of db20 are shorter than its 40 taps, and
    at 5x7 (db20), 3x130 (db8) and 130x3 (db4) the symmetric extension wraps around the line several times. Where lines are
    shorter than L - 1 (5x7, 20x20 and 33x47 with db20, 8x8 with db8) every level is longer than the one before it, so a
    level's row-filtered halves outgrow level 0's."""
    lo32, hi32, lo64, hi64 = dwt_filters32(wave)
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
    report(('dwt analysis', H, W, wave), [rel(y.cpu(), r) for y, r in zip(Ys, ref)], DWT_BAR * math.sqrt(max(1., len(lo32) / 12.)))


@pytest.mark.parametrize('H,W', [(720, 1280), (135, 241)])
def test_dwt_analysis_perfect_reconstruction(L, H, W):
    """coif2 analysis (bands divided by dwt_image's scales), then the synthesis multiplies them back: the image on its first
    H x W (the synthesis of an odd side is one pixel longer)."""
    from aphantasia_b200.image import DWTImage
    gen = DWTImage([1, 3, H, W], 'coif2', 0.3)
    x = torch.randn(3, H, W, generator=torch.Generator().manual_seed(W)).cuda()
    Ys = dwt_analyze(L, gen.plan, x, gen.level_hw, [float(np.float32(1. / s)) for s in gen.scales])
    oh, ow = gen.out_hw
    x_raw = torch.empty(3, oh, ow, device='cuda'); out = torch.empty_like(x_raw)
    stats = torch.empty(4, device='cuda', dtype=torch.float64)
    ptrs = (C.c_void_p * len(Ys))(*[y.data_ptr() for y in Ys])
    L.check(L.lib().aph_synth_dwt_fwd(gen.plan, ptrs, gen.scales_c, 1.0, None, 0, x_raw.data_ptr(), stats.data_ptr(), out.data_ptr(),
                                      L.stream_ptr()), 'aph_synth_dwt_fwd')
    torch.cuda.synchronize()
    assert (oh, ow) == (H + H % 2, W + W % 2)
    report(('dwt perfect reconstruction', H, W), [per_channel(x_raw[:, :H, :W].cpu(), x.cpu().double())], PR_BAR)


# ---------------------------------------------------------------------------------------------------------------- entry points
@pytest.mark.parametrize('name', ['rgb', 'grey', 'rgba', 'oddw'])
def test_fft_image_from_picture_file_vs_reference(L, fx, tmp_path, name):
    """fft_image(shape, 0.07, decay, path): the reference's parameters, the picture's size returned and written into shape,
    and a generator of that size; resume_fft(path, sd=1) as illustrip.py calls it."""
    from aphantasia_b200.image import fft_image, resume_fft
    img = fx['file_%s_img' % name]
    decay = float(fx['file_%s_decay' % name])
    path = picture_file(tmp_path, img)
    h, w = img.shape[:2]
    shape = [1, 3, 64, 48]
    params, image_f, size = fft_image(shape, 0.07, decay, path)
    assert tuple(size) == (h, w) and shape == [1, 3, h, w] and (image_f.h, image_f.w) == (h, w)
    assert tuple(params[0].shape) == (1, 3, h, w // 2 + 1, 2) and params[0].requires_grad and params[0].is_cuda
    report(('fft_image', name), RO.band_errors(params[0], fx['file_%s_fft' % name], h, w), ENTRY_BAR)
    assert bool(torch.isfinite(image_f()).all())
    if name == 'rgb':
        p1, size1 = resume_fft(path, None, decay, sd=1.)
        report(('resume_fft sd=1', name), RO.band_errors(p1, fx['file_rgb_resume_sd1'], h, w), ENTRY_BAR)


@pytest.mark.parametrize('name', ['even', 'oddh', 'oddw'])
def test_img2fft_and_un_rgb_vs_reference(L, fx, name):
    from aphantasia_b200.image import img2fft, un_rgb
    colors, decay = fx['arr_%s_cfg' % name]
    img = fx['arr_%s_img' % name]
    h, w = img.shape[:2]
    spec = img2fft(img, decay, colors)
    assert spec.is_cuda and tuple(spec.shape) == (1, 3, h, w // 2 + 1, 2)
    report(('img2fft', name), RO.band_errors(spec, fx['arr_%s_fft' % name], h, w), ENTRY_BAR)
    if name == 'even':
        report(('un_rgb', name), [per_channel(un_rgb(img, colors)[0].cpu(), torch.tensor(fx['arr_even_unrgb'][0]))], ENTRY_BAR)


@pytest.mark.parametrize('name', ['rgb', 'grey'])
def test_pixel_image_from_picture_file_vs_reference(L, fx, tmp_path, name):
    from aphantasia_b200.image import pixel_image, to_valid_rgb
    img = fx['file_%s_img' % name]
    path = picture_file(tmp_path, img)
    params, image_f, size = pixel_image([1, 3, 8, 8], path)
    assert tuple(size) == img.shape[:2] and params[0].requires_grad
    report(('pixel_image', name), [per_channel(params[0][0].detach().cpu(), torch.tensor(fx['file_%s_pixel' % name][0]))], ENTRY_BAR)
    rgb = to_valid_rgb(image_f, colors=1.5)(contrast=1.0, fixcontrast=True)                   # illustrip.py's mode for a picture
    assert tuple(rgb.shape) == (1, 3, *img.shape[:2]) and bool(torch.isfinite(rgb).all())


def test_dwt_image_from_picture_file(L, tmp_path):
    """dwt_image(shape, 'coif2', 0.5, 1.8, path): parameters of the picture's size, bands divided by init_dwt's sharp = 0.3
    scales (not 0.5), while the generator synthesises with sharp = 0.5; init_dwt and img2dwt give the same bits."""
    from aphantasia_b200.image import DWTImage, dwt_image, img2dwt, init_dwt
    img = smooth_picture(45, 64, 3)
    path = picture_file(tmp_path, img)
    shape = [1, 3, 96, 128]
    Ys, gen, size = dwt_image(shape, 'coif2', 0.5, 1.8, path)
    assert tuple(size) == (45, 64) and shape == [1, 3, 96, 128]
    assert [tuple(y.shape) for y in Ys] == DWTImage([1, 3, 45, 64], 'coif2', 0.5).param_shapes() == gen.param_shapes()
    assert gen.scales == [((gen.level_hw[0][0] * gen.level_hw[0][1]) / (h * w)) ** 0.5 for h, w in gen.level_hw]
    ref = RO.img2dwt(img, 'coif2', 0.3, 1.8)
    report(('dwt_image picture bands', 45, 64), [rel(y.detach().cpu(), r) for y, r in zip(Ys, ref)], DWT_BAR)
    for a, b in ((img2dwt(img, 'coif2', 0.3, 1.8), Ys), (init_dwt(path, shape, 'coif2', 1.8)[0], Ys)):
        assert all(torch.equal(x, y.detach()) for x, y in zip(a, b))
    r = init_dwt(path, shape, 'coif2', 1.8)
    assert r[1] is None and r[2] is None and tuple(r[3]) == (45, 64)
    rgb = to_valid_rgb_of(gen)
    assert tuple(rgb.shape) == (1, 3, *gen.out_hw) and bool(torch.isfinite(rgb).all())


def test_dwt_image_from_picture_smaller_than_the_filter(L, tmp_path):
    """A 9 x 11 picture with db20 (40 taps): the levels grow (9 -> 24 -> 31 -> 35 rows), the analysis still matches float64."""
    from aphantasia_b200.image import dwt_image
    img = smooth_picture(9, 11, 4)
    Ys, gen, size = dwt_image([1, 3, 64, 64], 'db20', 0.3, 1.5, picture_file(tmp_path, img))
    assert tuple(size) == (9, 11) and [tuple(y.shape) for y in Ys] == gen.param_shapes()
    assert [hw[0] for hw in gen.level_hw] == [24, 31, 35]
    ref = RO.img2dwt(img, 'db20', 0.3, 1.5)
    report(('dwt_image db20 picture bands', 9, 11), [rel(y.detach().cpu(), r) for y, r in zip(Ys, ref)], DWT_BAR * math.sqrt(40 / 12.))


def to_valid_rgb_of(gen):
    from aphantasia_b200.image import to_valid_rgb
    return to_valid_rgb(gen, colors=1.8)(contrast=1.1)


def test_web_size_picture_refused_by_fft_taken_by_dwt_and_pixel(L, tmp_path):
    """1000 x 667 (667 = 23 * 29): no FFT plan exists for it; the wavelet and pixel generators take any size."""
    from aphantasia_b200.image import dwt_image, fft_image, pixel_image
    img = smooth_picture(667, 1000, 9)
    path = picture_file(tmp_path, img)
    n0 = L.lib().aph_launch_count()
    with pytest.raises(ValueError, match='1000×667: 667 = 23·29'):
        fft_image([1, 3, 64, 64], 0.07, 1.5, path)
    assert L.lib().aph_launch_count() == n0
    Ys, gen, size = dwt_image([1, 3, 64, 64], 'coif2', 0.3, 1.8, path)
    assert tuple(size) == (667, 1000) and [tuple(y.shape) for y in Ys] == gen.param_shapes() and all(bool(torch.isfinite(y).all()) for y in Ys)
    params, _, size = pixel_image([1, 3, 64, 64], path)
    assert tuple(size) == (667, 1000) and tuple(params[0].shape) == (1, 3, 667, 1000)


# ---------------------------------------------------------------------------------------------------------------- unmodified script
needs_script = pytest.mark.skipif(not os.path.isfile(SCRIPT), reason='no copy of the original clip_fft.py: build() stages one into oracle/_ref/')


def frame_sizes(out_dir):
    return [Image.open(f).size for f in sorted(glob.glob(os.path.join(out_dir, '*', '*.jpg')))]


@needs_script
def test_unmodified_clip_fft_resume_from_picture(tmp_path):
    """--resume pic.png (320 x 240) with --size 224-224: the canvas takes the picture's size."""
    path = picture_file(tmp_path, smooth_picture(240, 320, 1))
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--resume', path, '--size', '224-224', '--samples', '8', '--steps', '3'])
    assert tr['encode_image_calls'] == 3 and len(tr['sims']) == 3 and all(math.isfinite(s) for s in tr['sims'])
    assert frame_sizes(out_dir) == [(320, 240)] * 3


@needs_script
def test_unmodified_clip_fft_dwt_resume_from_odd_picture(tmp_path):
    """--dwt --resume on a 241 x 321 picture: frames of the synthesis output size, one pixel larger on each odd side."""
    path = picture_file(tmp_path, smooth_picture(241, 321, 2))
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--dwt', '--resume', path, '--size', '224-224', '--samples', '8', '--steps', '3'])
    assert tr['encode_image_calls'] == 3 and all(math.isfinite(s) for s in tr['sims'])
    assert frame_sizes(out_dir) == [(322, 242)] * 3
