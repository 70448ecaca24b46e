"""Starting from an image file, host side (CPU only): the restatements of un_rgb / img2fft are pinned to the reference's own
outputs (tests/golden/reference_golden_resume.npz, made by tests/golden/make_golden_resume.py), and the host rules of the
drop-in entry points are checked without a GPU: which files count as pictures, resume_fft's own colors, sd folded into the
analysis scale, un_spectrum's odd-width frequencies, the refusal of picture sizes the FFT generator cannot take."""
import inspect
import os

import numpy as np
import pytest
import torch
from PIL import Image

import resume_oracle as RO
from aphantasia_b200 import image
from oracle import restate as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAR = 1e-6


@pytest.fixture(scope='module')
def fx():
    with np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_golden_resume.npz')) as z:
        return {k: z[k] for k in z.files}


def rel(a, b):
    a, b = torch.as_tensor(np.asarray(a)).double(), torch.as_tensor(np.asarray(b)).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def as_rgb(img):
    """utils.img_read's rules: grey stacked to 3 channels, alpha dropped"""
    return np.dstack([img] * 3) if img.ndim == 2 else img[..., :3]


def test_un_rgb_restatement_pinned(fx):
    colors, _ = fx['arr_even_cfg']
    assert rel(RO.un_rgb(fx['arr_even_img'], colors), fx['arr_even_unrgb']) < BAR


@pytest.mark.parametrize('name', ['even', 'oddh', 'oddw'])
def test_img2fft_restatement_pinned(fx, name):
    colors, decay = fx['arr_%s_cfg' % name]
    img = fx['arr_%s_img' % name]
    ref = fx['arr_%s_fft' % name]
    h, w = img.shape[:2]
    errs = RO.band_errors(RO.img2fft(img, decay, colors), ref, h, w)
    assert len(errs) >= 2 and max(errs) < BAR, errs


@pytest.mark.parametrize('name', ['rgb', 'grey', 'rgba', 'oddw'])
def test_picture_file_fixtures_pinned(fx, name):
    """fft_image(shape, 0.07, decay, path) of the reference = 0.07 * img2fft(img_read(path), decay, colors=1.6), at the
    picture's size, which it also writes into shape; the product's host-built analysis scale reproduces it from the fp32 DFT."""
    img = as_rgb(fx['file_%s_img' % name])
    decay = float(fx['file_%s_decay' % name])
    h, w = img.shape[:2]
    ref = fx['file_%s_fft' % name]
    assert tuple(fx['file_%s_size' % name]) == (h, w) and list(fx['file_%s_shape' % name]) == [1, 3, h, w]
    assert max(RO.band_errors(0.07 * RO.img2fft(img, decay, 1.6), ref, h, w)) < BAR
    dft = torch.view_as_real(torch.fft.rfftn(RO.un_rgb(img, 1.6), s=(h, w), dim=[2, 3], norm='ortho'))
    ours = dft * image._analysis_scale(h, w // 2 + 1, decay, 0.07)[None, None, ..., None]
    assert max(RO.band_errors(ours, ref, h, w)) < BAR
    if name == 'rgb':
        assert max(RO.band_errors(RO.img2fft(img, decay, 1.6), fx['file_rgb_resume_sd1'], h, w)) < BAR
    if name in ('rgb', 'grey'):
        assert tuple(fx['file_%s_pixel_size' % name]) == (h, w)
        assert rel(3.3 * RO.un_rgb(img, 2.), fx['file_%s_pixel' % name]) < BAR


def test_analysis_scale_odd_width_uses_w_minus_one():
    """un_spectrum recovers w = (Wh - 1) * 2: for W = 21 that is 20, whose frequencies differ from those of 21."""
    h, W = 16, 21
    ours = image._analysis_scale(h, W // 2 + 1, 1.5, 0.07).double()
    assert torch.allclose(ours, torch.tensor(0.07 * 500000. / RO.un_spectrum_scale(h, W // 2 + 1, 1.5)), rtol=1e-7, atol=0)
    naive = 1. / np.maximum(image.rfft2d_freqs(h, W), 1. / max(W, h)) ** 1.5 * np.sqrt(W * h)
    assert not np.allclose(ours.numpy(), 0.07 * 500000. / naive, rtol=1e-3)


def test_picture_extensions():
    for p in ('a.jpg', 'a.JPG', 'b.png', 'c.tif', 'd.bmp', 'x/y.Png'):
        assert image._is_image_file(p), p
    for p in ('a.jpeg', 'a.tiff', 'a.pt', 'a.gif', 'png'):
        assert not image._is_image_file(p), p


def test_resume_fft_uses_its_own_colors_and_folds_sd(tmp_path, monkeypatch):
    """fft_image never passes colors, so the picture is analysed with resume_fft's default 1.6; sd goes to the analysis."""
    assert inspect.signature(image.resume_fft).parameters['colors'].default == 1.6
    path = str(tmp_path / 'pic.png')
    Image.fromarray(np.zeros((12, 20, 3), np.uint8)).save(path)
    seen = []
    monkeypatch.setattr(image, '_img2fft', lambda img, decay, colors, sd: seen.append((img.shape, decay, colors, sd)) or 'spectrum')
    params, size = image.resume_fft(path, [1, 3, 64, 64], 1.5, sd=0.07)
    assert params == 'spectrum' and tuple(size) == (12, 20)
    assert seen == [((12, 20, 3), 1.5, 1.6, 0.07)]


def test_fft_image_refuses_sizes_with_large_prime_factors_before_gpu_work(tmp_path):
    from aphantasia_b200._lib import lib
    path = str(tmp_path / 'web.png')
    Image.fromarray(np.zeros((667, 1000, 3), np.uint8)).save(path)
    n0 = lib().aph_launch_count()
    shape = [1, 3, 64, 64]
    with pytest.raises(ValueError, match='1000×667: 667 = 23·29; the FFT generator needs prime factors ≤ 13'):
        image.fft_image(shape, 0.07, 1.5, path)
    assert lib().aph_launch_count() == n0 and shape == [1, 3, 64, 64]
    with pytest.raises(ValueError, match='17×16: 17 = 17;'):
        image.img2fft(np.zeros((16, 17, 3), np.uint8))


def test_picture_arrays_refused_or_converted():
    with pytest.raises(ValueError, match='uint8'):
        image._rgb_u8(np.zeros((4, 4, 3), np.float32))
    with pytest.raises(ValueError, match='uint8'):
        image._rgb_u8(np.zeros((4, 4), np.uint16))
    with pytest.raises(ValueError, match='shape'):
        image._rgb_u8(np.zeros((4, 4, 2), np.uint8))
    g = np.arange(12, dtype=np.uint8).reshape(3, 4)
    assert np.array_equal(image._rgb_u8(g), np.dstack([g] * 3))
    rgba = np.arange(48, dtype=np.uint8).reshape(3, 4, 4)
    out = image._rgb_u8(rgba)
    assert np.array_equal(out, rgba[..., :3]) and out.flags['C_CONTIGUOUS']


def test_img_read_without_imageio(tmp_path):
    """utils.img_read decodes with PIL when imageio is absent: grey -> 3 channels, RGBA -> RGB, palette -> its colours."""
    from aphantasia_b200.utils import img_read
    g = (np.arange(30) * 7 % 256).astype(np.uint8).reshape(5, 6)
    Image.fromarray(g).save(str(tmp_path / 'g.png'))
    assert np.array_equal(img_read(str(tmp_path / 'g.png')), np.dstack([g] * 3))
    rgba = (np.arange(120) * 5 % 256).astype(np.uint8).reshape(5, 6, 4)
    Image.fromarray(rgba).save(str(tmp_path / 'a.png'))
    assert np.array_equal(img_read(str(tmp_path / 'a.png')), rgba[..., :3])
    pal = Image.fromarray(g).convert('P')
    pal.save(str(tmp_path / 'p.png'))
    assert np.array_equal(img_read(str(tmp_path / 'p.png')), np.asarray(pal.convert('RGB')))


def test_dwt_scale_helpers_match_restatement():
    shapes = R.dwt_level_shapes(45, 64, 12)
    Ys = [torch.empty(1, 3, *shapes[-1])] + [torch.empty(1, 3, 3, *hw) for hw in shapes]
    assert image.dwt_scale(Ys, 0.3) == R.dwt_scales(shapes, 0.3) == image._dwt_scales(shapes, 0.3)


@pytest.mark.parametrize('wave,h,w', [('coif2', 24, 20), ('coif2', 15, 21), ('db3', 17, 26), ('haar', 16, 16)])
def test_img2dwt_restatement_perfect_reconstruction_unpinned(wave, h, w):
    """PARITY UNPINNED (pytorch_wavelets absent): the restated img2dwt, its bands multiplied back by their scales, goes through
    the restated DWTInverse to un_rgb(img) on its first H x W (the synthesis of an odd side is one pixel longer)."""
    img = np.random.RandomState(h * w).randint(0, 256, (h, w, 3)).astype(np.uint8)
    Ys = RO.img2dwt(img, wave, 0.3, 1.5)
    assert [tuple(y.shape[3:5]) for y in Ys[1:]] == R.dwt_level_shapes(h, w, len(R.wavelet_filters(wave)[0]))
    scales = R.dwt_scales([tuple(y.shape[3:5]) for y in Ys[1:]], 0.3)
    rec_lo, rec_hi = R.wavelet_filters(wave)
    x = R.dwt_inverse(Ys[0], [y * s for y, s in zip(Ys[1:], scales)], rec_lo, rec_hi)
    assert rel(x[..., :h, :w], RO.un_rgb(img, 1.5, torch.float64)) < 1e-9


@pytest.mark.parametrize('H,W,wave,L', [(5, 7, 'db20', 40), (20, 20, 'db20', 40), (33, 47, 'db20', 40), (8, 8, 'db8', 16)])
def test_dwt_analysis_levels_outgrow_level_zero_and_are_tested_on_the_gpu(H, W, wave, L):
    """Where lines are shorter than L - 1 a level is longer than its input ((h + L - 1) // 2 > h), so the row-filtered halves
    [3][2][h_in][w_out] of a later level are larger than level 0's: a scratch sized for level 0 would be overrun. These sizes
    are among the GPU cases that compare the analysis with float64 at every level."""
    import test_image_resume_gpu as G
    shapes = R.dwt_level_shapes(H, W, L)
    h_in = [H] + [hw[0] for hw in shapes[:-1]]
    rows = [6 * h * hw[1] for h, hw in zip(h_in, shapes)]
    assert max(rows) > rows[0], rows
    assert (H, W, wave) in G.DWT_CASES
