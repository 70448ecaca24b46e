"""CPU restatement of the reference's start-from-an-image analysis -- TEST INFRASTRUCTURE ONLY (never imported by the product).

un_rgb / img2fft follow aphantasia/image.py:185-220 (paths relative to the original project) and are pinned to the reference's
own outputs by tests/test_image_resume_host.py with tests/golden/reference_golden_resume.npz (tests/golden/make_golden_resume.py).
img2dwt follows image.py:82-94 on oracle/restate.py's afb1d_sym: pytorch_wavelets / PyWavelets are absent, so its parity with
them is unpinned (perfect reconstruction through the restated DWTInverse is what can be checked).
"""
import math

import numpy as np
import torch

from oracle import restate as R


def un_rgb(img, colors=1., dtype=torch.float32):
    """image.py:185-197 on a uint8 HWC picture: [1,3,H,W]. fp32 reproduces the reference's rounding; float64 is the exact value."""
    x = torch.tensor(np.asarray(img), dtype=dtype).permute(2, 0, 1)[None] / 255.
    mean = torch.tensor(R.CLIP_MEAN, dtype=torch.float32).to(dtype).view(1, 3, 1, 1)
    std = torch.tensor(R.CLIP_STD, dtype=torch.float32).to(dtype).view(1, 3, 1, 1)
    x = (x - mean) / std                                                  # transforms.py:106 (Normalize)
    inv = torch.linalg.inv(R.color_matrix(colors)).to(dtype)             # inv(colcorr_t), inverted in fp32
    return torch.einsum('nchw,cd->ndhw', x, inv)


def un_spectrum_scale(h, wh, decay):
    """image.py:199-206: float64 [h, wh]; w is recovered as (wh - 1) * 2, i.e. W - 1 for an odd width."""
    w = (wh - 1) * 2
    fy = np.fft.fftfreq(h)[:, None]
    fx = np.fft.fftfreq(w)[:w // 2 + 1]
    scale = 1. / np.maximum(np.sqrt(fx * fx + fy * fy), 1. / max(w, h)) ** decay
    return scale * np.sqrt(w * h)


def img2fft(img, decay=1., colors=1., dtype=torch.float32):
    """image.py:208-220: [1,3,H,W//2+1,2]."""
    x = un_rgb(img, colors, dtype)
    h, w = x.shape[2], x.shape[3]
    spectrum = torch.view_as_real(torch.fft.rfftn(x, s=(h, w), dim=[2, 3], norm='ortho'))
    scale = torch.tensor(un_spectrum_scale(h, w // 2 + 1, decay))
    scale = (scale.float() if dtype == torch.float32 else scale.to(dtype))[None, None, ..., None]
    return spectrum / scale * 500000.


def dwt_analysis(x, rec_lo, rec_hi):
    """DWTForward(J = floor(log2 min(H, W)), mode 'symmetric') of x [N,C,H,W]: [Yl, Yh_1 (finest) .. Yh_J], Yh_i [N,C,3,h,w]
    with bands (LH, HL, HH): rows (W) filtered before columns (H), as pytorch_wavelets' afb2d."""
    dec_lo, dec_hi = list(rec_lo)[::-1], list(rec_hi)[::-1]
    J = int(math.floor(math.log2(min(x.shape[2], x.shape[3]))))
    ll, yh = x, []
    for _ in range(J):
        lo, hi = R.afb1d_sym(ll, dec_lo, dec_hi, 3)
        ll, lh = R.afb1d_sym(lo, dec_lo, dec_hi, 2)
        hl, hh = R.afb1d_sym(hi, dec_lo, dec_hi, 2)
        yh.append(torch.stack([lh, hl, hh], 2))
    return [ll] + yh


def img2dwt(img, wave='coif2', sharp=0.3, colors=1., dtype=torch.float64):
    """image.py:82-94: each Yh_i divided by dwt_scale(Ys, sharp)[i]."""
    rec_lo, rec_hi = R.wavelet_filters(wave.replace('sym', 'db'))        # sym2 / sym3 are db2 / db3
    Ys = dwt_analysis(un_rgb(img, colors, dtype), rec_lo, rec_hi)
    scales = R.dwt_scales([tuple(y.shape[3:5]) for y in Ys[1:]], sharp)
    return [Ys[0]] + [y / s for y, s in zip(Ys[1:], scales)]


def radial_bands(h, w, bands=((0., 0.05), (0.05, 0.25), (0.25, 1.))):
    """boolean masks [h, w//2+1] of the radial frequency bands |f| in [lo, hi)"""
    fy = np.abs(np.fft.fftfreq(h))[:, None]
    fx = np.fft.rfftfreq(w)[None, :]
    f = np.sqrt(fx * fx + fy * fy)
    return [torch.tensor((f >= lo) & (f < hi)) for lo, hi in bands]


def band_errors(got, ref, h, w):
    """max over channels of ||got - ref|| / ||ref|| within each non-empty radial band of spectra [.., 3, h, w//2+1, 2]"""
    got = torch.as_tensor(np.asarray(got.detach().cpu() if torch.is_tensor(got) else got)).double().reshape(3, h, w // 2 + 1, 2)
    ref = torch.as_tensor(np.asarray(ref.detach().cpu() if torch.is_tensor(ref) else ref)).double().reshape(3, h, w // 2 + 1, 2)
    errs = []
    for m in radial_bands(h, w):
        if bool(m.any()):
            errs.append(max(float((got[c][m] - ref[c][m]).norm() / ref[c][m].norm().clamp_min(1e-300)) for c in range(3)))
    return errs
