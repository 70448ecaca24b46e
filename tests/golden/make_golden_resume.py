"""Generates tests/golden/reference_golden_resume.npz from the REAL reference (the original project), build container only.

    python tests/golden/make_golden_resume.py

Starting from an image: the reference's own un_rgb, img2fft, resume_fft / fft_image on a picture file and pixel_image on a
picture file (aphantasia/image.py:98-150, 185-220), run in place through oracle/ref_import.py with imageio's imread replaced by
a PIL reader (imageio is absent). The pictures are seeded uint8 arrays stored in the fixture; the tests write them back to
PNG files, which round-trip uint8 exactly. img2dwt needs pytorch_wavelets (absent): it is not pinned here.
"""
import os
import sys
import tempfile

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def picture(h, w, seed, channels=3):
    """smooth colour ramps plus noise, so the spectrum has both a strong low band and a populated high band"""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = [128 + 90 * np.sin(2 * np.pi * (xx / w * (k + 1) + yy / h * (2 - k)) + k) for k in range(max(channels, 3))]
    img = np.stack(base[:channels], -1) + rng.normal(0, 25, (h, w, channels))
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    return img[..., 0] if channels == 1 else img


def main():
    ref = ref_import.load()
    pil_read = lambda path: np.asarray(Image.open(path))
    ref.utils.imread = pil_read
    ref.image.imread = pil_read
    g = {}
    # un_rgb and img2fft on arrays: even x even, odd H, odd W (un_spectrum's W - 1 frequencies)
    for name, (h, w), colors, decay, seed in [('even', (24, 20), 1.5, 1.5, 1), ('oddh', (15, 20), 2.0, 1.0, 2), ('oddw', (16, 21), 1.6, 1.5, 3)]:
        img = picture(h, w, seed)
        g['arr_%s_img' % name] = img
        g['arr_%s_cfg' % name] = np.array([colors, decay])
        if name == 'even':
            g['arr_%s_unrgb' % name] = ref.image.un_rgb(img, colors=colors).numpy()
        g['arr_%s_fft' % name] = ref.image.img2fft(img, decay, colors).numpy()
    # picture files: RGB, grey (stacked to 3 channels by img_read), RGBA (alpha dropped), odd W
    files = [('rgb', picture(24, 20, 4), 1.5), ('grey', picture(18, 26, 5, 1), 1.0), ('rgba', picture(15, 22, 6, 4), 1.5),
             ('oddw', picture(12, 21, 7), 1.0)]
    with tempfile.TemporaryDirectory() as d:
        for name, img, decay in files:
            path = os.path.join(d, name + '.png')
            Image.fromarray(img).save(path)
            assert np.array_equal(pil_read(path), img)
            g['file_%s_img' % name] = img
            g['file_%s_decay' % name] = np.array(decay)
            shape = [1, 3, 7, 9]
            params, _, size = ref.image.fft_image(shape, 0.07, decay, path)          # resume_fft(path, sd=0.07), colors 1.6
            g['file_%s_fft' % name] = params[0].detach().numpy()
            g['file_%s_size' % name] = np.array(size)
            g['file_%s_shape' % name] = np.array(shape)
            if name == 'rgb':
                p1, _ = ref.image.resume_fft(path, None, decay, sd=1.)                     # illustrip.py's sd
                g['file_%s_resume_sd1' % name] = p1.numpy()
            if name in ('rgb', 'grey'):
                pix, _, psize = ref.image.pixel_image([1, 3, 5, 5], path)                  # 3.3 * un_rgb(img, colors=2)
                g['file_%s_pixel' % name] = pix[0].detach().numpy()
                g['file_%s_pixel_size' % name] = np.array(psize)
    path = os.path.join(OUT, 'reference_golden_resume.npz')
    np.savez_compressed(path, **g)
    print('wrote', path, os.path.getsize(path) // 1024, 'KiB,', len(g), 'arrays')


if __name__ == '__main__':
    main()
