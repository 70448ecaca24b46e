"""GPU integration: the unmodified clip_fft.py with --in_img and --sync (the LPIPS composition loss, clip_fft.py:219-222,268-270),
through the launcher, as in test_real_script.py (and skipped, as those tests are, without a staged copy of the script)."""
import glob
import os

import numpy as np
import pytest

from test_real_script import _run, needs_script

pytestmark = pytest.mark.gpu


def _picture(tmp_path, h, w):
    from PIL import Image
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([255 * xx / w, 255 * yy / h, 128 + 64 * np.sin(xx / 9.0)], -1).astype(np.uint8)
    p = str(tmp_path / 'picture.png')
    Image.fromarray(img).save(p)
    return p


@needs_script
def test_unmodified_clip_fft_sync(tmp_path):
    """-t "red square" --in_img picture.png --sync 0.5 --size 320-256 --samples 16 --steps 6: exits 0, writes its 6 frames and
    makes one LPIPS call per step; then a --resume of the same picture with --sync also runs."""
    pic = _picture(tmp_path, 200, 240)
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--in_img', pic, '--sync', '0.5', '--size', '320-256', '--samples', '16',
                                     '--steps', '6'])
    assert tr['lpips_calls'] == 6 and tr['launches'] > 0
    assert tr['encode_image_calls'] == 7                # one per step, and the picture's own crops once (clip_fft.py:216)
    assert all(np.isfinite(tr['sims']))
    assert len(glob.glob(os.path.join(out_dir, '*', '*.jpg'))) == 6
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--in_img', pic, '--resume', pic, '--sync', '0.3', '--size', '320-256',
                                     '--samples', '16', '--steps', '3'])
    assert tr['lpips_calls'] == 3
