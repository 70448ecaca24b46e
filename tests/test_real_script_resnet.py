"""GPU integration: the UNMODIFIED clip_fft.py, cppn.py and illustrip.py of eps696/aphantasia with `-m RN50` / `-m RN101` (the
ResNet image towers) end to end through the launcher, as tests/test_real_script.py runs them with the ViTs. The scripts belong to
the original project: build() stages copies into the git-ignored oracle/_ref/, and without them these tests are skipped."""
import glob
import json
import math
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')


def _run(tmp_path, script, args, nv=True, sims=True):
    path = os.path.join(REF, script)
    if not os.path.isfile(path):
        pytest.skip('no copy of the original %s: build() stages one into oracle/_ref/' % script)
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_RUN_VERBOSE='1')
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', path] + args + ['--out_dir', str(tmp_path / 'out')] + (['-nv'] if nv else [])
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    tr = json.load(open(trace))
    assert tr['encode_image_calls'] > 0 and tr['launches'] > 0
    assert all(math.isfinite(s) for s in tr['sims']) and (tr['sims'] or not sims)
    return tr


@pytest.mark.parametrize('args', [['-m', 'RN50', '--samples', '8'], ['-m', 'RN101', '-tf', 'custom', '--samples', '8'],
                                  ['-m', 'RN50', '--dualmod', '2', '--samples', '40']],
                         ids=['RN50', 'RN101-custom', 'RN50-dualmod'])
def test_clip_fft_resnet(tmp_path, args):
    """--dualmod makes the script itself switch to ViT-B/32 (with ViT-B/16 every other step) and scale the samples by 0.23,
    hence the larger --samples there."""
    _run(tmp_path, 'clip_fft.py', ['-t', 'red square', '--size', '256-224', '--steps', '3'] + args)
    assert len(glob.glob(str(tmp_path / 'out' / '*' / '*.jpg'))) == 3


def test_cppn_resnet(tmp_path):
    _run(tmp_path, 'cppn.py', ['-t', 'red square', '--size', '128-128', '--samples', '8', '--steps', '4', '-m', 'RN50'], nv=False, sims=False)
    assert glob.glob(str(tmp_path / 'out' / '**' / '*.jpg'), recursive=True)


def test_illustrip_resnet_fft(tmp_path):
    _run(tmp_path, 'illustrip.py', ['-t', 'red square', '--size', '256-224', '--steps', '4', '--samples', '8', '--fstep', '2', '-m', 'RN50',
                                    '--gen', 'FFT'])
    assert glob.glob(str(tmp_path / 'out' / '**' / '*.jpg'), recursive=True)
