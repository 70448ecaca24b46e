"""GPU integration: the UNMODIFIED clip_fft.py, illustrip.py and cppn.py of eps696/aphantasia with `-m RN50x4`, `-m RN50x16` and
`-m RN50x64` end to end through the launcher. These models load from an OpenAI checkpoint only, so each test writes a seeded
synthetic fp16 one in OpenAI's key layout to a temporary directory and points APH_CLIP_WEIGHTS_<NAME> at it. The scripts belong
to the original project: build() stages copies into the git-ignored oracle/_ref/, and without them these tests are skipped."""
import glob
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from aphantasia_b200 import clip

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
_CKPT = {}


def _checkpoint(tmp_path_factory, name):
    if name not in _CKPT:
        sd = clip.synthetic_resnet_state_dict(seed=3, **clip._MODELS[name])
        path = tmp_path_factory.mktemp('ckpt') / ('%s.pt' % name)
        torch.save({k: (v.half() if v.is_floating_point() else v) for k, v in sd.items()}, str(path))
        _CKPT[name] = str(path)
    return _CKPT[name]


def _run(tmp_path, tmp_path_factory, script, name, args, nv=True, sims=True):
    path = os.path.join(REF, script)
    if not os.path.isfile(path):
        pytest.skip('no copy of the original %s: build() stages one into oracle/_ref/' % script)
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_RUN_VERBOSE='1')
    env.pop('APH_CLIP_WEIGHTS', None)
    env[clip.weights_variable(name)] = _checkpoint(tmp_path_factory, name)
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', path] + args + ['-m', name, '--out_dir', str(tmp_path / 'out')] + \
        (['-nv'] if nv else [])
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    tr = json.load(open(trace))
    assert tr['encode_image_calls'] > 0 and tr['launches'] > 0
    assert all(math.isfinite(s) for s in tr['sims']) and (tr['sims'] or not sims)
    return tr


@pytest.mark.parametrize('name, tf', [('RN50x4', 'fast'), ('RN50x4', 'custom'), ('RN50x16', 'fast'), ('RN50x16', 'custom')])
def test_clip_fft_wide_resnet(tmp_path, tmp_path_factory, name, tf):
    """--samples 40 gives RN50x4 six crops and RN50x16 two after the script's per-model memory scale."""
    _run(tmp_path, tmp_path_factory, 'clip_fft.py', name, ['-t', 'red square', '--size', '480-480', '--steps', '3', '--samples', '40',
                                                           '-tf', tf])
    assert len(glob.glob(str(tmp_path / 'out' / '*' / '*.jpg'))) == 3


def test_illustrip_rn50x16(tmp_path, tmp_path_factory):
    _run(tmp_path, tmp_path_factory, 'illustrip.py', 'RN50x16', ['-t', 'red square', '--size', '480-480', '--steps', '4', '--samples', '40',
                                                                 '--fstep', '2', '--gen', 'FFT'])
    assert glob.glob(str(tmp_path / 'out' / '**' / '*.jpg'), recursive=True)


def test_cppn_rn50x64(tmp_path, tmp_path_factory):
    """--samples 100 gives RN50x64 three crops after the script's per-model memory scale (x 0.04) and its 0.95."""
    _run(tmp_path, tmp_path_factory, 'cppn.py', 'RN50x64', ['-t', 'red square', '--size', '456-456', '--samples', '100', '--steps', '3'],
         nv=False, sims=False)
    assert glob.glob(str(tmp_path / 'out' / '**' / '*.jpg'), recursive=True)
