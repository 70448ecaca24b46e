"""GPU integration: the UNMODIFIED cppn.py of eps696/aphantasia executed end to end against libaphb200.so through the launcher
(python -m aphantasia_b200.run), which replaces the script's own CPPN class by aphantasia_b200.cppn.CPPN. The script and the
shader export it imports (shader_expo.py) belong to the original project: build() stages copies into the git-ignored
oracle/_ref/ (__graft_entry__._stage_cppn_script) when the original project is readable, and without them these tests are skipped."""
import glob
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPPN_PY = os.path.join(ROOT, 'oracle', '_ref', 'cppn.py')
needs_script = pytest.mark.skipif(not (os.path.isfile(CPPN_PY) and os.path.isfile(os.path.join(ROOT, 'oracle', '_ref', 'shader_expo.py'))),
                                  reason='no copy of the original cppn.py / shader_expo.py: build() stages them into oracle/_ref/')
SHADERS = ('-td.glsl', '-shadertoy.glsl', '-bookofshaders.glsl', '.tfx', '.txt')


def _run(tmp_path, args):
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_RUN_VERBOSE='1')
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', CPPN_PY] + args + ['--out_dir', str(tmp_path / 'out')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert 'eps -> %s' % os.path.join(ROOT, 'dropin', 'eps') in r.stderr
    return r, json.load(open(trace))


def _check_outputs(base, steps):
    frames = sorted(glob.glob(os.path.join(base, '*.jpg')))
    snaps = sorted(glob.glob(os.path.join(base, '*.npy')))
    assert [os.path.basename(f) for f in frames] == ['%04d.jpg' % i for i in range(steps)], frames
    assert [os.path.basename(f) for f in snaps] == ['%04d.npy' % i for i in range(steps)], snaps
    assert os.path.isfile(base + '.npy') and os.path.isfile(base + '-%d.jpg' % steps)
    for sfx in SHADERS:
        assert os.path.getsize(base + sfx) > 0, sfx
    params = np.load(base + '.npy', allow_pickle=True)
    assert all(np.isfinite(p).all() for p in params)
    first = np.load(os.path.join(base, '0000.npy'), allow_pickle=True)
    assert any(not np.array_equal(a, b) for a, b in zip(first, params)), 'the weights did not move'


@needs_script
def test_cppn_default_text_run(tmp_path):
    r, tr = _run(tmp_path, ['-t', 'red square', '--size', '256-224', '--steps', '6', '--samples', '20'])
    _check_outputs(str(tmp_path / 'out' / 'cppn' / 'red_square-l10-n24'), 6)
    # one training forward and one preview forward per step
    assert tr['cppn_calls'] == 12 and tr['encode_image_calls'] == 6 and tr['launches'] > 0
    assert all(math.isfinite(s) for s in tr['sims'])


@needs_script
def test_cppn_sharp_aesthetic_relu(tmp_path):
    r, tr = _run(tmp_path, ['-t', 'red square', '--size', '256-224', '--steps', '3', '--samples', '20', '--sharp', '1', '--aest', '1',
                            '-act', 'relu'])
    _check_outputs(str(tmp_path / 'out' / 'cppn' / 'red_square-l10-n24-ae1'), 3)
    assert tr['cppn_calls'] == 6 and tr['encode_image_calls'] == 3


@needs_script
def test_cppn_resume_export_without_clip(tmp_path):
    """-r <snapshot> --export writes the shaders and a preview next to the snapshot and exits before clip.load."""
    _run(tmp_path, ['-t', 'red square', '--size', '128-128', '--steps', '2', '--samples', '8'])
    snap = str(tmp_path / 'out' / 'cppn' / 'red_square-l10-n24' / '0001.npy')
    os.makedirs(str(tmp_path / 'exp'))
    exp = str(tmp_path / 'exp' / 'snap.npy')
    os.replace(snap, exp)
    r, tr = _run(tmp_path, ['-r', exp, '--export', '--size', '160-96'])
    base = exp[:-4]
    for sfx in SHADERS + ('.jpg',):
        assert os.path.getsize(base + sfx) > 0, sfx
    assert tr['cppn_calls'] == 1 and tr['encode_image_calls'] == 0 and tr['encode_text_calls'] == 0


@needs_script
def test_cppn_dualmod(tmp_path):
    r, tr = _run(tmp_path, ['-t', 'red square', '--size', '256-224', '--steps', '4', '--samples', '20', '--dualmod', '2'])
    _check_outputs(str(tmp_path / 'out' / 'cppn' / 'red_square-l10-n24-dm2'), 4)
    assert tr['encode_image_calls'] == 4 and tr['cppn_calls'] == 8
