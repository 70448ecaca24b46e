"""GPU integration: the UNMODIFIED clip_fft.py of eps696/aphantasia executed end to end against libaphb200.so through the
launcher (python -m aphantasia_b200.run), SURVEY.md 8(b). The script belongs to the original project and is not part of this
repository: build() stages a copy into the git-ignored oracle/_ref/ (oracle/stage_ref.py) when the original project is readable,
APH_REF_SCRIPT may name another copy, and without either these tests are skipped."""
import glob
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.environ.get('APH_REF_SCRIPT') or os.path.join(ROOT, 'oracle', '_ref', 'clip_fft.py')
needs_script = pytest.mark.skipif(not os.path.isfile(SCRIPT), reason='no copy of the original clip_fft.py: build() stages one into oracle/_ref/')


def _run(tmp_path, args, env_add=None, nproc=1):
    out_dir = str(tmp_path / 'out')
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_RUN_VERBOSE='1')
    env.update(env_add or {})
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', SCRIPT] + args + ['--out_dir', out_dir, '-nv']
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert 'aphantasia -> %s' % os.path.join(ROOT, 'dropin', 'aphantasia') in r.stderr
    tr = json.load(open(trace))
    return r, tr, out_dir


@needs_script
def test_unmodified_clip_fft_config1(tmp_path):
    """BASELINE configs[0] flags: -t "red square" --size 224-224 --samples 4 --steps 10 (ViT-B/32), on the GPU."""
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--size', '224-224', '--samples', '4', '--steps', '10', '--save_pt'])
    assert tr['launches'] > 0 and tr['encode_image_calls'] == 10 and len(tr['sims']) == 10
    assert tr['sims'][-1] > tr['sims'][0], 'similarity did not increase over 10 steps: %s' % tr['sims']        # loss = -sim decreases
    frames = sorted(glob.glob(os.path.join(out_dir, '*', '*.jpg')))
    assert len(frames) == 10, frames
    assert len(glob.glob(os.path.join(out_dir, '*-10.jpg'))) == 1 and len(glob.glob(os.path.join(out_dir, '*.pt'))) == 1
    assert 'rate' in r.stdout                                                                                  # the reference's only speed read-out


@needs_script
def test_unmodified_clip_fft_enforce_sharp_aest_noise(tmp_path):
    """Optional loss terms of the script (clip_fft.py:238,255-256,271-278): two encode_image calls per step (--enforce), the
    finite-difference sharpness term, the aesthetic head, the spectrum noise shift."""
    r, tr, out_dir = _run(tmp_path, ['-t', 'red square', '--size', '256-224', '--samples', '16', '--steps', '4', '--enforce', '0.5',
                                     '--sharp', '0.3', '--aest', '1', '--noise', '0.02'])
    assert tr['encode_image_calls'] == 8 and tr['launches'] > 0
    assert len(glob.glob(os.path.join(out_dir, '*', '*.jpg'))) == 4


@needs_script
def test_unmodified_clip_fft_dualmod_dwt_fused_adam(tmp_path):
    """--dualmod 2 (BASELINE configs[3] on one GPU: ViT-B/16 every 2nd step, cosine similarity), then --dwt with the script's DEFAULT
    wavelet coif2 (clip_fft.py:61), then the fused-Adam opt-in."""
    r, tr, _ = _run(tmp_path, ['-t', 'red square', '--size', '320-256', '--samples', '40', '--steps', '4', '--dualmod', '2'])
    assert tr['encode_image_calls'] == 4 and 'dual model every 2 step' in r.stdout
    r, tr, _ = _run(tmp_path, ['-t', 'red square', '--size', '320-256', '--samples', '8', '--steps', '3', '--dwt'])
    assert tr['encode_image_calls'] == 3
    r, tr, _ = _run(tmp_path, ['-t', 'red square', '--size', '224-224', '--samples', '4', '--steps', '10'], env_add={'APH_FUSED_ADAM': '1'})
    assert tr['sims'][-1] > tr['sims'][0]
