"""GPU integration: the UNMODIFIED clip_fft.py, illustrip.py and illustra.py of eps696/aphantasia through the launcher with
APH_FUSED_ADAM=1, for the optimisers and generators the fused update covers: AdamW with AMSGrad over the FFT and the wavelet
generators, Adam over the pixel generator, AdamW across illustrip.py --smooth frames and illustra.py lines (state_dict /
load_state_dict). Each run must write its frames and report in its APH_TRACE that the updates ran inside the synthesis
backwards. The scripts belong to the original project: build() stages copies into the git-ignored oracle/_ref/, and without
them these tests are skipped."""
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
CLIP_FFT, ILLUSTRIP, ILLUSTRA = (os.path.join(REF, n) for n in ('clip_fft.py', 'illustrip.py', 'illustra.py'))
needs = lambda *scripts: pytest.mark.skipif(not all(os.path.isfile(s) for s in scripts),
                                            reason='no copy of the original script: build() stages it into oracle/_ref/')

# the launcher's main() after seeding every host RNG the scripts draw from (the crops, the initial picture) and pinning the
# motion timeline's clock seed (utils._clock_seed), so that two runs differ only in what the environment switches
_SEEDED = '''
import random, sys
import numpy as np, torch
sys.path.insert(0, {root!r})
random.seed(0); np.random.seed(0); torch.manual_seed(0)
from aphantasia_b200 import run, utils
utils._clock_seed = lambda: (np.random.seed(0), np.arange(1, 5, dtype=np.uint32))[1]
sys.exit(run.main(sys.argv[1:]))
'''


def _run(tmp_path, script, args, fused=True, seeded=False, tag='run'):
    trace = str(tmp_path / ('%s.json' % tag))
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_FUSED_ADAM='1' if fused else '0')
    if seeded:
        runner = tmp_path / 'seeded_run.py'
        runner.write_text(_SEEDED.format(root=ROOT))
        head = [sys.executable, str(runner)]
    else:
        head = [sys.executable, '-m', 'aphantasia_b200.run']
    out = tmp_path / tag
    r = subprocess.run(head + [script] + args + ['--out_dir', str(out), '-nv'], capture_output=True, text=True, timeout=900,
                       cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    return json.load(open(trace)), out


@needs(CLIP_FFT)
@pytest.mark.parametrize('gen', ['fft', 'dwt'])
def test_clip_fft_adamw_custom(tmp_path, gen):
    tr, out = _run(tmp_path, CLIP_FFT, ['-t', 'red square', '--size', '256-224', '--samples', '8', '--steps', '4', '-opt', 'adamw_custom']
                   + (['--dwt'] if gen == 'dwt' else []))
    assert len(glob.glob(str(out / '*' / '*.jpg'))) == 4
    assert tr['optim_steps_fused'] == 4 and tr['optim_steps_unfused'] == 0
    assert all(math.isfinite(s) for s in tr['sims'])


@needs(ILLUSTRIP)
def test_illustrip_default_rgb_matches_the_stock_optimiser(tmp_path):
    """--gen RGB (pixel_image) with the default -opt adam_custom, seeded, with and without the switch: the per-step similarity
    traces agree to 1e-3 (measured on an H100: 2.3e-4). What differs is the update's fp32 betas and operation order, and the
    backward's atomic sums, which are not run-to-run deterministic either; every frame starts a new optimiser, so each update
    is a first Adam step. With the motion timeline left to the clock the traces differ by ~1e-2."""
    args = ['-t', 'red square', '--size', '256-224', '--steps', '6', '--samples', '20', '--fstep', '3']
    tr, out = _run(tmp_path, ILLUSTRIP, args, fused=True, seeded=True, tag='fused')
    ref, _ = _run(tmp_path, ILLUSTRIP, args, fused=False, seeded=True, tag='stock')
    assert len(glob.glob(str(out / 'red_square-rgb' / 'ttt' / '*.jpg'))) == 6
    assert tr['optim_steps_fused'] == 6 and tr['optim_steps_unfused'] == 0
    assert ref['optim_steps_fused'] == ref['optim_steps_unfused'] == 0
    assert len(tr['sims']) == len(ref['sims']) == 12
    diff = max(abs(a - b) for a, b in zip(tr['sims'], ref['sims']))
    print('illustrip RGB similarity trace, fused vs stock: max |difference| %.2e' % diff)
    assert diff < 1e-3, (tr['sims'], ref['sims'])


@needs(ILLUSTRIP)
def test_illustrip_fft_smooth_adamw_custom(tmp_path):
    """--gen FFT --smooth: a new generator and optimiser every frame, the moments carried over by state_dict / load_state_dict."""
    tr, out = _run(tmp_path, ILLUSTRIP, ['-t', 'red square', '--gen', 'FFT', '--smooth', '-opt', 'adamw_custom', '--size', '256-224',
                                         '--steps', '4', '--samples', '20', '--fstep', '2'])
    assert len(glob.glob(str(out / 'red_square-fft' / 'ttt' / '*.jpg'))) == 4
    assert tr['optim_steps_fused'] == 4 and tr['optim_steps_unfused'] == 0


@needs(ILLUSTRA)
def test_illustra_adamw_two_lines(tmp_path):
    """-opt adamw (AdamW with AMSGrad); the second line loads the first line's optimiser state."""
    (tmp_path / 'lines.txt').write_text('red square\nblue circle\n')
    tr, out = _run(tmp_path, ILLUSTRA, ['-t', str(tmp_path / 'lines.txt'), '--size', '256-224', '--steps', '3', '--lsteps', '2',
                                        '--samples', '20', '-opt', 'adamw'])
    for name in ('0001-red_square-ViTB32', '0002-blue_circle-ViTB32'):
        assert len(glob.glob(str(out / name / '*.jpg'))) == 3
    assert tr['optim_steps_fused'] == 6 and tr['optim_steps_unfused'] == 0
