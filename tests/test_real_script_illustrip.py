"""GPU integration: the UNMODIFIED illustrip.py and illustra.py of eps696/aphantasia executed end to end against libaphb200.so
through the launcher (python -m aphantasia_b200.run), as tests/test_real_script.py does for clip_fft.py. The scripts belong to the
original project and are not part of this repository: build() stages copies into the git-ignored oracle/_ref/
(oracle/stage_video_scripts.py) when the original project is readable, and without them these tests are skipped."""
import glob
import json
import math
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, 'oracle', '_ref')
ILLUSTRIP, ILLUSTRA = os.path.join(REF, 'illustrip.py'), os.path.join(REF, 'illustra.py')
needs_scripts = pytest.mark.skipif(not (os.path.isfile(ILLUSTRIP) and os.path.isfile(ILLUSTRA)),
                                   reason='no copy of the original illustrip.py / illustra.py: build() stages them into oracle/_ref/')
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _run(tmp_path, script, args, ok=True):
    trace = str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_RUN_VERBOSE='1')
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', script] + args + ['--out_dir', str(tmp_path / 'out'), '-nv']
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    if not ok:
        return r, None
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    assert 'depth -> %s' % os.path.join(ROOT, 'dropin', 'depth') in r.stderr
    return r, json.load(open(trace))


@needs_scripts
def test_illustrip_default_rgb(tmp_path):
    r, tr = _run(tmp_path, ILLUSTRIP, ['-t', 'red square', '--size', '256-224', '--steps', '6', '--samples', '20', '--fstep', '3'])
    frames = sorted(glob.glob(str(tmp_path / 'out' / 'red_square-rgb' / 'ttt' / '*.jpg')))
    assert len(frames) == 6, frames
    assert tr['encode_image_calls'] == 6 and tr['affine_calls'] == 6 and tr['launches'] > 0
    # get_encs pairs the prompt with the next one (here itself), weighted (steps - i) / steps and i / steps: two similarities per step
    assert len(tr['sims']) == 12 and all(math.isfinite(s) for s in tr['sims'])
    assert os.path.isfile(str(tmp_path / 'out' / 'red_square-rgb' / 'config.txt'))


@needs_scripts
def test_illustrip_fft_smooth_over_two_prompts(tmp_path):
    """--gen FFT --smooth: every frame builds a new fft_image (one shared plan) and carries the Adam state over; with two prompt
    lines get_encs interpolates between them."""
    (tmp_path / 'prompts.txt').write_text('red square\nblue circle\n')
    r, tr = _run(tmp_path, ILLUSTRIP, ['-t', str(tmp_path / 'prompts.txt'), '--gen', 'FFT', '--smooth', '--size', '256-224', '--steps', '3',
                                       '--samples', '20', '--fstep', '2'])
    frames = sorted(glob.glob(str(tmp_path / 'out' / 'prompts-fft' / 'ttt' / '*.jpg')))
    assert len(frames) == 6, frames
    assert tr['encode_image_calls'] == 6 and tr['affine_calls'] == 6
    # each step sums two weighted similarities (the scene's prompt and the next one)
    assert len(tr['sims']) == 12 and all(math.isfinite(s) for s in tr['sims'])


@needs_scripts
def test_illustrip_depth_exits_with_the_reason(tmp_path):
    r, _ = _run(tmp_path, ILLUSTRIP, ['-t', 'red square', '--size', '256-224', '--steps', '2', '--samples', '8', '--depth', '0.5'], ok=False)
    assert r.returncode != 0
    assert 'NotImplementedError' in r.stderr and 'Depth Anything V2' in r.stderr


@needs_scripts
def test_illustra_two_lines(tmp_path):
    (tmp_path / 'lines.txt').write_text('red square\nblue circle\n')
    r, tr = _run(tmp_path, ILLUSTRA, ['-t', str(tmp_path / 'lines.txt'), '--size', '256-224', '--steps', '3', '--lsteps', '2',
                                      '--samples', '20'])
    out = tmp_path / 'out'
    pts = sorted(glob.glob(str(out / '*.pt')))
    assert [os.path.basename(p) for p in pts] == ['0001-red_square-ViTB32.pt', '0002-blue_circle-ViTB32.pt'], pts
    for name in ('0001-red_square-ViTB32', '0002-blue_circle-ViTB32'):
        assert len(glob.glob(str(out / name / '*.jpg'))) == 3
        assert os.path.isfile(str(out / ('%s-3.jpg' % name)))
    assert len(glob.glob(str(out / '_final' / '*.jpg'))) == 2 * 2
    assert tr['encode_image_calls'] == 6


_RANK_RUNNER = '''
import os, runpy, sys, torch
sys.path.insert(0, {root!r})
from aphantasia_b200 import run, motion
script, out = sys.argv[1], sys.argv[2]
run.install_dropin(os.path.dirname(script))
motion.install()
rank = int(os.environ.get('RANK', '0'))
sys.argv = [script] + sys.argv[3:] + ['--out_dir', os.path.join(out, 'rank%d' % rank)]
g = runpy.run_path(script, run_name='__main__')
torch.save(g['params_tmp'].detach().cpu(), os.path.join(out, 'canvas%d.pt' % rank))
'''


@needs_scripts
@pytest.mark.skipif(NGPU < 2, reason='needs at least 2 GPUs')
def test_illustrip_two_ranks_keep_identical_canvases(tmp_path):
    """Under torchrun every rank holds the whole canvas: the motion timeline (drawn from the clock without a seed) and the
    crop replay must agree across ranks, or the replicated canvases diverge."""
    runner = tmp_path / 'runner.py'
    runner.write_text(_RANK_RUNNER.format(root=ROOT))
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    env = {k: v for k, v in os.environ.items() if k not in ('RANK', 'WORLD_SIZE', 'LOCAL_RANK')}
    env['PYTHONPATH'] = ROOT
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(port), str(runner), ILLUSTRIP, str(tmp_path), '-t', 'red square', '--size', '256-224', '--steps', '6',
           '--samples', '20', '--fstep', '3', '-nv']
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    a, b = torch.load(str(tmp_path / 'canvas0.pt')), torch.load(str(tmp_path / 'canvas1.pt'))
    assert torch.equal(a, b)
