"""CLIP text encoder on the GPU (csrc/text.cu through aph_text_*): parity with the CPU restatement (tests/text_oracle.py) at
small geometries and at the ViT-B text configuration, causality of the attention mask, the public clip.load / tokenize /
encode_text path, and the unmodified clip_fft.py with a checkpoint that holds a text tower."""
import glob
import json
import os
import subprocess
import sys

import pytest
import torch

import text_oracle as TO
from aphantasia_b200 import _lib, clip

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VITB = dict(width=512, layers=12, heads=8, out_dim=512, context=77, vocab=49408)


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).norm() / b.detach().cpu().double().norm())


def _tokens(n, ctx, vocab, eots, seed):
    """[n, ctx] ids: sot, random ids, eot (= vocab - 1, the largest id) at eots[r], then zero padding."""
    g = torch.Generator().manual_seed(seed)
    t = torch.zeros(n, ctx, dtype=torch.long)
    for r in range(n):
        e = eots[r % len(eots)]
        t[r, 0] = vocab - 2
        t[r, 1:e] = torch.randint(1, vocab - 2, (e - 1,), generator=g)
        t[r, e] = vocab - 1
    return t


@pytest.mark.parametrize('cfg', [dict(width=128, layers=2, heads=2, out_dim=128, context=16, vocab=500),
                                 dict(width=256, layers=2, heads=4, out_dim=256, context=77, vocab=1000),
                                 VITB], ids=['w128-ctx16', 'w256-ctx77', 'vitb'])
def test_text_fwd_matches_restatement(cfg):
    sd = clip.synthetic_text_state_dict(seed=5, **cfg)
    ref = TO.build_text(sd)
    tower = clip.TextTransformer(sd)
    ctx = cfg['context']
    eots = [1, ctx // 2, ctx - 1, 3, ctx - 2]
    before = _lib.lib().aph_launch_count()
    for n in (1, 3, 5):                    # growing n re-creates the handle; the largest n comes last
        toks = _tokens(n, ctx, cfg['vocab'], eots, seed=n)
        got = tower(toks.cuda())
        with torch.no_grad():
            want = ref(toks)
        assert got.shape == (n, cfg['out_dim']) and got.dtype == torch.float32 and got.is_cuda
        assert _rel(got, want) < 2e-2, (cfg, n, _rel(got, want))
    assert _lib.lib().aph_launch_count() > before
    # a smaller batch after a larger one reuses the handle
    toks = _tokens(2, ctx, cfg['vocab'], eots[::-1], seed=9)
    with torch.no_grad():
        assert _rel(tower(toks.cuda()), ref(toks)) < 2e-2


def test_text_attention_is_causal():
    """Tokens after each row's EOT do not change the embedding (bit for bit); a token before it does."""
    cfg = dict(width=256, layers=2, heads=4, out_dim=256, context=77, vocab=1000)
    sd = clip.synthetic_text_state_dict(seed=7, **cfg)
    tower = clip.TextTransformer(sd)
    toks = _tokens(3, 77, cfg['vocab'], [4, 20, 40], seed=1)
    base = tower(toks.cuda()).cpu()
    after = toks.clone()
    g = torch.Generator().manual_seed(2)
    for r, e in enumerate([4, 20, 40]):
        after[r, e + 1:] = torch.randint(1, cfg['vocab'] - 2, (76 - e,), generator=g)       # all below the EOT id
    assert torch.equal(tower(after.cuda()).cpu(), base)
    before = toks.clone()
    before[:, 2] = (before[:, 2] + 17) % (cfg['vocab'] - 2) + 1
    changed = tower(before.cuda()).cpu()
    assert all(not torch.equal(changed[r], base[r]) for r in range(3))


def test_text_rejects_bad_input():
    cfg = dict(width=128, layers=1, heads=2, out_dim=128, context=16, vocab=500)
    tower = clip.TextTransformer(clip.synthetic_text_state_dict(seed=1, **cfg))
    toks = _tokens(2, 16, 500, [5], seed=0)
    with pytest.raises(RuntimeError, match='CUDA tensor'):
        tower(toks)
    bad = toks.clone(); bad[1, 3] = 500
    with pytest.raises(ValueError, match=r'\[0, 500\)'):
        tower(bad.cuda())
    with pytest.raises(ValueError):
        tower(toks[:, :8].cuda())


def test_public_path_and_two_models(tmp_path, monkeypatch):
    """CLIP with visual + text weights (synthetic=False), tokenize with a BPE vocabulary, encode_text on the GPU; two models
    side by side (as --dualmod holds ViT-B/32 and ViT-B/16) keep independent handles."""
    gz, _, _, n_vocab = TO.write_vocab(str(tmp_path / 'vocab'))
    monkeypatch.setenv('APH_CLIP_BPE', gz)
    models, refs = [], []
    for name, patch, seed in (('ViT-B/32', 32, 0), ('ViT-B/16', 16, 1)):
        sd = clip.synthetic_visual_state_dict(patch=patch, seed=seed)
        sd.update(clip.synthetic_text_state_dict(seed=10 + seed))
        models.append(clip.CLIP(name, sd, False))
        refs.append(TO.build_text(sd))
    toks = clip.tokenize(['red square', 'blue circle'])
    assert toks[0, 0] == n_vocab - 2 and (toks == n_vocab - 1).sum() == 2
    outs = []
    for m, ref in zip(models + models[::-1], refs + refs[::-1]):            # interleaved calls
        e = m.encode_text(toks.cuda())
        assert not e.requires_grad and e.shape == (2, 512)
        with torch.no_grad():
            assert _rel(e, ref(toks)) < 2e-2
        outs.append(e.cpu())
    assert torch.equal(outs[0], outs[3]) and torch.equal(outs[1], outs[2])
    assert _rel(outs[0], outs[1]) > 0.1


SCRIPT = os.environ.get('APH_REF_SCRIPT') or os.path.join(ROOT, 'oracle', '_ref', 'clip_fft.py')


@pytest.mark.skipif(not os.path.isfile(SCRIPT), reason='no copy of the original clip_fft.py: build() stages one into oracle/_ref/')
def test_unmodified_clip_fft_with_text_tower(tmp_path):
    """clip_fft.py -t "red square" with a checkpoint holding the text tower and a BPE vocabulary: the prompt goes through the
    CUDA text encoder and the optimisation follows it."""
    gz, _, _, _ = TO.write_vocab(str(tmp_path / 'vocab'))
    sd = clip.synthetic_visual_state_dict(patch=32, layers=2, seed=0)
    sd.update(clip.synthetic_text_state_dict(layers=2, seed=3))
    weights = str(tmp_path / 'ViT-B-32.pt')
    torch.save({k: v.half() for k, v in sd.items()}, weights)
    out_dir, trace = str(tmp_path / 'out'), str(tmp_path / 'trace.json')
    env = dict(os.environ, PYTHONPATH=ROOT, APH_TRACE=trace, APH_CLIP_WEIGHTS=weights, APH_CLIP_BPE=gz)
    cmd = [sys.executable, '-m', 'aphantasia_b200.run', SCRIPT, '-t', 'red square', '--size', '224-224', '--samples', '4',
           '--steps', '10', '--out_dir', out_dir, '-nv']
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    tr = json.load(open(trace))
    assert tr['text_tower'] == 'cuda' and tr['encode_text_calls'] >= 1 and tr['encode_image_calls'] == 10
    assert tr['sims'][-1] > tr['sims'][0], 'similarity did not increase over 10 steps: %s' % tr['sims']
    assert len(glob.glob(os.path.join(out_dir, '*', '*.jpg'))) == 10
