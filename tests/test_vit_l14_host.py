"""ViT-L/14 on the host side: the model table, the refused @336px variant, and the streaming-attention test hook's declaration
and binding. No GPU needed."""
import os
import re

import pytest

from aphantasia_b200 import _lib, clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_vitl14_is_listed_with_its_geometry():
    assert 'ViT-L/14' in clip.available_models()
    m = clip._MODELS['ViT-L/14']
    assert m == dict(patch=14, width=1024, layers=24, heads=16, out_dim=768, res=224)
    assert (m['res'] // m['patch']) ** 2 + 1 == 257          # the sequence the streaming attention serves
    assert m['heads'] * 64 == m['width']


def test_vitl14_336px_is_refused():
    with pytest.raises(RuntimeError, match='not available'):
        clip.load('ViT-L/14@336px')


def test_vitl14_synthetic_state_dict_layout():
    """the existing generator at ViT-L/14 geometry: conv1 is [1024, 3, 14, 14] (588 values per row), 257 positions"""
    sd = clip.synthetic_visual_state_dict(seed=0, **dict(clip._MODELS['ViT-L/14'], layers=1))
    assert tuple(sd['visual.conv1.weight'].shape) == (1024, 3, 14, 14)
    assert tuple(sd['visual.positional_embedding'].shape) == (257, 1024)
    assert tuple(sd['visual.proj'].shape) == (1024, 768)


def test_attn_long_test_is_declared_and_bound():
    with open(os.path.join(ROOT, 'include', 'aphb200.h')) as f:
        header = f.read()
    assert re.search(r'int aph_attn_long_test\(int fwd, const void\* qkv, const void\* dout, void\* out, int S, int T, int D, int heads,\s*'
                     r'void\* stream\);', header)
    assert 'aph_attn_long_test' in _lib.EXPORTS
    res, args = _lib._SIGS['aph_attn_long_test']
    assert len(args) == 9
