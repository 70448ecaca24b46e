"""CPU tests of the wide CPPN nets (72 <= nf <= 256): the range aph_cppn_create accepts, and the seeded initialisation at nf 256
against the original module's draws."""
import os

import numpy as np
import pytest
import torch

import cppn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_TREE = os.path.join(ROOT, 'oracle', '_ref')


@pytest.mark.parametrize('nf', [72, 128, 200, 256])
def test_wide_nets_are_accepted(nf):
    from aphantasia_b200.cppn import CPPN
    for act in ('unbias', 'comp', 'relu'):
        net = CPPN(2, nf, 3, 3, act_fn=act)
        assert net.net[1].conv.weight.shape == (nf, nf if act == 'relu' else 2 * nf, 1, 1)


def test_refusals_name_the_new_limit():
    from aphantasia_b200.cppn import CPPN
    for nf in (264, 100, 20):
        with pytest.raises(NotImplementedError, match=r'multiple of 8 in \[8, 256\]'):
            CPPN(2, nf, 10, 3)
    with pytest.raises(NotImplementedError, match=r'layers = 33'):
        CPPN(2, 256, 33, 3)


@pytest.mark.parametrize('act', ['unbias', 'relu'])
def test_seeded_init_at_nf_256_equals_the_originals_draws(act):
    from oracle import ref_import
    from aphantasia_b200.cppn import CPPN
    path = os.path.join(REF_TREE, 'cppn.py')
    if not (ref_import.available() and os.path.isfile(path)):
        pytest.skip('the original project is not readable here')
    mod = O.load_original_script(path)
    torch.manual_seed(5)
    want = mod.CPPN(2, 256, 10, 3, act_fn=act).state_dict()
    torch.manual_seed(5)
    got = CPPN(2, 256, 10, 3, act_fn=act).state_dict()
    assert list(got) == list(want)
    for k in want:
        assert got[k].shape == want[k].shape and np.array_equal(got[k].numpy(), want[k].numpy()), k
