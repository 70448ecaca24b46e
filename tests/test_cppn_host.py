"""CPU tests of cppn.py's path: the float64 restatement (tests/cppn_oracle.py) against the original classes' values
(tests/golden/reference_golden_cppn.npz), the seeded initialisation of aphantasia_b200.cppn.CPPN, the script's own .npy
convention, the launcher's detection of scripts that define their CPPN, and the `eps` drop-in."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cppn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_TREE = os.path.join(ROOT, 'oracle', '_ref')
GOLDEN = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_golden_cppn.npz'))
ACTS = ('unbias', 'comp', 'relu')
CASES = sorted({int(k[1:].split('_')[0]) for k in GOLDEN.files})


def _case(i):
    act, nf, layers, H, W, seed = (int(v) for v in GOLDEN['c%d_meta' % i])
    n = 2 * (layers + 1)
    return dict(act=ACTS[act], nf=nf, layers=layers, H=H, W=W, seed=seed, params=[GOLDEN['c%d_p%d' % (i, k)] for k in range(n)],
                grads=[GOLDEN['c%d_g%d' % (i, k)] for k in range(n)], coords=GOLDEN['c%d_coords' % i], out=GOLDEN['c%d_out' % i],
                gout=GOLDEN['c%d_gout' % i])


@pytest.mark.parametrize('i', CASES)
def test_restatement_equals_the_original_network(i):
    """Without TF32 rounding, the float64 restatement is the original's fp32 CPU result up to fp32 rounding."""
    c = _case(i)
    out, cache = O.forward(c['coords'], c['params'], c['act'], tf32_ops=False)
    np.testing.assert_allclose(out, c['out'], rtol=0, atol=2e-6)
    for k, (g, want) in enumerate(zip(O.backward(cache, c['gout']), c['grads'])):
        g = g.reshape(want.shape)
        assert np.linalg.norm(g - want) <= 1e-5 * max(np.linalg.norm(want), 1e-3), (k, np.abs(g - want).max())


def test_tf32_rounding_is_round_to_nearest_ties_away():
    x = np.array([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -12, 1.0 + 3 * 2 ** -12, -(1.0 + 2 ** -11), 1.0 + 2 ** -11 - 2 ** -23], np.float32)
    # TF32's ulp at 1 is 2^-10: a tie (2^-11) rounds away from zero, a quarter ulp down, three quarters up
    want = np.array([1.0, 1.0 + 2 ** -10, 1.0, 1.0 + 2 ** -10, -(1.0 + 2 ** -10), 1.0])
    np.testing.assert_array_equal(O.tf32(x), want)


@pytest.mark.parametrize('i', CASES)
def test_seeded_init_equals_the_originals_bit_for_bit(i):
    from aphantasia_b200.cppn import CPPN
    c = _case(i)
    torch.manual_seed(c['seed'])
    sd = CPPN(2, c['nf'], c['layers'], 3, act_fn=c['act']).state_dict()
    keys = list(sd)
    assert keys == ['net.%d.conv.%s' % (l, k) for l in range(c['layers'] + 1) for k in ('weight', 'bias')]
    for k, want in zip(keys, c['params']):
        assert sd[k].shape == want.shape and np.array_equal(sd[k].numpy(), want), k


def test_unsupported_shapes_raise_not_implemented_naming_the_limit():
    from aphantasia_b200.cppn import CPPN
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        CPPN(2, 20, 10, 3)
    with pytest.raises(NotImplementedError, match=r'\[1, 32\]'):
        CPPN(2, 24, 33, 3)
    with pytest.raises(NotImplementedError, match='nf_in'):
        CPPN(3, 24, 10, 3)


def _original_script():
    from oracle import ref_import
    path = os.path.join(REF_TREE, 'cppn.py')
    if not (ref_import.available() and os.path.isfile(path)):
        pytest.skip('the original project is not readable here')
    return O.load_original_script(path)


def test_npy_snapshot_of_the_scripts_export_loads_back_into_our_class(tmp_path, monkeypatch):
    """export_data (cppn.py:150-168) writes the weights permuted to [1,1,in,out]; load_cppn (cppn.py:118-133) reads them back into
    `CPPN`, which the launcher rebinds to ours."""
    from aphantasia_b200.cppn import CPPN
    mod = _original_script()
    monkeypatch.setattr(torch.nn.Module, 'cuda', lambda self, *a, **k: self)      # load_cppn builds CPPN(...).cuda()
    for act, nf in (('unbias', 24), ('relu', 16)):
        torch.manual_seed(7)
        net = CPPN(2, nf, 4, 3, act_fn=act)
        name = str(tmp_path / act)
        mod.export_data(net.state_dict(), name, [64, 64], npy=True)
        mod.CPPN = CPPN
        back = mod.load_cppn(name + '.npy', verbose=False)
        assert isinstance(back, CPPN) and back.act_fn == act
        for k, v in net.state_dict().items():
            assert torch.equal(back.state_dict()[k], v), k


def test_launcher_equivalence_check_accepts_the_scripts_cppn_and_refuses_a_different_one():
    from aphantasia_b200 import cppn, run
    mod = _original_script()
    state = torch.get_rng_state()
    run.check_cppn_equivalence(mod.CPPN, cppn.CPPN)
    assert torch.equal(state, torch.get_rng_state())

    class Other(cppn.CPPN):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            with torch.no_grad():
                self.net[1].conv.bias.add_(1e-3)
    with pytest.raises(NotImplementedError, match='net.1.conv.bias'):
        run.check_cppn_equivalence(mod.CPPN, Other)


def test_launcher_detects_cppn_py_and_no_other_staged_script():
    from aphantasia_b200 import run
    scripts = sorted(f for f in os.listdir(REF_TREE) if f.endswith('.py')) if os.path.isdir(REF_TREE) else []
    if 'cppn.py' not in scripts:
        pytest.skip('no copy of the original cppn.py: build() stages one into oracle/_ref/')
    assert [s for s in scripts if run.cppn_script(os.path.join(REF_TREE, s))] == ['cppn.py']
    assert {'clip_fft.py', 'illustrip.py', 'illustra.py', 'shader_expo.py'} <= set(scripts)


def test_eps_resolves_to_dropin():
    if not os.path.isfile(os.path.join(REF_TREE, 'cppn.py')):
        pytest.skip('no copy of the original cppn.py: build() stages one into oracle/_ref/')
    env = dict(os.environ, APH_RUN_VERBOSE='1', PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, '-m', 'aphantasia_b200.run', os.path.join(REF_TREE, 'cppn.py'), '--help'], capture_output=True,
                         text=True, timeout=300, cwd=REF_TREE, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    assert '--actfn' in out.stdout
    for name in ('aphantasia', 'clip', 'eps'):
        assert '%s -> %s' % (name, os.path.join(ROOT, 'dropin', name)) in out.stderr, out.stderr[-2000:]
    sys.path.insert(0, os.path.join(ROOT, 'dropin'))
    try:
        from eps import data_load, progress_bar
        from aphantasia_b200 import progress_bar as pb, utils
        assert progress_bar.ProgressBar is pb.ProgressBar
        for n in ('basename', 'img_list', 'img_read', 'file_list', 'save_cfg'):
            assert getattr(data_load, n) is getattr(utils, n)
    finally:
        sys.path.remove(os.path.join(ROOT, 'dropin'))
        for k in [k for k in sys.modules if k == 'eps' or k.startswith('eps.')]:
            del sys.modules[k]


def test_sobel_restatement_unpinned_on_known_images():
    """kornia is absent, so this checks the restatement against hand values, not against kornia. A horizontal ramp of slope 1 has gx = 1 inside and 1/2 on the replicated edge columns, gy = 0; a constant image has 0."""
    H, W = 5, 6
    img = np.tile(np.arange(W, dtype=np.float64), (1, 2, H, 1))
    g = O.sobel_gradient(img)
    assert np.allclose(g[:, :, 0, :, 1:-1], 1.) and np.allclose(g[:, :, 0, :, [0, -1]], .5) and np.allclose(g[:, :, 1], 0.)
    v, d = O.sobel_derivat(np.full((1, 3, 4, 4), .25))
    assert v == 0. and not d.any()
    # the adjoint against central differences on a random image
    rng = np.random.default_rng(0)
    x = rng.standard_normal((1, 2, 4, 5))
    _, d = O.sobel_derivat(x)
    for idx in [(0, 0, 0, 0), (0, 1, 3, 4), (0, 0, 2, 0), (0, 1, 1, 2)]:
        e = np.zeros_like(x); e[idx] = 1e-6
        num = (O.sobel_derivat(x + e)[0] - O.sobel_derivat(x - e)[0]) / 2e-6
        assert abs(num - d[idx]) < 1e-6, idx
