"""CPU tests of what illustrip.py and illustra.py need from the drop-in: their imports through the launcher, the helpers
they call (against the original's, loaded by oracle/ref_import.py where the original project is readable), the `depth` stand-in,
and the host side of the motion route (its inverse matrix and the calls it leaves to torchvision)."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_TREE = os.path.join(ROOT, 'oracle', '_ref')          # the original scripts + aphantasia/ as build() staged them


_REF = {}


def _ref_utils():
    """The original's utils module. The loader's stand-ins for packages absent here (imageio, kornia, ...) and its
    `.cuda()` shim are taken back afterwards, so that they do not leak into the tests that run after this file."""
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip('the original project is not readable here')
    if 'utils' not in _REF:
        before = set(sys.modules)
        cuda_t, cuda_m = torch.Tensor.cuda, torch.nn.Module.cuda
        try:
            _REF['utils'] = ref_import.load().utils
        finally:
            for k in [k for k in sys.modules if k not in before and getattr(sys.modules[k], '__aph_stub__', False)]:
                del sys.modules[k]
            torch.Tensor.cuda, torch.nn.Module.cuda = cuda_t, cuda_m
    return _REF['utils']


def _launch_help(script):
    env = dict(os.environ, APH_RUN_VERBOSE='1', PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, '-m', 'aphantasia_b200.run', os.path.join(REF_TREE, script), '--help'], capture_output=True,
                          text=True, timeout=300, cwd=REF_TREE, env=env)


@pytest.mark.parametrize('script,flag', [('illustrip.py', '--fstep'), ('illustra.py', '--lsteps')])
def test_launcher_resolves_every_import_of_the_video_scripts(script, flag):
    """Started from inside a tree with the original `aphantasia/` and `depth/` packages beside it, every top-level import of the
    unmodified script resolves to dropin/ (argparse --help exits before any GPU work)."""
    if not os.path.isfile(os.path.join(REF_TREE, script)):
        pytest.skip('no copy of the original %s: build() stages one into oracle/_ref/' % script)
    out = _launch_help(script)
    assert out.returncode == 0, out.stderr[-3000:]
    assert flag in out.stdout
    for name in ('aphantasia', 'clip', 'depth'):
        assert '%s -> %s' % (name, os.path.join(ROOT, 'dropin', name)) in out.stderr, out.stderr[-2000:]


@pytest.mark.parametrize('cubic', [True, False])
@pytest.mark.parametrize('uniform', [True, False])
@pytest.mark.parametrize('start_lat', [None, [0.6, 0.5, 0.5]])
def test_latent_anima_equals_the_original_with_a_seed(cubic, uniform, start_lat):
    ref = _ref_utils()
    from aphantasia_b200 import utils
    for frames, transit in ((40, 7), (300, 100), (9, 20), (12, 1)):
        kw = dict(uniform=uniform, cubic=cubic, start_lat=start_lat, seed=1234, verbose=False)
        a = utils.latent_anima([3], frames, transit, **kw)
        b = ref.latent_anima([3], frames, transit, **kw)
        assert a.shape == b.shape and np.array_equal(a, b), (frames, transit)


def test_latent_anima_without_a_seed_reseeds_numpys_stream_from_the_clock(monkeypatch):
    """The original reseeds NumPy's global stream from the clock; the draws that follow (the crop replay's) must continue from
    the same state. The key latents come from the OS's entropy in both, so only their shape is compared."""
    ref = _ref_utils()
    from aphantasia_b200 import utils
    monkeypatch.setattr(time, 'time', lambda: 1700000000.4321)
    a = utils.latent_anima([2], 30, 10, uniform=True, cubic=True, start_lat=[0.5, 0.5])
    after_ours = np.random.rand(5)
    b = ref.latent_anima([2], 30, 10, uniform=True, cubic=True, start_lat=[0.5, 0.5])
    after_ref = np.random.rand(5)
    assert a.shape == b.shape == (30, 2)
    assert np.array_equal(after_ours, after_ref)


def test_slerp_intrl_and_pad_up_to_equal_the_original():
    ref = _ref_utils()
    from aphantasia_b200 import utils
    g = torch.Generator().manual_seed(5)
    z1, z2 = torch.randn(1, 512, generator=g), torch.randn(1, 512, generator=g) * 3
    for kw in (dict(num_steps=7), dict(num_steps=5, smooth=0.), dict(x=0.3), dict(x=0.8, smooth=1.5)):
        assert torch.equal(utils.slerp(z1, z2, **kw), ref.slerp(z1, z2, **kw)), kw
    a, b = list(range(11)), [-v for v in range(11)]
    for step in (2, 3, 5):
        assert utils.intrl(list(a), b, step) == ref.intrl(list(a), b, step)
    x = torch.randn(1, 3, 7, 10, generator=g)
    for size, kind in (((12, 15), 'centr'), ((7, 10), 'centr'), ((30, 41), 'centr'), ((12, 15), 'side'), ((25, 9 + 31), 'symm'),
                       ((16, 17), 'side symm')):
        assert torch.equal(utils.pad_up_to(x, size, kind), ref.pad_up_to(x, size, kind)), (size, kind)
    assert torch.equal(utils.tile_pad(x, [3, 20, 9, 1], symm=True), ref.tile_pad(x, [3, 20, 9, 1], symm=True))


def test_file_list_and_save_cfg_equal_the_original(tmp_path):
    ref = _ref_utils()
    from aphantasia_b200 import utils
    for name in ('b.pt', 'a.pt', '10.jpg', '9.PNG', 'c.txt', 'sub/z.pt', 'sub/y.jpg'):
        p = tmp_path / name
        p.parent.mkdir(exist_ok=True)
        p.write_text('x')
    for args in ((), ('pt',), (['jpg', 'png'],), ('pt', True), (None, True)):
        assert utils.file_list(str(tmp_path), *args) == ref.file_list(str(tmp_path), *args), args
    a = argparse.Namespace(size=[720, 1280], in_txt='red square', lrate=0.1, invert=1., gen='RGB', depth_dir=None,
                           nested={'b': 2, 'a': {'x': [1, 2]}})
    utils.save_cfg(a, str(tmp_path / 'ours'))
    ref.save_cfg(a, str(tmp_path / 'ref'))
    utils.save_cfg(vars(a), str(tmp_path / 'ours'), 'cfg.txt')
    ref.save_cfg(vars(a), str(tmp_path / 'ref'), 'cfg.txt')
    for f in ('config.txt', 'cfg.txt'):
        assert (tmp_path / 'ours' / f).read_text() == (tmp_path / 'ref' / f).read_text()


def test_depth_stand_in_raises_with_its_reason():
    sys.path.insert(0, os.path.join(ROOT, 'dropin'))
    try:
        sys.modules.pop('depth', None); sys.modules.pop('depth.depth', None)
        from depth import depth
        assert depth.__file__.startswith(os.path.join(ROOT, 'dropin', 'depth'))
        with pytest.raises(NotImplementedError, match='Depth Anything V2'):
            depth.InferDepthAny('b')
        with pytest.raises(NotImplementedError, match='--depth 0'):
            depth.depthwarp(None, None, None, 0.5)
    finally:
        sys.path.remove(os.path.join(ROOT, 'dropin'))
        sys.modules.pop('depth', None); sys.modules.pop('depth.depth', None)


def test_motion_matrix_is_torchvisions_for_the_scripts_argument_types():
    """illustrip.py passes numpy.float64 angle and shear, a tuple of numpy scalars and a shape-(1,) array for the scale."""
    import torchvision.transforms.functional as TF
    from aphantasia_b200 import motion
    angle, shear, shift, scale = np.float64(-0.37), np.float64(0.21), np.array([3.25, -7.5]), np.array([1.0113])
    want = TF._get_inverse_affine_matrix([0., 0.], float(angle), [3.25, -7.5], 1.0113, [float(shear), 0.])
    assert motion.inverse_matrix(angle, tuple(shift), scale, shear) == want
    assert motion.inverse_matrix(30, [4, 5], 0.5, [2., 3.]) == TF._get_inverse_affine_matrix([0., 0.], 30., [4., 5.], 0.5, [2., 3.])
    assert motion.inverse_matrix(1., [0, 0], 2., [7.]) == TF._get_inverse_affine_matrix([0., 0.], 1., [0., 0.], 2., [7., 7.])


def test_motion_leaves_cpu_calls_to_torchvision():
    import torchvision.transforms.functional as TF
    from torchvision.transforms import InterpolationMode as IM
    from aphantasia_b200 import motion
    x = torch.rand(1, 3, 20, 24)
    got = motion.affine(x, np.float64(3.), (np.float64(1.), np.float64(-2.)), np.array([1.05]), np.float64(0.4), fill=0,
                        interpolation=IM.BILINEAR)
    assert torch.equal(got, motion.stock_affine(x, np.float64(3.), (np.float64(1.), np.float64(-2.)), np.array([1.05]),
                                                np.float64(0.4), fill=0, interpolation=IM.BILINEAR))
    assert motion.stock_affine is not motion.affine and TF.affine in (motion.stock_affine, motion.affine)
