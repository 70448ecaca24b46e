"""CPU tests of transforms_custom / transforms_elastic: the host replay of their random draws (Python specification and native),
the CPU restatement against the reference's fixtures (tests/golden/reference_golden_transforms.npz, written by
make_golden_transforms.py from the real reference), the rotation convention against OpenCV, and the C-ABI surface."""
import os
import re

import numpy as np
import pytest
import torch

from aphantasia_b200 import _rng

import kornia_oracle as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_golden_transforms.npz'))
CASES = sorted({k[len('trf_'):-len('_table')] for k in G.files if k.startswith('trf_') and k.endswith('_table')})
VALUES = sorted({k[len('val_'):-len('_out')] for k in G.files if k.startswith('val_') and k.endswith('_out')})
# every field the reference fixes directly: offsets, size, flags, erase rectangle, angle, jitter shift
EXACT = [_rng.F_OFFY, _rng.F_OFFX, _rng.F_CSIZE, _rng.F_FLAGS, _rng.F_ER_I, _rng.F_ER_J, _rng.F_ER_H, _rng.F_ER_W, _rng.F_ANGLE,
         _rng.F_JIT_DX, _rng.F_JIT_DY]


def _replay(name, mode):
    H, W, cnt, size, kind, macro, s = G['trf_%s_cfg' % name]
    torch.manual_seed(int(s)); np.random.seed(int(s))
    if mode == 'py':
        tabs, _ = _rng.draw_crop_table_py(int(cnt), (int(H), int(W)), int(size), int(kind), str(G['trf_%s_align' % name]), float(macro))
    else:
        _rng._NP_INPLACE = False if mode == 'native_copy' else None
        try:
            tabs, _ = _rng.draw_crop_table_native(int(cnt), (int(H), int(W)), int(size), int(kind), str(G['trf_%s_align' % name]), float(macro))
        finally:
            _rng._NP_INPLACE = None
    _, key, pos = np.random.get_state()[:3]
    return tabs[0], torch.get_rng_state().numpy(), np.append(np.asarray(key, np.int64), pos)


@pytest.mark.parametrize('mode', ['py', 'native', 'native_copy'])
@pytest.mark.parametrize('name', CASES)
def test_replay_reproduces_reference_tables_and_generator_states(name, mode):
    tab, tstate, nstate = _replay(name, mode)
    ref = G['trf_%s_table' % name]
    assert tab.shape == ref.shape
    np.testing.assert_array_equal(tab[:, EXACT], ref[:, EXACT])
    # the inverse of the rotation matrix the reference passes to warp_affine (its stub records the angle)
    want = np.array([_rng.kornia_inverse_rotation(a) for a in ref[:, _rng.F_ANGLE]], np.float32)
    np.testing.assert_array_equal(tab[:, _rng.F_ROT:_rng.F_ROT + 4], want)
    np.testing.assert_array_equal(tstate, G['trf_%s_torch_after' % name])
    np.testing.assert_array_equal(nstate, G['trf_%s_np_after' % name])


def test_fixture_cases_exercise_every_branch():
    extra = {n: G['trf_%s_extra' % n] for n in CASES}
    flags = np.concatenate([G['trf_%s_table' % n][:, _rng.F_FLAGS].astype(int) for n in CASES])
    assert ((flags & _rng.FLAG_ERASE) > 0).sum() >= 10 and ((flags & _rng.FLAG_ELASTIC) > 0).sum() >= 100
    tabs = np.concatenate([G['trf_%s_table' % n] for n in CASES])
    assert set(np.unique(tabs[:, _rng.F_JIT_DX])) == set(range(8)) and set(np.unique(tabs[:, _rng.F_JIT_DY])) == set(range(8))
    assert (tabs[:, _rng.F_ANGLE] == 0).sum() > 0 and (tabs[:, _rng.F_ANGLE] != 0).sum() > 0
    for n in CASES:
        size = int(G['trf_%s_cfg' % n][3])
        e = extra[n]
        assert np.all(e[:, 0:2] == (size + 7) / 2) and np.all(e[:, 9] == size + 8)     # rotation centre (s - 1) / 2, dsize s
        el = G['trf_%s_table' % n][:, _rng.F_FLAGS].astype(int) & _rng.FLAG_ELASTIC > 0
        assert np.all(e[el, 8] == 0)                                                    # the reference passes zero noise
        assert np.all((e[el, 2] >= 17) & (e[el, 2] <= 127) & (e[el, 2] % 2 == 1))         # k = randint(8, 64) * 2 + 1


def test_fast_tables_unchanged():
    """The RandomErasing draw is shared with the new kinds: transforms_fast must draw exactly what the reference drew."""
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_golden.npz'))
    for name in ('c2', 'c1', 'central', 'small'):
        H, W, cnt, size, kind, macro, s = g['rng_%s_cfg' % name]
        for fn in (_rng.draw_crop_table_py, _rng.draw_crop_table_native):
            torch.manual_seed(int(s)); np.random.seed(int(s))
            tabs, _ = fn(int(cnt), (int(H), int(W)), int(size), int(kind), str(g['rng_%s_align' % name]), float(macro))
            after = np.array([torch.rand(1).item(), float(np.random.rand())])
            ref = g['rng_%s_table' % name]
            np.testing.assert_array_equal(tabs[0][:, :4], ref[:, :4])
            np.testing.assert_array_equal(tabs[0][:, 12:16], ref[:, 12:16])                 # the shared RandomErasing draw
            np.testing.assert_allclose(tabs[0][:, 4:12], ref[:, 4:12], atol=1e-4)           # float32 perspective solve
            np.testing.assert_allclose(tabs[0][:, 16:21], ref[:, 16:21], atol=1e-6)
            np.testing.assert_array_equal(after, g['rng_%s_after' % name])


@pytest.mark.parametrize('name', VALUES)
def test_oracle_reproduces_reference_values(name):
    H, W, cnt, size, kind, macro, s = G['val_%s_cfg' % name]
    size, kind = int(size), int(kind)
    canvas = torch.from_numpy(G['val_%s_canvas' % name].astype(np.float32))
    torch.manual_seed(int(s)); np.random.seed(int(s))
    tabs, frame = _rng.draw_crop_table_py(int(cnt), (int(H), int(W)), size, kind, str(G['val_%s_align' % name]), float(macro))
    tab = tabs[0]
    params = G['val_%s_params' % name]
    np.testing.assert_array_equal(tab[:, EXACT[3:]], params[:, EXACT[3:]])
    # pad + erase: the input of the reference's warp_affine, crop by crop
    framed = KO.R.wrap_pad(canvas, frame)
    warp_in = []
    for row in tab:
        oy, ox, cs = int(row[_rng.F_OFFY]), int(row[_rng.F_OFFX]), int(row[_rng.F_CSIZE])
        cut = torch.nn.functional.interpolate(framed[:, :, oy:oy + cs, ox:ox + cs], (size, size), mode='bicubic', align_corners=True)
        warp_in.append(KO.pad_erase(cut, row, kind == 4))
    np.testing.assert_array_equal(torch.cat(warp_in).numpy(), G['val_%s_warp_in' % name])
    out = KO.sample_crops(canvas, tab, size, kind, frame)
    assert out.shape == (int(cnt), 3, size + 8, size + 8)
    np.testing.assert_allclose(out.numpy(), G['val_%s_out' % name], atol=2e-6, rtol=0)


def test_restated_rotation_matches_opencv():
    cv2 = pytest.importorskip('cv2')
    s = 232
    c = (s - 1) / 2
    yy, xx = np.meshgrid(np.arange(s), np.arange(s), indexing='ij')
    img = (np.sin(xx / 17.) * np.cos(yy / 23.) + 0.1 * xx / s).astype(np.float32)
    for angle in (-30, -7, 0, 13, 29):
        M = cv2.getRotationMatrix2D((c, c), angle, 1.0)
        want = cv2.warpAffine(img, M, (s, s), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        Mi = cv2.invertAffineTransform(M)
        sx = Mi[0, 0] * xx + Mi[0, 1] * yy + Mi[0, 2]; sy = Mi[1, 0] * xx + Mi[1, 1] * yy + Mi[1, 2]
        inner = (np.abs(sx - c) < c - 2) & (np.abs(sy - c) < c - 2)
        got = KO.warp_affine(torch.from_numpy(img)[None, None], KO.kornia_rotation_matrix(angle, c))[0, 0].numpy()
        assert np.abs(got - want)[inner].max() < 2e-3, angle
        # the table's pixel-space inverse is the same map
        r = _rng.kornia_inverse_rotation(angle)
        np.testing.assert_allclose(c + r[0] * (xx - c) + r[1] * (yy - c), sx, atol=1e-9)
        np.testing.assert_allclose(c + r[2] * (xx - c) + r[3] * (yy - c), sy, atol=1e-9)
        if angle != 0:       # the opposite sign is far off
            wrong = KO.warp_affine(torch.from_numpy(img)[None, None], KO.kornia_rotation_matrix(-angle, c))[0, 0].numpy()
            assert np.abs(wrong - want)[inner].max() > 0.1, angle


def test_elastic_zero_noise_is_the_stretch():
    s = 40
    img = torch.rand(1, 1, s, s, dtype=torch.float64).float()
    out = KO.elastic_zero_noise(img)[0, 0].double()
    j = np.arange(s); src = j * s / (s - 1) - 0.5
    x0 = np.floor(src).astype(int); t = src - x0
    Wm = np.zeros((s, s))
    for k in range(s):
        if 0 <= x0[k] < s: Wm[k, x0[k]] += 1 - t[k]
        if 0 <= x0[k] + 1 < s: Wm[k, x0[k] + 1] += t[k]
    np.testing.assert_allclose(out.numpy(), Wm @ img[0, 0].double().numpy() @ Wm.T, atol=1e-5)
    assert float((out - img[0, 0]).abs().max()) > 0.1           # not an identity


def test_header_exports_and_bindings_for_the_new_kinds():
    from aphantasia_b200 import _lib, transforms
    hdr = open(os.path.join(ROOT, 'include', 'aphb200.h')).read()
    get = lambda n: int(re.search(r'#define %s\s+(\d+)' % n, hdr).group(1))
    assert (get('APH_TF_CUSTOM'), get('APH_TF_ELASTIC')) == (_rng.TF_CUSTOM, _rng.TF_ELASTIC) == (3, 4)
    assert (get('APH_F_JIT_DX'), get('APH_F_JIT_DY')) == (_rng.F_JIT_DX, _rng.F_JIT_DY) == (21, 22)
    assert (get('APH_FLAG_JITTER'), get('APH_FLAG_ELASTIC')) == (_rng.FLAG_JITTER, _rng.FLAG_ELASTIC)
    for name in ('aph_vit_fwd_sized', 'aph_vit_bwd_sized'):
        assert re.search(r'\b%s\s*\(' % name, hdr) and name in _lib.EXPORTS and hasattr(_lib.lib(), name)
    assert transforms.transforms_custom.kind == _rng.TF_CUSTOM and transforms.transforms_elastic.kind == _rng.TF_ELASTIC
    assert _rng.out_side(224, _rng.TF_CUSTOM) == _rng.out_side(224, _rng.TF_ELASTIC) == 232 and _rng.out_side(224, _rng.TF_FAST) == 224
    with pytest.raises(NotImplementedError):
        transforms.transforms_lucent(torch.zeros(1, 3, 8, 8))


def test_patchlink_accepts_the_window_only_when_asked():
    from aphantasia_b200 import _patchlink

    class Vis:
        input_resolution, patch_size = 224, 32
    v = Vis()
    saved = list(_patchlink._consumers)
    for x in saved:
        _patchlink._consumers.discard(x)
    try:
        _patchlink.register(v)
        assert _patchlink.target(224) is v and _patchlink.target(232) is None
        assert _patchlink.target(232, windowed=True) is v and _patchlink.target(255, windowed=True) is v
        assert _patchlink.target(256, windowed=True) is None and _patchlink.target(223, windowed=True) is None
    finally:
        _patchlink._consumers.discard(v)
        for x in saved:
            _patchlink.register(x)
