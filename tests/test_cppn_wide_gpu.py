"""GPU tests of the wide CPPN nets (72 <= nf <= 256, csrc/cppn.cu: layer by layer, the hidden layers as TF32 wgmma GEMMs)
against the float64 restatement with TF32-rounded operands (tests/cppn_oracle.py).

The bars are the narrow path's (tests/test_cppn_gpu.py derives them): on the contracted nets (hidden weights x 1/4), forward
max-abs <= 1e-4 and every weight and bias gradient <= max(1e-3, 2^-10 sqrt(L - 1)) norm-wise. The wider K (up to 512 terms) only
adds fp32 accumulation error, about sqrt(K) 2^-24 relative per product, three orders below the TF32 flips the bars are sized for,
so they stay as they are. Each case prints its measured maxima.

One thing the bars cannot absorb: a `relu` layer-0 pre-activation within fp32 rounding of 0 (layer 0 runs in fp32, the
restatement in float64) takes opposite signs in the two, so relu' and with it one term of dW_0 / db_0 differ whole. With seed
nf + layers, nf 256 / 2 layers at 37x53 has one (z_0 = 6.4e-9 in float64, -5.0e-9 in fp32; dW_0 off by 3.8e-3 norm-wise, every
other gradient within 2e-5). The small-frame cases therefore draw seed 1000 + nf + layers, under which no relu case has such a
pre-activation (checked from the parameters on the CPU).
"""
import gc
import math
import os

import pytest
import torch

from test_cppn_gpu import _check, _net, _raw, mgrid

pytestmark = pytest.mark.gpu

ACTS = ('unbias', 'comp', 'relu')


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('nf', [72, 128, 200, 256])
@pytest.mark.parametrize('layers', [1, 2, 10, 32])
@pytest.mark.parametrize('HW', [(1, 1), (37, 53)])
def test_wide_cppn_against_tf32_restatement_small_frames(act, nf, layers, HW):
    _check(nf, layers, act, *HW, seed=1000 + nf + layers)


@pytest.mark.parametrize('act,nf,layers', [('unbias', 128, 2), ('comp', 72, 3), ('relu', 256, 2)])
def test_wide_cppn_against_tf32_restatement_512(act, nf, layers):
    _check(nf, layers, act, 512, 512, seed=9)


def test_wide_cppn_batch_of_two_frames_matches_each_frame_alone():
    net = _net(200, 10, 'unbias', 4, 0.25)
    coords = mgrid(45, 67, 2).cuda()
    gout = torch.randn(2, 3, 45, 67, generator=torch.Generator().manual_seed(3)).cuda()
    out, grads = _raw(net, coords, gout)
    outs, gsum = [], None
    for n in range(2):
        o, g = _raw(net, coords[n:n + 1].contiguous(), gout[n:n + 1].contiguous())
        outs.append(o)
        gsum = g if gsum is None else [a + b for a, b in zip(gsum, g)]
    assert float((out - torch.cat(outs)).abs().max()) <= 1e-4
    for a, b in zip(grads, gsum):
        assert float((a - b).norm()) <= 1e-3 * max(float(b.norm()), 1e-30)
    _check(200, 10, 'unbias', 45, 67, N=2, seed=4)


def test_module_forward_backward_and_preview_at_nf_256():
    """CPPN(2, 256, 10, 3) through autograd gives the C entry points' values; under no_grad it returns a PreviewTensor."""
    from aphantasia_b200.utils import PreviewTensor
    net = _net(256, 10, 'unbias', 11)
    coords = mgrid(64, 80).cuda()
    gout = torch.randn(1, 3, 64, 80, generator=torch.Generator().manual_seed(2)).cuda()
    out = net(coords)
    (out * gout).sum().backward()
    raw_out, raw_grads = _raw(net, coords, gout)
    assert torch.equal(out.detach(), raw_out)
    for p, g in zip(net._params(), raw_grads):
        assert torch.equal(p.grad, g)
    with torch.no_grad():
        prev = net(coords)
    assert isinstance(prev, PreviewTensor) and torch.equal(prev.as_subclass(torch.Tensor), raw_out)


def test_unsupported_nets_raise_and_launch_nothing():
    from aphantasia_b200._lib import lib
    from aphantasia_b200.cppn import CPPN
    before = lib().aph_launch_count()
    for nf in (264, 100):
        with pytest.raises(NotImplementedError, match=r'multiple of 8 in \[8, 256\]'):
            CPPN(2, nf, 10, 3)
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        CPPN(2, 20, 10, 3)
    with pytest.raises(NotImplementedError, match=r'layers = 33'):
        CPPN(2, 256, 33, 3)
    assert lib().aph_launch_count() == before


def _launches(fn):
    from aphantasia_b200._lib import lib
    torch.cuda.synchronize()
    before = lib().aph_launch_count()
    fn()
    torch.cuda.synchronize()
    return lib().aph_launch_count() - before


def test_nf_64_still_runs_the_narrow_kernels():
    """nf 64: one launch forward, two backward (k_cppn_fwd; k_cppn_bwd + k_cppn_reduce). nf 72: layers + 2 forward."""
    coords = mgrid(32, 48).cuda()
    gout = torch.randn(1, 3, 32, 48, device='cuda')
    net = _net(64, 10, 'unbias', 1)
    _raw(net, coords, gout)                       # warm the scratch
    assert _launches(lambda: _raw(net, coords)) == 1
    assert _launches(lambda: _raw(net, coords, gout)) == 1 + 2
    wide = _net(72, 10, 'unbias', 1)
    assert _launches(lambda: _raw(wide, coords)) == 10 + 2


def _wide_bytes(nf, L, act, P, bwd):
    """the handle's bytes as include/aphb200.h states them"""
    kh = nf if act == 'relu' else 2 * nf
    chunk = max(4096, math.ceil(math.ceil(P / 256) / 128) * 128)
    S = math.ceil(P / chunk)
    Pp = S * chunk
    R = Pp // 16
    khp = math.ceil(kh / (128 if kh <= 128 else 256)) * (128 if kh <= 128 else 256)
    Q = 3 * kh + 8 + nf
    F = 2 * Pp * kh + (L - 1) * nf * kh
    if bwd:
        F += (L - 1) * nf * kh + L * nf * Pp + khp * Pp + nf * Pp + max(R * Q, S * nf * kh) + 2 * math.ceil(R / 256) * Q
    return 4 * F


def test_handle_bytes_follow_the_documented_formula_and_come_back_on_destroy():
    from aphantasia_b200._lib import lib
    gc.collect()
    gc.disable()
    try:
        torch.cuda.synchronize()
        start = lib().aph_device_bytes()
        net = _net(256, 10, 'unbias', 2)
        assert lib().aph_cppn_bytes(net._handle) == 0
        for (N, H, W) in ((1, 37, 53), (2, 300, 400)):
            coords = mgrid(H, W, N).cuda()
            _raw(net, coords)
            assert lib().aph_cppn_bytes(net._handle) == _wide_bytes(256, 10, 'unbias', N * H * W, False)
            _raw(net, coords, torch.randn(N, 3, H, W, device='cuda'))
            assert lib().aph_cppn_bytes(net._handle) == _wide_bytes(256, 10, 'unbias', N * H * W, True)
        torch.cuda.synchronize()
        assert lib().aph_device_bytes() - start == lib().aph_cppn_bytes(net._handle)
        net._handle.close()
        torch.cuda.synchronize()
        assert lib().aph_device_bytes() == start
    finally:
        gc.enable()


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPPN_PY = os.path.join(ROOT, 'oracle', '_ref', 'cppn.py')
needs_script = pytest.mark.skipif(not (os.path.isfile(CPPN_PY) and os.path.isfile(os.path.join(ROOT, 'oracle', '_ref', 'shader_expo.py'))),
                                  reason='no copy of the original cppn.py / shader_expo.py: build() stages them into oracle/_ref/')


@needs_script
def test_unmodified_script_at_nf_256_and_shader_export(tmp_path):
    """python -m aphantasia_b200.run cppn.py --nf 256 trains, writes its frames and snapshots; -r <snapshot> -ex exports from it."""
    from test_real_script_cppn import SHADERS, _check_outputs, _run
    r, tr = _run(tmp_path, ['-t', 'red square', '--nf', '256', '-s', '256-256', '--steps', '3', '--samples', '4'])
    base = str(tmp_path / 'out' / 'cppn' / 'red_square-l10-n256')
    _check_outputs(base, 3)
    assert tr['cppn_calls'] == 6 and tr['encode_image_calls'] == 3
    os.makedirs(str(tmp_path / 'exp'))
    exp = str(tmp_path / 'exp' / 'snap.npy')
    os.replace(os.path.join(base, '0002.npy'), exp)
    r, tr = _run(tmp_path, ['-r', exp, '-ex', '-s', '256-256'])
    for sfx in SHADERS + ('.jpg',):
        assert os.path.getsize(exp[:-4] + sfx) > 0, sfx
    assert tr['cppn_calls'] == 1 and tr['encode_image_calls'] == 0
