"""GPU tests of the CPPN generator (csrc/cppn.cu) against the float64 restatement with TF32-rounded operands
(tests/cppn_oracle.py), and of derivat(img, mode='sobel') (csrc/loss.cu).

Rounding model behind the bars. Kernel and restatement round the same fp32 operands to TF32 for the hidden layers' products, so
what remains is (i) fp32 accumulation over K <= 128 terms and the fp32 activations (atanf / expf within 2 ulp): about 1e-6
relative per layer; (ii) the rare operand whose fp32 value lands on the other side of a TF32 rounding boundary in the two
computations (probability about a few 2^-24 / 2^-10, i.e. 1e-4, per activation operand; the weights are the same fp32 values in
both and round alike), which moves one product term by one TF32 ulp (2^-10 relative, up to about 4e-3 of a |w x| <= 4) in that
pixel. (ii) then propagates through the remaining layers with the network's gain.

The seeded networks of cppn.py are chaotic at depth: their gain per layer exceeds 1, so TF32 itself moves the output of a
32-layer `unbias` net by up to 0.8 from plain float64, and one flip in an early layer moves a pixel by as much. Bars on such a
pixel would bound the chaos, not the kernel. So:
  * the strict bars apply to the same networks with the hidden layers' weights scaled by 1/4 (gain below 1): forward max-abs
    <= 1e-4, as a flip then stays within a few 1e-5 at the output (sigmoid slope <= 1/4 times the output weights). The backward
    is linear in dz, so a flip in it keeps its relative size (2^-10) in every layer below, and each of the L - 1 TF32 layers the
    signal crosses can add one: each weight and bias gradient <= max(1e-3, 2^-10 sqrt(L - 1)) norm-wise (measured first against
    a flat 1e-3, which 32-layer nets exceeded at up to 3.5e-3);
  * the seeded default networks (nf 24, 10 layers) are compared by the share of output elements off by more than 1e-4: with
    432 activation operands per pixel, about 5 % of the pixels see a flip; the bar is 10 %.
The distance from plain float64 (no TF32 rounding) is printed, not asserted.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import cppn_oracle as O

pytestmark = pytest.mark.gpu

ACTS = ('unbias', 'comp', 'relu')


def mgrid(H, W, N=1):
    """cppn.py's get_mgrid: channel 0 runs along W, channel 1 along H, np.linspace in float64, then fp32."""
    xs, ys = np.linspace(-1, 1, num=W), np.linspace(-1, 1, num=H)
    g = np.stack(np.meshgrid(xs, ys), axis=0)[None].astype(np.float32)
    if N > 1:
        g = np.concatenate([g * (1. - 0.1 * n) for n in range(N)], 0).astype(np.float32)
    return torch.from_numpy(g)


def _net(nf, layers, act, seed=0, hidden_scale=1.):
    from aphantasia_b200.cppn import CPPN
    torch.manual_seed(seed)
    net = CPPN(2, nf, layers, 3, act_fn=act)
    with torch.no_grad():
        for layer in net.net[1:-1]:
            layer.conv.weight.mul_(hidden_scale)
    return net.cuda()


def _raw(net, coords, gout=None):
    """The C entry points on NaN-filled outputs: (out, [dparams] or None)."""
    from aphantasia_b200._lib import check, lib, stream_ptr
    params = net._params()
    ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
    N, _, H, W = coords.shape
    out = torch.full((N, 3, H, W), float('nan'), device='cuda')
    check(lib().aph_cppn_fwd(net._handle, coords.data_ptr(), N, H, W, ptrs, out.data_ptr(), stream_ptr()), 'aph_cppn_fwd')
    grads = None
    if gout is not None:
        grads = [torch.full_like(p, float('nan')) for p in params]
        gp = (C.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        check(lib().aph_cppn_bwd(net._handle, coords.data_ptr(), N, H, W, ptrs, gout.data_ptr(), gp, stream_ptr()), 'aph_cppn_bwd')
    torch.cuda.synchronize()
    return out, grads


def _check(nf, layers, act, H, W, N=1, seed=0, seeded_init=False):
    """Strict bars on the contracted net (hidden weights x 1/4); seeded_init=True: the script's own init, share-of-pixels bar."""
    net = _net(nf, layers, act, seed, 1. if seeded_init else 0.25)
    coords = mgrid(H, W, N).cuda()
    g = torch.Generator().manual_seed(seed + 1)
    gout = torch.randn(N, 3, H, W, generator=g).cuda()
    out, grads = _raw(net, coords, gout)
    _, grads2 = _raw(net, coords, gout)
    assert torch.isfinite(out).all(), 'an output element was not written or is not finite'
    params = [p.detach().cpu().numpy() for p in net._params()]
    c64 = coords.cpu().numpy()
    ref, cache = O.forward(c64, params, act, tf32_ops=True)
    d = np.abs(out.cpu().numpy() - ref)
    err, share = float(d.max()), float((d > 1e-4).mean())
    plain, _ = O.forward(c64, params, act, tf32_ops=False)
    want = O.backward(cache, gout.cpu().numpy())
    rels = []
    for k, (a, b, w) in enumerate(zip(grads, grads2, want)):
        assert torch.equal(a, b), 'gradient %d differs between two backward calls' % k
        a = a.cpu().numpy().reshape(w.shape).astype(np.float64)
        assert np.isfinite(a).all()
        rels.append(np.linalg.norm(a - w) / max(np.linalg.norm(w), 1e-30))
    print('cppn nf %d layers %d %s %dx%dx%d %s: forward max-abs %.2e (share > 1e-4: %.4f) vs TF32 restatement, %.2e vs plain float64; '
          'worst gradient %.2e norm-wise' % (nf, layers, act, N, H, W, 'seeded' if seeded_init else 'contracted', err, share,
                                             float(np.abs(out.cpu().numpy() - plain).max()), max(rels)))
    if seeded_init:
        assert share <= 0.1
    else:
        assert err <= 1e-4
        assert max(rels) <= max(1e-3, 2. ** -10 * np.sqrt(layers - 1)), rels


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('nf', [8, 24, 64])
@pytest.mark.parametrize('layers', [1, 2, 10, 32])
@pytest.mark.parametrize('HW', [(1, 1), (37, 53)])
def test_cppn_against_tf32_restatement_small_frames(act, nf, layers, HW):
    _check(nf, layers, act, *HW, seed=nf + layers)


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('HW', [(512, 512), (720, 1280)])
def test_cppn_against_tf32_restatement_full_frames(act, HW):
    _check(24, 10, act, *HW, seed=3)


@pytest.mark.parametrize('act', ACTS)
def test_cppn_seeded_default_net_share_of_flipped_pixels(act):
    _check(24, 10, act, 512, 512, seed=3, seeded_init=True)


def test_cppn_batch_of_two_frames_and_the_largest_net():
    _check(64, 32, 'unbias', 67, 45, N=2, seed=5)
    _check(64, 10, 'comp', 128, 96, N=1, seed=6)     # z_l beyond the shared-memory budget: the scratch path


def test_module_forward_backward_and_preview():
    """CPPN.forward through autograd gives the C entry points' values; under no_grad it returns a PreviewTensor."""
    from aphantasia_b200.utils import PreviewTensor
    net = _net(24, 10, 'unbias', 11)
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
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        CPPN(2, 20, 10, 3)
    with pytest.raises(NotImplementedError, match=r'layers = 33'):
        CPPN(2, 24, 33, 3)
    assert lib().aph_launch_count() == before


@pytest.mark.parametrize('shape', [(1, 3, 37, 53), (2, 3, 64, 64), (1, 3, 1, 1), (1, 1, 2, 7)])
def test_sobel_derivat_against_unpinned_restatement(shape):
    from aphantasia_b200.utils import derivat
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=g).cuda().requires_grad_(True)
    v = derivat(x, mode='sobel')
    (v * 0.7).backward()
    rv, rg = O.sobel_derivat(x.detach().cpu().numpy(), 0.7)
    assert abs(v.item() - rv) <= 1e-5 * max(abs(rv), 1e-30) or rv == 0.
    gg = x.grad.cpu().numpy()
    assert np.linalg.norm(gg - rg) <= 1e-5 * max(np.linalg.norm(rg), 1e-30) or not rg.any()


def test_sobel_derivat_of_a_constant_image_is_zero():
    from aphantasia_b200.utils import derivat
    x = torch.full((1, 3, 40, 30), 0.37, device='cuda', requires_grad=True)
    v = derivat(x, mode='sobel')
    v.backward()
    assert v.item() == 0. and not x.grad.any()
    with pytest.raises(NotImplementedError, match='scharr'):
        derivat(x, mode='scharr')
