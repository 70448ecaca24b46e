"""GPU tests of the LPIPS kernels (csrc/lpips.cu, csrc/conv_tc.cuh) against float64.

Bars. Each kernel is compared with float64 computed from the SAME bf16-rounded inputs and weights, so what remains is the fp32
accumulation and the bf16 rounding of the stored output: one rounding of 2^-9 relative per element, 2e-3 norm-wise at most.
The layer bars are 6e-3 norm-wise (three times that).

The whole LPIPS value is held to the project's bf16-path bar of 2e-2 norm-wise against the float64 restatement. The canvas
gradient cannot meet that bar: a bf16 activation moves the argmax of a few max-pool windows (0.2 % of the relu1_2 windows up
to 1.2 % of the relu4_3 ones, for the synthetic weights at 64 x 64), and each move sends a whole window's gradient to another
pixel. Emulated on the CPU in float64, those roundings alone put the canvas gradient 5.2 % (norm-wise) from float64 at 64 x 64,
and the CUDA result is 5.2 % from it too. So the gradient is checked twice:
  - against the restatement run with the CUDA path's rounding model (lpips_oracle.lpips(bf16=True): bf16 weights, activations
    and activation gradients), bar 5e-2. Measured on an H100: 2.0 % to 4.0 % over these cases. The remainder comes from fp32
    accumulation crossing a bf16 rounding boundary where float64 does not, which moves a few more argmaxes;
  - against plain float64, bar 1.5e-1: a bound on the bf16 design rather than on the kernels.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from aphantasia_b200 import _lib
from aphantasia_b200 import lpips as L
import lpips_oracle as O

pytestmark = pytest.mark.gpu


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _nhwc(x):                 # NCHW -> bf16 NHWC contiguous
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def _nchw(x):
    return x.permute(0, 3, 1, 2).double()


@pytest.mark.parametrize('cin, cout', [(64, 64), (64, 128), (256, 256), (512, 512)])
@pytest.mark.parametrize('h, w', [(7, 9), (45, 80), (22, 40)])
def test_conv_layer_fwd_and_data_gradient(cin, cout, h, w):
    """One 3x3 layer, forward (bias + ReLU) and data gradient (with and without the ReLU-mask select), against float64 from
    the same bf16 operands. Sizes are not multiples of the 8 x 16 pixel tile. Outputs are pre-filled with NaN: every element
    must be written and finite. Bar 6e-3 norm-wise (module docstring)."""
    torch.manual_seed(cin + cout + h)
    N = 2
    x = torch.randn(N, cin, h, w, device='cuda').bfloat16()
    wt = (torch.randn(cout, cin, 3, 3, device='cuda') * (2.0 / (9 * cin)) ** 0.5)
    wb = wt.bfloat16().double()
    bias = torch.randn(cout, device='cuda') * 0.1
    out = torch.full((N, h, w, cout), float('nan'), device='cuda', dtype=torch.bfloat16)
    xh = _nhwc(x)                 # operands are held in names: a temporary's memory could be handed to the next one
    _lib.check(_lib.lib().aph_lpips_conv_test(1, xh.data_ptr(), wt.data_ptr(), bias.data_ptr(), None, out.data_ptr(),
                                              N, h, w, cin, cout, _st()), 'conv fwd')
    ref = F.relu(F.conv2d(x.double(), wb, bias.double(), padding=1))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert _rel(_nchw(out), ref) < 6e-3

    dy = torch.randn(N, cout, h, w, device='cuda').bfloat16()
    mask = torch.randn(N, cin, h, w, device='cuda').bfloat16()
    dx_ref = torch.nn.grad.conv2d_input((N, cin, h, w), wb, dy.double(), padding=1)
    dyh, mh = _nhwc(dy), _nhwc(mask)
    for m in (None, mask):
        dx = torch.full((N, h, w, cin), float('nan'), device='cuda', dtype=torch.bfloat16)
        _lib.check(_lib.lib().aph_lpips_conv_test(0, dyh.data_ptr(), wt.data_ptr(), None, None if m is None else mh.data_ptr(),
                                                  dx.data_ptr(), N, h, w, cin, cout, _st()), 'conv bwd')
        want = dx_ref if m is None else torch.where(m.double() > 0, dx_ref, torch.zeros_like(dx_ref))
        torch.cuda.synchronize()
        assert torch.isfinite(dx).all()
        assert _rel(_nchw(dx), want) < 6e-3
        if m is not None:
            assert (_nchw(dx)[m.double() <= 0] == 0).all()


@pytest.mark.parametrize('h, w', [(7, 9), (33, 50)])
def test_conv1_1_fwd_and_canvas_gradient(h, w):
    """conv1_1 in fp32 with the input scaling (normalize=True): forward against float64 (only the bf16 store rounds: 6e-3), and
    the canvas gradient from a bf16 dz against float64 of the same dz (fp32 only: 1e-5)."""
    torch.manual_seed(h)
    N = 2
    img = torch.rand(N, 3, h, w, device='cuda')
    wt = torch.randn(64, 3, 3, 3, device='cuda') * 0.3
    bias = torch.randn(64, device='cuda') * 0.1
    out = torch.full((N, h, w, 64), float('nan'), device='cuda', dtype=torch.bfloat16)
    _lib.check(_lib.lib().aph_lpips_conv0_test(1, img.data_ptr(), wt.data_ptr(), bias.data_ptr(), out.data_ptr(), N, h, w, 1, _st()), 'conv0')
    shift = torch.tensor(O.SHIFT, device='cuda', dtype=torch.float64).view(1, 3, 1, 1)
    scale = torch.tensor(O.SCALE, device='cuda', dtype=torch.float64).view(1, 3, 1, 1)
    xi = ((2 * img.double() - 1) - shift) / scale
    ref = F.relu(F.conv2d(xi, wt.double(), bias.double(), padding=1))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and _rel(_nchw(out), ref) < 6e-3
    dz = torch.randn(N, 64, h, w, device='cuda').bfloat16()
    g = torch.full((N, 3, h, w), float('nan'), device='cuda')
    dzh = _nhwc(dz)
    _lib.check(_lib.lib().aph_lpips_conv0_test(0, dzh.data_ptr(), wt.data_ptr(), None, g.data_ptr(), N, h, w, 1, _st()), 'conv0 bwd')
    gref = torch.nn.grad.conv2d_input((N, 3, h, w), wt.double(), dz.double(), padding=1) * 2 / scale
    torch.cuda.synchronize()
    assert torch.isfinite(g).all() and _rel(g, gref) < 1e-5


@pytest.mark.parametrize('h, w', [(7, 9), (22, 40), (45, 80)])
def test_max_pool_and_adjoint(h, w):
    """2x2 max-pool (floor) and its adjoint against torch.max_pool2d's, exactly (no arithmetic). Values are drawn from a few
    levels so that ties occur: the first element of the window wins, as in torch. Dropped rows / columns get exactly zero."""
    torch.manual_seed(w)
    N, C = 2, 64
    x = torch.randint(0, 3, (N, C, h, w), device='cuda').float().bfloat16()
    out = torch.empty(N, h // 2, w // 2, C, device='cuda', dtype=torch.bfloat16)
    xh = _nhwc(x)
    _lib.check(_lib.lib().aph_lpips_pool_test(1, xh.data_ptr(), None, out.data_ptr(), N, h, w, C, _st()), 'pool')
    xd = x.double().requires_grad_(True)
    ref = F.max_pool2d(xd, 2, 2)
    dy = torch.randn(N, C, h // 2, w // 2, device='cuda').bfloat16()
    gref, = torch.autograd.grad(ref, xd, dy.double())
    dx = torch.full((N, h, w, C), float('nan'), device='cuda', dtype=torch.bfloat16)
    dyh = _nhwc(dy)
    _lib.check(_lib.lib().aph_lpips_pool_test(0, xh.data_ptr(), dyh.data_ptr(), dx.data_ptr(), N, h, w, C, _st()), 'pool adj')
    torch.cuda.synchronize()
    assert torch.equal(_nchw(out), ref.detach())
    assert torch.equal(_nchw(dx), gref)
    if h % 2:
        assert (_nchw(dx)[:, :, -1, :] == 0).all()
    if w % 2:
        assert (_nchw(dx)[:, :, :, -1] == 0).all()


def _perturbed(seed):
    sd = L.synthetic_vgg_state_dict()
    g = torch.Generator().manual_seed(seed)
    for k in sd:
        sd[k] = 0.05 * torch.randn(sd[k].shape, generator=g) if k.endswith('.bias') else sd[k] * (1 + 0.3 * torch.randn(sd[k].shape, generator=g))
    lin = {k: v * (0.5 + torch.rand(v.shape, generator=g)) for k, v in L.synthetic_lin_state_dict().items()}
    return sd, lin


def _check_against_oracle(m, vgg, lin, in0, in1, plain_gbar=1.5e-1):
    """Bars in the module docstring: 2e-2 for the value; 5e-2 for the gradient against the rounding model, 1.5e-1 against plain
    float64."""
    x = in0.clone().requires_grad_(True)
    v = m(x, in1, normalize=True)
    up = torch.linspace(0.5, 1.5, in0.shape[0], device='cuda').view(-1, 1, 1, 1)
    g, = torch.autograd.grad(v, x, up)
    assert v.shape == (in0.shape[0], 1, 1, 1) and torch.isfinite(g).all()
    for bf16, gbar in ((True, 5e-2), (False, plain_gbar)):
        xd = in0.double().clone().requires_grad_(True)
        vr = O.lpips(xd, in1.double(), vgg, lin, bf16=bf16)
        gr, = torch.autograd.grad(vr, xd, up.double())
        assert _rel(v.detach(), vr.detach()) < 2e-2, (bf16, v.flatten().tolist(), vr.flatten().tolist())
        assert _rel(g, gr) < gbar, (bf16, _rel(g, gr))
    return v, g


@pytest.mark.parametrize('h, w', [(64, 64), (45, 70), (360, 640)])
@pytest.mark.parametrize('weights', ['synthetic', 'perturbed'])
def test_lpips_against_oracle(h, w, weights):
    """The whole LPIPS, value and canvas gradient (per-sample upstream gradients), against float64 (bars: module docstring)."""
    vgg, lin = (L.synthetic_vgg_state_dict(), L.synthetic_lin_state_dict()) if weights == 'synthetic' else _perturbed(11)
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    torch.manual_seed(h + w)
    N = 1 if h > 100 else 2
    in1 = torch.rand(N, 3, h, w, device='cuda')
    in0 = (in1 + 0.3 * torch.randn_like(in1)).clamp(0, 1)
    _check_against_oracle(m, vgg, lin, in0, in1)


def test_lpips_fp64_inputs():
    """fp64 inputs (the script's img_in is float64 before .float()) give an fp64 value and gradient equal to the fp32 run's."""
    vgg, lin = _perturbed(2)
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    torch.manual_seed(0)
    a, b = torch.rand(1, 3, 48, 40, device='cuda', dtype=torch.float64), torch.rand(1, 3, 48, 40, device='cuda', dtype=torch.float64)
    x = a.clone().requires_grad_(True)
    v = m(x, b, normalize=True)
    g, = torch.autograd.grad(v.sum(), x)
    assert v.dtype == torch.float64 and g.dtype == torch.float64
    x32 = a.float().requires_grad_(True)
    v32 = m(x32, b.float(), normalize=True)
    g32, = torch.autograd.grad(v32.sum(), x32)
    assert torch.equal(v.float(), v32) and torch.equal(g.float(), g32)


def test_zero_norm_pixels():
    """A flat image region under a negative conv1_2 bias leaves whole relu1_2 pixels at zero, where the norm's derivative is
    singular. The canvas gradient is finite and matches the oracle's (whose ReLU select removes the NaN) within the rounding-model
    bar. Against plain float64 the bar is 3e-1 (measured 22.9 % on an H100): around the flat region many pre-activations sit near
    zero, and bf16 flips their ReLU masks and max-pool argmaxes far more often than in a textured image."""
    vgg, lin = L.synthetic_vgg_state_dict(), L.synthetic_lin_state_dict()
    vgg['features.2.bias'] = torch.full((64,), -0.4)
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    g0 = torch.Generator().manual_seed(1)
    in0 = torch.full((1, 3, 64, 64), 0.5)
    in0[..., 16:48, 16:48] = torch.rand(3, 32, 32, generator=g0)
    in1 = torch.rand(1, 3, 64, 64, generator=g0)
    in0, in1 = in0.cuda(), in1.cuda()
    f = O.taps(O.vgg_features(vgg).cuda(), (2 * in0.double() - 1 - torch.tensor(O.SHIFT, device='cuda', dtype=torch.float64).view(1, 3, 1, 1))
               / torch.tensor(O.SCALE, device='cuda', dtype=torch.float64).view(1, 3, 1, 1))[0]
    assert (f.abs().sum(dim=1) == 0).any()
    _check_against_oracle(m, vgg, lin, in0, in1, plain_gbar=3e-1)


def test_reproducible_and_reference_cache():
    """Two runs are bit-identical; the second call with the same in1 runs no reference pass (fewer launches: exactly the 14 of
    one VGG16 forward); a cached result equals a recomputed one bit for bit; changing in1 in place recomputes, correctly."""
    vgg, lin = _perturbed(5)
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    m2 = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    torch.manual_seed(3)
    in1 = torch.rand(1, 3, 90, 120, device='cuda')
    in0 = torch.rand(1, 3, 90, 120, device='cuda')

    def run(model):
        x = in0.clone().requires_grad_(True)
        v = model(x, in1, normalize=True)
        g, = torch.autograd.grad(v.sum(), x)
        torch.cuda.synchronize()
        return v, g

    lib = _lib.lib()
    m._ensure()                                                        # weights packed: not counted below
    c0 = lib.aph_launch_count()
    v1, g1 = run(m)
    c1 = lib.aph_launch_count()
    v2, g2 = run(m)
    c2 = lib.aph_launch_count()
    assert torch.equal(v1, v2) and torch.equal(g1, g2)
    assert (c1 - c0) - (c2 - c1) == 13 + 4, (c1 - c0, c2 - c1)        # conv1_1 + 12 convs + 4 pools of the reference pass
    v3, g3 = run(m2)                                                   # a fresh handle computes the reference features
    assert torch.equal(v1, v3) and torch.equal(g1, g3)
    in1.mul_(0.5)                                                      # in place: the version counter moves
    c3 = lib.aph_launch_count()
    v4, g4 = run(m)
    assert lib.aph_launch_count() - c3 == c1 - c0
    _check_against_oracle(m, vgg, lin, in0, in1)
    assert not torch.equal(v4, v1)


def test_stale_backward_is_detected():
    """A forward after a grad-tracked forward overwrites the handle's saved activations: the earlier backward raises."""
    vgg, lin = L.synthetic_vgg_state_dict(), L.synthetic_lin_state_dict()
    m = L.LPIPS(net='vgg', verbose=False, vgg_state_dict=vgg, lin_state_dict=lin)
    in1 = torch.rand(1, 3, 32, 32, device='cuda')
    x = torch.rand(1, 3, 32, 32, device='cuda', requires_grad=True)
    v = m(x, in1, normalize=True)
    m(torch.rand(1, 3, 32, 32, device='cuda'), in1, normalize=True)
    with pytest.raises(RuntimeError, match='overwritten'):
        v.sum().backward()
