"""GPU: illustrip.py's per-frame motion (aphantasia_b200.motion, csrc/motion.cu) against a float64 restatement of torchvision's
tensor `affine` and against stock torchvision on the same device; the calls the route leaves to torchvision; and the FFT plan that
fft_image generators of one size share."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from torchvision.transforms import InterpolationMode as IM  # noqa: E402


def reference_f64(img, matrix):
    """torchvision's tensor path in float64: _gen_affine_grid (pixel-centre base grid, normalised by the size), grid_sample
    bilinear / zeros / align_corners=False of the image with a ones-plane, and the fill-0 blend image * mask."""
    n, c, h, w = img.shape
    x = img.double()
    theta = torch.tensor(matrix, dtype=torch.float64, device=x.device).reshape(1, 2, 3)
    xs = torch.linspace(-w * 0.5 + 0.5, w * 0.5 - 0.5, w, dtype=torch.float64, device=x.device)
    ys = torch.linspace(-h * 0.5 + 0.5, h * 0.5 - 0.5, h, dtype=torch.float64, device=x.device)
    base = torch.stack([xs.expand(h, w), ys[:, None].expand(h, w), torch.ones(h, w, dtype=torch.float64, device=x.device)], -1)
    grid = (base.reshape(1, h * w, 3) @ (theta.transpose(1, 2) / torch.tensor([0.5 * w, 0.5 * h], dtype=torch.float64,
                                                                               device=x.device))).reshape(1, h, w, 2)
    both = torch.cat([x, torch.ones(n, 1, h, w, dtype=torch.float64, device=x.device)], 1)
    s = F.grid_sample(both, grid.expand(n, h, w, 2), mode='bilinear', padding_mode='zeros', align_corners=False)
    return s[:, :c] * s[:, c:]


def _lib():
    from aphantasia_b200 import _lib
    return _lib.lib()


ILLUSTRIP = [(np.float64(0.8), (np.float64(10.), np.float64(-10.)), np.array([1.012]), np.float64(0.4)),
             (np.float64(-0.8), (np.float64(-7.3), np.float64(4.1)), np.array([0.988]), np.float64(-0.4)),
             (np.float64(0.13), (np.float64(0.25), np.float64(0.5)), np.array([1.0031]), np.float64(0.05))]
LARGE = [(30., [0., 0.], 1., 0.), (0., [0., 0.], 0.5, 0.), (-12., [3., -5.], 2., 0.), (0., [5000., 0.], 1., 0.),
         (0., [0., -900.], 1.2, 3.)]


@pytest.mark.parametrize('hw', [(224, 224), (720, 1280), (255, 333)])
@pytest.mark.parametrize('planes', [1, 3])
def test_routed_affine_matches_torchvision(hw, planes):
    from aphantasia_b200 import motion
    h, w = hw
    g = torch.Generator(device='cuda').manual_seed(h * 7 + w + planes)
    img = torch.randn(1, planes, h, w, device='cuda', generator=g)
    for angle, shift, scale, shear in ILLUSTRIP + LARGE:
        kw = dict(interpolation=IM.BILINEAR, fill=0)
        got = motion.affine(img, angle, shift, scale, shear, **kw)
        stock = motion.stock_affine(img, angle, shift, scale, shear, **kw)
        want = reference_f64(img, motion.inverse_matrix(angle, shift, scale, shear))
        e64, est = float((got.double() - want).abs().max()), float((got - stock).abs().max())
        assert got.shape == img.shape and got.dtype == torch.float32
        assert e64 < 2e-5, ('float64', hw, planes, angle, shift, scale, shear, e64)
        # torchvision forms the source point in fp32 through the normalised grid: up to ~1e-4 pixel at these sizes, times the
        # difference between neighbouring N(0, 1) pixels
        assert est < 5e-3, ('stock', hw, planes, angle, shift, scale, shear, est)
        if shift == [5000., 0.]:
            assert not got.any()                                   # shifted past the frame: the fill everywhere


def test_routed_affine_is_one_launch_and_deterministic():
    from aphantasia_b200 import motion
    img = torch.rand(1, 3, 720, 1280, device='cuda')
    motion.affine(img, 0.3, (1., 2.), 1.01, 0.2, interpolation=IM.BILINEAR, fill=0)
    torch.cuda.synchronize()
    n0 = _lib().aph_launch_count()
    a = motion.affine(img, np.float64(0.31), (np.float64(4.5), np.float64(-2.25)), np.array([1.007]), np.float64(0.12),
                      interpolation=IM.BILINEAR, fill=[0., 0., 0.])
    assert _lib().aph_launch_count() - n0 == 1
    b = motion.affine(img, np.float64(0.31), (np.float64(4.5), np.float64(-2.25)), np.array([1.007]), np.float64(0.12),
                      interpolation=IM.BILINEAR, fill=0)
    assert _lib().aph_launch_count() - n0 == 2
    assert torch.equal(a, b)


def test_forms_the_kernel_does_not_compute_go_to_torchvision_unchanged():
    from aphantasia_b200 import motion
    img = torch.rand(1, 3, 64, 80, device='cuda')
    args = (7., (3, -2), 1.1, 0.5)
    cases = [(img, dict(interpolation=IM.NEAREST, fill=0)),
             (img, dict(interpolation=IM.BILINEAR, fill=0.5)),
             (img, dict(interpolation=IM.BILINEAR, fill=[0., 1., 0.])),
             (img, dict(interpolation=IM.BILINEAR, fill=None)),
             (img.cpu(), dict(interpolation=IM.BILINEAR, fill=0)),
             (img.double(), dict(interpolation=IM.BILINEAR, fill=0)),
             (img, dict(interpolation=IM.BILINEAR, fill=0, center=[10, 20])),
             (img[0], dict(interpolation=IM.BILINEAR, fill=0)),
             (img[..., ::2], dict(interpolation=IM.BILINEAR, fill=0))]
    for x, kw in cases:
        n0 = _lib().aph_launch_count()
        assert torch.equal(motion.affine(x, *args, **kw), motion.stock_affine(x, *args, **kw)), kw
        assert _lib().aph_launch_count() == n0
    x = img.clone().requires_grad_(True)
    got = motion.affine(x, *args, interpolation=IM.BILINEAR, fill=0)
    assert got.requires_grad and torch.equal(got, motion.stock_affine(x, *args, interpolation=IM.BILINEAR, fill=0))


def test_fft_image_of_one_size_shares_its_plan_and_computes_the_same():
    from aphantasia_b200 import image
    from aphantasia_b200.image import fft_image, to_valid_rgb
    h, w = 360, 640
    torch.manual_seed(0)
    p0 = 0.01 * torch.randn(1, 3, h, w // 2 + 1, 2, device='cuda')
    g_out = torch.rand(1, 3, h, w, device='cuda')

    def run(params_in):
        params, image_f, _ = fft_image([1, 3, h, w], sd=1, resume=params_in.clone())
        out = to_valid_rgb(image_f, colors=2.3)()
        out.backward(g_out)
        return out.detach(), params[0].grad.clone()

    o1, g1 = run(p0)                            # creates the plan for this size (or finds one an earlier test made)
    made = image.fft_plans_created
    o2, g2 = run(p0)
    assert image.fft_plans_created == made
    shared = image._fft_plans.pop((h, w))       # the next generator of this size gets a fresh plan
    o3, g3 = run(p0)
    assert image.fft_plans_created == made + 1
    torch.cuda.synchronize()
    from aphantasia_b200 import _lib
    _lib.lib().aph_fft_plan_destroy(shared)
    assert torch.equal(o1, o2) and torch.equal(o1, o3) and torch.equal(g1, g2) and torch.equal(g1, g3)
    run_other = fft_image([1, 3, h, w + 8], sd=1)
    assert image.fft_plans_created == made + 2 and run_other[1].plan.value != image._shared_fft_plan(h, w).value
